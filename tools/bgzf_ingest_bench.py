"""A BGZF-compressed BAM file into a context, two ways, on the same synthetic records (SURVEY.md 8f row 2):
  A  host inflate (elp_bgzf_inflate, zlib on every host thread) + elp_bam_header_size + elp_append_bam
  B  elp_append_bgzf in 64 MiB chunks of the compressed file + elp_append_bgzf_end (inflate, CRC, header walk and framing on the device)
at deflate levels 1 and 6.  Wall times end in a device synchronise; per-kernel ms and GB/s of bgzf_inflate, bgzf_crc and bam_frame come
from elp_kernel_stats (algorithmic bytes: compressed in + inflated out for inflate, inflated bytes for CRC and framing); H2D bytes are the
bytes each path uploads.  Asserts that A and B give identical elp_fetch_bam bytes.  Card name and power limit are read in the same run.
usage: python tools/bgzf_ingest_bench.py [n_pairs] [reps] > bgzf_ingest_bench.json"""
import json, os, struct, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from elprep_b200 import bgzf, device, synth
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
CHUNK = 64 << 20
threads = os.cpu_count() or 1
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
except (OSError, ValueError):
    card, power = "?", "?"

contigs = synth.scaled_hg38(bench.GENOME_SCALE)
w = synth.make_workload(n_pairs, contigs, seed=20260924, threads=32, want_reference=False)
raw, _ = synth.encode_bam(w.batch, w.header, threads=32)
n = w.batch.n
text = b"@HD\tVN:1.6\tSO:unsorted\n"
hdr = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(contigs)) + b"".join(
    struct.pack("<i", len(nm) + 1) + nm.encode() + b"\0" + struct.pack("<i", int(ln)) for nm, ln in contigs)
plain = np.concatenate([np.frombuffer(hdr, np.uint8), raw])
ctx = device.Context(w.header, profile=True)
out = dict(card=card, power_limit_w=power, reads=n, record_bytes=int(raw.size), bytes_per_read=raw.size / n, host_threads=threads, chunk_bytes=CHUNK, levels={})


def fetch_all():
    ctx.sort_markdup(mark_duplicates=False)
    return ctx.fetch_bam()[0]


for level in (1, 6):
    data = bgzf.deflate(plain, level=level, n_threads=threads)
    ta, tb, stats = [], [], {}
    ref = got = None
    for rep in range(reps + 1):
        ctx.reset(); ctx.synchronize()
        t0 = time.perf_counter()
        inflated = bgzf.inflate(data, n_threads=threads)                    # A
        h0, _ = bgzf.bam_header_size(inflated)
        ctx.append_bam(inflated[h0:], None); ctx.synchronize()
        t1 = time.perf_counter()
        if rep == reps:
            ref = fetch_all().copy()
        ctx.reset(); ctx.synchronize()
        if rep == 1:
            ctx.reset_stats()
        t2 = time.perf_counter()
        for a in range(0, data.size, CHUNK):                                 # B
            ctx.append_bgzf(data[a:a + CHUNK])
        ctx.append_bgzf_end(); ctx.synchronize()
        t3 = time.perf_counter()
        if rep == reps:
            st = ctx.kernel_stats()
            got = fetch_all().copy()
        if rep >= 1:
            ta.append(t1 - t0); tb.append(t3 - t2)
    assert ref is not None and got is not None and np.array_equal(ref, got), "paths A and B give different elp_fetch_bam bytes"
    k = {name: dict(ms_per_file=st[name]["ms"] / reps, GBps=st[name]["alg_bytes"] / st[name]["ms"] / 1e6 if st[name]["ms"] > 0 else None)
         for name in ("bgzf_inflate", "bgzf_crc", "bam_frame", "bam_header") if name in st}
    out["levels"][str(level)] = dict(compressed_bytes=int(data.size), ratio=plain.size / data.size,
                                     wall_A_s=min(ta), wall_B_s=min(tb), wall_A_runs=ta, wall_B_runs=tb, B_over_A=min(tb) / min(ta),
                                     h2d_A_bytes=int(plain.size - len(hdr)), h2d_B_bytes=int(data.size), kernels=k, fetch_bam_identical=True)
ctx.close()
print(json.dumps(out))
