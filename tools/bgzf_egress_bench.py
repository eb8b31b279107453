"""The output records as a BGZF-compressed BAM file, two ways, on the same sorted, duplicate-marked synthetic reads (SURVEY.md 8f row 2):
  A  elp_fetch_bam (every uncompressed record to the host) + host elp_bgzf_deflate (zlib on every host thread), at levels 1 and 6
  B  elp_fetch_bgzf with the BAM header as prefix and the EOF marker (deflate, CRC and compaction on the device, compressed bytes to the host)
Wall times end in a device synchronise; per-kernel ms and GB/s of bgzf_deflate, bgzf_deflate_crc and bgzf_compact come from elp_kernel_stats
(algorithmic bytes: input + output for deflate, input for CRC, 2 x output for compaction); D2H bytes are the bytes each path downloads.
Asserts that the files of A and B inflate to identical bytes.  Card name and power limit are read in the same run.
usage: python tools/bgzf_egress_bench.py [n_pairs] [reps] > bgzf_egress_bench.json"""
import json, os, struct, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from elprep_b200 import bgzf, device, synth
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
threads = os.cpu_count() or 1
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
except (OSError, ValueError):
    card, power = "?", "?"

contigs = synth.scaled_hg38(bench.GENOME_SCALE)
w = synth.make_workload(n_pairs, contigs, seed=20260924, threads=32, want_reference=False)
raw, off = synth.encode_bam(w.batch, w.header, threads=32)
text = b"@HD\tVN:1.6\tSO:coordinate\n"
hdr = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(contigs)) + b"".join(
    struct.pack("<i", len(nm) + 1) + nm.encode() + b"\0" + struct.pack("<i", int(ln)) for nm, ln in contigs)
ctx = device.Context(w.header, profile=True)
ctx.append_bam(raw, off)
ctx.sort_markdup(device.SO_COORDINATE, True)
n = ctx.n_output()
nb = int(ctx.L.elp_fetch_bam_bytes(ctx.h, 0, n))
out = dict(card=card, power_limit_w=power, reads=int(n), record_bytes=nb, host_threads=threads, paths={})
inflated = {}

for level in (1, 6):                                                        # A
    ts = []
    for rep in range(reps + 1):
        ctx.synchronize()
        t0 = time.perf_counter()
        recs = ctx.fetch_bam()[0]
        f = bgzf.deflate(np.concatenate([np.frombuffer(hdr, np.uint8), recs]), level=level, n_threads=threads)
        ctx.synchronize()
        if rep >= 1:
            ts.append(time.perf_counter() - t0)
    inflated[f"A{level}"] = bgzf.inflate(f, n_threads=threads)
    out["paths"][f"A_level{level}"] = dict(wall_s=min(ts), wall_runs=ts, d2h_bytes=nb, file_bytes=int(f.size), ratio=(nb + len(hdr)) / f.size)

ts = []                                                                     # B
for rep in range(reps + 1):
    if rep == 1:
        ctx.reset_stats()
    ctx.synchronize()
    t0 = time.perf_counter()
    f = ctx.fetch_bgzf(prefix=hdr, eof=True)
    ctx.synchronize()
    if rep >= 1:
        ts.append(time.perf_counter() - t0)
st = ctx.kernel_stats()
inflated["B"] = bgzf.inflate(f, n_threads=threads)
k = {name: dict(ms_per_file=st[name]["ms"] / reps, GBps=st[name]["alg_bytes"] / st[name]["ms"] / 1e6 if st[name]["ms"] > 0 else None)
     for name in ("bgzf_deflate", "bgzf_deflate_crc", "bgzf_compact", "bam_format", "scan") if name in st}
out["paths"]["B"] = dict(wall_s=min(ts), wall_runs=ts, d2h_bytes=int(f.size) - 28, file_bytes=int(f.size), ratio=(nb + len(hdr)) / f.size, kernels=k,
                         other_kernels=sorted(set(st) - set(k)))
assert np.array_equal(inflated["A1"], inflated["B"]) and np.array_equal(inflated["A6"], inflated["B"]), "paths A and B inflate to different bytes"
out["inflate_identical"] = True
out["B_over_A_level6"] = out["paths"]["B"]["wall_s"] / out["paths"]["A_level6"]["wall_s"]
ctx.close()
print(json.dumps(out))
