"""End-to-end timing of the path with BAM records at both ends (SURVEY.md 8f row 1): elp_append_bam -> sort + markdup ->
BQSR gather / finalize / apply -> elp_fetch_bam, host buffers pinned, copies inside the timed region.
usage: python tools/bam_bench.py [n_pairs] > bam_bench.json"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from elprep_b200 import synth, device
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 15_000_000
contigs = synth.scaled_hg38(bench.GENOME_SCALE)
w = synth.make_workload(n_pairs, contigs, seed=20260924, threads=32)
raw, offs = synth.encode_bam(w.batch, w.header, threads=32)
n = w.batch.n
praw = torch.empty(raw.size, dtype=torch.uint8).pin_memory().numpy(); praw[:] = raw
pout = torch.empty(raw.size, dtype=torch.uint8).pin_memory().numpy()
poff = np.empty(n + 1, np.uint64)
ctx = device.Context(w.header, profile=True)
for ci in range(len(contigs)):
    ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], True)
CH = 8
cuts = [n * i // CH for i in range(CH + 1)]
times = []
for rep in range(4):
    ctx.reset(); ctx.synchronize()
    if rep == 1:
        ctx.reset_stats()
    t0 = time.perf_counter()
    for a, b in zip(cuts[:-1], cuts[1:]):
        ctx.append_bam(praw[int(offs[a]):int(offs[b])], offs[a:b + 1] - offs[a])
    t1 = time.perf_counter()
    ctx.sort_markdup(); ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply(); ctx.synchronize()
    t2 = time.perf_counter()
    pos = 0
    for a, b in zip(cuts[:-1], cuts[1:]):
        nb = int(ctx.L.elp_fetch_bam_bytes(ctx.h, a, b - a))
        ctx._ck(ctx.L.elp_fetch_bam(ctx.h, a, b - a, pout[pos:].ctypes.data, nb, poff[a:].ctypes.data))
        pos += nb
    t3 = time.perf_counter()
    if rep >= 1:
        times.append((t1 - t0, t2 - t1, t3 - t2))
st = ctx.kernel_stats()
reps = len(times)
ing, cmp_, egr = (sum(t[k] for t in times) / reps for k in range(3))
ok = int(pos) == int(raw.size)
print(json.dumps({"workload": f"{n} synthetic reads as BAM alignment records ({raw.size / n:.0f} B/read), hg38/{bench.GENOME_SCALE:g}-shaped genome, 1 x H100",
                  "e2e_reads_per_s": n / (ing + cmp_ + egr), "ingest_ms": 1e3 * ing, "compute_ms": 1e3 * cmp_, "egress_ms": 1e3 * egr,
                  "h2d_bytes": int(raw.size), "d2h_bytes": int(pos), "bytes_roundtrip_ok": ok,
                  "kernels_ms_per_step": {k: st[k]["ms"] / reps for k in ("bam_fixed", "bam_copy", "bam_format") if k in st},
                  "kernels_GBps": {k: st[k]["alg_bytes"] / st[k]["ms"] / 1e6 for k in ("bam_fixed", "bam_copy", "bam_format") if k in st and st[k]["ms"] > 0}}))
