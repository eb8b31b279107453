"""Ingest rate of SAM text (elp_append_sam) against BAM records (elp_append_bam) of the same reads, in one process.
Whole-call time: host clock around the appends of one context, ending in a device synchronise, the two paths alternated.
Device-kernel time: CUDA events of every kernel of the appends (kernel_stats), in separate runs with profiling on.
With an ingest filter (mask and min_mapq of elp_set_ingest_filter), both paths run the fused filter on every append.
usage: python tools/sam_ingest_bench.py [n_pairs] [reps] [filter_mask] [min_mapq]   -> one JSON line on stdout"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch

from elprep_b200 import device, synth
from samtext import sam_text

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
filter_mask = int(sys.argv[3]) if len(sys.argv) > 3 else 0
min_mapq = int(sys.argv[4]) if len(sys.argv) > 4 else 0
CH = 8                                                          # appends per pass, cut at line / record boundaries


def pinned(a):
    p = torch.empty(a.size, dtype=torch.uint8).pin_memory().numpy()
    p[:] = a
    return p


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    return name, float(pl)


w = synth.make_workload(n_pairs, synth.scaled_hg38(20.0), seed=20261015, L=150, want_reference=False, threads=32)
n = w.batch.n
text = pinned(sam_text(w.batch, w.header))
raw, offs = synth.encode_bam(w.batch, w.header, threads=32)
raw = pinned(raw)
nl = np.nonzero(text == 10)[0]
line_cut = [0] + [int(nl[n * i // CH - 1]) + 1 for i in range(1, CH)] + [text.size]
rec_cut = [n * i // CH for i in range(CH + 1)]


def run_sam(ctx):
    for a, b in zip(line_cut[:-1], line_cut[1:]):
        ctx.append_sam(text[a:b])


def run_bam(ctx):
    for a, b in zip(rec_cut[:-1], rec_cut[1:]):
        ctx.append_bam(raw[int(offs[a]):int(offs[b])], offs[a:b + 1] - offs[a])


paths = {"sam": run_sam, "bam": run_bam}
ctx = device.Context(w.header)
ctx.set_ingest_filter(filter_mask, min_mapq)
wall = {k: [] for k in paths}
for rep in range(reps + 1):                                     # rep 0 warms up every shape and allocation
    for k, f in paths.items():
        ctx.reset(); ctx.synchronize()
        t0 = time.perf_counter()
        f(ctx)
        ctx.synchronize()
        dt = time.perf_counter() - t0
        assert ctx.n + ctx.n_filtered() == n and (ctx.n == n or filter_mask or min_mapq)
        kept = ctx.n
        if rep:
            wall[k].append(dt)
ctx.close()

prof = device.Context(w.header, profile=True)
prof.set_ingest_filter(filter_mask, min_mapq)
kern = {}
for k, f in paths.items():
    for rep in range(2):
        prof.reset(); prof.synchronize(); prof.reset_stats()
        f(prof)
        prof.synchronize()
    kern[k] = prof.kernel_stats()
prof.close()

name, power = card()
out = {"tool": "sam_ingest_bench", "gpu": name, "power_limit_w": power, "reads": n, "read_length": 150, "appends_per_pass": CH,
       "sam_text_bytes": int(text.size), "bam_record_bytes": int(raw.size), "reps": reps,
       "filter_mask": filter_mask, "min_mapq": min_mapq, "reads_kept": kept}
for k in paths:
    best, med = min(wall[k]), float(np.median(wall[k]))
    kms = sum(v["ms"] for v in kern[k].values())
    nbytes = text.size if k == "sam" else raw.size
    out[k] = {"call_s_median": med, "call_s_best": best, "reads_per_s": n / med, "input_GBps": nbytes / med / 1e9,
              "kernel_ms": kms, "kernel_reads_per_s": n / (kms / 1e3), "kernel_input_GBps": nbytes / (kms / 1e3) / 1e9,
              "kernels": {name_: round(v["ms"], 3) for name_, v in sorted(kern[k].items(), key=lambda kv: -kv[1]["ms"])}}
print(json.dumps(out))
