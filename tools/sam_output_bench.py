"""Output rate of SAM text (elp_fetch_sam) against BAM records (elp_fetch_bam) of the same sorted, duplicate-marked reads, in one process.
Whole-call time: host clock around the fetches of all reads in chunks into page-locked host buffers (each call ends in a device
synchronise), the two formats alternated.  Device-kernel time: CUDA events of every kernel of the fetches (kernel_stats), in a separate
run with profiling on.  Workloads: the reads as they come from synth (no float tags), and the same reads with one f tag each (bounds the
host float step).
usage: python tools/sam_output_bench.py [n_pairs] [reps]   -> one JSON line on stdout"""
import ctypes as C
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
CHUNK = 1 << 20                                                  # reads per fetch call


def pinned(n):
    return torch.empty(max(n, 1), dtype=torch.uint8).pin_memory().numpy()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    return name, float(pl)


w = synth.make_workload(n_pairs, synth.scaled_hg38(20.0), seed=20261015, L=150, want_reference=False, threads=32)
n = w.batch.n
raw, offs = synth.encode_bam(w.batch, w.header, threads=32)
ftext = sam_text(w.batch, w.header, const_tags=b"XF:f:0.73914623")
cuts = list(range(0, n, CHUNK)) + [n]


def load(ctx, kind):
    if kind == "plain":
        ctx.append_bam(raw, offs)
    else:
        nl = np.nonzero(ftext == 10)[0]
        half = int(nl[nl.size // 2]) + 1
        ctx.append_sam(ftext[:half])
        ctx.append_sam(ftext[half:])
    ctx.sort_markdup()


def sizes(ctx):
    s = [int(ctx.L.elp_fetch_sam_bytes(ctx.h, a, b - a)) for a, b in zip(cuts[:-1], cuts[1:])]
    m = [int(ctx.L.elp_fetch_bam_bytes(ctx.h, a, b - a)) for a, b in zip(cuts[:-1], cuts[1:])]
    return s, m


def run(ctx, fmt, buf, off):
    f = ctx.L.elp_fetch_sam if fmt == "sam" else ctx.L.elp_fetch_bam
    total = 0
    for a, b in zip(cuts[:-1], cuts[1:]):
        rc = f(ctx.h, a, b - a, buf.ctypes.data_as(C.c_void_p), buf.size, off.ctypes.data_as(C.c_void_p))
        assert rc == 0, ctx.L.elp_last_error(ctx.h)
        total += int(off[b - a])
    return total


out = {"tool": "sam_output_bench", "reads": n, "read_length": 150, "reads_per_call": CHUNK, "reps": reps}
for kind in ("plain", "one_f_tag"):
    ctx = device.Context(w.header)
    load(ctx, kind)
    ss, bs = sizes(ctx)
    buf = pinned(max(max(ss), max(bs)))
    off = torch.empty((CHUNK + 1) * 8, dtype=torch.uint8).pin_memory().numpy().view(np.uint64)
    wall = {"sam": [], "bam": []}
    nbytes = {}
    for rep in range(reps + 1):                                  # rep 0 warms up every shape and allocation
        for fmt in ("sam", "bam"):
            ctx.synchronize()
            t0 = time.perf_counter()
            nbytes[fmt] = run(ctx, fmt, buf, off)
            dt = time.perf_counter() - t0
            if rep:
                wall[fmt].append(dt)
    ctx.close()
    prof = device.Context(w.header, profile=True)
    load(prof, kind)
    kern = {}
    for fmt in ("sam", "bam"):
        run(prof, fmt, buf, off)                                  # warm-up
        prof.synchronize(); prof.reset_stats()
        run(prof, fmt, buf, off)
        kern[fmt] = prof.kernel_stats()
    prof.close()
    res = {"sam_text_bytes": nbytes["sam"], "bam_record_bytes": nbytes["bam"], "text_over_bam": nbytes["sam"] / nbytes["bam"]}
    for fmt in ("sam", "bam"):
        med = float(np.median(wall[fmt]))
        kms = sum(v["ms"] for v in kern[fmt].values())
        res[fmt] = {"call_s_median": med, "call_s_best": min(wall[fmt]), "reads_per_s": n / med, "output_GBps": nbytes[fmt] / med / 1e9,
                    "kernel_ms": kms, "kernel_output_GBps": nbytes[fmt] / (kms / 1e3) / 1e9,
                    "kernels": {k: round(v["ms"], 3) for k, v in sorted(kern[fmt].items(), key=lambda kv: -kv[1]["ms"])}}
    out[kind] = res
name, power = card()
out.update(gpu=name, power_limit_w=power)
print(json.dumps(out))
