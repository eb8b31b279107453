"""Cost of the write-phase filters (elp_set_output_filter) on elp_fetch_bam and elp_fetch_sam, and the unfiltered fetches against an earlier
build of the library, in one process.
Workload: sorted, duplicate-marked reads of 150 bp, appended as SAM text with RG:Z plus two constant fields (MD:Z, NM:i).
Variants per format: no filter, REMOVE_DUPLICATES, keep RG, both.  Whole-call time: host clock around the fetches of all output records in
chunks into page-locked host buffers (each call ends in a device synchronise), every variant alternated with the others.  Device-kernel
time: CUDA events of every kernel of the fetches (kernel_stats), in a separate run with profiling on.
With --parent LIB (a libelprep_b200.so built from an earlier commit), the unfiltered calls of that library run on a second context holding the
same reads, alternated with the rest.
usage: python tools/output_filter_bench.py [--pairs N] [--reps R] [--parent LIB]   -> one JSON line on stdout"""
import argparse
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

from elprep_b200 import _lib, device, synth
from samtext import sam_text

ap = argparse.ArgumentParser()
ap.add_argument("--pairs", type=int, default=5_000_000)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--parent", default=None)
args = ap.parse_args()
CHUNK = 1 << 20                                                  # output records per fetch call
VARIANTS = {"none": (0, None), "remove_duplicates": (_lib.OUT_REMOVE_DUPLICATES, None), "keep_RG": (0, ("RG",)),
            "both": (_lib.OUT_REMOVE_DUPLICATES, ("RG",))}
PARENT_FNS = ("elp_create", "elp_destroy", "elp_last_error", "elp_append_sam", "elp_sort_markdup", "elp_n_reads", "elp_fetch_bam", "elp_fetch_bam_bytes",
              "elp_fetch_sam", "elp_fetch_sam_bytes", "elp_synchronize")


def pinned(n):
    return torch.empty(max(n, 1), dtype=torch.uint8).pin_memory().numpy()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    return name, float(pl)


def parent_context(header, path):
    """a Context whose calls go to another build of the library (only the calls this tool makes)"""
    L = _lib.load()
    P = C.CDLL(os.path.abspath(path))
    for f in PARENT_FNS:
        getattr(P, f).argtypes, getattr(P, f).restype = getattr(L, f).argtypes, getattr(L, f).restype
    load = _lib.load
    _lib.load = lambda: P
    try:
        return device.Context(header)
    finally:
        _lib.load = load


w = synth.make_workload(args.pairs, synth.scaled_hg38(20.0), seed=20261015, L=150, want_reference=False, threads=32)
text = sam_text(w.batch, w.header, const_tags=b"MD:Z:75A74\tNM:i:1")
nl = np.nonzero(text == 10)[0]
half = int(nl[nl.size // 2]) + 1
del nl


def load(ctx):
    ctx.append_sam(text[:half])
    ctx.append_sam(text[half:])
    ctx.sort_markdup()


def run(ctx, fmt, buf, off, m):
    f = ctx.L.elp_fetch_sam if fmt == "sam" else ctx.L.elp_fetch_bam
    total = 0
    for a in range(0, m, CHUNK):
        b = min(m, a + CHUNK)
        rc = f(ctx.h, a, b - a, buf.ctypes.data_as(C.c_void_p), buf.size, off.ctypes.data_as(C.c_void_p))
        assert rc == 0, ctx.L.elp_last_error(ctx.h)
        total += int(off[b - a])
    return total


ctx = device.Context(w.header)
load(ctx)
n = ctx.n
par = None
if args.parent:
    par = parent_context(w.header, args.parent)
    load(par)
buf = pinned(int(ctx.L.elp_fetch_sam_bytes(ctx.h, 0, min(n, CHUNK))) + (1 << 24))
off = torch.empty((CHUNK + 1) * 8, dtype=torch.uint8).pin_memory().numpy().view(np.uint64)
jobs = [(fmt, v) for v in VARIANTS for fmt in ("bam", "sam")] + ([("bam", "parent"), ("sam", "parent")] if par else [])
wall = {j: [] for j in jobs}
nbytes, nout = {}, {}
for rep in range(args.reps + 1):                                  # rep 0 warms up every shape and allocation
    for fmt, v in jobs:
        c = par if v == "parent" else ctx
        if v != "parent":
            mask, keep = VARIANTS[v]
            ctx.set_output_filter(mask, keep=keep)
        m = c.n if v == "parent" else ctx.n_output()
        c.synchronize()
        t0 = time.perf_counter()
        nbytes[(fmt, v)] = run(c, fmt, buf, off, m)
        dt = time.perf_counter() - t0
        nout[(fmt, v)] = m
        if rep:
            wall[(fmt, v)].append(dt)
ctx.close()
if par:
    par.close()
prof = device.Context(w.header, profile=True)
load(prof)
kern = {}
for fmt, v in jobs:
    if v == "parent":
        continue
    mask, keep = VARIANTS[v]
    prof.set_output_filter(mask, keep=keep)
    m = prof.n_output()
    run(prof, fmt, buf, off, m)                                   # warm-up (and the selection of this setting)
    prof.synchronize(); prof.reset_stats()
    run(prof, fmt, buf, off, m)
    kern[(fmt, v)] = prof.kernel_stats()
prof.close()
out = {"tool": "output_filter_bench", "reads": n, "read_length": 150, "records_per_call": CHUNK, "reps": args.reps}
for fmt, v in jobs:
    med = float(np.median(wall[(fmt, v)]))
    r = {"records": nout[(fmt, v)], "bytes": nbytes[(fmt, v)], "call_s_median": med, "call_s_best": min(wall[(fmt, v)]),
         "output_GBps": nbytes[(fmt, v)] / med / 1e9}
    if (fmt, v) in kern:
        kms = sum(x["ms"] for x in kern[(fmt, v)].values())
        r.update(kernel_ms=round(kms, 3), kernels={k: round(x["ms"], 3) for k, x in sorted(kern[(fmt, v)].items(), key=lambda kv: -kv[1]["ms"])})
    out[f"{fmt}_{v}"] = r
name, power = card()
out.update(gpu=name, power_limit_w=power)
print(json.dumps(out))
