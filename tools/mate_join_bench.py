"""Times elp_sort_markdup (coordinate sort + MarkDuplicates) on the flagship reads in their arrival order and under a seeded permutation,
for this library and, with --parent LIB, a libelprep_b200.so built from an earlier commit, alternated call by call in one process.

    python tools/mate_join_bench.py [--pairs N] [--reps R] [--parent LIB]   -> one JSON line on stdout

Aligners write the two mates of a pair next to each other, and so does the generator; the permuted order leaves no mates adjacent, the
case where the mate join's adjacency pass finds nothing.  Per library and order: elp_sort_markdup in ms (CUDA events on the library's
stream around the call, median and spread of R calls), the mate-join kernels and the radix sort kernels in ms per call (from the
profiled stats of the same calls), and a SHA-256 of the FLAG column in arrival order, which must be equal across the libraries.  The
card's name and power limit are printed with the numbers, since every number belongs to them."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elprep_b200 import _lib, device, synth  # noqa: E402

KERNELS = ("join_adjacent", "prefix_scan", "join_compact", "join_keys", "join", "pair_flag", "radix_onesweep_u64", "radix_hist_u64")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip().split("\n")[0]


def parent_context(header, path):
    """a Context whose calls go to another build of the library"""
    L = _lib.load()
    P = C.CDLL(os.path.abspath(path))
    for f in _lib.EXPORTS:
        if hasattr(P, f) and hasattr(L, f):
            getattr(P, f).argtypes, getattr(P, f).restype = getattr(L, f).argtypes, getattr(L, f).restype
    load = _lib.load
    _lib.load = lambda: P
    try:
        return device.Context(header, profile=True)
    finally:
        _lib.load = load


def one_call(ctx, batch):
    ctx.reset()
    ctx.append(batch)
    ctx.synchronize()
    ctx.timer_start()
    ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP)
    return ctx.timer_stop()


def flag_digest(ctx, n):
    idx, flag, _, _ = ctx.fetch(want_qual=False)
    out = np.empty(n, np.uint16)
    out[idx.astype(np.int64)] = flag
    return hashlib.sha256(out.tobytes()).hexdigest()[:16], int(((out & 0x400) != 0).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=15_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent", default=None)
    args = ap.parse_args()
    print("card:", card(), file=sys.stderr, flush=True)
    w = synth.make_workload(args.pairs, synth.scaled_hg38(20.0), seed=20260924, want_reference=False, threads=min(32, os.cpu_count() or 1))
    orders = {"arrival": w.batch, "permuted": synth.take(w.batch, np.random.default_rng(20261018).permutation(w.batch.n))}
    libs = {"this": device.Context(w.header, profile=True)}
    if args.parent:
        libs["parent"] = parent_context(w.header, args.parent)
    res = {}
    for oname, b in orders.items():
        for lname, ctx in libs.items():       # warm-up: allocations and module loads
            one_call(ctx, b)
            ctx.reset_stats()
        times = {k: [] for k in libs}
        for _ in range(args.reps):
            for lname, ctx in libs.items():
                times[lname].append(one_call(ctx, b))
        for lname, ctx in libs.items():
            st = ctx.kernel_stats()
            ctx.reset_stats()
            digest, dups = flag_digest(ctx, b.n)
            t = np.asarray(times[lname])
            res[f"{oname}/{lname}"] = {"sort_markdup_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3),
                                      "kernels_ms_per_call": {k: round(st[k]["ms"] / args.reps, 3) for k in KERNELS if k in st},
                                      "launches_per_call": {k: st[k]["launches"] / args.reps for k in KERNELS if k in st},
                                      "join_elements": st["join"]["alg_bytes"] / 12 / args.reps if "join" in st else None,
                                      "flag_sha256": digest, "duplicates": dups}
            print(oname, lname, json.dumps(res[f"{oname}/{lname}"]), file=sys.stderr, flush=True)
    for ctx in libs.values():
        ctx.close()
    same = {o: len({res[k]["flag_sha256"] for k in res if k.startswith(o + "/")}) == 1 for o in orders}
    print(json.dumps({"card": card(), "reads": int(w.batch.n), "reps": args.reps, "flag_equal_across_libraries": same, "results": res}))


if __name__ == "__main__":
    main()
