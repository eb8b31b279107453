"""Times elp_bqsr_gather on the flagship workload (bench.py's reads, seed and genome scale), kernel by kernel, for this library and,
with --parent LIB or --lib NAME=LIB, other builds of libelprep_b200.so, alternated call by call in one process.

    python tools/count_bench.py [--reps R] [--parent LIB] [--lib NAME=LIB ...]   -> one JSON line on stdout

Each library gets its own context holding the same reads, sorted and duplicate-marked once; then R gathers per library run in turn.
Per library: the gather call in ms (CUDA events on the library's stream, median and spread), and per kernel (bqsr_g_count,
bqsr_g_count_indel, bqsr_g_prep2, ...) the ms per call and the algorithmic GB/s the library charges it with, from its profiled stats.
A SHA-256 of the gathered tables says whether two builds count the same; builds made by tools/ablate.sh count wrong tables by design.
The card's name and power limit are printed with the numbers, since every number belongs to them."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from elprep_b200 import device, synth  # noqa: E402
from mate_join_bench import card, parent_context  # noqa: E402


def make_ctx(w, hb, path):
    ctx = device.Context(w.header, profile=True) if path is None else parent_context(w.header, path)
    for ci in range(len(w.contig_bases)):
        ctx.set_reference(ci, w.contig_bases[ci])
        ctx.set_known_sites(ci, w.sites[ci], already_flat=True)
    ctx.append(hb)
    ctx.sort_markdup()
    ctx.synchronize()
    return ctx


def one_call(ctx):
    ctx.synchronize()
    ctx.timer_start()
    ctx.bqsr_gather()
    return ctx.timer_stop()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=bench.DEFAULT_READS // 2)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--parent", default=None, help="libelprep_b200.so of another commit")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=LIB", help="another build, e.g. from tools/ablate.sh")
    args = ap.parse_args()
    print("card:", card(), file=sys.stderr, flush=True)
    w = synth.make_workload(args.pairs, synth.scaled_hg38(bench.GENOME_SCALE), seed=20260924, threads=min(32, os.cpu_count() or 1))
    hb = bench.pinned(w.batch)
    paths = {"this": None}
    if args.parent:
        paths["parent"] = args.parent
    for spec in args.lib:
        name, _, path = spec.partition("=")
        paths[name] = path
    libs = {name: make_ctx(w, hb, p) for name, p in paths.items()}
    for ctx in libs.values():      # warm-up: allocations and module loads
        one_call(ctx)
        ctx.reset_stats()
    times = {k: [] for k in libs}
    for _ in range(args.reps):
        for name, ctx in libs.items():
            times[name].append(one_call(ctx))
    res = {}
    for name, ctx in libs.items():
        st = ctx.kernel_stats()
        t = np.asarray(times[name])
        kern = {k: {"ms": round(v["ms"] / args.reps, 3), "GBps": round(v["alg_bytes"] / (v["ms"] / 1e3) / 1e9, 1) if v["ms"] > 0 and v["alg_bytes"] > 0 else None}
                for k, v in sorted(st.items(), key=lambda kv: -kv[1]["ms"]) if k.startswith("bqsr_g_")}
        res[name] = {"gather_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3),
                     "kernels": kern, "tables_sha256": hashlib.sha256(np.ascontiguousarray(ctx.tables_get()).tobytes()).hexdigest()[:16]}
        print(name, json.dumps(res[name]), file=sys.stderr, flush=True)
    for ctx in libs.values():
        ctx.close()
    print(json.dumps({"card": card(), "reads": int(hb.n), "reps": args.reps, "results": res}))


if __name__ == "__main__":
    main()
