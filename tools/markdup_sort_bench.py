"""Times elp_sort_markdup (coordinate sort + MarkDuplicates) with the smaller duplicate-marking sorts and with
ELPREP_B200_MARKDUP=exact, alternated call by call in one process, on the flagship reads in arrival order, under a seeded permutation,
and on workloads with many more mate-unmapped pairs (true fragments), where the set pass, the probe pass and the path choice show.

    python tools/markdup_sort_bench.py [--pairs N] [--reps R] [--mate-unmapped F ...]   -> one JSON line on stdout

Per workload and setting: elp_sort_markdup in ms (CUDA events on the library's stream around the call, median and spread of R calls),
the duplicate-marking and radix sort kernels in ms per call (from the profiled stats of the same calls), the true-fragment share of
the entering reads, and a SHA-256 of the FLAG column in arrival order, which must be equal across the two settings.  The card's name
and power limit are printed with the numbers, since every number belongs to them."""
import argparse
import gc
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from elprep_b200 import device, synth  # noqa: E402
from mate_join_bench import card, flag_digest, one_call  # noqa: E402

KERNELS = ("frag_keys", "frag_mark", "frag_set_insert", "frag_set_probe", "frag_sparse_mark", "pair_keys", "pair_mark", "pair_hash_mark",
           "radix_onesweep_u64", "radix_hist_u64", "radix_onesweep_u32", "radix_hist_u32", "radix_onesweep_u128", "radix_hist_u128")
SETTINGS = {"smaller": None, "exact": "exact"}


def fragment_share(b):
    f = b.flag.astype(np.int64)
    entering = (f & 0x904) == 0
    frag = entering & ((f & 0x9) != 0x1)
    return float(frag.sum()) / max(1, int(entering.sum()))


def set_mode(mode):
    if mode is None:
        os.environ.pop("ELPREP_B200_MARKDUP", None)
    else:
        os.environ["ELPREP_B200_MARKDUP"] = mode


def bench(name, b, header, reps, res):
    ctxs = {s: device.Context(header, profile=True) for s in SETTINGS}
    for s, ctx in ctxs.items():       # warm-up: allocations and module loads
        set_mode(SETTINGS[s])
        one_call(ctx, b)
        ctx.reset_stats()
    times = {s: [] for s in SETTINGS}
    for _ in range(reps):
        for s, ctx in ctxs.items():
            set_mode(SETTINGS[s])
            times[s].append(one_call(ctx, b))
    set_mode(None)
    share = fragment_share(b)
    for s, ctx in ctxs.items():
        st = ctx.kernel_stats()
        digest, dups = flag_digest(ctx, b.n)
        t = np.asarray(times[s])
        res[f"{name}/{s}"] = {"sort_markdup_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3),
                              "kernels_ms_per_call": {k: round(st[k]["ms"] / reps, 3) for k in KERNELS if k in st},
                              "launches_per_call": {k: st[k]["launches"] / reps for k in KERNELS if k in st},
                              "fragment_share": round(share, 4), "flag_sha256": digest, "duplicates": dups}
        print(name, s, json.dumps(res[f"{name}/{s}"]), file=sys.stderr, flush=True)
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=15_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mate-unmapped", type=float, nargs="*", default=[0.2, 0.35])
    args = ap.parse_args()
    print("card:", card(), file=sys.stderr, flush=True)
    threads = min(32, os.cpu_count() or 1)
    res = {}
    w = synth.make_workload(args.pairs, synth.scaled_hg38(20.0), seed=20260924, want_reference=False, threads=threads)
    bench("arrival", w.batch, w.header, args.reps, res)
    bench("permuted", synth.take(w.batch, np.random.default_rng(20261018).permutation(w.batch.n)), w.header, args.reps, res)
    del w
    gc.collect()
    for f in args.mate_unmapped:
        w = synth.make_workload(args.pairs, synth.scaled_hg38(20.0), seed=20260924, want_reference=False, threads=threads, mate_unmapped_frac=f)
        bench(f"mate_unmapped_{f}", w.batch, w.header, args.reps, res)
        del w
        gc.collect()
    names = sorted({k.split("/")[0] for k in res})
    same = {n: res[f"{n}/smaller"]["flag_sha256"] == res[f"{n}/exact"]["flag_sha256"] for n in names}
    print(json.dumps({"card": card(), "reps": args.reps, "flag_equal_across_settings": same, "results": res}))


if __name__ == "__main__":
    main()
