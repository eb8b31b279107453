"""Cost of `--target-regions` on the device (elp_filter_target_regions) and what it saves in the BQSR gather and apply.
Workload: synth.make_workload(exome=True) -- fragments around 300-base exons every 15 kbp -- over a scaled human genome; the regions are the
generator's exons padded on both sides, with the padding chosen from the reads so that about 70 % of them are kept.
Two contexts hold the same reads, sorted and duplicate-marked: one calls the filter, the other does not.  Per repetition (alternating):
  filter   CUDA events of every kernel of the call (kernel_stats, profile on) and the host clock around the call (it ends in a synchronise)
  gather   elp_timer (device events on the library's stream) around elp_bqsr_gather, with and without the filter
  apply    the same around elp_bqsr_apply (finalize is not timed)
Achieved bandwidth: each kernel's algorithmic bytes (the figures in DESIGN.md section 3) over its event time.  A smaller workload runs through
the device and through the reference order composed from the oracle (tests/targetregions_ref.py) and must match bit for bit.
usage: python tools/target_regions_bench.py [--pairs N] [--reps R] [--check-pairs M]   -> one JSON line on stdout"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np

from elprep_b200 import device, synth
from util import oracle_tables_dense, set_side_inputs

ap = argparse.ArgumentParser()
ap.add_argument("--pairs", type=int, default=15_000_000)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--check-pairs", type=int, default=100_000)
ap.add_argument("--keep", type=float, default=0.70, help="target share of reads kept")
args = ap.parse_args()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    return name, float(pl)


def regions_for(w, contigs, seed, share):
    """the generator's exons with the smallest padding (steps of 10 bases) that keeps at least `share` of a sample of the reads"""
    import targetregions_ref as T
    sample = w.batch.take(np.arange(0, w.batch.n, max(1, w.batch.n // 50_000)))
    spans = [(r.refid, *T.R.aln_span(r)) for r in T.recs_of(sample)]
    rid = np.array([x[0] for x in spans]); st = np.array([x[1] for x in spans], np.int64); en = np.array([x[2] for x in spans], np.int64)
    for pad in range(0, 5000, 10):
        ex = synth.exome_regions(contigs, seed=seed, pad=pad)
        keep = np.zeros(rid.size, bool)
        for c, iv in enumerate(ex):
            fl = np.array(T.flatten({0: iv})[0], np.int64).reshape(-1, 2)
            m = rid == c
            j = np.searchsorted(fl[:, 1], st[m], side="left")            # first region ending at or after the read's start
            keep[m] = (j < len(fl)) & (fl[np.minimum(j, len(fl) - 1), 0] < en[m])   # intervals.Overlap: start <= alnEnd - 1
        if keep.mean() >= share:
            return pad, {c: ex[c] for c in range(len(contigs))}
    raise RuntimeError("no padding keeps that many reads")


def loaded(w, reg, filt):
    ctx = device.Context(w.header, profile=True)
    set_side_inputs(ctx, w)
    ctx.append(w.batch)
    ctx.sort_markdup(device.SO_COORDINATE, 1)
    for c, iv in reg.items():
        ctx.set_bqsr_target_regions(c, iv)
    ctx.reset_stats()
    out = {}
    if filt:
        t0 = time.perf_counter()
        out["removed"] = ctx.filter_target_regions()
        out["filter_host_ms"] = (time.perf_counter() - t0) * 1e3
        out["filter_kernels"] = ctx.kernel_stats()
    return ctx, out


def timed(ctx, fn):
    ctx.timer_start()
    fn()
    return ctx.timer_stop()


def check(contigs, seed, share):
    import targetregions_ref as T
    w = synth.make_workload(args.check_pairs, contigs, seed=seed + 1, exome=True)
    pad, reg = regions_for(w, contigs, seed + 1, share)
    ctx = device.Context(w.header)
    try:
        set_side_inputs(ctx, w)
        ctx.append(w.batch)
        ctx.sort_markdup(device.SO_COORDINATE, 1)
        for c, iv in reg.items():
            ctx.set_bqsr_target_regions(c, iv)
        removed = ctx.filter_target_regions()
        ctx.bqsr_gather()
        tables = ctx.tables_get()
        ctx.bqsr_finalize(None)
        ctx.bqsr_apply()
        idx, flag, qoff, qual = ctx.fetch()
    finally:
        ctx.close()
    o = T.mark_then_filter(w, reg)
    d, _ = oracle_tables_dense(o["tables"])
    ok = (removed == o["n_removed"] and np.array_equal(idx, o["perm"]) and np.array_equal(flag, o["flag"]) and np.array_equal(tables, d)
          and np.array_equal(qual[:int(qoff[-1])], o["qual"]))
    return dict(reads=int(w.batch.n), kept=int(o["perm"].size), pad=pad, identical=bool(ok))


def main():
    name, pl = card()
    contigs = synth.scaled_hg38(20.0)
    seed = 20261016
    chk = check(contigs, seed, args.keep)        # (also the first launch of every kernel the timed runs use)
    w = synth.make_workload(args.pairs, contigs, seed=seed, exome=True, threads=32)
    pad, reg = regions_for(w, contigs, seed, args.keep)
    n = int(w.batch.n)
    A, a = loaded(w, reg, True)
    B, _ = loaded(w, reg, False)
    kept = n - a["removed"]
    for ctx in (A, B):                           # warm-up of every shape
        ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply()
    res = {k: [] for k in ("gather_filtered_ms", "gather_all_ms", "apply_filtered_ms", "apply_all_ms")}
    for _ in range(args.reps):
        res["gather_filtered_ms"].append(timed(A, A.bqsr_gather)); res["gather_all_ms"].append(timed(B, B.bqsr_gather))
        A.bqsr_finalize(None); B.bqsr_finalize(None)
        res["apply_filtered_ms"].append(timed(A, A.bqsr_apply)); res["apply_all_ms"].append(timed(B, B.bqsr_apply))
    A.close(); B.close()
    filt = {k: dict(ms=v["ms"], gb_per_s=(v["alg_bytes"] / (v["ms"] * 1e-3) / 1e9) if v["ms"] > 0 else None, alg_bytes=v["alg_bytes"])
            for k, v in a["filter_kernels"].items()}
    out = dict(card=name, power_limit_w=pl, reads=n, kept=kept, kept_share=kept / n, pad=pad, regions=int(sum(len(v) for v in reg.values())),
               filter_host_ms=a["filter_host_ms"], filter_kernel_ms=sum(v["ms"] for v in a["filter_kernels"].values()), filter_kernels=filt,
               **{k: dict(median=float(np.median(v)), all=v) for k, v in res.items()}, check=chk)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
