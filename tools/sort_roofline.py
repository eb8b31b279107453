"""Times the sort machinery at the flagship shapes, per library build, against the HBM roof.

    python tools/sort_roofline.py default [variant ...]

`default` is elprep_b200/lib/libelprep_b200.so, a directory is another source tree as its build() left it (an older
commit, say: its own Python package drives its own library), and any other name is elprep_b200/lib/exp/lib_<name>.so
(variants built with -DRS64_THREADS/-DRS64_ITEMS/-DRS64_MINCTAS, or -DRS_TIMING for the onesweep phase cycles, which go to
stderr).  Each build runs in a child process of its own.  Per build and shape: ms per onesweep pass (median of 5 sorts), GB/s over the
algorithmic 2 * (K + 4) bytes per element and pass, the fraction of 3350 GB/s (the H100 SXM data sheet's HBM3 figure,
not a measured peak), the histogram kernel and one 30 M u32 -> u64 exclusive scan.  Builds without the u32 sort or the
scan entry point skip those lines.  Prints the card's name, power limit and SM clocks first, since every number here
belongs to them.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_GBPS = 3350.0

CHILD = r'''
import json, os, sys
sys.path.insert(0, sys.argv[2])
import numpy as np
from elprep_b200 import device, sam
PEAK = %r
name = sys.argv[1]
ctx = device.Context(sam.Header(sq=[{"SN": "c", "LN": 10}]), profile=True)
rng = np.random.default_rng(1)

def med(xs):
    return float(np.median(np.asarray(xs)))

def sort_shape(kind, n, bits, reps=5):
    dt = np.uint32 if kind == "u32" else np.uint64
    keys = rng.integers(0, 1 << bits, size=n, dtype=np.uint64).astype(dt)
    vals = np.arange(n, dtype=np.uint32)
    per, hist = [], []
    for _ in range(reps):
        ctx.reset_stats()
        k2, v2 = (ctx.debug_sort_u32(keys, vals, bits) if kind == "u32" else ctx.debug_sort_u64(keys, vals, bits))
        st = ctx.kernel_stats()
        o, h = st["radix_onesweep_" + kind], st["radix_hist_" + kind]
        per.append(o["ms"] / o["launches"]); hist.append(h["ms"])
    ok = bool(np.array_equal(v2, np.argsort(keys, kind="stable").astype(np.uint32)))
    kb = 4 if kind == "u32" else 8
    p = med(per)
    gbps = n * 2 * (kb + 4) / p / 1e6
    hms = med(hist)
    return dict(lib=name, shape="%%s keys, %%d M, %%d bits" %% (kind, n // 1_000_000, bits), stable_sorted=ok, passes=o["launches"],
                ms_per_pass=round(p, 4), GBps=round(gbps, 1), frac_of_peak=round(gbps / PEAK, 3),
                hist_ms=round(hms, 4), hist_GBps=round(n * kb / hms / 1e6, 1), sort_ms=round(p * o["launches"] + hms, 3))

print(json.dumps(sort_shape("u64", 30_000_000, 32)), flush=True)
print(json.dumps(sort_shape("u64", 15_000_000, 62)), flush=True)
if hasattr(ctx.L, "elp_debug_sort_u32_range"):
    print(json.dumps(sort_shape("u32", 30_000_000, 32)), flush=True)
if hasattr(ctx.L, "elp_debug_scan_u32"):
    n = 30_000_000
    x = rng.integers(0, 400, size=n, dtype=np.uint32)
    ts = []
    for _ in range(5):
        ctx.reset_stats(); out = ctx.debug_scan_u32(x, 7)
        s = ctx.kernel_stats()["prefix_scan"]; ts.append(s["ms"] / s["launches"])
    ok = bool(out[0] == 7 and np.array_equal(np.diff(out.astype(np.int64)), x.astype(np.int64)))
    t = med(ts)
    print(json.dumps(dict(lib=name, shape="exclusive scan u32 -> u64, 30 M", correct=ok, ms=round(t, 4), GBps=round(n * 12 / t / 1e6, 1),
                          frac_of_peak=round(n * 12 / t / 1e6 / PEAK, 3))), flush=True)
ctx.close()
''' % (PEAK_GBPS,)


def tree_and_lib(name):
    if os.path.isdir(name):
        root = os.path.abspath(name)
        return root, os.path.join(root, "elprep_b200", "lib", "libelprep_b200.so")
    lib = os.path.join(ROOT, "elprep_b200", "lib")
    return ROOT, os.path.join(lib, "libelprep_b200.so") if name == "default" else os.path.join(lib, "exp", f"lib_{name}.so")


def main(names):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    print("card:", q.stdout.strip(), flush=True)
    for name in names or ["default"]:
        root, lib = tree_and_lib(name)
        env = dict(os.environ, ELPREP_B200_LIB=lib)
        subprocess.run([sys.executable, "-c", CHILD, name, root], env=env, check=True)


if __name__ == "__main__":
    main(sys.argv[1:])
