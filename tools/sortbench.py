"""times the u64 onesweep radix sort (30 M keys, 34 significant bits, u32 payload) for each library variant"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
child = r'''
import sys, os
sys.path.insert(0, %r)
import numpy as np
from elprep_b200 import device, sam
n = int(os.environ.get("SORT_N", 30_000_000)); bits = int(os.environ.get("SORT_BITS", 34))
rng = np.random.default_rng(1)
keys = rng.integers(0, 1 << bits, size=n, dtype=np.uint64); vals = np.arange(n, dtype=np.uint32)
mode = os.environ.get("SORT_MODE", "random")
if mode == "sorted": keys.sort()
if mode == "const": keys[:] = 12345
if mode == "few": keys = (keys & np.uint64(0x0303030303))          # 4 distinct digits per pass: long write runs
ctx = device.Context(sam.Header(sq=[{"SN": "c", "LN": 10}]), profile=True)
for rep in range(3):
    ctx.reset_stats(); k2, v2 = ctx.debug_sort_u64(keys, vals, bits)
st = ctx.kernel_stats()
ok = bool((np.diff(k2.astype(np.int64)) >= 0).all())
o = st["radix_onesweep_u64"]; h = st["radix_hist_u64"]
per = o["ms"] / o["launches"]
print("%%-28s sorted=%%s passes=%%d  %%.3f ms/pass = %%.0f GB/s (%%.1f%%%% of the 3350 GB/s H100 SXM data sheet)  hist %%.3f ms  total %%.2f ms -> %%.1f Gkeys/s" %% (
    os.environ.get("ELPREP_B200_LIB", "default").split("/")[-1] + ":" + mode, ok, o["launches"], per, n * 24 / per / 1e6, 100 * n * 24 / per / 1e6 / 3350.0, h["ms"], o["ms"] + h["ms"], n / (o["ms"] + h["ms"]) / 1e6), flush=True)
''' % ROOT
for name in sys.argv[1:]:
    env = dict(os.environ)
    env["ELPREP_B200_LIB"] = os.path.join(ROOT, "elprep_b200", "lib", "libelprep_b200.so" if name == "default" else os.path.join("exp", f"lib_{name}.so"))
    subprocess.run([sys.executable, "-c", child], env=env)
