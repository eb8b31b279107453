"""times the gather phase with each ablation variant of the library (one process per variant)"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
child = r'''
import sys, time, os
sys.path.insert(0, %r)
import numpy as np
from elprep_b200 import synth, device
import bench
contigs = synth.scaled_hg38(20.0)
w = synth.make_workload(15_000_000, contigs, seed=20260924, threads=32)
hb = bench.pinned(w.batch)
ctx = device.Context(w.header, profile=True)
for ci in range(len(contigs)):
    ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], True)
for rep in range(3):
    ctx.reset(); ctx.append(hb); ctx.reset_stats(); ctx.sort_markdup(); ctx.bqsr_gather(); ctx.bqsr_finalize(None); ctx.bqsr_apply(); ctx.synchronize()
st = ctx.kernel_stats()
print(os.environ.get("ELPREP_B200_LIB","default").split("/")[-1], "  ".join("%%s %%.2f" %% (k, st[k]["ms"]) for k in ("bqsr_gather", "bqsr_gather_indel", "bqsr_gather_general", "bqsr_gen_list", "bqsr_prep", "bqsr_apply", "bqsr_apply_gmem", "adapt") if k in st), flush=True)
''' % ROOT
for name in sys.argv[1:]:
    env = dict(os.environ)
    env["ELPREP_B200_LIB"] = os.path.join(ROOT, "elprep_b200", "lib", "libelprep_b200.so" if name == "default" else os.path.join("exp", f"lib_{name}.so"))
    subprocess.run([sys.executable, "-c", child], env=env)
