import sys, time, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
from elprep_b200 import synth, device
import bench
contigs = synth.scaled_hg38(20.0)
w = synth.make_workload(15_000_000, contigs, seed=20260924, threads=32)
hb = bench.pinned(w.batch)
ctx = device.Context(w.header, profile=False)
for ci in range(len(contigs)):
    ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], True)
ctx.reserve(hb.n, int(hb.qual.size), int(hb.cigar.size), int(hb.qname.size))
for rep in range(3):
    ctx.reset(); ctx.synchronize()
    t=[time.perf_counter()]
    ctx.append(hb); ctx.synchronize(); t.append(time.perf_counter())
    ctx.sort_markdup(); ctx.synchronize(); t.append(time.perf_counter())
    ctx.bqsr_gather(); ctx.synchronize(); t.append(time.perf_counter())
    ctx.bqsr_finalize(None); ctx.synchronize(); t.append(time.perf_counter())
    ctx.bqsr_apply(); ctx.synchronize(); t.append(time.perf_counter())
    out = ctx.fetch(); t.append(time.perf_counter())
    names=["append","sort_markdup","gather","finalize","apply","fetch(pageable)"]
    print(" | ".join("%s %.1f ms"%(n,1e3*(b-a)) for n,a,b in zip(names,t[:-1],t[1:])), flush=True)
