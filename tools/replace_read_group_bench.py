"""The cost of --replace-read-group on the byte outputs (elp_set_replace_read_group): the same sorted, duplicate-marked synthetic reads fetched
with the replacement off and on.  Off, elp_fetch_bam / elp_fetch_bgzf copy the stored records (bam_format); on, they run the field
measure / emit pair that rewrites the RG field (bam_out_fields_measure, bam_out_fields_emit), and elp_fetch_sam writes RG:Z:id in its lines.
Two contexts hold the same reads, one with the setting; each rep times the off call and the on call back to back, each ending in a device
synchronise.  Per-kernel ms come from elp_kernel_stats of one more profiled call per path.  Card name and power limit are read in the same run.
usage: python tools/replace_read_group_bench.py [n_pairs] [reps] > replace_read_group_bench.json"""
import json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from elprep_b200 import device, sam, synth
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
except (OSError, ValueError):
    card, power = "?", "?"

contigs = synth.scaled_hg38(bench.GENOME_SCALE)
w = synth.make_workload(n_pairs, contigs, seed=20260924, threads=32, want_reference=False)
raw, off = synth.encode_bam(w.batch, w.header, threads=32)                # RG:Z of one of four @RG IDs behind NM:C
h = sam.Header(sq=w.header.SQ, rg=[{"ID": "grp", "LB": "lib1", "PU": "unit1"}])
ctxs = {}
for mode in ("off", "on"):
    c = device.Context(h if mode == "on" else w.header)                     # off: the input's own read groups
    if mode == "on":
        c.set_replace_read_group(True)
    c.append_bam(raw, off)
    c.sort_markdup(device.SO_COORDINATE, True)
    ctxs[mode] = c
n = ctxs["off"].n_output()
out = dict(card=card, power_limit_w=power, reads=int(n), reps=reps,
           record_bytes={m: int(c.L.elp_fetch_bam_bytes(c.h, 0, n)) for m, c in ctxs.items()}, calls={})
calls = {"fetch_bgzf": lambda c: c.fetch_bgzf(eof=True), "fetch_bam": lambda c: c.fetch_bam(), "fetch_sam": lambda c: c.fetch_sam()}
for name, f in calls.items():
    ts = {"off": [], "on": []}
    for rep in range(reps + 1):                                            # rep 0 warms up
        for mode in ("off", "on"):
            c = ctxs[mode]
            c.synchronize()
            t0 = time.perf_counter()
            f(c)
            c.synchronize()
            if rep:
                ts[mode].append(time.perf_counter() - t0)
    out["calls"][name] = {m: dict(wall_s=min(v), wall_runs=v) for m, v in ts.items()}
    print(name, {m: min(v) for m, v in ts.items()}, file=sys.stderr, flush=True)
    out["calls"][name]["on_over_off"] = min(ts["on"]) / min(ts["off"])

for mode in ("off", "on"):                                                 # per-kernel times: one profiled call of each kind
    c = device.Context(h if mode == "on" else w.header, profile=True)
    if mode == "on":
        c.set_replace_read_group(True)
    c.append_bam(raw, off)
    c.sort_markdup(device.SO_COORDINATE, True)
    for name, f in calls.items():
        c.reset_stats()
        f(c)
        st = c.kernel_stats()
        out["calls"][name][mode]["kernels"] = {k: dict(ms=v["ms"], launches=v["launches"], GBps=v["alg_bytes"] / v["ms"] / 1e6 if v["ms"] > 0 else None)
                                               for k, v in st.items() if v["ms"] > 0.05}
    c.close()
for c in ctxs.values():
    c.close()
print(json.dumps(out))
