"""The cost of --rename-chromosomes and --replace-reference-sequences on the byte paths (elp_set_input_dictionary): the same sorted,
duplicate-marked synthetic reads ingested with elp_append_bgzf and fetched with elp_fetch_bgzf / elp_fetch_bam / elp_fetch_sam, with the
setting off, with rename (the file's names lack "chr") and with replace (the output dictionary is the input's, reversed).  With the setting
on, bam_keep runs at ingest with the one extra predicate, and the BAM egress patches refID / next_refID in its copy kernel.  Three contexts
hold the reads; each rep times the three modes back to back, each call ending in a device synchronise.  Card name and power limit are read
in the same run.
usage: python tools/reference_dictionary_bench.py [n_pairs] [reps] > reference_dictionary_bench.json"""
import json, os, struct, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from elprep_b200 import _lib, device, sam, synth
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
except (OSError, ValueError):
    card, power = "?", "?"


def bam_header(names, lens):
    text = b"@HD\tVN:1.6\tSO:coordinate\n"
    return b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(names)) + b"".join(
        struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", int(l)) for n, l in zip(names, lens))


contigs = synth.scaled_hg38(bench.GENOME_SCALE)
w = synth.make_workload(n_pairs, contigs, seed=20260924, threads=32, want_reference=False)
raw, off = synth.encode_bam(w.batch, w.header, threads=32)
names, lens = w.header.contig_names(), w.header.contig_lengths()
short = [n[3:] if n.startswith("chr") else n for n in names]
src = device.Context(w.header)                                             # the input file: the reads sorted and duplicate-marked, as BGZF
src.append_bam(raw, off)
src.sort_markdup(device.SO_COORDINATE, True)
files = {"full": src.fetch_bgzf(prefix=bam_header(names, lens)).tobytes(), "short": src.fetch_bgzf(prefix=bam_header(short, lens)).tobytes()}
src.close()
del raw, off

rev = sam.Header(sq=w.header.SQ[::-1], rg=w.header.RG)
modes = {"off": (w.header, 0, None, "full"),
         "rename": (sam.Header(sq=[{"SN": "chr" + s, "LN": l} for s, l in zip(short, lens)], rg=w.header.RG), _lib.DICT_RENAME_CHROMOSOMES, short, "short"),
         "replace": (rev, _lib.DICT_REPLACE, names, "full")}
ctxs = {}
for m, (h, mode, inp, _) in modes.items():
    c = device.Context(h)
    if mode:
        c.set_input_dictionary(mode, inp, lens)
    ctxs[m] = c


def ingest(m):
    c = ctxs[m]
    c.reset()
    f = files[modes[m][3]]
    c.synchronize()
    t0 = time.perf_counter()
    c.append_bgzf(f)
    c.append_bgzf_end()
    c.synchronize()
    return time.perf_counter() - t0


out = dict(card=card, power_limit_w=power, pairs=n_pairs, reps=reps, file_bytes=len(files["full"]), calls={})
ts = {m: [] for m in modes}
for rep in range(reps + 1):                                                # rep 0 warms up
    for m in modes:
        t = ingest(m)
        if rep:
            ts[m].append(t)
out["calls"]["append_bgzf"] = {m: dict(wall_s=min(v), wall_runs=v) for m, v in ts.items()}
print("append_bgzf", {m: min(v) for m, v in ts.items()}, file=sys.stderr, flush=True)
for c in ctxs.values():
    c.sort_markdup(device.SO_COORDINATE, True)
out["reads"] = int(ctxs["off"].n_output())
calls = {"fetch_bgzf": lambda c: c.fetch_bgzf(eof=True), "fetch_bam": lambda c: c.fetch_bam(), "fetch_sam": lambda c: c.fetch_sam()}
for name, f in calls.items():
    ts = {m: [] for m in modes}
    for rep in range(reps + 1):
        for m in modes:
            c = ctxs[m]
            c.synchronize()
            t0 = time.perf_counter()
            f(c)
            c.synchronize()
            if rep:
                ts[m].append(time.perf_counter() - t0)
    out["calls"][name] = {m: dict(wall_s=min(v), wall_runs=v) for m, v in ts.items()}
    print(name, {m: min(v) for m, v in ts.items()}, file=sys.stderr, flush=True)
for c in ctxs.values():
    c.close()
print(json.dumps(out))
