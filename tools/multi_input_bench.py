"""The cost of ingesting several lane files into one context (elp_add_input / elp_select_input / elp_set_tag_rename): the same synthetic
reads as N BGZF lane files, each with its own @SQ order and colliding @RG IDs, against one BGZF file of the same reads with the merged
header.  With several inputs every record goes through the rewrite (relabel_measure, relabel_emit) before bam_ingest_core.  One context
per setting; each rep times the two back to back, each ending in a device synchronise.  Card name and power limit are read in the same run.
usage: python tools/multi_input_bench.py [n_pairs] [lanes] [reps] > multi_input_bench.json"""
import json, os, struct, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from elprep_b200 import bgzf, device, sam, synth
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
n_lanes = int(sys.argv[2]) if len(sys.argv) > 2 else 4
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
except (OSError, ValueError):
    card, power = "?", "?"


def bam_file(h, raw):
    text = b"@HD\tVN:1.6\n"
    hb = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(h.SQ)) + b"".join(
        struct.pack("<i", len(s["SN"]) + 1) + s["SN"].encode() + b"\0" + struct.pack("<i", int(s["LN"])) for s in h.SQ)
    return bgzf.deflate(np.concatenate([np.frombuffer(hb, np.uint8), raw]), level=1, write_eof=True).tobytes()


def to(b, m):
    b.refid[:] = np.where(b.refid >= 0, m[np.maximum(b.refid, 0)], b.refid)
    b.nref[:] = np.where(b.nref >= 0, m[np.maximum(b.nref, 0)], b.nref)


contigs = synth.scaled_hg38(bench.GENOME_SCALE)
w = synth.make_workload(n_pairs, contigs, seed=20260924, threads=32, want_reference=False)
names = w.header.contig_names()
heads = []
for k in range(n_lanes):          # lane k: its own extra contig in front (a different merged index for every name), @RG "1" and "2" in all
    sq = [{"SN": f"lane{k}", "LN": 1000}] + [dict(s) for s in w.header.SQ]
    heads.append(sam.Header(sq=sq, rg=[dict(w.header.RG[j], ID=str(j + 1)) for j in range(len(w.header.RG))]))
merged, sq_maps, rg_map, _ = sam.MergeInputs(heads, "1700000000")
lane = (np.arange(w.batch.n) * n_lanes) // w.batch.n
files, order = [], []
for k in range(n_lanes):
    idx = np.nonzero(lane == k)[0]
    lb = w.batch.take(idx)
    to(lb, np.arange(1, len(names) + 1, dtype=np.int32))
    files.append(bam_file(heads[k], synth.encode_bam(lb, heads[k], threads=32)[0]))
    order.append(idx)
mb = w.batch.take(np.concatenate(order))
to(mb, np.array([merged.contig_names().index(n) for n in names], np.int32))
ids = [r["ID"] for r in merged.RG]
# the RG filters apply to the reads of every lane, the first included: every read's ID becomes its renamed one
mb.rg[:] = np.array([ids.index(rg_map.get(str(j + 1), str(j + 1))) for j in range(len(w.header.RG))], np.int32)[mb.rg]
one = bam_file(merged, synth.encode_bam(mb, merged, threads=32)[0])

h = sam.Header(sq=merged.SQ, rg=merged.RG)
multi, single = device.Context(h), device.Context(h)
for hk in heads:
    multi.add_input([s["SN"] for s in hk.SQ], [int(s["LN"]) for s in hk.SQ])
multi.set_tag_rename("RG", rg_map)


def ingest_multi():
    multi.reset()
    multi.synchronize()
    t0 = time.perf_counter()
    for k, f in enumerate(files):
        multi.select_input(k)
        multi.append_bgzf(f)
        multi.append_bgzf_end()
    multi.synchronize()
    return time.perf_counter() - t0


def ingest_single():
    single.reset()
    single.synchronize()
    t0 = time.perf_counter()
    single.append_bgzf(one)
    single.append_bgzf_end()
    single.synchronize()
    return time.perf_counter() - t0


t = {"lanes": [], "one_file": []}
for _ in range(reps):
    t["lanes"].append(ingest_multi())
    t["one_file"].append(ingest_single())
assert multi.n == single.n == w.batch.n
print(json.dumps({"card": card, "power_limit_w": power, "reads": int(w.batch.n), "lanes": n_lanes,
                  "bytes": sum(len(f) for f in files), "bytes_one_file": len(one),
                  "append_bgzf_lanes_s": min(t["lanes"]), "append_bgzf_one_file_s": min(t["one_file"]), "runs": t}))
