"""Runs one several-rank scenario through the library's collective path on ONE GPU, over the in-process NCCL stand-in
(tests/c/nccl_loopback.cpp): one thread and one device.Context per rank, all on the same device.

    LD_LIBRARY_PATH=<dir of the stand-in's libnccl.so.2> python tests/comm_loopback.py SCENARIO.pkl OUT.npz

It must not import torch, which would load the real libnccl.so.2 first; it asserts that the NCCL the library loaded is the stand-in.
The scenario (a pickled dict, see tests/test_gpu_comm_loopback.py) holds the header, the whole input, the side inputs, the contig ->
rank table and the world size.  The driver runs the whole input through one context, then every rank's share through the phases of
tools/multigpu_check.py: comm_init, comm_set_partition, append, sort_markdup(ELP_MARKDUP_OPTICAL), gather, tables_allreduce,
finalize, apply, optical_allreduce, fetch.  It writes the per-read results of both runs to OUT.npz and prints one JSON line: per rank
the return code, error text and time of sort_markdup and the kernels it ran, the equality of FLAG, QUAL, tables, metrics and metrics
file text with the one-context run, and the stand-in's counters."""
import json
import os
import pickle
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elprep_b200 import _lib, device, multi  # noqa: E402

CMDLINE, STARTED = "elprep filter in out", "T"


def qual_in_arrival_order(whole_qoff, read_idx, qoff, qual):
    """QUAL bytes fetched in output order (record k is read read_idx[k]) -> one arena in the input's arrival-order layout"""
    out = np.zeros(int(whole_qoff[-1]), np.uint8)
    lens = (qoff[1:] - qoff[:-1]).astype(np.int64)
    dst = np.repeat(whole_qoff[read_idx].astype(np.int64) - qoff[:-1].astype(np.int64), lens) + np.arange(int(qoff[-1]), dtype=np.int64)
    out[dst] = qual[:int(qoff[-1])]
    return out


def same_metrics(a, b):
    """(percent_duplication is NaN in a slot without reads, and NaN != NaN)"""
    return json.dumps(a, sort_keys=True) == json.dumps(b, sort_keys=True)


def setup(ctx, sc):
    if sc["bqsr"]:
        for ci in range(len(sc["header"].SQ)):
            ctx.set_reference(ci, sc["contig_bases"][ci])
            ctx.set_known_sites(ci, sc["sites"][ci], already_flat=True)


def after_markdup(ctx, sc, whole, reads, allreduce):
    """the phases after sort_markdup; -> dict of results by input read (reads: the input index of every read of ctx)"""
    res = {}
    if sc["bqsr"]:
        ctx.bqsr_gather()
        if allreduce:
            ctx.tables_allreduce()
        res["tables"] = ctx.tables_get()
        ctx.bqsr_finalize(None)
        ctx.bqsr_apply()
    if allreduce:
        ctx.optical_allreduce()
    res["metrics"] = ctx.optical_metrics()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.txt")
        ctx.print_duplicates_metrics(p, CMDLINE, STARTED)
        res["metrics_text"] = open(p).read()
    idx, flag, qoff, qual = ctx.fetch()
    gidx = reads[idx.astype(np.int64)]
    res["gidx"], res["flag"] = gidx, flag
    if sc["bqsr"]:
        res["qual"] = qual_in_arrival_order(whole.qual_off, gidx, qoff, qual)
    return res


def run_whole(sc):
    whole = sc["batch"]
    ctx = device.Context(sc["header"], optical_pixel_distance=sc["pixel"], profile=True)
    try:
        setup(ctx, sc)
        ctx.append(whole)
        try:
            ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
        except device.ElprepError as e:
            return {"rc": e.code, "err": str(e)}
        res = after_markdup(ctx, sc, whole, np.arange(whole.n, dtype=np.int64), allreduce=False)
        res["rc"], res["err"] = 0, ""
        res["kernels"] = {k: v["launches"] for k, v in ctx.kernel_stats().items()}
        return res
    finally:
        ctx.close()


def run_rank(sc, uid, rank, parts, out):
    whole, world = sc["batch"], sc["world"]
    reads = parts[rank]
    r = out[rank] = {"rank": rank, "reads": int(reads.size)}
    ctx = device.Context(sc["header"], optical_pixel_distance=sc["pixel"], profile=True)
    try:
        setup(ctx, sc)
        ctx.comm_init(uid, rank, world)
        ctx.comm_set_partition(sc["owner"])
        mine = whole.take(reads)
        if reads.size:
            ctx.append(mine)
        for attempt in range(2 if sc.get("rerun") else 1):
            if attempt:                                   # a second run on the same communicator after elp_reset
                r["first"] = {k: r[k] for k in ("flag", "gidx")}
                ctx.reset()
                if reads.size:
                    ctx.append(mine)
            t0 = time.monotonic()
            try:
                ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
                r["rc"], r["err"] = 0, ""
            except device.ElprepError as e:
                r["rc"], r["err"] = e.code, str(e)
            r["seconds"] = time.monotonic() - t0
            r["kernels"] = {k: v["launches"] for k, v in ctx.kernel_stats().items()}
            ctx.reset_stats()
            if r["rc"]:
                # the refused call left the context unsorted: read the FLAG column back in arrival order (a read the sort itself
                # refuses, such as a negative POS, makes that impossible: the refusal is recorded instead)
                try:
                    ctx.sort_markdup(device.SO_KEEP, 0)
                    idx, flag, _, _ = ctx.fetch(want_qual=False)
                    r["flag_after_failure"] = flag[np.argsort(idx)] if reads.size else flag
                    r["flag_in"] = mine.flag.copy()
                except device.ElprepError as e:
                    r["readback_error"] = str(e)
                return
            r.update(after_markdup(ctx, sc, whole, reads, allreduce=True))
    except Exception as e:                               # any other failure of this rank is reported, not raised in the thread
        r.setdefault("rc", 0)
        r["exception"] = f"{type(e).__name__}: {e}"
    finally:
        ctx.close()


def loaded_nccl():
    """paths of every libnccl mapped into this process"""
    with open("/proc/self/maps") as f:
        return sorted({ln.split()[-1] for ln in f if "libnccl" in ln})


def main(scenario_path, out_path):
    with open(scenario_path, "rb") as f:
        sc = pickle.load(f)
    sc.setdefault("bqsr", True)
    sc.setdefault("pixel", 100)
    whole, world = sc["batch"], sc["world"]
    assert "torch" not in sys.modules
    one = run_whole(sc)
    parts = sc.get("parts")
    if parts is None:
        parts = [multi.partition(whole, sc["owner"], r, world) for r in range(world)]
    parts = [np.asarray(p, np.int64) for p in parts]
    uid = device.Context.comm_unique_id()
    out = [None] * world
    th = [threading.Thread(target=run_rank, args=(sc, uid, r, parts, out)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    import ctypes
    stand_in = ctypes.CDLL("libnccl.so.2")                # the copy already loaded (same SONAME)
    assert hasattr(stand_in, "loopback_stats"), "the library loaded a real libnccl.so.2, not the stand-in"
    stand_in.loopback_stats.restype = ctypes.c_char_p
    stats = json.loads(stand_in.loopback_stats().decode())
    nccl_paths = loaded_nccl()

    arrays = {"one_rc": one["rc"]}
    summary = {"world": world, "one": {"rc": one["rc"], "err": one["err"], "kernels": one.get("kernels")}, "ranks": [], "stats": stats, "nccl": nccl_paths}
    ok = all(r["rc"] == 0 and "exception" not in r for r in out) and one["rc"] == 0
    if ok:
        flag = np.zeros(whole.n, np.uint16)
        seen = np.zeros(whole.n, np.int64)
        qual = np.zeros(int(whole.qual_off[-1]), np.uint8)
        for r in out:
            flag[r["gidx"]] = r["flag"]
            seen[r["gidx"]] += 1
            if sc["bqsr"]:
                qual |= r["qual"]                         # (zero outside the rank's reads, and the ranks' reads are disjoint)
        one_flag = np.zeros(whole.n, np.uint16)
        one_flag[one["gidx"]] = one["flag"]
        arrays.update(flag=flag, one_flag=one_flag)
        eq = {"every_read_once": bool((seen == 1).all()), "flag": bool(np.array_equal(flag, one_flag)),
              "metrics": all(same_metrics(r["metrics"], one["metrics"]) for r in out), "metrics_text": all(r["metrics_text"] == one["metrics_text"] for r in out)}
        if sc["bqsr"]:
            arrays.update(qual=qual, one_qual=one["qual"], tables=out[0]["tables"], one_tables=one["tables"])
            eq["qual"] = bool(np.array_equal(qual, one["qual"]))
            eq["tables"] = all(np.array_equal(r["tables"], one["tables"]) for r in out)
        if sc.get("rerun"):
            eq["rerun_flag"] = all(np.array_equal(r["first"]["flag"], r["flag"]) and np.array_equal(r["first"]["gidx"], r["gidx"]) for r in out)
        summary["equal"] = eq
        summary["metrics"] = out[0]["metrics"]
        arrays["metrics_text"] = np.frombuffer(out[0]["metrics_text"].encode(), np.uint8)
    for r in out:
        summary["ranks"].append({k: r.get(k) for k in ("rank", "reads", "rc", "err", "seconds", "kernels", "exception", "readback_error")})
        if "flag_after_failure" in r:
            summary["ranks"][-1]["flag_untouched"] = bool(np.array_equal(r["flag_after_failure"], r["flag_in"]))
    np.savez(out_path, **arrays)
    print(json.dumps(summary, default=lambda x: x.tolist() if hasattr(x, "tolist") else str(x)))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
