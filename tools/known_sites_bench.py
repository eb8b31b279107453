"""--known-sites files into a context with elp_load_known_sites, on seeded dbSNP-shaped data:
  dbsnp.elsites   the hg38 primary contigs (chr1-22, X, Y, M at their real lengths), one site per ~50 bp, sorted, mostly SNPs (end == start)
  mills.elsites   one indel per ~2 kb, end = start + 1..50
Reports, after a warm-up load: the load's wall time (ends in a device synchronise), the file read alone (the same files read into host
memory), a page-locked H2D copy of the same bytes timed with CUDA events, the per-kernel times of elp_kernel_stats with their algorithmic
bytes over kernel time, and the card's name and power limit, read in the same run.  The files go to a temporary directory.
usage: python tools/known_sites_bench.py [bp_per_site] [reps] > known_sites_bench.json"""
import json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from elprep_b200 import device, sam

HG38 = [("chr1", 248956422), ("chr2", 242193529), ("chr3", 198295559), ("chr4", 190214555), ("chr5", 181538259), ("chr6", 170805979),
        ("chr7", 159345973), ("chr8", 145138636), ("chr9", 138394717), ("chr10", 133797422), ("chr11", 135086622), ("chr12", 133275309),
        ("chr13", 114364328), ("chr14", 107043718), ("chr15", 101991189), ("chr16", 90338345), ("chr17", 83257441), ("chr18", 80373285),
        ("chr19", 58617616), ("chr20", 64444167), ("chr21", 46709983), ("chr22", 50818468), ("chrX", 156040895), ("chrY", 57227415),
        ("chrM", 16569)]
HEADER = b"# elsites format version 1.0\n"


def _digits(v):
    """non-negative int64 -> (ascii digits right-aligned in 10 columns, digit counts)"""
    d = np.empty((len(v), 10), np.uint8)
    x = v.copy()
    for k in range(9, -1, -1):
        d[:, k] = (x % 10 + 48).astype(np.uint8)
        x //= 10
    n = np.ones(len(v), np.int64)
    for p in range(1, 10):
        n += v >= 10 ** p
    return d, n


def format_lines(name, s, e):
    """"name\\tstart\\tend\\n" for every row, vectorised"""
    nb = np.frombuffer(name.encode(), np.uint8)
    ds, ns = _digits(s)
    de, ne = _digits(e)
    L = len(nb)
    m = np.empty((len(s), L + 23), np.uint8)
    m[:, :L] = nb; m[:, L] = 9; m[:, L + 1:L + 11] = ds; m[:, L + 11] = 9; m[:, L + 12:L + 22] = de; m[:, L + 22] = 10
    keep = np.ones_like(m, dtype=bool)
    col = np.arange(10)
    keep[:, L + 1:L + 11] = col[None, :] >= 10 - ns[:, None]
    keep[:, L + 12:L + 22] = col[None, :] >= 10 - ne[:, None]
    return m[keep].tobytes()


def write_files(d, bp_per_site, seed=20261017):
    rng = np.random.default_rng(seed)
    paths, lines = [], 0
    for fname, per, indel in (("dbsnp.elsites", bp_per_site, False), ("mills.elsites", 2000, True)):
        p = os.path.join(d, fname)
        with open(p, "wb") as f:
            f.write(HEADER)
            for name, ln in HG38:
                k = max(1, ln // per)
                s = np.sort(rng.integers(1, ln, size=k)).astype(np.int64)
                e = s + (rng.integers(1, 51, size=k) if indel else (rng.random(k) < 0.08) * rng.integers(1, 6, size=k))
                f.write(format_lines(name, s, e))
                lines += k
        paths.append(p)
    return paths, lines


def main():
    bp = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
        card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    except (OSError, ValueError):
        card, power = "?", "?"
    hdr = sam.Header(sq=[{"SN": n, "LN": ln} for n, ln in HG38])
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        paths, lines = write_files(d, bp)
        gen_s = time.perf_counter() - t0
        nbytes = sum(os.path.getsize(p) for p in paths)
        out = dict(card=card, power_limit_w=power, lines=lines, file_bytes=nbytes, bp_per_site=bp, generate_s=round(gen_s, 2))
        # file read alone (page cache warm, as for the load that follows)
        buf = np.empty(max(os.path.getsize(p) for p in paths), np.uint8)
        rd = []
        for _ in range(reps):
            t0 = time.perf_counter()
            for p in paths:
                with open(p, "rb", buffering=0) as f:
                    f.readinto(memoryview(buf)[:os.path.getsize(p)])
            rd.append(time.perf_counter() - t0)
        out["file_read_s"] = min(rd)
        # page-locked H2D copy of the same bytes
        h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        g = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g.copy_(h, non_blocking=True); torch.cuda.synchronize()
        h2d = []
        for _ in range(reps):
            a.record(); g.copy_(h, non_blocking=True); b.record(); b.synchronize()
            h2d.append(a.elapsed_time(b) / 1e3)
        out["h2d_pinned_s"] = min(h2d); out["h2d_pinned_GBps"] = nbytes / min(h2d) / 1e9
        del g, h
        torch.cuda.empty_cache()
        # the load: wall time without profiling, then one profiled run for the kernel split
        ctx = device.Context(hdr)
        nu = ctx.load_known_sites(paths)      # warm-up (staging allocation, module load)
        wall = []
        for _ in range(reps):
            t0 = time.perf_counter()
            ctx.load_known_sites(paths)
            ctx.synchronize()
            wall.append(time.perf_counter() - t0)
        n_sites = sum(len(ctx.known_sites(i)) for i in range(len(HG38)))
        ctx.close()
        out.update(load_s=min(wall), load_all_s=wall, unmatched=nu, flattened_sites=n_sites, load_GBps=nbytes / min(wall) / 1e9)
        ctx = device.Context(hdr, profile=True)
        ctx.load_known_sites(paths)
        ctx.reset_stats()
        t0 = time.perf_counter()
        ctx.load_known_sites(paths)
        out["load_profiled_s"] = time.perf_counter() - t0
        st = ctx.kernel_stats()
        ctx.close()
    kern = {k: dict(launches=v["launches"], ms=round(v["ms"], 3), GBps=round(v["alg_bytes"] / v["ms"] / 1e6, 1) if v["ms"] > 0 else None)
            for k, v in st.items() if k.startswith("sites_") or k == "prefix_scan" or k.startswith("radix_")}
    out["kernels"] = kern
    own = [k for k in kern if k.startswith("sites_")]
    out["kernel_ms_sites"] = round(sum(kern[k]["ms"] for k in own), 3)   # sites_sort spans the radix_*_sites launches: counted once
    out["split"] = dict(file_read_s=out["file_read_s"], upload_s_if_alone=out["h2d_pinned_s"], kernels_s=out["kernel_ms_sites"] / 1e3, load_s=out["load_s"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
