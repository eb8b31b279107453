"""--reference into a context with elp_load_reference, on a seeded hg38-shaped reference (chr1-22, X, Y, M at their real lengths, about
3.1 Gbp of random bases with lower-case and N runs, 60-column lines), written to a temporary directory in three forms:
  ref.fa        FASTA text
  ref.fa.gz     the same text as BGZF (level 6)
  ref.elfasta   the ToElfasta layout
Reports, after a warm-up load of each form: the load's wall time (it ends in a device synchronise), the present path for comparison (the
.elfasta's sequences already in host memory, as fasta.OpenElfasta maps them, then elp_set_reference per contig), reading each file alone
(page cache warm), the per-kernel times of elp_kernel_stats, and the card's name and power limit, read in the same run.
usage: python tools/reference_load_bench.py [scale] [reps] > reference_load_bench.json   (scale < 1 shortens every contig)"""
import json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from elprep_b200 import bgzf, device, sam
from fasta_ref import MAGIC, put_varint
from known_sites_bench import HG38

W = 60
ALPHA = np.frombuffer(b"ACGTACGTACGTACGTACGTacgtN", np.uint8)


def contig(i, ln):
    """contig i's bases, seeded per contig: random ACGT with lower-case runs and a few N runs"""
    rng = np.random.default_rng(1000 + i)
    s = ALPHA[rng.integers(0, 20, size=ln)]
    for a in rng.integers(0, max(1, ln - 5000), size=max(1, ln // 2_000_000)):
        s[a:a + 5000] = ord("N")
    return s


def lines(s):
    """60-column FASTA lines of s, each ended by '\\n'"""
    full = len(s) // W
    m = np.empty((full, W + 1), np.uint8)
    m[:, :W] = s[:full * W].reshape(full, W)
    m[:, W] = 10
    tail = s[full * W:].tobytes()
    return m.tobytes() + (tail + b"\n" if tail else b"")


def write_files(d, contigs):
    paths = {k: os.path.join(d, "ref." + k) for k in ("fa", "fa.gz", "elfasta")}
    table = len(MAGIC) + sum(len(n) + 21 for n, _ in contigs) + 1
    with open(paths["fa"], "wb") as fa, open(paths["fa.gz"], "wb") as gz, open(paths["elfasta"], "wb") as el:
        el.write(MAGIC)
        at = table
        for n, ln in contigs:
            el.write(n.encode() + b"\t" + put_varint(at).ljust(10, b"\0") + put_varint(ln).ljust(10, b"\0"))
            at += ln
        el.write(b"\n")
        for i, (n, ln) in enumerate(contigs):
            s = contig(i, ln)
            text = b">" + n.encode() + b"  AC:XX000000.0  gi|0|ref|rl:Chromosome  as:hg38\n" + lines(s)
            fa.write(text)
            gz.write(bgzf.deflate(text, level=6, n_threads=os.cpu_count() or 8, write_eof=False).tobytes())
            el.write(s.tobytes())
        gz.write(bgzf.deflate(b"", write_eof=True).tobytes())
    return paths


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
        card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    except (OSError, ValueError):
        card, power = "?", "?"
    contigs = [(n, max(1000, int(ln * scale))) for n, ln in HG38]
    hdr = sam.Header(sq=[{"SN": n, "LN": ln} for n, ln in contigs])
    out = dict(card=card, power_limit_w=power, contigs=len(contigs), bases=sum(ln for _, ln in contigs), scale=scale)
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        paths = write_files(d, contigs)
        out["generate_s"] = round(time.perf_counter() - t0, 1)
        print(f"generated in {out['generate_s']} s", file=sys.stderr, flush=True)
        out["file_bytes"] = {k: os.path.getsize(p) for k, p in paths.items()}
        ctx = device.Context(hdr)
        try:
            for form, p in paths.items():
                rd = []
                buf = np.empty(os.path.getsize(p), np.uint8)
                for _ in range(reps):
                    t0 = time.perf_counter()
                    with open(p, "rb", buffering=0) as f:
                        f.readinto(memoryview(buf))
                    rd.append(time.perf_counter() - t0)
                del buf
                assert ctx.load_reference(p) == (0, 0)          # warm-up
                wall = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    ctx.load_reference(p)
                    ctx.synchronize()
                    wall.append(time.perf_counter() - t0)
                out[form] = dict(load_s=min(wall), load_all_s=wall, file_read_s=min(rd), bases_per_s=out["bases"] / min(wall))
                print(form, out[form], file=sys.stderr, flush=True)
            # the present path: the .elfasta's sequences in host memory (mapped, page cache warm), then elp_set_reference per contig
            m = np.memmap(paths["elfasta"], dtype=np.uint8, mode="r")
            table = len(MAGIC) + sum(len(n) + 21 for n, _ in contigs) + 1
            offs = np.cumsum([table] + [ln for _, ln in contigs])
            nib0 = ctx.reference(0)[1]
            wall = []
            for _ in range(reps):
                t0 = time.perf_counter()
                for ci in range(len(contigs)):
                    ctx.set_reference(ci, m[offs[ci]:offs[ci + 1]])
                ctx.synchronize()
                wall.append(time.perf_counter() - t0)
            assert np.array_equal(ctx.reference(0)[1], nib0)
            out["set_reference_per_contig"] = dict(load_s=min(wall), load_all_s=wall)
            del m
        finally:
            ctx.close()
        stats = {}
        for form, p in paths.items():
            ctx = device.Context(hdr, profile=True)
            try:
                ctx.load_reference(p)
                ctx.reset_stats()
                ctx.load_reference(p)
                stats[form] = {k: dict(launches=v["launches"], ms=round(v["ms"], 3)) for k, v in ctx.kernel_stats().items()}
            finally:
                ctx.close()
        out["kernels"] = stats
    print(json.dumps(out))


if __name__ == "__main__":
    main()
