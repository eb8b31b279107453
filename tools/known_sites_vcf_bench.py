"""--known-sites VCF files into a context with elp_load_known_sites, on a seeded dbSNP-shaped VCF:
  the hg38 primary contigs (chr1-22, X, Y, M at their real lengths), one site per bp_per_site bp, sorted; rs IDs, dbSNP-style INFO of
  ~100 bytes; 90% SNVs, the rest indels with REF of 2..40 bases
written as plain text and as BGZF (level 1), plus the .elsites of the same sites.  Reports, after a warm-up load of each: the load's wall
time (ends in a device synchronise), the file read alone (the same file read into host memory), the per-kernel times of
elp_kernel_stats with their algorithmic bytes over kernel time, the .elsites load of the same sites, and the card's name and power limit,
read in the same run.  The files go to a temporary directory.
usage: python tools/known_sites_vcf_bench.py [bp_per_site] [reps] > known_sites_vcf_bench.json"""
import json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
from elprep_b200 import bgzf, device, sam
from known_sites_bench import HG38, HEADER, format_lines


def write_vcf(d, bp_per_site, seed=20261018):
    rng = np.random.default_rng(seed)
    head = (b"##fileformat=VCFv4.2\n##source=dbSNP\n##dbSNP_BUILD_ID=154\n##reference=GRCh38.p12\n"
            b"##INFO=<ID=RS,Number=1,Type=Integer,Description=\"dbSNP ID (i.e. rs number)\">\n"
            b"##INFO=<ID=dbSNPBuildID,Number=1,Type=Integer,Description=\"First dbSNP Build for RS\">\n"
            b"##INFO=<ID=VC,Number=1,Type=String,Description=\"Variation Class\">\n"
            b"##INFO=<ID=COMMON,Number=0,Type=Flag,Description=\"common\">\n"
            + b"".join(b"##contig=<ID=%s,length=%d>\n" % (n.encode(), ln) for n, ln in HG38)
            + b"#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
    parts, sites, lines = [head], [], 0
    for name, ln in HG38:
        k = max(1, ln // bp_per_site)
        pos = np.sort(rng.integers(1, ln, size=k))
        rl = np.where(rng.random(k) < 0.9, 1, rng.integers(2, 41, size=k))
        rs = rng.integers(1, 1_500_000_000, size=k)
        fr = rng.integers(1, 999, size=k)
        nb = name.encode()
        parts.append(b"".join(
            b"%s\t%d\trs%d\t%s\t%s\t.\t.\tRS=%d;dbSNPBuildID=154;SSR=0;VC=%s;GENEINFO=GENE:%d;FREQ=1000Genomes:0.%03d,0.%03d|GnomAD:0.%03d\n"
            % (nb, p, i, b"A" * r, b"G" if r == 1 else b"A", i, b"SNV" if r == 1 else b"DEL", i % 100000, f, 1000 - f, f)
            for p, r, i, f in zip(pos.tolist(), rl.tolist(), rs.tolist(), fr.tolist())))
        sites.append((name, pos, pos - 1 + rl))
        lines += k
    text = b"".join(parts)
    p_vcf, p_gz, p_el = os.path.join(d, "dbsnp.vcf"), os.path.join(d, "dbsnp.vcf.gz"), os.path.join(d, "dbsnp.elsites")
    with open(p_vcf, "wb") as f:
        f.write(text)
    with open(p_gz, "wb") as f:
        f.write(bgzf.deflate(text, level=1).tobytes())
    with open(p_el, "wb") as f:
        f.write(HEADER)
        for name, s, e in sites:
            f.write(format_lines(name, s, e))
    return dict(vcf=p_vcf, vcf_gz=p_gz, elsites=p_el), lines


def read_s(p, reps):
    n = os.path.getsize(p)
    buf = np.empty(n, np.uint8)
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        with open(p, "rb", buffering=0) as f:
            f.readinto(memoryview(buf))
        t.append(time.perf_counter() - t0)
    return min(t)


def main():
    bp = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
        card, power = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    except (OSError, ValueError):
        card, power = "?", "?"
    hdr = sam.Header(sq=[{"SN": n, "LN": ln} for n, ln in HG38])
    out = dict(card=card, power_limit_w=power, bp_per_site=bp)
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        paths, lines = write_vcf(d, bp)
        out.update(lines=lines, generate_s=round(time.perf_counter() - t0, 2))
        for tag, p in paths.items():
            nbytes = os.path.getsize(p)
            r = dict(file_bytes=nbytes, file_read_s=read_s(p, reps))
            ctx = device.Context(hdr)
            ctx.load_known_sites([p])           # warm-up (staging allocation, module load)
            wall = []
            for _ in range(reps):
                t0 = time.perf_counter()
                ctx.load_known_sites([p])
                ctx.synchronize()
                wall.append(time.perf_counter() - t0)
            r["flattened_sites"] = sum(len(ctx.known_sites(i)) for i in range(len(HG38)))
            ctx.close()
            r.update(load_s=min(wall), load_all_s=wall, load_GBps=nbytes / min(wall) / 1e9)
            ctx = device.Context(hdr, profile=True)
            ctx.load_known_sites([p])
            ctx.reset_stats()
            ctx.load_known_sites([p])
            st = ctx.kernel_stats()
            ctx.close()
            r["kernels"] = {k: dict(launches=v["launches"], ms=round(v["ms"], 3), GBps=round(v["alg_bytes"] / v["ms"] / 1e6, 1) if v["ms"] > 0 else None)
                            for k, v in st.items() if k.startswith(("sites_", "vcf_", "bgzf_", "radix_")) or k == "prefix_scan"}
            out[tag] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
