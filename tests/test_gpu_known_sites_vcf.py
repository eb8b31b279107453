"""elp_load_known_sites on VCF files: plain and BGZF VCF parsed on the device into the known-sites table, against the restatement of
ParseHeader / ParseVariant / FromVcfFile (vcf_ref), at staging-chunk sizes that put lines, the header's end and BGZF block edges on chunk
edges."""
import numpy as np
import pytest

import elsites_ref as er
import vcf_cases as vc
import vcf_ref as vr
from elprep_b200 import _lib, bgzf, device, sam, synth
from util import gpu_phases

pytestmark = pytest.mark.gpu

CHUNKS = [1, 7, 64, 0]   # 0: the default

REASON_TEXT = {vr.LONG: "65536 bytes or more", vr.TAB: "missing tabulator", vr.POS: "POS: strconv.ParseInt", vr.QUAL: "(syntax)",
               vr.QUAL_RANGE: "(value out of range)", vr.INFO: "INFO: a declared key", vr.END: "END key", vr.CHROM: "empty CHROM", vr.HEADER: ""}


def _header(names, ln=1 << 30):
    return sam.Header(sq=[{"SN": n, "LN": ln} for n in names])


def _write(tmp_path, files, tag):
    paths = []
    for i, data in enumerate(files):
        p = tmp_path / f"{tag}{i}.vcf"
        p.write_bytes(data)
        paths.append(str(p))
    return paths


def _tables(ctx, n):
    return [ctx.known_sites(ci) for ci in range(n)]


def _assert_tables(got, want):
    assert len(got) == len(want)
    for ci, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), (ci, g[:8].tolist(), w[:8].tolist(), len(g), len(w))


def _forms(files):
    """the files as given, and (when every file is plain VCF text) as BGZF with 17-byte blocks, so blocks end inside lines and inside
    the header"""
    out = [("plain", files)]
    if all(d.startswith(vr.PREFIX) for d in files):
        out.append(("bgzf", [vr.bgzf(d, block=17) for d in files]))
    return out


@pytest.mark.parametrize("chunk", CHUNKS)
def test_known_answers(tmp_path, chunk):
    ctx = device.Context(_header(vc.NAMES))
    try:
        ctx.debug_set_sites_chunk(chunk)
        for cid, files, _, _ in vc.VALID:
            if chunk == 1 and cid == "line_65535":
                continue   # 64 KiB one byte at a time: covered at 7 bytes
            want, wu = vr.load(files, vc.NAMES)
            for form, fs in _forms(files):
                nu = ctx.load_known_sites(_write(tmp_path, fs, f"{cid}_{form}"))
                assert nu == wu, (cid, form)
                _assert_tables(_tables(ctx, len(vc.NAMES)), want)
    finally:
        ctx.close()


@pytest.mark.parametrize("chunk", [7, 0])
def test_refusals(tmp_path, chunk):
    """every malformed form is ELP_EVCF naming the file and the 1-based line; the previous table stays"""
    ctx = device.Context(_header(vc.NAMES))
    try:
        ctx.debug_set_sites_chunk(chunk)
        ctx.load_known_sites(_write(tmp_path, vc.VALID[1][1], "good"))
        before = _tables(ctx, len(vc.NAMES))
        for cid, files, (fi, line, reason) in vc.INVALID:
            for form, fs in _forms(files):
                with pytest.raises(device.ElprepError) as ei:
                    ctx.load_known_sites(_write(tmp_path, fs, f"{cid}_{form}"))
                msg = str(ei.value)
                assert ei.value.code == _lib.EVCF, (cid, form, msg)
                assert f"(file {fi}), line {line} " in msg and REASON_TEXT[reason] in msg, (cid, form, msg)
                _assert_tables(_tables(ctx, len(vc.NAMES)), before)
    finally:
        ctx.close()


def test_bgzf_violations(tmp_path):
    """a plain gzip file, a truncated BGZF file and one without the EOF marker are ELP_EBGZF; the table stays"""
    import gzip
    text = vc.H + vc.row() + b"\n"
    ctx = device.Context(_header(vc.NAMES))
    try:
        ctx.load_known_sites(_write(tmp_path, [text], "ok"))
        before = _tables(ctx, len(vc.NAMES))
        z = vr.bgzf(text, block=40)
        for tag, data in [("gzip", gzip.compress(text)), ("truncated", z[:-40]), ("no_eof", z[:-28]), ("header_cut", vr.bgzf(text, block=40)[:30])]:
            with pytest.raises(device.ElprepError) as ei:
                ctx.load_known_sites(_write(tmp_path, [data], tag))
            assert ei.value.code == _lib.EBGZF, (tag, str(ei.value))
            _assert_tables(_tables(ctx, len(vc.NAMES)), before)
    finally:
        ctx.close()


# ---- a seeded dbSNP-shaped file ----
RANDOM_NAMES = [f"chr{i}" for i in range(1, 23)] + ["chrX", "chrY", "chrM", "dupA", "dupA"]
EXTRA = ["chrUn_gl000220", "chr1_KI270706v1_random"]   # not @SQ SN: unmatched


def dbsnp_like(seed, n_lines):
    """VCF text shaped like dbSNP: sorted per contig, rs IDs, SNVs and indels, long INFO; some CRLF lines, some QUAL values, some
    declared INFO flags -> (text, [(chrom, start, end)] arrays)"""
    rng = np.random.default_rng(seed)
    names = sorted(set(RANDOM_NAMES)) + EXTRA
    w = rng.random(len(names)) + 0.2
    cnt = rng.multinomial(n_lines, w / w.sum())
    head = (b"##fileformat=VCFv4.2\n##source=dbSNP\n##INFO=<ID=RS,Number=1,Type=Integer,Description=\"dbSNP ID\">\n"
            b"##INFO=<ID=COMMON,Number=0,Type=Flag,Description=\"common\">\n##INFO=<ID=VC,Number=1,Type=String,Description=\"class\">\n"
            + b"".join(b"##contig=<ID=%s>\n" % n.encode() for n in names) + b"#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
    out, chrom, st, en = [head], [], [], []
    for name, k in zip(names, cnt):
        pos = np.sort(rng.integers(1, 250_000_000, size=k))
        rl = np.where(rng.random(k) < 0.9, 1, rng.integers(2, 40, size=k))
        rs = rng.integers(1, 2_000_000_000, size=k)
        qual = rng.random(k)
        nb = name.encode()
        for p, r, i, q in zip(pos.tolist(), rl.tolist(), rs.tolist(), qual.tolist()):
            info = (b"RS=%d;dbSNPBuildID=154;SSR=0;VC=%s;GENEINFO=ABC1:123;FREQ=1000Genomes:0.99,0.01|GnomAD:0.98,0.02" % (i, b"SNV" if r == 1 else b"INDEL")
                    if q > 0.02 else b"COMMON")
            out.append(b"%s\t%d\trs%d\t%s\tG\t%s\t%s\t%s%s" % (nb, p, i, b"A" * r, b"." if q < 0.9 else b"%.2f" % (q * 100), b"." if q < 0.5 else b"PASS",
                                                              info, b"\r\n" if q < 0.01 else b"\n"))
        chrom.append(np.full(k, names.index(name)))
        st.append(pos)
        en.append(pos - 1 + rl)
    return b"".join(out), names, np.concatenate(chrom), np.concatenate(st), np.concatenate(en)


def _expect(names, chrom, st, en, ctx_names):
    tabs = []
    for n in ctx_names:
        i = names.index(n)
        m = chrom == i
        tabs.append(er.sort_flatten_fast(np.stack([st[m], en[m]], axis=1)))
    unmatched = int(sum((chrom == names.index(n)).sum() for n in EXTRA))
    return tabs, unmatched


def test_random_dbsnp_like(tmp_path):
    text, names, chrom, st, en = dbsnp_like(20261018, 2_000_000)
    want, wu = _expect(names, chrom, st, en, RANDOM_NAMES)
    plain = tmp_path / "dbsnp.vcf"; plain.write_bytes(text)
    gz = tmp_path / "dbsnp.vcf.gz"; gz.write_bytes(bgzf.deflate(text, level=1).tobytes())
    ctx = device.Context(_header(RANDOM_NAMES))
    try:
        for chunk, p in [(0, plain), (0, gz), (1 << 20, plain), ((1 << 20) + 13, gz)]:
            ctx.debug_set_sites_chunk(chunk)
            assert ctx.load_known_sites([str(p)]) == wu, (chunk, p)
            _assert_tables(_tables(ctx, len(RANDOM_NAMES)), want)
    finally:
        ctx.close()


def test_bqsr_same_as_elsites(tmp_path):
    """one gather + finalize + apply: the tables, the report and QUAL are identical whether the known sites come from a VCF or from
    the .elsites vcf-to-elsites writes for it"""
    w = synth.make_workload(4000, [("chr20", 400_000), ("chr21", 200_000)], seed=1)
    lines = [vc.H]
    for sq, t in zip(w.header.SQ, w.sites):
        for s, e in np.asarray(t).reshape(-1, 2).tolist():
            if e >= s:
                lines.append(b"%s\t%d\t.\t%s\tG\t.\tPASS\tRS=1\n" % (sq["SN"].encode(), s, b"A" * (e - s + 1)))
    text = b"".join(lines)
    res = {}
    for tag, data in [("vcf", text), ("vcf.gz", vr.bgzf(text, block=4000)), ("elsites", vr.vcf_to_elsites(text))]:
        ctx = device.Context(w.header)
        try:
            for ci, b in enumerate(w.contig_bases):
                ctx.set_reference(ci, b)
            ctx.load_known_sites(_write(tmp_path, [data], tag))
            ctx.append(w.batch)
            res[tag] = gpu_phases(ctx)
        finally:
            ctx.close()
    for tag in ("vcf", "vcf.gz"):
        for k in ("tables", "emp", "qual", "perm"):
            assert np.array_equal(res[tag][k], res["elsites"][k]), (tag, k)
        assert res[tag]["report"] == res["elsites"]["report"], tag
