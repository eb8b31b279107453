"""elp_load_reference on the device: .elfasta, FASTA and BGZF FASTA files read into every contig's one-hot reference, against the
restatement of ParseFasta / OpenElfasta (fasta_ref) and against elp_set_reference, at chunk sizes that put every case on a staging-chunk
edge."""
import ctypes as C

import numpy as np
import pytest

import elsites_ref as er
import fasta_cases as fc
import fasta_ref as fr
from elprep_b200 import _lib, bgzf, device, sam, synth
from util import compare_bqsr, gpu_phases, gpu_pipeline, oracle_pipeline

pytestmark = pytest.mark.gpu

CHUNKS = [1, 7, 64, 0]   # 0: the default


def _header(names, ln=1 << 30):
    return sam.Header(sq=[{"SN": n, "LN": ln} for n in names])


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def _elfasta_of(fasta):
    """an .elfasta of a parsed FASTA; names the table cannot hold (a leading '\\n' ends it, a '\\t' ends the name) are left out"""
    return fr.to_elfasta({k: v for k, v in fasta.items() if not k.startswith(b"\n") and b"\t" not in k})


def _forms(text):
    """the three forms of one FASTA text: (tag, file bytes)"""
    return [("fa", text), ("fa.gz", fr.bgzf_blocks(text, level=6, block=4000)), ("elfasta", _elfasta_of(fr.parse_fasta(text)))]


def _check(ctx, names, data):
    """the device's references after a load of `data` equal the restatement's, contig by contig"""
    seqs, nu, nm = fr.load(data, names)
    for ci, s in enumerate(seqs):
        n, nib = ctx.reference(ci)
        want = b"" if s is None else s
        assert n == len(want), (ci, n, len(want))
        assert nib.tobytes() == fr.hot_nibbles(want), ci
    return nu, nm


@pytest.mark.parametrize("chunk", CHUNKS)
def test_known_answers(tmp_path, chunk):
    ctx = device.Context(_header(fc.NAMES))
    try:
        ctx.debug_set_reference_chunk(chunk)
        cases = [(cid, f) for cid, text, _ in fc.FASTA_VALID for f in _forms(text)]
        cases += [(cid, ("elfasta", data)) for cid, data, _ in fc.ELFASTA_VALID]
        for cid, (tag, data) in cases:
            got = ctx.load_reference(_write(tmp_path, f"{cid}.{tag}", data))
            assert got == _check(ctx, fc.NAMES, data), (cid, tag)
    finally:
        ctx.close()


def _snapshot(ctx, n):
    return [(ctx.reference(ci)[0], ctx.reference(ci)[1].tobytes()) for ci in range(n)]


@pytest.mark.parametrize("chunk", [7, 0])
def test_refusals(tmp_path, chunk):
    """every refusal names the file and the line (FASTA) or offset (.elfasta, BGZF); the previous references stay"""
    import gzip
    ctx = device.Context(_header(fc.NAMES))
    try:
        ctx.debug_set_reference_chunk(chunk)
        ctx.load_reference(_write(tmp_path, "good.fa", fc.FASTA_VALID[0][1] + b">dup\nACGTTT\n"))
        before = _snapshot(ctx, len(fc.NAMES))
        bad = []
        for cid, text, (line, reason) in fc.FASTA_INVALID:
            bad.append((f"{cid}.fa", text, _lib.EFASTA, f"line {line}: ", reason))
            bad.append((f"{cid}.fa.gz", fr.bgzf_blocks(text, block=5000), _lib.EFASTA, f"line {line}: ", reason))
        for cid, data, (off, reason) in fc.ELFASTA_INVALID:
            bad.append((f"{cid}.elfasta", data, _lib.EFASTA, f"byte offset {off}: ", reason))
        good = b">chr1\nACGT\n" * 3000
        z = fr.bgzf_blocks(good, block=3000)
        crc = bytearray(z)
        crc[len(z) - 28 - 8] ^= 1                                      # the CRC32 of the last data block
        bad += [("plain.gz", gzip.compress(good), _lib.EBGZF, "offset", ""),
                ("crc.fa.gz", bytes(crc), _lib.EBGZF, "offset", ""),
                ("no_eof.fa.gz", fr.bgzf_blocks(good, eof=False), _lib.EBGZF, "offset", "EOF marker"),
                ("truncated.fa.gz", z[:-40], _lib.EBGZF, "offset", "")]
        for name, data, code, where, reason in bad:
            p = _write(tmp_path, name, data)
            with pytest.raises(device.ElprepError) as ei:
                ctx.load_reference(p)
            msg = str(ei.value)
            assert ei.value.code == code and p in msg and where in msg and reason in msg, (name, msg)
            assert _snapshot(ctx, len(fc.NAMES)) == before, name
        missing = str(tmp_path / "does_not_exist.fa")
        with pytest.raises(device.ElprepError) as ei:
            ctx.load_reference(missing)
        assert ei.value.code == _lib.EINVAL and missing in str(ei.value)
        assert _snapshot(ctx, len(fc.NAMES)) == before
    finally:
        ctx.close()


def test_context_without_contig_names(tmp_path):
    L = _lib.load()
    lens = np.full(2, 1000, np.int32)
    cfg = _lib.ElpConfig(0, 2, None, lens.ctypes.data_as(C.c_void_p), 0, None, None, None, 500, 0, None, 0, b"GATK", 100, 0)
    h = C.c_void_p()
    assert L.elp_create(C.byref(cfg), C.byref(h)) == 0
    try:
        p = _write(tmp_path, "a.fa", b">chr1\nACGT\n")
        assert L.elp_load_reference(h, p.encode(), None, None) == _lib.EINVAL
        assert b"contig_names" in L.elp_last_error(h)
        assert L.elp_reference_get(h, 0, None, 0) == 0
    finally:
        L.elp_destroy(h)


# ---- a seeded FASTA of about 100 Mbp ----
WIDTHS = [60, 50, 61, 80, 60, 61, 50, 80]


def _random_fasta(seed, total=100_000_000):
    rng = np.random.default_rng(seed)
    names = [f"chr{i}" for i in range(1, 8)] + ["chrUn_x"]
    w = rng.random(len(names)) + 0.3
    lens = (w / w.sum() * total).astype(np.int64)
    alpha = np.frombuffer(b"ACGTACGTACGTacgtNNnRYKMSWBDHV", np.uint8)
    seqs = {}
    for i, (n, L) in enumerate(zip(names, lens)):
        s = alpha[rng.integers(0, len(alpha), size=L)]
        if i == 2:   # every byte value but '\n' (and no '>' that starts a line, no '\r' that ends one: the widths are fixed below)
            s = rng.integers(0, 256, size=L).astype(np.uint8)
            s[s == 0x0A] = 0x0B
        seqs[n.encode()] = s
    parts = []
    for i, (n, s) in enumerate(seqs.items()):
        W, eol = WIDTHS[i], (b"\r\n" if i in (1, 5) else b"\n")
        s = s.copy()
        s[0::W][s[0::W] == ord(">")] = ord("A")                      # a line never starts with '>'
        s[W - 1::W][s[W - 1::W] == 0x0D] = ord("C")                  # nor ends with '\r'
        if len(s) and s[-1] == 0x0D:
            s[-1] = ord("C")
        seqs[n] = s
        b = s.tobytes()
        parts.append(b">" + n + b" LN:%d random description\t%d" % (len(s), i) + eol)
        parts.append(eol.join(b[j:j + W] for j in range(0, len(b), W)) + eol)
        if i % 3 == 1:
            parts.append(eol * 2)                                      # empty lines between contigs
    return b"".join(parts), {k: v.tobytes() for k, v in seqs.items()}


def test_random_fasta(tmp_path):
    text, seqs = _random_fasta(seed=7)
    names = list(k.decode() for k in seqs if k != b"chrUn_x") + ["chr3", "absent"]   # chr3 twice; chrUn_x unmatched; absent missing
    hdr_at = text.index(b">chr2")
    paths = {"fa": _write(tmp_path, "r.fa", text)}
    paths["fa.gz1"] = _write(tmp_path, "r1.fa.gz", bgzf.deflate(text, level=1).tobytes())
    paths["fa.gz9"] = _write(tmp_path, "r9.fa.gz", bgzf.deflate(text, level=9).tobytes())
    paths["elfasta"] = _write(tmp_path, "r.elfasta", fr.to_elfasta(seqs, data_order=sorted(seqs)))
    runs = [("fa", 0), ("fa", len(text) // 50 + 1), ("fa", hdr_at + 5), ("fa.gz1", 0), ("fa.gz9", 0), ("fa.gz1", len(text) // 53 + 1),
            ("elfasta", 0), ("elfasta", 1_000_003)]
    ctx = device.Context(_header(names), profile=True)
    try:
        for form, chunk in runs:
            ctx.debug_set_reference_chunk(chunk)
            assert ctx.load_reference(paths[form]) == (1, 1), (form, chunk)
            for ci, n in enumerate(names):
                got_n, nib = ctx.reference(ci)
                want = seqs.get(n.encode(), b"")
                assert got_n == len(want) and nib.tobytes() == fr.hot_nibbles(want), (form, chunk, n)
        st = ctx.kernel_stats()
        for k in ("fasta_lines", "fasta_classify", "fasta_scatter", "ref_pack", "bgzf_inflate"):
            assert k in st and st[k]["launches"] > 0, sorted(st)
        ref = device.Context(_header(names[:3]))
        try:
            for ci in range(3):
                ref.set_reference(ci, np.frombuffer(seqs[names[ci].encode()], np.uint8))
                assert ref.reference(ci)[1].tobytes() == ctx.reference(ci)[1].tobytes(), ci
        finally:
            ref.close()
    finally:
        ctx.close()


def test_every_byte_value_elfasta(tmp_path):
    """.elfasta sequences may hold any byte, '\\n' included; odd-sized pieces at chunk 7 start at odd bases"""
    rng = np.random.default_rng(3)
    a = np.concatenate([np.arange(256, dtype=np.uint8), rng.integers(0, 256, size=100_001).astype(np.uint8)]).tobytes()
    data = fr.to_elfasta({b"chr1": a, b"chr2": a[5:77_777]}, data_order=[b"chr2", b"chr1"])
    ctx = device.Context(_header(["chr1", "chr2"]))
    ref = device.Context(_header(["chr1", "chr2"]))
    try:
        ref.set_reference(0, np.frombuffer(a, np.uint8))
        ref.set_reference(1, np.frombuffer(a[5:77_777], np.uint8))
        for chunk in (7, 1000, 0):
            ctx.debug_set_reference_chunk(chunk)
            assert ctx.load_reference(_write(tmp_path, "b.elfasta", data)) == (0, 0)
            for ci in range(2):
                assert ctx.reference(ci)[0] == ref.reference(ci)[0]
                assert ctx.reference(ci)[1].tobytes() == ref.reference(ci)[1].tobytes(), (chunk, ci)
    finally:
        ctx.close(); ref.close()


def test_counts_and_duplicates(tmp_path):
    """n_unmatched and n_missing with duplicate names (the later wins, even an empty one) and duplicate SNs"""
    text = b">a\nAC\n>b\nGG\n>zz\nT\n>a\nTTT\n>b\n>\nA\n"
    names = ["a", "b", "a", "c"]
    ctx = device.Context(_header(names))
    try:
        for tag, data in _forms(text):
            nu, nm = ctx.load_reference(_write(tmp_path, "d." + tag, data))
            assert (nu, nm) == _check(ctx, names, data), tag
            assert ctx.reference(0)[0] == 3 and ctx.reference(2)[0] == 3 and ctx.reference(1)[0] == 0, tag
        assert fr.load(text, names)[1:] == (2, 1)
    finally:
        ctx.close()


def _workload():
    return synth.make_workload(4000, [("chr20", 400_000), ("chr21", 200_000)], seed=1)


def _fasta_of(w, skip=()):
    out = []
    for sq, b in zip(w.header.SQ, w.contig_bases):
        if sq["SN"] in skip:
            continue
        s = np.asarray(b, np.uint8).tobytes()
        out.append(b">%s\n" % sq["SN"].encode() + b"\n".join(s[j:j + 60] for j in range(0, len(s), 60)) + b"\n")
    return b"".join(out)


def _elsites_of(w):
    return er.write([(sq["SN"], int(s), int(e)) for sq, t in zip(w.header.SQ, w.sites) for s, e in np.asarray(t).reshape(-1, 2)])


def test_end_to_end(tmp_path):
    """load_reference + load_known_sites, then sort, duplicate marking, gather, finalize and apply: bit-exact against the oracle and
    against the elp_set_reference path, also after a refused load"""
    w = _workload()
    text = _fasta_of(w)
    sites = _write(tmp_path, "s.elsites", _elsites_of(w))
    o = oracle_pipeline(w)
    g_set = gpu_pipeline(w)
    compare_bqsr(g_set, o)
    for tag, data in [("fa", text), ("fa.gz", fr.bgzf_blocks(text)), ("elfasta", fr.to_elfasta(fr.parse_fasta(text)))]:
        ctx = device.Context(w.header)
        try:
            assert ctx.load_reference(_write(tmp_path, "w." + tag, data)) == (0, 0)
            ctx.load_known_sites([sites])
            with pytest.raises(device.ElprepError):
                ctx.load_reference(_write(tmp_path, "bad.fa", text + b"\nACGT\n"))   # an empty line inside the last contig
            ctx.append(w.batch)
            g = gpu_phases(ctx)
        finally:
            ctx.close()
        compare_bqsr(g, o)
        for k in ("tables", "emp", "qual", "perm"):
            assert np.array_equal(g[k], g_set[k]), (tag, k)
        assert g["report"] == g_set["report"], tag


def test_missing_contig_is_refend(tmp_path):
    """a contig whose SN has no sequence in the file has none: a recalibrated read on it fails with ELP_EREFEND, as for a contig never set"""
    w = _workload()
    ctx = device.Context(w.header)
    try:
        assert ctx.load_reference(_write(tmp_path, "m.fa", _fasta_of(w, skip=("chr21",)))) == (0, 1)
        ctx.load_known_sites([_write(tmp_path, "s.elsites", _elsites_of(w))])
        ctx.append(w.batch)
        ctx.sort_markdup(device.SO_COORDINATE, True)
        with pytest.raises(device.ElprepError) as ei:
            ctx.bqsr_gather()
        assert ei.value.code == _lib.EREFEND
    finally:
        ctx.close()


def test_lifetime(tmp_path):
    names = ["c0", "c1", "c2"]
    f1 = _write(tmp_path, "l1.fa", b">c0\nACGT\n>c1\nGGGCC\n>c2\nT\n")
    f2 = _write(tmp_path, "l2.fa", b">c1\nAA\n")
    ctx = device.Context(_header(names))
    hot = fr.hot_nibbles
    try:
        ctx.set_reference(2, np.frombuffer(b"CCCC", np.uint8))
        ctx.load_reference(f1)                          # replaces every contig
        assert [ctx.reference(i)[1].tobytes() for i in range(3)] == [hot(b"ACGT"), hot(b"GGGCC"), hot(b"T")]
        ctx.set_reference(1, np.frombuffer(b"TTT", np.uint8))   # one contig, inside the loaded block
        assert [ctx.reference(i)[1].tobytes() for i in range(3)] == [hot(b"ACGT"), hot(b"TTT"), hot(b"T")]
        ctx.reset()                                     # the references survive elp_reset
        assert [ctx.reference(i)[0] for i in range(3)] == [4, 3, 1]
        assert ctx.load_reference(f2) == (0, 2)         # load -> load: contigs without a sequence are emptied
        assert [ctx.reference(i)[0] for i in range(3)] == [0, 2, 0]
        ctx.set_reference(0, np.frombuffer(b"GA", np.uint8))
        ctx.load_reference(f1)
        assert [ctx.reference(i)[0] for i in range(3)] == [4, 5, 1]
    finally:
        ctx.close()                                     # load -> destroy
    ctx = device.Context(_header(names))
    ctx.load_reference(f1)
    ctx.close()
    with pytest.raises(device.ElprepError):
        device.Context(_header(names)).reference(3)
