"""The VCF restatement (vcf_ref) against hand-derived known answers (vcf_cases), strconv.ParseFloat's syntax and range edges, and the
composition the loader stands for: a VCF in the --known-sites list gives the table of vcf-to-elsites on it (sort + ParallelFlatten per
chromosome, the .elsites written) followed by loading that .elsites in the same position of the list."""
import numpy as np
import pytest

import elsites_ref as er
import vcf_cases as vc
import vcf_ref as vr


@pytest.mark.parametrize("cid,files,expect,unmatched", vc.VALID, ids=[c[0] for c in vc.VALID])
def test_valid_known_answers(cid, files, expect, unmatched):
    tables, nu = vr.load(files, vc.NAMES)
    assert nu == unmatched
    for name, t in zip(vc.NAMES, tables):
        want = np.array(expect.get(name, []) if name != "*" else [], dtype=np.int32).reshape(-1, 2)
        assert np.array_equal(t, want), (name, t.tolist(), want.tolist())


@pytest.mark.parametrize("cid,files,where", vc.INVALID, ids=[c[0] for c in vc.INVALID])
def test_invalid_known_answers(cid, files, where):
    with pytest.raises(vr.VcfError) as ei:
        vr.load(files, vc.NAMES)
    assert (ei.value.file, ei.value.line, ei.value.reason) == where


def test_bgzf_cases_are_bgzf():
    """the BGZF-only cases start with 0x1f, every other VCF case with the plain prefix (else the content rule would not pick VCF)"""
    for cid, files, *_ in vc.VALID + vc.INVALID:
        for d in files:
            assert d.startswith(er.HEADER) or d[:1] == b"\x1f" or d.startswith(vr.PREFIX), cid


@pytest.mark.parametrize("s,v", [(b"1_000.5", 1000.5), (b"0x1p-2", 0.25), (b"0X1.8P+1", 3.0), (b"+INF", float("inf")), (b"-infinity", float("-inf")),
                                 (b"1e-400", 0.0), (b".5", 0.5), (b"5.", 5.0), (b"0x_1p0", 1.0), (b"1e1_0", 1e10), (b"0x1.fffffffffffff7p1023", 1.7976931348623157e308),
                                 (b"00.0012", 0.0012), (b"0x00.8p1", 1.0), (b"0e99999999", 0.0)])
def test_parse_float_accepts(s, v):
    """atof.go: special(), readFloat() with underscoreOK, hex mantissas with a 'p' exponent; underflow is no error"""
    assert vr.parse_float(s) == v


@pytest.mark.parametrize("s", [b"", b"+", b".", b"e5", b"1e", b"1e+", b"0x", b"0x1", b"0x1.8", b"0xp1", b"1__0", b"_1", b"1_", b"1_.5", b"1e_5",
                               b"+nan", b"-nan", b"infx", b"infin", b"infinityx", b"nanx", b"1.5.", b" 1", b"1 ", b"1d", b"0b101", b"0o7", b"1e5_",
                               b"\xd9\xa1"])
def test_parse_float_rejects(s):
    with pytest.raises(ValueError):
        vr.parse_float(s)


@pytest.mark.parametrize("s", [b"1e309", b"-1e309", b"1.7976931348623159e308", b"0x1.fffffffffffff8p1023", b"0x1p1024", b"1e99999999",
                               b"0.0000000001e319", b"1797693134862315807937289714053034150799341327100378269361737789804449682927647509466490179775872070963302864166928879109465555478519404026306574886715058206819089020007083836762738548458177115317644757302700698555713669596228429148198608349364752927190741684443655107043427115596995080930428801779041744977920e-1"])
def test_parse_float_range(s):
    """a value that rounds to +-Inf is strconv's range error (at the bound 2^1024 - 2^970 itself, round-half-even goes up)"""
    with pytest.raises(OverflowError):
        vr.parse_float(s)


def test_utf8_rules():
    """utf8.DecodeRune: valid forms decode; overlong forms, surrogates, code points above U+10FFFF and truncated forms are RuneError"""
    assert vr._decode_rune(b"\xc3\xa9x") == (0xE9, 2)
    assert vr._decode_rune(b"\xf0\x9f\x98\x80") == (0x1F600, 4)
    for bad in (b"\xc0\x80", b"\xe0\x80\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\xe2\x82", b"\x80", b"\xff"):
        assert vr._decode_rune(bad)[0] == 0xFFFD, bad
    assert vr._decode_rune(b"\xef\xbf\xbd") == (0xFFFD, 3)   # a valid encoding of U+FFFD is refused by the caller as well


# ---- the composition, on seeded random files ----
CHROMS = [b"chr1", b"chr10", b"chrX", b"dup", b"chrZ", b"*", b"."]


def random_vcf(rng, n):
    """a small VCF: unsorted positions, equal starts, REFs of length 0..6 (so end < start happens), missing fields, CRLF lines"""
    lines = []
    for _ in range(n):
        c = CHROMS[rng.integers(len(CHROMS))]
        pos = b"." if rng.random() < 0.05 else b"%d" % rng.integers(-3, 40)
        ref = b"A" * int(rng.integers(0, 7))
        info = [b"RS=1", b"DB", b"X Y", b"DP=1:DB", b"."][rng.integers(5)]
        ln = b"\t".join([c, pos, b".", ref if ref or rng.random() < 0.5 else b".", b"G", b".", b"PASS", info])
        if rng.random() < 0.05:
            ln = b"\t".join([c, pos, b"."])
        lines.append(ln + (b"\r\n" if rng.random() < 0.1 else b"\n"))
    return vc.H + b"".join(lines)


@pytest.mark.parametrize("seed", range(40))
def test_composition_equals_single_flatten(seed):
    rng = np.random.default_rng(seed)
    files = []
    for _ in range(int(rng.integers(1, 4))):
        if rng.random() < 0.3:
            rows = [(CHROMS[rng.integers(4)], int(rng.integers(0, 40)), int(rng.integers(0, 45))) for _ in range(int(rng.integers(0, 20)))]
            files.append(er.write(rows))
        else:
            files.append(random_vcf(rng, int(rng.integers(0, 60))))
    direct, du = vr.load(files, vc.NAMES)
    composed = [f if f.startswith(er.HEADER) else vr.vcf_to_elsites(f) for f in files]
    via, _ = er.load(composed, vc.NAMES)
    for a, b in zip(direct, via):
        assert np.array_equal(a, b), (a.tolist(), b.tolist())
    # n_unmatched counts VCF data lines, not flattened .elsites lines
    want_u = 0
    for f in files:
        for chrom, _, _ in vr.rows(f):
            want_u += chrom not in {b"chr1", b"chr10", b"chrX", b"dup", b"."}
    assert du == want_u
