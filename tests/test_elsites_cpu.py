"""The .elsites restatement (elsites_ref) against hand-derived known answers: the header and line rules of
intervals.FromElsitesFile (intervals/intervals.go:199-254), bufio.ScanLines, strconv.ParseInt(s, 10, 32), and the per-contig sort and
flatten of NewBaseRecalibrator (filters/bqsr.go:424-443).  Each case in elsites_cases cites the rule it pins."""
import numpy as np
import pytest

import elsites_cases as ec
import elsites_ref as er
import knownsites_ref as ks


@pytest.mark.parametrize("cid,files,expect,unmatched", ec.VALID, ids=[c[0] for c in ec.VALID])
def test_valid_known_answers(cid, files, expect, unmatched):
    tables, nu = er.load(files, ec.NAMES)
    assert nu == unmatched
    for name, t in zip(ec.NAMES, tables):
        want = np.array(expect.get(name, []) if name != "*" else [], dtype=np.int32).reshape(-1, 2)
        assert np.array_equal(t, want), (name, t.tolist(), want.tolist())


@pytest.mark.parametrize("cid,files,where", ec.INVALID, ids=[c[0] for c in ec.INVALID])
def test_invalid_known_answers(cid, files, where):
    with pytest.raises(er.ElsitesError) as ei:
        er.load(files, ec.NAMES)
    assert (ei.value.file, ei.value.line, ei.value.reason) == where


@pytest.mark.parametrize("s,v", [(b"0", 0), (b"+5", 5), (b"-0", 0), (b"007", 7), (b"2147483647", 2147483647), (b"-2147483648", -2147483648)])
def test_parse_int32_accepts(s, v):
    """strconv.ParseInt(s, 10, 32): optional sign, decimal digits, int32 range"""
    assert er.parse_int32(s) == v


@pytest.mark.parametrize("s", [b"", b"+", b"-", b" 5", b"5 ", b"1_000", b"0x10", b"2147483648", b"-2147483649", b"++1", b"1e3", b"\xd9\xa1"])
def test_parse_int32_rejects(s):
    """underscores are only allowed with base 0 (strconv/atoi.go underscoreOK), so base 10 rejects them like every other non-digit"""
    with pytest.raises(ValueError):
        er.parse_int32(s)


def test_scan_lines():
    """bufio.ScanLines: '\\n' ends a line, dropCR removes one '\\r', the final segment is a line only when non-empty"""
    assert er.scan_lines(b"a\nb\r\n\r\nc") == [(1, b"a"), (2, b"b"), (1, b""), (1, b"c")]
    assert er.scan_lines(b"a\n") == [(1, b"a")]
    assert er.scan_lines(b"") == []
    assert er.scan_lines(b"x\r") == [(2, b"x")]
    assert er.scan_lines(b"x\r\r\n") == [(3, b"x\r")]


def test_swallowing_case_takes_the_serial_flatten():
    """ParallelFlatten panics when a left interval swallows the whole right half (knownsites_ref raises IndexError); the load keeps the
    serial Flatten result there, like elp_set_known_sites"""
    n = 2 * ks.GRAIN
    pairs = np.array([(0, 10 * n)] + [(i, i) for i in range(1, n)], dtype=np.int64)
    with pytest.raises(IndexError):
        ks.sort_and_flatten(pairs)
    assert er.sort_flatten(pairs).tolist() == [[0, 10 * n]]


def test_write_round_trip():
    rows = [("chr1", 5, 9), ("chrX", -3, 4)]
    for crlf in (False, True):
        for fin in (False, True):
            got = er.from_elsites(er.write(rows, crlf=crlf, final_newline=fin))
            assert got == [(b"chr1", 5, 9), (b"chrX", -3, 4)]


@pytest.mark.parametrize("seed", range(6))
def test_fast_flatten_equals_sort_flatten(seed):
    """the vectorised restatement the large GPU test uses against sort_and_flatten / Flatten, with reversed, touching and swallowing
    intervals on both sides of ParallelFlatten's grain"""
    rng = np.random.default_rng(seed)
    n = [10, 500, ks.GRAIN - 1, ks.GRAIN + 7, 3 * ks.GRAIN, 2 * ks.GRAIN][seed]
    s = rng.integers(-50, 10 * n, size=n)
    e = s + rng.integers(-5, 12, size=n)
    if seed % 2:
        s[0], e[0] = -100, 20 * n        # swallows everything
    pairs = np.stack([s, e], 1)
    assert np.array_equal(er.sort_flatten_fast(pairs), er.sort_flatten(pairs))
