"""The restatement of ApplyBQSR's per-base rule (apply_ref.py) against the oracle's bqsr_apply, on every case of apply_cases.py, with
tables gathered from the cases and with crafted tables; plus hand-derived keys for contextWith and the cycle covariate."""
import numpy as np
import pytest

import apply_cases as AC
import apply_ref
from elprep_b200 import sam

ERR = {"ENORG": "BQSR requires input with read groups", "ECYCLE": "cycle value exceeds maximum cycle value",
       "ECONTEXT": "context covariate would panic"}


@pytest.fixture(scope="module")
def ref():
    return AC.genome()


def _oracle(w, t, **kw):
    import oracle
    b = w.batch.copy()
    try:
        oracle.bqsr_apply(b, w.header, t, n_threads=1, **kw)
    except ValueError as e:
        return None, str(e)
    return b.qual, None


def _gathered(w, max_cycle):
    import oracle
    t = oracle.bqsr_gather(w.batch, w.header, oracle.Reference(w.header, w.contig_bases, w.sites), max_cycle=max_cycle)
    oracle.bqsr_finalize(t)
    return t


def _check(w, t, **kw):
    got, err = apply_ref.apply(w.batch, w.header, t, **kw)
    oq, oerr = _oracle(w, t, **kw)
    if err is None:
        assert oerr is None, oerr
        assert np.array_equal(got, oq), int(np.count_nonzero(got != oq))
    else:
        assert oerr is not None and ERR[err] in oerr, (err, oerr)
    return got, err


CONTEXTS = {
    "len32": lambda r: AC.lengths_context(32), "len33": lambda r: AC.lengths_context(33), "len100": lambda r: AC.lengths_context(100),
    "len1024": lambda r: AC.lengths_context(1024), "tails": lambda r: AC.tail_context(), "bases": lambda r: AC.base_context(r),
    "quals": lambda r: AC.qual_context(), "read_groups": lambda r: AC.read_group_context(),
}


@pytest.mark.parametrize("name", sorted(CONTEXTS))
def test_restatement_matches_oracle_gathered(name, ref):
    specs = CONTEXTS[name](ref)
    w, _ = AC.build(specs, AC.header(), ref)
    mc = max(1, max(s["L"] for s in specs))
    t = _gathered(w, mc)
    got, err = _check(w, t)
    assert err is None
    if name == "quals":
        assert int(np.count_nonzero(got != w.batch.qual)) > 0
    if name == "read_groups":    # rg4 has no table entries: its reads keep their QUAL, 200 included
        qo = w.batch.qual_off.astype(np.int64)
        for i in np.nonzero(w.batch.rg == 3)[0]:
            assert np.array_equal(got[qo[i]:qo[i + 1]], w.batch.qual[qo[i]:qo[i + 1]])


@pytest.mark.parametrize("levels,sqq", [(0, None), (16, None), (0, [10, 20, 30])])
def test_restatement_matches_oracle_crafted(levels, sqq, ref):
    specs = AC.lengths_context(100) + AC.qual_context() + AC.tail_context()
    w, _ = AC.build(specs, AC.header(), ref)
    t = AC.oracle_tables(AC.crafted_dense(3, 100, range(6, 94), empty_covs=(2,), longest=100), 100)
    _check(w, t, quantize_levels=levels, sqq=sqq)


def test_errors(ref):
    hdr = AC.header()
    t = AC.oracle_tables(AC.crafted_dense(3, 40, range(6, 94), empty_covs=(2,), longest=40), 40)
    for specs, err in (([AC.spec(20), AC.spec(20, rg=None)], "ENORG"), ([AC.spec(20), AC.spec(0, qual=[], seq="", rg=None)], "ENORG"),
                       ([AC.spec(41, 0)], "ECYCLE"), ([AC.spec(41, 0x10)], "ECYCLE"),
                       ([AC.spec(41, 0, qual=[30] * 40 + [5])], None), ([AC.spec(41, 0x10, qual=[5] + [30] * 40)], None),
                       ([AC.spec(41, 0x10, qual=[30] * 40 + [5])], "ECYCLE"), ([AC.spec(40, 0x1 | 0x80 | 0x10)], None)):
        w, _ = AC.build(specs, hdr, ref)
        assert _check(w, t)[1] == err, specs


def test_context_quirks(ref):
    """contextWith at the read start: the panic and the TT keys, as the oracle restates them"""
    hdr = AC.header()
    t = AC.oracle_tables(AC.crafted_dense(3, 10, range(6, 94), longest=10), 10)
    for seq, q, f in AC.quirk_reads():
        assert apply_ref.context_quirk(seq, q, f), seq
        w, _ = AC.build([AC.spec(len(seq), f, qual=q, seq=seq)], hdr, ref)
        _check(w, t)
    assert apply_ref.context_with(list("NRACGT"))[2:4] == [0xF2, 2 | (3 << 4) | (1 << 6)]   # TT, then T as the previous base
    with pytest.raises(apply_ref.ContextPanic):
        apply_ref.context_with(list("RACG"))


def test_keys_by_hand():
    A, C, G, T = 0, 1, 2, 3
    k = lambda p, c: 2 | (p << 4) | (c << 6)
    assert apply_ref.context_with(list("ACGT")) == [-1, k(A, C), k(C, G), k(G, T)]
    assert apply_ref.context_with(list("ACNGTA")) == [-1, k(A, C), -1, -1, k(G, T), k(T, A)]
    assert apply_ref.context_with(list("NACG")) == [-1, -1, k(A, C), k(C, G)]
    assert apply_ref.context_with(list("A")) == [-1] and apply_ref.context_with([]) == []
    # reverse strand: complemented, reversed, keys reversed back; tails read as N; 0xFF is not a tail
    assert apply_ref.context_covariates("AACG", [30] * 4, sam.Reversed) == [k(T, T), k(G, T), k(C, G), -1]
    assert apply_ref.context_covariates("AACG", [2, 30, 30, 1], 0) == [-1, -1, k(A, C), -1]
    assert apply_ref.stranded_clipped_seq("AC", [255, 255], False) == ["A", "C"]
    assert apply_ref.stranded_clipped_seq("AC", [2, 2], False) is None
    # cycles: 0x80 means "last" whether or not 0x1 is set
    assert apply_ref.cycle_covariates(0, 10) == (1, 1) and apply_ref.cycle_covariates(0x10, 10) == (10, -1)
    assert apply_ref.cycle_covariates(0x80, 10) == (-1, -1) and apply_ref.cycle_covariates(0x80 | 0x10, 10) == (-10, 1)


def test_read_group_covariate():
    hdr = AC.header()
    assert [apply_ref.read_group_covariate(hdr, g) for g in (0, 1, 2, 3, -1)] == ["FC1.1", "FC1.1", "rg3", "FC9.9", None]
    assert hdr.rg_cov_ids()[1] == ["FC1.1", "rg3", "FC9.9"]
