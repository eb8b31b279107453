"""The CIGAR-geometry cases of the BQSR gather (gather_cigar_cases.py) through the oracle alone: every family has reads that count, the
error reads fail in the oracle with the codes the device must match, and the reads at the count kernel's record limits and the prep kernel's
64-operation limit are built as intended."""
import numpy as np
import pytest

import gather_cigar_cases as gc
import oracle
from knownsites_ref import parse_cigar


@pytest.fixture(scope="module", params=gc.FAMILIES)
def fam(request):
    return request.param, gc.family(request.param, gc.GENERAL)


def _ops(b, i):
    co = b.cigar_off.astype(np.int64)
    return [(int(x) >> 4, "MIDNSHP=X"[int(x) & 15]) for x in b.cigar[co[i]:co[i + 1]]]


def test_family_contributes(fam):
    name, F = fam
    d = gc.oracle_dense(F.good)
    assert d[:, :, 0, 0].sum() > 0
    idx = range(F.good.batch.n) if F.good.batch.n <= 1000 else range(0, F.good.batch.n, 7)    # a sample of the large families
    contrib = gc.contributions(F.good, reads=idx)
    n_in = sum(1 for v in contrib.values() if v[:, :, 0, 0].sum() > 0)
    assert n_in >= 0.75 * len(contrib), (name, n_in, len(contrib))


def test_error_reads(fam):
    name, F = fam
    expected = {"indel": set(), "indel_over_record": set(), "complex": {"ops65", "ops65_rev"}, "adaptor": {"2D58M_fwd_b1", "2D58M_rev_b1"},
                "contig_end": {c["name"] for c in gc.contig_end_cases() if c["contig_end"] > 0}}
    assert {n for n, *_ in F.errors} == expected[name]
    for n, w, ocode, dcode in F.errors:
        assert w.batch.n == 1
        if ocode is None:
            assert dcode == gc.ELP_ELIMIT
            assert gc.oracle_dense(w)[:, :, 0, 0].sum() > 0, n          # the oracle accepts the read and counts it
        else:
            with pytest.raises(ValueError, match=oracle.ERRORS[ocode]):
                gc.oracle_dense(w)


def test_indel_family_geometry():
    F, O = gc.family("indel", gc.FAST), gc.family("indel_over_record", gc.FAST)
    for fam, big in ((F, False), (O, True)):
        b = fam.good.batch
        seen = set()
        for i in range(b.n):
            ops = _ops(b, i)
            ind = [(n, op) for n, op in ops if op in "ID"]
            assert len(ind) == 1
            n, op = ind[0]
            assert (n == (256 if op == "I" else 4096)) == big
            lead = ops[1][0] if ops[0][1] == "H" and ops[1][1] == "S" else (ops[0][0] if ops[0][1] == "S" else 0)
            trail = ops[-2][0] if ops[-1][1] == "H" and ops[-2][1] == "S" else (ops[-1][0] if ops[-1][1] == "S" else 0)
            f = int(b.flag[i])
            seen.add((op, lead, trail, ops[0][1] == "H", ops[-1][1] == "H", bool(f & 0x10), bool(f & 0x80)))
            assert int(b.tlen[i]) == 0                                   # no adaptor clipping: the indel stays in the kept read
        ops_seen = {s[0] for s in seen}
        assert ops_seen == {"I", "D"}
        for k, values in ((1, gc.CLIPS), (2, gc.CLIPS), (3, (False, True)), (4, (False, True)), (5, (False, True)), (6, (False, True))):
            assert {s[k] for s in seen} == set(values), k
    lens = {(op, n) for fam in (F, O) for i in range(fam.good.batch.n) for n, op in _ops(fam.good.batch, i) if op in "ID"}
    assert lens == {("I", n) for n in gc.INS} | {("D", n) for n in gc.DEL}
    # every offset for 48, 64 and 100 aligned bases; 16k +- 1 and 32k +- 1 from both ends for 151 and 300
    assert gc.indel_offsets(64) == list(range(1, 64))
    for L in (151, 300):
        offs = set(gc.indel_offsets(L))
        for b in (16, 32):
            for k in range(1, L // b + 1):
                for d in (-1, 0, 1):
                    if 1 <= b * k + d <= L - 1:
                        assert b * k + d in offs and L - (b * k + d) in offs


def test_operation_limits():
    F = gc.family("complex", gc.GENERAL)
    b = F.good.batch
    nc = {n: int(b.cigar_off[i + 1] - b.cigar_off[i]) for i, n in enumerate(F.names)}
    assert nc["ops64"] == 64 and nc["ops64_adaptor_fwd"] == 64 and nc["ops64_split_first_rev"] == 64 and nc["ten_ops"] == 10
    assert all(w.batch.cigar.size == 65 for n, w, *_ in F.errors)
    # the adaptor clips of the 64-operation reads split an operation; the reverse one without soft clips leaves 65 operations
    for i, n in enumerate(F.names):
        if n.startswith("ops64_adaptor") or n.startswith("ops64_split"):
            rc, lo, hi, npos, cg = gc.probe_clip(b, i)
            lens = [int(x) >> 4 for x in cg if int(x) & 15 == 0]
            assert rc > 0 and 0 < hi - lo < int(b.lseq[i]), n
            if not n.endswith("in_del"):
                assert min(lens) < 3, n                                   # part of a 3M is kept
    i = F.names.index("ops64_split_first_rev")
    assert gc.probe_clip(b, i)[0] == 65


def test_contig_end_geometry():
    cases = gc.contig_end_cases()
    w, names = gc.build(cases, gc.FAST)
    b = w.batch
    clen = w.header.contig_lengths()
    for i, c in enumerate(cases):
        pos, ops = int(b.pos[i]), parse_cigar(c["cigar"])
        last_m = max(k for k, (op, _) in enumerate(ops) if op in "M=X")
        last = pos - 1 + sum(n for op, n in ops[:last_m + 1] if op in "MDN=X")
        assert last - int(clen[b.refid[i]]) == c["contig_end"], c["name"]
        assert pos <= clen[b.refid[i]]                                    # eligible: POS inside the contig (alignmentAgreesWithHeader)
        assert int(b.refid[i]) == i + 1                                   # a contig of its own
        q = b.qual[int(b.qual_off[i]):int(b.qual_off[i + 1])]
        if c["name"] in ("past_counted", "past_after_deletion"):
            assert q[-1] >= 6
        if c["name"] == "past_qual_below_6":
            assert q[-1] == 5
