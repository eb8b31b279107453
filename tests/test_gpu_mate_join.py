"""The mate join of duplicate marking: adjacent mates paired in one streaming pass, the rest through the hash sort.

Reads i and i+1 pair up at once when both are entering true-pair reads with equal (library, QNAME) hashes, neither neighbour
outside them is another such read with that hash, and their libraries and name bytes are equal.  Every other true-pair read, and one
element per adjacent pair, goes into the reduced list that is sorted by 31 hash bits and matched on bytes in arrival order.  Every
case compares FLAG, output order and the duplication metrics with the oracle (markdup_check.check), checks that the three join
kernels ran, and checks the size of the reduced list against a numpy restatement of the adjacency rule (the `join` kernel counts 12
algorithmic bytes per element)."""
import numpy as np
import pytest

from elprep_b200 import sam, synth
from markdup_check import check
from markdup_edges import COLLIDING_PAIRS, COLLIDING_TRIPLE, join_hash

pytestmark = pytest.mark.gpu

JOIN_KERNELS = ("join_adjacent", "join_compact", "join")


def _header(n_libs=1):
    return sam.Header(sq=[{"SN": "c0", "LN": 1_000_000}, {"SN": "c1", "LN": 1_000_000}],
                      rg=[{"ID": f"rg{i}", "LB": f"lib{i}"} for i in range(n_libs)])


def R(q, flag, pos, score=30, rg="rg0", rname="c0", **kw):
    return dict(QNAME=q, FLAG=flag, RNAME=rname, POS=pos, MAPQ=60, CIGAR="4M", SEQ="ACGT", QUAL=[score] * 4, RG=rg, **kw)


def pair(q, p1, p2, s1=30, s2=None, rg="rg0"):
    return [R(q, 99, p1, s1, rg=rg, RNEXT="=", PNEXT=p2), R(q, 147, p2, s1 if s2 is None else s2, rg=rg, RNEXT="=", PNEXT=p1)]


def _dup(flag, recs, name):
    return [bool(flag[i] & 0x400) for i, r in enumerate(recs) if r["QNAME"] == name]


def reduced_size(b, h):
    """(elements of the reduced list, adjacent pairs) by the adjacency rule of join_adjacent_kernel"""
    f = b.flag.astype(np.int64)
    inn = ((f & 0x904) == 0) & ((f & 0x9) == 0x1)
    libs = {}
    for rg in h.RG:
        if rg.get("LB"):
            libs.setdefault(rg["LB"], len(libs))
    rg_lib = np.array([libs[rg["LB"]] if rg.get("LB") else -1 for rg in h.RG] + [-1], np.int64)
    g = b.rg.astype(np.int64)
    lib = rg_lib[np.where((g >= 0) & (g < len(h.RG)), g, len(h.RG))]
    qo = b.qname_off.astype(np.int64)
    names = [bytes(b.qname[qo[i]:qo[i + 1]]) for i in range(b.n)]
    qh = np.zeros(b.n, np.uint64)
    sel = np.flatnonzero(inn)
    if sel.size:
        qh[sel] = join_hash([names[i] for i in sel], lib[sel])
    n = b.n
    in_p = np.r_[False, inn, False, False]                     # read k at index k + 1
    qh_p = np.r_[np.uint64(0), qh, np.uint64(0), np.uint64(0)]
    u = np.arange(n - 1) + 1 if n > 1 else np.zeros(0, np.int64)
    same = lambda a, c: in_p[a] & in_p[c] & (qh_p[a] == qh_p[c])
    hp = same(u, u + 1) & ~same(u - 1, u) & ~same(u + 2, u)
    adj = [int(k) - 1 for k in u[hp] if lib[k - 1] == lib[k] and names[k - 1] == names[k]]
    return int(inn.sum()) - len(adj), len(adj)


def run(recs, h, optical=True, b=None):
    b = b if b is not None else sam.AlignmentBatch.from_records(h, recs)
    flag, stats = check(b, h, optical=optical)
    for k in JOIN_KERNELS:
        assert stats[k]["launches"] == 1, (k, sorted(stats))
    assert "join_keys" not in stats
    m, adj = reduced_size(b, h)
    assert stats["join"]["alg_bytes"] == 12 * m, (stats["join"]["alg_bytes"] / 12, m)
    return flag, m, adj


# ---------------------------------------------------------------- arrival orders
def _pairs_for_orders():
    """24 pairs in 8 signatures of 3 pairs each (scores 20 / 35 / 25: the 35 survives)"""
    out = []
    for s in range(8):
        for k, sc in enumerate((20, 35, 25)):
            out.append(pair(f"s{s}p{k}", 1000 + 1000 * s, 1300 + 1000 * s, sc))
    return out


@pytest.mark.parametrize("order", ["adjacent", "shuffled", "half"])
def test_same_pairs_in_three_arrival_orders(order):
    h = _header()
    pairs = _pairs_for_orders()
    rng = np.random.default_rng(7)
    if order == "adjacent":
        recs = [r for p in pairs for r in p]
    else:
        k = len(pairs) if order == "shuffled" else len(pairs) // 2
        tail = [r for p in pairs[len(pairs) - k:] for r in p]
        firsts, seconds = tail[0::2], tail[1::2]
        rng.shuffle(firsts); rng.shuffle(seconds)
        recs = [r for p in pairs[:len(pairs) - k] for r in p] + firsts + seconds    # every first mate before every second mate
    flag, m, adj = run(recs, h)
    assert adj == {"adjacent": 24, "shuffled": 0, "half": 12}[order]
    assert m == 48 - adj
    for s in range(8):
        assert _dup(flag, recs, f"s{s}p0") == [True, True] and _dup(flag, recs, f"s{s}p1") == [False, False] and _dup(flag, recs, f"s{s}p2") == [True, True]


# ---------------------------------------------------------------- a third read of the name elsewhere
@pytest.mark.parametrize("where", ["before", "after"])
def test_adjacent_pair_with_a_third_read_elsewhere(where):
    """DeleteOrStore pairs the first two arrivals: a third read before the adjacent pair takes its first read"""
    h = _header()
    third = R("q", 65, 9000, 40, RNEXT="=", PNEXT=9300)
    body = pair("q", 5000, 5300, 30) + pair("w", 5000, 5300, 32) + pair("z", 9000, 9300, 31)
    recs = ([third] + pair("o", 100, 400) + body) if where == "before" else (pair("o", 100, 400) + body + [third])
    flag, m, adj = run(recs, h, optical=False)
    assert adj == 4 and m == 4 + 1                                  # q's pair counts as one element, the third read as another
    if where == "after":                                            # (q 1st, q 2nd) has w's signature and the lower score
        assert _dup(flag, recs, "q") == [True, True, False] and _dup(flag, recs, "w") == [False, False]
    else:                                                           # (third, q 1st) pairs; q 2nd is left alone
        assert not any(_dup(flag, recs, "q")) and _dup(flag, recs, "w") == [False, False]


@pytest.mark.parametrize("k", [3, 4, 5])
def test_same_name_reads_in_a_row(k):
    """k same-name true-pair reads next to each other: no read has a disjoint same-hash pair, so all go through the sort"""
    h = _header()
    recs = pair("o", 100, 400)
    for j in range(k):
        recs.append(R("same", 99 if j % 2 == 0 else 147, 1000 + 500 * (j // 2) if j % 2 == 0 else 1300 + 500 * (j // 2), 30 + j))
    recs += pair("x", 1000, 1300, 20) + pair("y", 1500, 1800, 20)   # the signatures of (1st, 2nd) and (3rd, 4th) of "same"
    flag, m, adj = run(recs, h, optical=False)
    assert adj == 3 and m == 3 + k
    assert _dup(flag, recs, "same") == [False] * k
    assert _dup(flag, recs, "x") == [True, True] and _dup(flag, recs, "y") == ([True, True] if k >= 4 else [False, False])


def test_adjacent_same_name_reads_of_two_libraries():
    h = _header(2)
    recs = [R("q", 99, 1000, 30, rg="rg0", RNEXT="=", PNEXT=1300), R("q", 147, 1300, 30, rg="rg1", RNEXT="=", PNEXT=1000),
            R("q", 147, 1300, 30, rg="rg0", RNEXT="=", PNEXT=1000), R("q", 99, 1000, 30, rg="rg1", RNEXT="=", PNEXT=1300)]
    recs += pair("r", 1000, 1300, 20, rg="rg0") + pair("s", 1000, 1300, 40, rg="rg1")
    flag, m, adj = run(recs, h, optical=False)
    # the hashes include the library, so no two neighbouring q reads are hash-equal: (0, 2) pair in lib0 and beat r, (1, 3) in lib1 lose to s
    assert adj == 2 and m == 4 + 2
    assert _dup(flag, recs, "q") == [False, True, False, True] and _dup(flag, recs, "r") == [True, True] and _dup(flag, recs, "s") == [False, False]


@pytest.mark.parametrize("where", ["between", "before", "after"])
def test_adjacent_pair_with_a_secondary_or_supplementary_copy(where):
    h = _header()
    a, b_ = pair("q", 1000, 1300, 30)
    sec, sup = R("q", 0x100 | 0x41, 5000, 30), R("q", 0x800 | 0x81, 6000, 30)
    core = {"between": [a, sec, b_], "before": [sec, sup, a, b_], "after": [a, b_, sup, sec]}[where]
    recs = pair("o", 100, 400) + core + pair("w", 1000, 1300, 35)
    flag, m, adj = run(recs, h)
    assert adj == (2 if where == "between" else 3) and m == adj + (2 if where == "between" else 0)
    assert [bool(flag[i] & 0x400) for i, r in enumerate(recs) if r["QNAME"] == "q" and r["FLAG"] in (99, 147)] == [True, True]
    assert _dup(flag, recs, "w") == [False, False]


# ---------------------------------------------------------------- colliding 31-bit keys
@pytest.mark.parametrize("adjacent", [True, False])
def test_colliding_pairs(adjacent):
    """pairs whose 31-bit join keys collide: adjacent pairs land in one run of the sorted list and are expanded and matched on bytes"""
    h = _header()
    recs = []
    for k, (x, y) in enumerate(COLLIDING_PAIRS):
        x, y = x.decode(), y.decode()
        px, py = pair(x, 1000, 1300, 30 + k), pair(y, 1000, 1300, 20 + k)
        if adjacent:
            recs += px + py
        else:
            recs += [px[0], py[0]] + pair(f"gap{k}", 8000 + 500 * k, 8300 + 500 * k) + [py[1], px[1]]
    flag, m, adj = run(recs, h)
    assert adj == (6 if adjacent else 3)
    best = COLLIDING_PAIRS[-1][0].decode()                          # the highest score sum
    assert [nm for nm in dict.fromkeys(r["QNAME"] for r in recs) if nm.startswith("pA") and not any(_dup(flag, recs, nm))] == [best]


# adjacent pairs per order: B and C share the whole 64-bit hash, so BB next to CC are four reads of one hash and neither pair is adjacent
TRIPLE_ORDERS = {"AA BB CC": 1, "AA B C B C": 1, "A BB A CC": 2, "CC AA BB": 3}


@pytest.mark.parametrize("order", list(TRIPLE_ORDERS))
def test_colliding_triple(order):
    h = _header()
    names = dict(zip("ABC", (x.decode() for x in COLLIDING_TRIPLE)))
    pos = {"A": (1000, 1400), "B": (1000, 1400), "C": (2000, 2400)}
    score = {"A": 30, "B": 35, "C": 30}
    seen, recs = {}, []
    for who in order.replace(" ", ""):
        mate = seen.get(who, 0) + 1
        seen[who] = mate
        p1, p2 = pos[who]
        recs.append(R(names[who], 99 if mate == 1 else 147, p1 if mate == 1 else p2, score[who], RNEXT="=", PNEXT=p2 if mate == 1 else p1))
    flag, m, adj = run(recs, h)
    assert join_hash([names["B"].encode()])[0] == join_hash([names["C"].encode()])[0]
    assert adj == TRIPLE_ORDERS[order]
    assert _dup(flag, recs, names["A"]) == [True, True] and not any(_dup(flag, recs, names["B"])) and not any(_dup(flag, recs, names["C"]))


# ---------------------------------------------------------------- block edges
@pytest.mark.parametrize("offset", [0, 1])
def test_adjacent_pairs_across_block_edges(offset):
    """1100 adjacent pairs after `offset` fragment reads: with 256 threads per block, pairs straddle the block edges when offset = 1"""
    h = _header()
    recs = [R(f"f{k}", 0, 50 + k) for k in range(offset)]
    for k in range(1100):
        recs += pair(f"p{k:05d}", 1000 + 10 * (k // 4), 1300 + 10 * (k // 4), 20 + k % 4)
    flag, m, adj = run(recs, h, optical=False)
    assert adj == 1100 and m == 1100
    for k in range(1100):
        assert _dup(flag, recs, f"p{k:05d}") == ([False, False] if k % 4 == 3 else [True, True])


# ---------------------------------------------------------------- a generated workload
@pytest.mark.parametrize("permuted", [False, True])
def test_generated_workload(permuted):
    w = synth.make_workload(1_000_000, synth.scaled_hg38(400.0), seed=11, want_reference=False)
    b = w.batch
    if permuted:
        b = synth.take(b, np.random.default_rng(5).permutation(b.n))
    flag, m, adj = run(None, w.header, optical=False, b=b)
    assert b.n >= 2_000_000
    if permuted:
        assert adj < m // 1000
    else:
        assert adj > 0.45 * b.n
