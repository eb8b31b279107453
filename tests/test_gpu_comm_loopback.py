"""The several-GPU path of the library (csrc/comm.cu: the cross-group pair exchange inside elp_sort_markdup, elp_bqsr_tables_allreduce,
elp_optical_allreduce) on ONE GPU: ranks are threads of tests/comm_loopback.py, NCCL is the in-process stand-in tests/c/nccl_loopback.cpp.

Every scenario compares, read by read, the ranks' FLAG and QUAL, the summed tables, the duplication metrics and the metrics file text with
one context holding the whole input, and FLAG, tables and metrics with the oracle.  It also checks from the stand-in's counters and the
ranks' kernel_stats() which exchanges moved records: the owner of a pair's smaller REFID appends the visiting mate (ghost_append), every
other rank holding a mate of a cross-group pair ships it (spread_fill), and the grouped send / receive bytes are 128 per record plus one
per reply.  The error cases check that every rank fails together, within the stand-in's timeout, with FLAG untouched.

Out of scope (an N-rank run legitimately differs from one context, as the arrival order changes when mates become ghosts): a QNAME
reused by several pairs, mates whose RNEXT does not name the other mate's contig, full ties between pairs with equal QNAMEs."""
import json
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from elprep_b200 import _lib, multi, sam
from test_nccl_loopback_cpu import build_loopback
from util import oracle_tables_dense

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT_S = 20          # the stand-in's rendezvous limit in these runs
LN = 1_000_000
SEQ = "ACGTTGCA"
EQUAL = -10             # ELP_EQUAL: "Invalid QUAL character"


@pytest.fixture(scope="module")
def loopback_dir(tmp_path_factory):
    return build_loopback(str(tmp_path_factory.mktemp("nccl")), host_only=False)


def header(n_contigs):
    return sam.Header(sq=[{"SN": f"c{i}", "LN": LN} for i in range(n_contigs)],
                      rg=[{"ID": "rg0", "LB": "lib0", "PU": "u0"}, {"ID": "rg1", "LB": "lib1", "PU": "u1"}, {"ID": "rg2", "LB": "lib0", "PU": "u2"}])


class Reads:
    """records with QNAMEs given as bytes (0x80-0xFF included)"""

    def __init__(self, h):
        self.h, self.recs, self.names = h, [], []

    def add(self, name, flag, contig, pos, q=30, rg="rg0", mate=None, n=8):
        """mate: (contig, pos) of the mate, or None; contig -1 is '*'"""
        rname = f"c{contig}" if contig >= 0 else "*"
        r = dict(QNAME="?" * len(name), FLAG=flag, RNAME=rname, POS=pos if contig >= 0 or mate else 0, MAPQ=60 if contig >= 0 else 0,
                 CIGAR=f"{n}M" if contig >= 0 and not flag & 4 else "*", SEQ=(SEQ * (n // 8 + 1))[:n], QUAL=[q] * n, RG=rg)
        if mate is not None:
            r["RNEXT"], r["PNEXT"] = (f"c{mate[0]}" if mate[0] >= 0 else "*"), mate[1]
        self.recs.append(r)
        self.names.append(name)

    def pair(self, name, c1, p1, c2, p2, q1=30, q2=30, rg="rg0", rev=False):
        f1, f2 = (163, 83) if rev else (99, 147)
        self.add(name, f1, c1, p1, q1, rg, (c2, p2))
        self.add(name, f2, c2, p2, q2, rg, (c1, p1))

    def batch(self):
        b = sam.AlignmentBatch.from_records(self.h, self.recs)
        b.qname = np.frombuffer(b"".join(self.names), np.uint8).copy()
        assert b.qname.size == int(b.qname_off[-1])
        return b


def scenario(h, b, owner, world, seed=1, **kw):
    rng = np.random.default_rng(seed)
    bases = [rng.choice(np.frombuffer(b"ACGT", np.uint8), LN) for _ in h.SQ]
    sites = [np.zeros(0, np.int32) for _ in h.SQ]
    return dict(header=h, batch=b, contig_bases=bases, sites=sites, owner=np.asarray(owner, np.int32), world=world, **kw)


def run(sc, loopback_dir, lib=None):
    with tempfile.TemporaryDirectory() as d:
        sp, op = os.path.join(d, "sc.pkl"), os.path.join(d, "out.npz")
        with open(sp, "wb") as f:
            pickle.dump(sc, f)
        env = dict(os.environ, LD_LIBRARY_PATH=loopback_dir + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""), LOOPBACK_NCCL_TIMEOUT=str(TIMEOUT_S))
        if lib:
            env["ELPREP_B200_LIB"] = lib
        p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "comm_loopback.py"), sp, op], capture_output=True, text=True, timeout=900, env=env)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
        res = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])
        arrays = dict(np.load(op))
    assert res["nccl"] and all(x.startswith(loopback_dir) for x in res["nccl"]), res["nccl"]
    assert res["stats"]["calls"]["ncclCommInitRank"] == sc["world"]
    return res, arrays


def spread_records(sc):
    """per rank: (records it ships, records it receives) -- the exchange restated on the host (multi.spread_reads)"""
    b, owner, world = sc["batch"], sc["owner"], sc["world"]
    parts = sc.get("parts") or [multi.partition(b, owner, r, world) for r in range(world)]
    send, recv = [0] * world, [0] * world
    for r in range(world):
        idx, powner = multi.spread_reads(b.take(parts[r]), owner, r)
        for d in powner[powner != r]:
            send[r] += 1
            recv[int(d)] += 1
    return send, recv


def oracle_results(sc, pixel=100):
    import oracle
    b, h = sc["batch"].copy(), sc["header"]
    perm = oracle.coordinate_sort(b.copy(), n_threads=4)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "o.txt")
        om = oracle.markdup_optical(b, h, order=perm, pixel_distance=pixel, metrics_path=p, command_line="elprep filter in out", started_on="T")
        text = open(p).read()
    srt = b.take(perm)
    t = oracle.bqsr_gather(srt, h, oracle.Reference(h, sc["contig_bases"], sc["sites"]), n_threads=4)
    return b.flag, oracle_tables_dense(t)[0], om, text


def check_equal(sc, loopback_dir):
    res, a = run(sc, loopback_dir)
    for r in res["ranks"]:
        assert r["rc"] == 0 and not r["exception"], r
    eq = res["equal"]
    assert all(eq.values()), eq
    # the oracle on the whole input
    import oracle
    flag, tables, om, text = oracle_results(sc)
    assert np.array_equal(a["flag"], flag), np.nonzero(a["flag"] != flag)[0][:20]
    assert np.array_equal(a["tables"], tables)
    for slot, g in enumerate(res["metrics"]):
        for k_g, k_o in zip(_lib.ElpDupMetrics.COUNTERS, oracle.COUNTERS):
            assert g[k_g] == om.counters[slot][k_o], (slot, k_g)
        assert [{int(k): v for k, v in x.items()} for x in g["hist"]] == om.hist[slot]
        assert g["estimated_library_size"] == om.library_size[slot]
    assert bytes(a["metrics_text"]).decode() == text
    # which exchanges moved records
    send, recv = spread_records(sc)
    st = res["stats"]
    assert st["bytes"]["ncclSend"] == 129 * sum(send) * (2 if sc.get("rerun") else 1), (st, send)
    assert st["timeouts"] == st["mismatches"] == st["p2p_mismatches"] == st["other_failures"] == 0, st
    for r, rr in enumerate(res["ranks"]):
        assert ("spread_fill" in rr["kernels"]) == (send[r] > 0), (r, rr["kernels"], send)
        assert ("ghost_append" in rr["kernels"]) == (recv[r] > 0), (r, rr["kernels"], recv)
    return res, a, send, recv


# ---------------------------------------------------------------- workloads
def name_of(k, style):
    if style == "hi":                                     # bytes 0x80-0xFF
        return bytes([0x80 + (k * 7) % 128, 0xFF, 0x80 + k % 128]) + b"n%d" % k
    if style == "long91":
        return (b"L%d_" % k).ljust(91, b"x")
    if style == "long92":
        return (b"M%d_" % k).ljust(92, b"y")
    if style == "opt":
        return b"M:%d:FC:1:%d:%d:%d" % (k, 1101 + k % 2, 1000 + (k % 5) * 30, 2000 + (k % 3) * 40)
    return b"p%d" % k


def mixed(n_contigs, seed):
    """pairs over every ordered pair of contigs (duplicate sets of 1-5 pairs with tied and untied score sums, several libraries and read
    groups, optical names), fragments shadowed by pair mates, secondary / supplementary reads pointing at other contigs, mate-unmapped
    pairs with the unmapped mate placed at its mate, and unmapped reads"""
    rng = np.random.default_rng(seed)
    h = header(n_contigs)
    R = Reads(h)
    k = 0
    styles = ["plain", "hi", "long91", "long92", "opt", "opt"]
    for a in range(n_contigs):
        for b in range(n_contigs):
            for rep in range(2):
                pa, pb = int(rng.integers(1000, LN - 1000)), int(rng.integers(1000, LN - 1000))
                style = styles[(2 * (a * n_contigs + b) + rep) % len(styles)]   # every style occurs, on local and cross-group pairs
                rev = bool(rng.integers(0, 2))
                rgs = ["rg0", "rg2"] if rep else ["rg0"]             # lib0 through two read groups
                for j in range(int(rng.integers(1, 6))):
                    q1, q2 = (int(x) for x in rng.choice([20, 30, 40], 2))
                    R.pair(name_of(k, style), a, pa, b, pb, q1, q2, rgs[j % len(rgs)], rev)
                    k += 1
                if rep == 0 and rng.integers(0, 2):                  # a fragment at the first mate: a duplicate of the pair read
                    R.add(b"f%d" % k, 32 if rev else 0, a, pa, 40, "rg0"); k += 1
            if a != b:
                R.add(b"s%d" % k, 0x1 | 0x40 | 0x100, a, int(rng.integers(1000, LN - 1000)), 30, "rg1", (b, 500)); k += 1
                R.add(b"u%d" % k, 0x1 | 0x40 | 0x800, a, int(rng.integers(1000, LN - 1000)), 30, "rg1", (b, 700)); k += 1
        pm = int(rng.integers(1000, LN - 1000))
        R.add(b"m%d" % k, 0x1 | 0x8 | 0x40, a, pm, 30, "rg1", (a, pm))
        R.add(b"m%d" % k, 0x1 | 0x4 | 0x80, a, pm, 30, "rg1", (a, pm)); k += 1
    # one QNAME in two libraries, mates on contigs 0 and 1 each time
    R.pair(b"twolib", 0, 5000, 1, 6000, 30, 30, "rg0")
    R.pair(b"twolib", 0, 5000, 1, 6000, 40, 40, "rg1")
    R.pair(b"a", 0, 5000, 1, 6000, 20, 20, "rg0")          # a 1-byte name, a loser of twolib's lib0 set
    for j in range(3):
        R.add(b"x%d" % j, 4, -1, 0, 30, "rg0")
    return h, R.batch()


@pytest.mark.parametrize("world,owner", [(2, [0, 1, 0]), (2, [1, 0, 1]), (3, [0, 1, 2, 1]), (3, [2, 0, 1, 0]), (4, [0, 1, 2, 3, 0]), (4, [3, 2, 1, 0, 2])])
def test_pairs_across_every_pair_of_ranks(loopback_dir, world, owner):
    h, b = mixed(len(owner), seed=world * 10 + owner[0])
    sc = scenario(h, b, owner, world)
    _, _, send, recv = check_equal(sc, loopback_dir)
    # pairs cross every pair of contigs in both REFID orders: the owner of the smaller REFID of a pair of contigs on two ranks receives
    n = len(owner)
    owners_of_smaller = {owner[a] for a in range(n) for b in range(a + 1, n) if owner[a] != owner[b]}
    assert {r for r in range(world) if recv[r]} == owners_of_smaller
    assert {r for r in range(world) if send[r]} == {owner[b] for a in range(n) for b in range(a + 1, n) if owner[a] != owner[b]}


def test_second_run_after_reset(loopback_dir):
    h, b = mixed(3, seed=5)
    check_equal(scenario(h, b, [0, 1, 0], 2, rerun=True), loopback_dir)


def test_rank_without_reads_and_rank_without_entering_reads(loopback_dir):
    """rank 1 holds nothing; rank 2 holds unmapped, secondary and supplementary reads only (some pointing at other ranks' contigs)"""
    h = header(4)
    R = Reads(h)
    R.pair(b"a1", 0, 100, 3, 300, 30, 30)
    R.pair(b"a2", 0, 100, 3, 300, 20, 30)
    R.pair(b"b1", 3, 900, 0, 700, 40, 20, rev=True)
    R.add(b"sec", 0x1 | 0x40 | 0x100, 2, 400, 30, "rg0", (0, 100))
    R.add(b"sup", 0x1 | 0x80 | 0x800, 2, 450, 30, "rg0", (3, 300))
    R.add(b"um", 0x1 | 0x4 | 0x80, 2, 460, 30, "rg0", (2, 460))
    R.add(b"um", 0x1 | 0x8 | 0x40 | 0x100, 2, 460, 30, "rg0", (2, 460))
    check_equal(scenario(h, R.batch(), [0, 1, 2, 0], 3), loopback_dir)


def test_rank_that_only_sends_and_rank_that_only_receives(loopback_dir):
    """rank 1 holds c1 only, whose reads all pair with c0 (rank 0): rank 1 only sends, rank 0 only receives"""
    h = header(2)
    R = Reads(h)
    for j in range(6):
        R.pair(b"q%d" % j, 0, 1000 + 10 * (j % 2), 1, 5000, 20 + 5 * (j % 3), 30)
    _, _, send, recv = check_equal(scenario(h, R.batch(), [0, 1], 2), loopback_dir)
    assert send == [0, 6] and recv == [6, 0]


def test_ghosts_without_local_entering_reads(loopback_dir):
    """rank 0 owns c0 and holds no read there; rank 1 holds reads on c1 whose mates (absent from the input) would lie on c0: they travel
    to rank 0, which then marks ghosts only (phase_markdup with n_entering == 0 and n_ghost > 0)"""
    h = header(2)
    R = Reads(h)
    for j in range(4):
        R.add(b"o%d" % j, 147, 1, 5000, 30, "rg0", (0, 100))
    R.pair(b"t1", 1, 800, 1, 900, 30, 30)
    sc = scenario(h, R.batch(), [0, 1], 2)
    _, _, send, recv = check_equal(sc, loopback_dir)
    assert send == [0, 4] and recv == [4, 0]


def test_mixed_groups_winner_and_ties(loopback_dir):
    """duplicate sets over c0 (rank 0) x c1 (rank 1): the winner's score sum comes mostly from the ghost mate, or from the local one; score
    sums tie so that the smallest QNAME decides (the winner's name on either side); a losing pair gets 0x400 on both real mates"""
    h = header(2)
    R = Reads(h)
    R.pair(b"g_win", 0, 1000, 1, 2000, 20, 40)           # ghost (c1 mate) carries the score
    R.pair(b"g_lose", 0, 1000, 1, 2000, 40, 10)
    R.pair(b"l_win", 0, 3000, 1, 4000, 40, 20)           # local mate carries the score
    R.pair(b"l_lose", 0, 3000, 1, 4000, 10, 40)
    R.pair(b"tie_b", 0, 5000, 1, 6000, 30, 30)           # ties: 'tie_a' wins on the name, arriving later
    R.pair(b"tie_c", 0, 5000, 1, 6000, 20, 40)
    R.pair(b"tie_a", 0, 5000, 1, 6000, 40, 20)
    R.pair(b"tie_z", 1, 7000, 0, 8000, 30, 30, rev=True)  # the first mate on the larger REFID
    R.pair(b"tie_y", 1, 7000, 0, 8000, 30, 30, rev=True)
    sc = scenario(h, R.batch(), [0, 1], 2)
    res, a, _, _ = check_equal(sc, loopback_dir)
    names = [bytes(n) for n in R.names]
    dup = {}
    for i, nm in enumerate(names):
        dup.setdefault(nm, []).append(bool(a["flag"][i] & 0x400))
    assert dup[b"g_win"] == [False, False] and dup[b"g_lose"] == [True, True]
    assert dup[b"l_win"] == [False, False] and dup[b"l_lose"] == [True, True]
    assert dup[b"tie_a"] == [False, False] and dup[b"tie_b"] == [True, True] and dup[b"tie_c"] == [True, True]
    assert dup[b"tie_y"] == [False, False] and dup[b"tie_z"] == [True, True]


def test_names_on_shipped_records(loopback_dir):
    """QNAMEs of 1, 91 and 92 bytes and with bytes 0x80-0xFF on pairs whose c1 mate (rank 1) travels to rank 0.  Within each duplicate set
    the score sums tie, so the smallest name wins, decided by the last byte of 91- and 92-byte names, and the ghost joins its local mate
    only if every name byte arrived"""
    h = header(2)
    R = Reads(h)
    sets = [[b"b", b"a", b"c"],
            [b"N" * 90 + b"b", b"N" * 90 + b"a"],
            [b"N" * 91 + b"z", b"N" * 91 + b"\xff", b"N" * 91 + b"y"],
            [b"\x80q", b"\xffq", b"\x7fq"]]                 # bytes compare unsigned
    for k, names in enumerate(sets):
        for nm in names:
            R.pair(nm, 0, 1000 + 1000 * k, 1, 50_000 + 1000 * k, 30, 30)
    assert {len(nm) for names in sets for nm in names} >= {1, 91, 92}
    _, a, send, recv = check_equal(scenario(h, R.batch(), [0, 1], 2), loopback_dir)
    assert send == [0, 11] and recv == [11, 0]
    for names in sets:
        for nm in names:
            i = [j for j, x in enumerate(R.names) if x == nm]
            assert [bool(a["flag"][j] & 0x400) for j in i] == [nm != min(names)] * 2, nm


def test_spread_read_in_fragment_group_and_skipped_reads(loopback_dir):
    """a cross-group mate shadows the fragments at its position on its home rank; secondary / supplementary reads with RNEXT on another
    rank, mate-unmapped pairs and unmapped reads placed at their mate are never shipped"""
    h = header(3)
    R = Reads(h)
    R.pair(b"sp", 0, 1000, 2, 3000, 20, 20)
    R.add(b"fr1", 0, 0, 1000, 40)                        # fragments at the forward mate on c0 (rank 0) ...
    R.add(b"fr2", 0, 0, 1000, 30)
    R.add(b"fr3", 16, 2, 3000, 40)                        # ... and at the reverse mate on c2 (rank 1)
    R.add(b"sec", 0x1 | 0x40 | 0x100, 1, 1000, 30, "rg0", (0, 1000))
    R.add(b"sup", 0x1 | 0x80 | 0x800, 1, 1000, 30, "rg0", (2, 3000))
    R.add(b"mu", 0x1 | 0x8 | 0x40, 2, 5000, 30, "rg0", (0, 5000))     # mate unmapped, RNEXT on another rank
    R.add(b"un", 0x1 | 0x4 | 0x80, 1, 6000, 30, "rg0", (1, 6000))
    R.add(b"un", 0x1 | 0x40, 1, 6000, 30, "rg0", (1, 6000))
    sc = scenario(h, R.batch(), [0, 1, 1], 2)
    res, a, send, recv = check_equal(sc, loopback_dir)
    assert send == [0, 1] and recv == [1, 0]
    names = [bytes(n) for n in R.names]
    for nm in (b"fr1", b"fr2", b"fr3"):
        assert a["flag"][names.index(nm)] & 0x400


def test_optical_clusters_of_ghost_and_local_reads(loopback_dir):
    """duplicate sets whose first-of-pair reads are on either rank, in clusters by tile, x and y, in one and in two read groups of a library"""
    h = header(2)
    R = Reads(h)
    k = 0
    for (c1, c2, rgs) in [(0, 1, ["rg0"]), (1, 0, ["rg0"]), (0, 1, ["rg0", "rg2"]), (1, 0, ["rg2", "rg0"])]:
        base = 10_000 * (k + 1)
        for j in range(12):
            x, y = 1000 + (j // 3) * 150 + j % 3, 2000 + (j % 2) * 50
            R.pair(b"M:%d:FC:1:%d:%d:%d" % (k, 1101 + j % 2, x, y), c1, base, c2, base + 300, 20 + j % 4, 30, rgs[j % len(rgs)], rev=bool(j % 5 == 0))
        k += 1
    res, _, _, _ = check_equal(scenario(h, R.batch(), [0, 1], 2), loopback_dir)
    assert sum(m["read_pair_optical_duplicates"] for m in res["metrics"]) > 0


def test_optical_allreduce_with_many_oversized_keys(loopback_dir):
    """70 duplicate sets of 1024 .. 1093 pairs on rank 0 (histogram keys above the dense bins), and a few small sets on rank 1"""
    h = header(2)
    sizes = list(range(1024, 1094))
    n = sum(sizes)
    names = [b"p%d" % k for k in range(n)]
    qn = np.frombuffer(b"".join(nm for nm in names for _ in (0, 1)), np.uint8)
    lens = np.repeat(np.array([len(x) for x in names], np.uint64), 2)
    qoff = np.zeros(2 * n + 1, np.uint64)
    np.cumsum(lens, out=qoff[1:])
    set_of = np.repeat(np.arange(len(sizes)), sizes)
    p1 = (10_000 + 1000 * set_of).astype(np.int32)
    pos = np.empty(2 * n, np.int32); pos[0::2] = p1; pos[1::2] = p1 + 300
    pnext = np.empty(2 * n, np.int32); pnext[0::2] = p1 + 300; pnext[1::2] = p1
    flag = np.tile(np.array([99, 147], np.uint16), n)
    score = (20 + np.arange(2 * n) % 7).astype(np.uint8)
    big = sam.AlignmentBatch(refid=np.zeros(2 * n, np.int32), pos=pos, flag=flag, mapq=np.full(2 * n, 60, np.uint8), nref=np.zeros(2 * n, np.int32),
                             pnext=pnext, tlen=np.zeros(2 * n, np.int32), rg=np.zeros(2 * n, np.int32), qname_off=qoff, qname=qn,
                             cigar_off=np.arange(2 * n + 1, dtype=np.uint64), cigar=np.full(2 * n, 8 << 4, np.uint32), lseq=np.full(2 * n, 8, np.int32),
                             seq=np.full(8 * n, 0x12, np.uint8), qual=np.repeat(score, 8))
    R = Reads(h)
    for j in range(5):
        R.pair(b"s%d" % j, 1, 5000, 0, 900_000, 30, 20 + j)
    b = sam.AlignmentBatch.concat([big, R.batch()])
    res, _, _, _ = check_equal(scenario(h, b, [0, 1], 2), loopback_dir)
    assert sum(1 for k in res["metrics"][1]["hist"][0] if int(k) >= 1024) == 70


def test_two_million_reads_over_four_ranks(loopback_dir):
    from elprep_b200 import synth
    world = 4
    contigs = synth.scaled_hg38(400.0)
    groups = multi.contig_groups(contigs, world)
    h = synth.make_header(contigs)
    owner = multi.owner_table(h, groups)
    parts, ref_w = [], None
    for r in range(world):
        home = np.array([1 if owner[i] == r else 0 for i in range(len(contigs))], np.uint8)
        w = synth.make_workload(250_000, contigs, seed=700 + r, home=home, pair_id_base=r * 10**9, genome_seed=77, cross_contig_frac=0.05,
                                optical_frac=0.4, dup_frac=0.2, want_reference=(r == 0))
        if r == 0:
            ref_w = w
        parts.append(w.batch)
    whole = sam.AlignmentBatch.concat(parts)
    assert whole.n >= 2_000_000
    sc = dict(header=h, batch=whole, contig_bases=ref_w.contig_bases, sites=ref_w.sites, owner=owner, world=world)
    _, _, send, recv = check_equal(sc, loopback_dir)
    assert sum(send) > 0.01 * whole.n


# ---------------------------------------------------------------- every rank fails together
def failing(kind):
    """(scenario, the rank expected to fail first, the code, a part of its text); rank 0 owns c0, rank 1 c1, rank 2 c2"""
    h = header(3)
    R = Reads(h)
    R.pair(b"ok1", 0, 1000, 1, 2000)
    R.pair(b"ok2", 0, 1000, 1, 2000, 20, 20)
    R.pair(b"ok3", 1, 3000, 2, 4000)
    R.pair(b"ok4", 2, 5000, 0, 6000, rev=True)
    if kind == "invalid_qual":
        R.add(b"badq", 0, 1, 9000, 100)
        fail, code, text = 1, EQUAL, "Invalid QUAL character"
    elif kind == "negative_pos":
        R.add(b"negpos", 0, 2, -5, 30)
        fail, code, text = 2, _lib.ELIMIT, "negative POS"
    else:                                                 # a 93- or 254-byte QNAME on a cross-group read: c2's mate ships to rank 1
        L = 93 if kind == "qname93" else 254
        R.pair(b"N".ljust(L, b"n"), 1, 7000, 2, 8000)
        fail, code, text = 2, _lib.ELIMIT, "QNAME longer than 92 bytes"
    return scenario(h, R.batch(), [0, 1, 2], 3), fail, code, text


@pytest.mark.parametrize("kind", ["invalid_qual", "negative_pos", "qname93", "qname254"])
def test_every_rank_fails_together(loopback_dir, kind):
    sc, fail, code, text = failing(kind)
    res, _ = run(sc, loopback_dir)
    for r in res["ranks"]:
        assert not r["exception"], r
        assert r["rc"] == code, r
        assert r["seconds"] < TIMEOUT_S / 2, r                              # agreed in a collective, not by the stand-in's timeout
        if r["rank"] == fail and kind == "negative_pos":                    # the coordinate sort refuses the read as well
            assert text in r["readback_error"], r
        else:
            assert r["flag_untouched"], r
        if r["rank"] == fail:
            assert text in r["err"] and "on rank" not in r["err"], r
        else:
            assert f"on rank {fail}" in r["err"], r
    st = res["stats"]
    assert st["timeouts"] == st["mismatches"] == st["p2p_mismatches"] == 0, st
    assert st["bytes"]["ncclSend"] == 0, st                                  # nothing was shipped
    if kind.startswith("qname"):                                             # one context has no QNAME limit
        assert res["one"]["rc"] == 0
    else:
        assert res["one"]["rc"] == code
