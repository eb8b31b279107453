"""The CPU restatement of the device sort (coordsort_ref.py) against the oracle, on every input of test_gpu_coordsort_edges.py that the
oracle orders the same way (no empty QNAME: the device compares it as the smallest name, the reference skips the clause); and the
restated chunk keys against the order they are meant to produce."""
import numpy as np
import pytest

import coordsort_ref as R
from coordsort_cases import CASES, NUL_NAMES, columns


def _nonempty(b):
    return bool((np.diff(b.qname_off.astype(np.int64)) > 0).all())


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_oracle(name):
    import oracle
    b, n_contigs = CASES[name]()
    assert _nonempty(b)
    assert np.array_equal(R.coordinate_order(b, n_contigs), oracle.coordinate_sort(b, n_threads=4))
    assert np.array_equal(R.queryname_order(b), oracle.queryname_sort(b))


def _device_algorithm(b, n_contigs):
    """the device's coordinate sort done with the restated keys: a stable sort by the primary key, runs of <= 32 by the comparator
    tuple, the reads of all longer runs together by LSD rounds over tie_rounds' chunks and bit ranges"""
    key = R.primary_key(b, n_contigs)
    perm = np.argsort(key, kind="stable")
    full = R.coordinate_order(b, n_contigs)
    rank = np.empty(b.n, np.int64)
    rank[full] = np.arange(b.n)
    ks = key[perm]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    lens = np.diff(np.r_[starts, ks.size])
    long_pos = []
    for s, n in zip(starts, lens):
        if n > R.SHORT_RUN:
            long_pos += range(s, s + n)
        else:
            perm[s:s + n] = perm[s:s + n][np.argsort(rank[perm[s:s + n]], kind="stable")]
    long_pos = np.array(long_pos, np.int64)
    elem = perm[long_pos]
    nq = R.n_qname_chunks(b)
    for ch, lo, bits in R.tie_rounds(b, n_contigs):
        field = (R.chunk_keys(b, ch, nq, n_contigs)[elem] >> np.uint64(lo)) & np.uint64((1 << bits) - 1 if bits < 64 else 2 ** 64 - 1)
        elem = elem[np.argsort(field, kind="stable")]
    perm[long_pos] = elem
    return perm


@pytest.mark.parametrize("name", [k for k in CASES if k != "names_40k"])
def test_chunk_rounds_give_the_order(name):
    b, n_contigs = CASES[name]()
    assert np.array_equal(_device_algorithm(b, n_contigs), R.coordinate_order(b, n_contigs))


def test_trailing_nul_chunk():
    """zero-padded QNAME chunks cannot tell "a" from "a\\0"; the trailing-NUL count breaks exactly those ties, and is 0 for the rest"""
    b = columns(NUL_NAMES, 0, 1)
    nq = R.n_qname_chunks(b)
    assert list(R.chunk_keys(b, 3, nq, 1)) == [0, 1, 2, 0, 0, 1, 0, 0]
    q = R.chunk_keys(b, R.QC0, nq, 1)
    assert q[0] == q[1] == q[2] == int.from_bytes(b"a".ljust(8, b"\0"), "big")
    assert R.queryname_order(b).tolist() == [0, 1, 2, 6, 4, 5, 3, 7]


def test_unpaired_mate_fields_do_not_order():
    b = columns([b"q"] * 3, 0, 5, flag=0, nref=[0, -1, 0], pnext=[9, 1, 3])
    assert R.coordinate_order(b, 1).tolist() == [0, 1, 2]
    assert not R.chunk_keys(b, 1, 1, 1).any()
    paired = columns([b"q"] * 3, 0, 5, flag=1, nref=[0, -1, 0], pnext=[9, 1, 3])
    assert R.coordinate_order(paired, 1).tolist() == [1, 2, 0]
