"""The onesweep radix sort and the single-pass prefix sum at their tile edges.

Each sort key width runs at n = T-1, T, T+1 and 3T+1 for its tile size T (one tile short of full, exactly full, one
element into the next tile, and a run whose look-back crosses several tiles), on inputs that stress stability and the
digit histogram: heavy duplicates, all-equal keys, already-sorted and reversed keys, and bit ranges above lo_bit.  The scan
runs at n = 0 and 1, at its tile edges, past 32 tiles (the look-back window of one warp), with a non-zero base and with a
total above 2^32.
"""
import numpy as np
import pytest

from elprep_b200 import sam

pytestmark = pytest.mark.gpu

# tile sizes: THREADS * ITEMS of rs::Cfg<K32/K64/K128> in elprep_b200/csrc/radix_sort.cuh
TILE_U32 = 384 * 16
TILE_U64 = 384 * 16
TILE_U128 = 256 * 8
# SCAN_TILE in elprep_b200/csrc/sort.cu
SCAN_TILE = 256 * 16


@pytest.fixture(scope="module")
def ctx():
    from elprep_b200 import device
    c = device.Context(sam.Header(sq=[{"SN": "c", "LN": 1000}]))
    yield c
    c.close()


def _edges(t):
    return [t - 1, t, t + 1, 3 * t + 1]


def _keys(rng, n, bits, pattern, dtype=np.uint64):
    keys = rng.integers(0, 1 << min(bits, 63), size=n, dtype=np.uint64)
    if pattern == "dups":
        keys[rng.integers(0, n, size=n // 2)] = keys[0]
    elif pattern == "equal":
        keys[:] = keys[0]
    elif pattern == "sorted":
        keys.sort()
    elif pattern == "reversed":
        keys = np.sort(keys)[::-1].copy()
    return keys.astype(dtype)


def _expect(keys, lo_bit, bits):
    field = (keys.astype(np.uint64) >> np.uint64(lo_bit)) & np.uint64((1 << bits) - 1)
    return np.argsort(field, kind="stable").astype(np.uint32)


PATTERNS = ["dups", "equal", "sorted", "reversed"]


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("n", _edges(TILE_U64))
def test_sort_u64_tile_edges(ctx, n, pattern):
    rng = np.random.default_rng(n)
    keys = _keys(rng, n, 40, pattern)
    vals = np.arange(n, dtype=np.uint32)
    k2, v2 = ctx.debug_sort_u64(keys, vals, 40)
    perm = _expect(keys, 0, 40)
    assert np.array_equal(v2, perm)
    assert np.array_equal(k2, keys[perm])


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("n", _edges(TILE_U32))
def test_sort_u32_tile_edges(ctx, n, pattern):
    rng = np.random.default_rng(n + 1)
    keys = _keys(rng, n, 32, pattern, np.uint32)
    vals = np.arange(n, dtype=np.uint32)
    k2, v2 = ctx.debug_sort_u32(keys, vals, 32)
    perm = _expect(keys, 0, 32)
    assert np.array_equal(v2, perm)
    assert np.array_equal(k2, keys[perm])


@pytest.mark.parametrize("n", _edges(TILE_U128))
def test_sort_u128_tile_edges(ctx, n):
    rng = np.random.default_rng(n + 2)
    lo = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64)
    hi = rng.integers(0, 1 << 20, size=n, dtype=np.uint64)
    hi[rng.integers(0, n, size=n // 2)] = hi[0]
    lo[hi == hi[0]] &= np.uint64(0xff)           # equal keys among the duplicates: stability decides their order
    h2, l2, v2 = ctx.debug_sort_u128(hi, lo, np.arange(n, dtype=np.uint32), 84)
    perm = np.lexsort((lo, hi)).astype(np.uint32)   # lexsort is stable
    assert np.array_equal(v2, perm)
    assert np.array_equal(h2, hi[perm]) and np.array_equal(l2, lo[perm])


@pytest.mark.parametrize("lo_bit,bits", [(3, 17), (9, 7), (31, 1), (0, 1)])
@pytest.mark.parametrize("n", [TILE_U32 + 1, 3 * TILE_U32 + 1])
def test_sort_u32_bit_range(ctx, n, lo_bit, bits):
    rng = np.random.default_rng(n + lo_bit)
    keys = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    k2, v2 = ctx.debug_sort_u32(keys, np.arange(n, dtype=np.uint32), bits, lo_bit)
    perm = _expect(keys, lo_bit, bits)
    assert np.array_equal(v2, perm)
    assert np.array_equal(k2, keys[perm])


@pytest.mark.parametrize("lo_bit,bits", [(5, 20), (40, 24), (63, 1)])
def test_sort_u64_bit_range_tiles(ctx, lo_bit, bits):
    n = 3 * TILE_U64 + 1
    rng = np.random.default_rng(lo_bit)
    keys = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    k2, v2 = ctx.debug_sort_u64(keys, np.arange(n, dtype=np.uint32), bits, lo_bit)
    perm = _expect(keys, lo_bit, bits)
    assert np.array_equal(v2, perm)
    assert np.array_equal(k2, keys[perm])


def _scan_expect(x, base):
    out = np.zeros(x.size + 1, np.uint64)
    out[1:] = np.cumsum(x, dtype=np.uint64)
    return out + np.uint64(base)


@pytest.mark.parametrize("n", [0, 1, 2, SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1, 2 * SCAN_TILE, 33 * SCAN_TILE + 5, 100 * SCAN_TILE - 1])
@pytest.mark.parametrize("base", [0, 123_456_789_012])
def test_scan_tile_edges(ctx, n, base):
    rng = np.random.default_rng(n)
    x = rng.integers(0, 1000, size=n, dtype=np.uint32)
    assert np.array_equal(ctx.debug_scan_u32(x, base), _scan_expect(x, base))


def test_scan_total_above_2_32(ctx):
    n = 3_000_017
    rng = np.random.default_rng(5)
    x = rng.integers(1 << 12, 1 << 13, size=n, dtype=np.uint32)
    x[-1] = 0xffffffff
    out = ctx.debug_scan_u32(x, 17)
    assert int(out[-1]) > (1 << 32)
    assert np.array_equal(out, _scan_expect(x, 17))
