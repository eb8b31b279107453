"""The colliding QNAMEs the mate-join tests rely on still collide under the numpy restatement of the join hash, and the restatement
agrees with a plain scalar one (Python integers, one byte at a time)."""
from markdup_edges import COLLIDING_LENGTHS, COLLIDING_PAIRS, COLLIDING_TRIPLE, candidates, find_colliding, join_hash, join_key


def _scalar_join_hash(name, lib):
    m64, m32 = (1 << 64) - 1, (1 << 32) - 1
    h = 0
    for k in range(0, len(name), 4):
        w = int.from_bytes(name[k:k + 4].ljust(4, b"\0"), "little")
        m = ((w ^ ((k * 0x9E3779B1) & m32)) * 0x85EBCA6B) & m32
        m ^= m >> 15
        m = (m * 0xC2B2AE35) & m32
        m ^= m >> 13
        h = (h + m * 0x9E3779B97F4A7C15) & m64
    x = (h + (lib + 1) * 0x9E3779B97F4A7C15 + len(name)) & m64
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & m64
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & m64
    x ^= x >> 33
    return x


def test_restatement_matches_scalar():
    names = [bytes((i * 7 + j * 13 + 33) % 94 + 33 for j in range(L)) for i, L in enumerate(list(range(0, 40)) + [127, 128, 253, 254])]
    for lib in (-1, 0, 1, 5):
        got = join_hash(names, lib)
        assert [int(v) for v in got] == [_scalar_join_hash(s, lib) for s in names], lib


def test_colliding_names_collide():
    for a, b in COLLIDING_PAIRS:
        assert a != b and len(a) == len(b)
        ka, kb = join_key([a, b])
        assert ka == kb
        assert join_hash([a])[0] != join_hash([b])[0]          # equal join keys, different full hashes
    t = join_key(list(COLLIDING_TRIPLE))
    assert len(set(COLLIDING_TRIPLE)) == 3 and t[0] == t[1] == t[2]
    a, b = COLLIDING_LENGTHS
    assert len(a) != len(b) and join_key([a])[0] == join_key([b])[0]
    # the library is part of the key: in another library the names no longer share it
    assert join_key([COLLIDING_PAIRS[0][0]], 1)[0] != join_key([COLLIDING_PAIRS[0][1]], 1)[0]


def test_pair_search_finds_the_committed_pairs():
    found = find_colliding(candidates("pA:", 1 << 17))
    assert sorted(tuple(g) for g in found) == sorted(COLLIDING_PAIRS)
