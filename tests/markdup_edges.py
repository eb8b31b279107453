"""The mate join's (library, QNAME) hash restated in numpy, and the QNAMEs whose join keys collide.

Duplicate marking pairs the mates of true-pair reads by sorting them on a 31-bit key, the low bits of a 64-bit hash of the
library and the QNAME (markdup.cu: qname_hash, mix64, the library/length term of adapt_kernel), and compares bytes inside runs of
equal key.  A run that is not a mate pair is rare at test sizes, so the names below are searched for once (find_colliding, a
birthday search) and committed: test_markdup_edges_cpu.py checks that they still collide under this restatement and the GPU tests
check the restatement against the device hash."""
import numpy as np

M64 = (1 << 64) - 1
GOLD64 = 0x9E3779B97F4A7C15


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def mix64(x):
    x = _u64(x).copy()
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xff51afd7ed558ccd)
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xc4ceb9fe1a85ec53)
    x ^= x >> np.uint64(33)
    return x


def name_hash(names, length):
    """qname_hash of names given as a uint8 matrix [n, >= length] (bytes past `length` are ignored): little-endian 4-byte
    words, zero past the name's end, each mixed with its offset and summed with a 64-bit wrapping product"""
    names = np.asarray(names, dtype=np.uint8)
    n = names.shape[0]
    nw = (length + 3) // 4
    buf = np.zeros((n, 4 * nw), np.uint8)
    buf[:, :length] = names[:, :length]
    words = buf.view("<u4").astype(np.uint32)
    h = np.zeros(n, np.uint64)
    with np.errstate(over="ignore"):
        for w in range(nw):
            m = (words[:, w] ^ np.uint32((4 * w * 0x9E3779B1) & 0xffffffff)) * np.uint32(0x85EBCA6B)
            m ^= m >> np.uint32(15)
            m *= np.uint32(0xC2B2AE35)
            m ^= m >> np.uint32(13)
            h += m.astype(np.uint64) * np.uint64(GOLD64)
    return h


def join_hash(names, lib=0):
    """the 64-bit hash adapt_kernel stores for a true-pair read: names is a list of bytes, lib the library index of the read's
    read group (-1: none)"""
    libs = np.broadcast_to(np.asarray(lib, dtype=np.int64), (len(names),))
    out = np.zeros(len(names), np.uint64)
    lens = np.array([len(s) for s in names], dtype=np.int64)
    for L in np.unique(lens):
        sel = np.flatnonzero(lens == L)
        mat = np.frombuffer(b"".join(names[i] for i in sel), np.uint8).reshape(sel.size, int(L)) if L else np.zeros((sel.size, 0), np.uint8)
        h = name_hash(mat, int(L))
        with np.errstate(over="ignore"):
            t = h + (libs[sel] + 1).astype(np.uint64) * np.uint64(GOLD64) + np.uint64(L)
        out[sel] = mix64(t)
    return out


def join_key(names, lib=0):
    return join_hash(names, lib) & np.uint64(0x7fffffff)


def candidates(prefix, count, start=0):
    """`count` distinct names prefix + a fixed-width base-36 number"""
    digits = "0123456789abcdefghijklmnopqrstuvwxyz"
    width = 1
    while 36 ** width < start + count:
        width += 1
    v = np.arange(start, start + count, dtype=np.int64)
    cols = []
    for _ in range(width):
        cols.append(v % 36)
        v //= 36
    table = np.frombuffer(digits.encode(), np.uint8)
    body = table[np.stack(cols[::-1], axis=1)]
    pre = np.broadcast_to(np.frombuffer(prefix.encode(), np.uint8), (count, len(prefix)))
    mat = np.ascontiguousarray(np.concatenate([pre, body], axis=1))
    return [bytes(r) for r in mat]


def find_colliding(names, lib=0, k=2):
    """groups of >= k names (in input order) with equal join keys"""
    key = join_key(names, lib)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    lens = np.diff(np.r_[starts, ks.size])
    return [[names[i] for i in sorted(order[s:s + l])] for s, l in zip(starts, lens) if l >= k]


# Found with find_colliding (library 0):
#   pairs    candidates("pA:", 1 << 17)
#   triples  candidates("tR:", 1 << 22)
#   lengths  candidates("dL:", 1 << 16) + candidates("dL:x", 1 << 16): one name one byte longer than the other
COLLIDING_PAIRS = [(b"pA:0zk3", b"pA:2om5"), (b"pA:1dsr", b"pA:1xw9"), (b"pA:1syy", b"pA:1ujf")]
COLLIDING_TRIPLE = (b"tR:00ley", b"tR:06udp", b"tR:1k5cr")
COLLIDING_LENGTHS = (b"dL:0j16", b"dL:x08m5")
