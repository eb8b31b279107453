"""FLAG, output order and duplication metrics of one duplicate-marking run against the oracle, and the radix-sort launches it
should take: a Python restatement of the packed key widths of phase_markdup (fragment groups, mate join, pair groups) and of the
coordinate sort's long-tie rounds."""
import os
import tempfile

import numpy as np

from coordsort_ref import F_NEXTUNMAPPED, F_PAIRED, passes as _passes, tie_rounds


def _tie_passes(b, n_contigs, bP):
    """digit passes of the long-tie rounds: for every chunk of the secondary key (coordsort_ref.chunk_keys), the bits that differ
    among the elements of runs of more than 32 equal coordinate keys"""
    return sum(_passes(bits) for _, _, bits in tie_rounds(b, n_contigs, bP))


def _joined_pairs(b, h, true_pair):
    """pairs the mate join forms: DeleteOrStore on (library, QNAME) over the true-pair reads in arrival order"""
    lib_of = {}
    for rg in h.RG:
        if rg.get("LB"):
            lib_of.setdefault(rg["LB"], len(lib_of))
    rg_lib = [lib_of[rg["LB"]] if rg.get("LB") else -1 for rg in h.RG]
    stored, n = set(), 0
    for i in np.flatnonzero(true_pair):
        g = int(b.rg[i])
        k = (rg_lib[g] if 0 <= g < len(rg_lib) else -1, bytes(b.qname[b.qname_off[i]:b.qname_off[i + 1]]))
        if k in stored:
            stored.remove(k)
            n += 1
        else:
            stored.add(k)
    return n


def expected_sorts(b, h, optical=True):
    """(u64 passes, u128 passes) of one elp_sort_markdup(coordinate, optical or not) over batch b, whose FLAG already carries the
    duplicate bits (the coordinate sort runs after duplicate marking and its modFlag chunk sees them)"""
    import oracle
    n_contigs = len(h.SQ)
    n_lib = len({rg["LB"] for rg in h.RG if rg.get("LB")})
    bR, bL = n_contigs.bit_length(), (n_lib + 1).bit_length()
    upos, _ = oracle.mark_duplicates(b.copy(), h, want_adapt=True)
    entering = (b.flag & 0x904) == 0
    true_pair = entering & ((b.flag & (F_PAIRED | F_NEXTUNMAPPED)) == F_PAIRED)
    bU = int(upos[entering].astype(np.int64).max() - upos[entering].astype(np.int64).min()).bit_length() if entering.any() else 0
    bP = int(max(0, b.pos.max())).bit_length()
    u64 = _passes(1 + bP + bR) + _tie_passes(b, n_contigs, bP)
    u128 = 0
    if entering.any():
        u64 += _passes(1 + bU + bR + bL)
    if true_pair.sum() >= 2:
        u64 += 4                                   # mate join: 32-bit keys
        pair_bits = 2 * bU + 2 + 2 * bR + bL
        if _joined_pairs(b, h, true_pair) < (1 if optical else 2):
            pass                                   # no pair signature to sort (optical marking still visits a single pair)
        elif pair_bits <= 64:
            u64 += _passes(pair_bits)
        else:
            u128 += _passes(pair_bits)
    return u64, u128


def check(b, h, pixel=100, optical=True):
    """FLAG, order, duplication metrics and the metrics file text against the oracle; the sort widths and pass counts against
    expected_sorts.  optical=False: MarkDuplicates alone, for inputs on which the reference's optical pass panics (a QNAME used by
    more than one pair re-joins differently in coordinate order: "origin for duplicate read pair unknown").
    Returns (the FLAG column in arrival order, kernel_stats())"""
    import oracle
    from elprep_b200 import device, _lib
    b1 = b.copy()
    oracle.mark_duplicates(b1, h, n_threads=1)
    perm = oracle.coordinate_sort(b1, n_threads=4)
    b2 = b.copy()
    if not optical:
        return _check_markdup_only(b, h, b1, perm)
    with tempfile.TemporaryDirectory() as tmp:
        om = oracle.markdup_optical(b2, h, order=perm, pixel_distance=pixel, metrics_path=os.path.join(tmp, "o.txt"), command_line="elprep filter in out", started_on="T")
        assert np.array_equal(b1.flag, b2.flag)
        ctx = device.Context(h, optical_pixel_distance=pixel, profile=True)
        try:
            ctx.append(b)
            ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
            idx, flag, _, _ = ctx.fetch()
            assert np.array_equal(idx, perm.astype(np.uint64)), "output order differs"
            assert np.array_equal(flag, b2.flag[perm]), "FLAG differs"
            for slot, g in enumerate(ctx.optical_metrics()):
                for k_g, k_o in zip(_lib.ElpDupMetrics.COUNTERS, oracle.COUNTERS):
                    assert g[k_g] == om.counters[slot][k_o], (slot, k_g)
                assert g["hist"] == om.hist[slot], slot
                assert g["estimated_library_size"] == om.library_size[slot]
            ctx.print_duplicates_metrics(os.path.join(tmp, "g.txt"), "elprep filter in out", "T")
            stats = ctx.kernel_stats()
        finally:
            ctx.close()
        with open(os.path.join(tmp, "g.txt")) as fg, open(os.path.join(tmp, "o.txt")) as fo:
            assert fg.read() == fo.read(), "metrics file text differs"
    u64, u128 = expected_sorts(b2, h)
    assert stats.get("radix_onesweep_u64", {}).get("launches", 0) == u64
    assert stats.get("radix_onesweep_u128", {}).get("launches", 0) == u128
    return b2.flag, stats


def _check_markdup_only(b, h, b1, perm):
    from elprep_b200 import device, _lib
    ctx = device.Context(h, profile=True)
    try:
        ctx.append(b)
        ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP)
        idx, flag, _, _ = ctx.fetch()
        assert np.array_equal(idx, perm.astype(np.uint64)), "output order differs"
        assert np.array_equal(flag, b1.flag[perm]), "FLAG differs"
        stats = ctx.kernel_stats()
    finally:
        ctx.close()
    u64, u128 = expected_sorts(b1, h, optical=False)
    assert stats.get("radix_onesweep_u64", {}).get("launches", 0) == u64
    assert stats.get("radix_onesweep_u128", {}).get("launches", 0) == u128
    return b1.flag, stats
