"""elp_load_known_sites on the device: .elsites files parsed, sorted and flattened into the known-sites table, against the restatement of
intervals.FromElsitesFile + NewBaseRecalibrator (elsites_ref), at chunk sizes that put every case on a staging-chunk edge."""
import ctypes as C

import numpy as np
import pytest

import elsites_cases as ec
import elsites_ref as er
import knownsites_cases as kc
from elprep_b200 import _lib, device, sam
from util import gpu_phases

pytestmark = pytest.mark.gpu

CHUNKS = [1, 7, 64, 0]   # 0: the default


def _header(names, ln=1 << 30):
    return sam.Header(sq=[{"SN": n, "LN": ln} for n in names])


def _write(tmp_path, files, tag="f"):
    paths = []
    for i, data in enumerate(files):
        p = tmp_path / f"{tag}{i}.elsites"
        p.write_bytes(data)
        paths.append(str(p))
    return paths


def _tables(ctx, n):
    return [ctx.known_sites(ci) for ci in range(n)]


def _assert_tables(got, want):
    assert len(got) == len(want)
    for ci, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), (ci, g[:8].tolist(), w[:8].tolist(), len(g), len(w))


@pytest.mark.parametrize("chunk", CHUNKS)
def test_known_answers(tmp_path, chunk):
    ctx = device.Context(_header(ec.NAMES))
    try:
        ctx.debug_set_sites_chunk(chunk)
        for cid, files, _, _ in ec.VALID:
            want, wu = er.load(files, ec.NAMES)
            nu = ctx.load_known_sites(_write(tmp_path, files, cid))
            assert nu == wu, cid
            _assert_tables(_tables(ctx, len(ec.NAMES)), want)
    finally:
        ctx.close()


@pytest.mark.parametrize("chunk", [7, 0])
def test_refusals(tmp_path, chunk):
    """every malformed form is ELP_ESITES naming the file and line; the previous table stays, and a valid load succeeds afterwards"""
    ctx = device.Context(_header(ec.NAMES))
    try:
        ctx.debug_set_sites_chunk(chunk)
        good = ec.VALID[0][1]
        ctx.load_known_sites(_write(tmp_path, good, "good"))
        before = _tables(ctx, len(ec.NAMES))
        for cid, files, (fi, line, reason) in ec.INVALID:
            with pytest.raises(er.ElsitesError):
                er.load(files, ec.NAMES)
            with pytest.raises(device.ElprepError) as ei:
                ctx.load_known_sites(_write(tmp_path, files, cid))
            msg = str(ei.value)
            assert ei.value.code == _lib.ESITES, (cid, msg)
            assert f"(file {fi}), line {line} " in msg, (cid, msg)
            _assert_tables(_tables(ctx, len(ec.NAMES)), before)
        missing = str(tmp_path / "does_not_exist.elsites")
        with pytest.raises(device.ElprepError) as ei:
            ctx.load_known_sites([_write(tmp_path, good, "g2")[0], missing])
        assert ei.value.code == _lib.EINVAL and missing in str(ei.value)
        _assert_tables(_tables(ctx, len(ec.NAMES)), before)
        want, _ = er.load(ec.VALID[1][1], ec.NAMES)
        ctx.load_known_sites(_write(tmp_path, ec.VALID[1][1], "after"))
        _assert_tables(_tables(ctx, len(ec.NAMES)), want)
    finally:
        ctx.close()


def test_context_without_contig_names(tmp_path):
    L = _lib.load()
    lens = np.full(2, 1000, np.int32)
    cfg = _lib.ElpConfig(0, 2, None, lens.ctypes.data_as(C.c_void_p), 0, None, None, None, 500, 0, None, 0, b"GATK", 100, 0)
    h = C.c_void_p()
    assert L.elp_create(C.byref(cfg), C.byref(h)) == 0
    try:
        paths = _write(tmp_path, ec.VALID[0][1])
        arr = (C.c_char_p * 1)(paths[0].encode())
        assert L.elp_load_known_sites(h, arr, 1, None) == _lib.EINVAL
        assert b"contig_names" in L.elp_last_error(h)
        assert L.elp_known_sites_get(h, 0, None, 0) == 0
    finally:
        L.elp_destroy(h)


# ---- seeded random files ----
RANDOM_NAMES = [f"chr{i}" for i in range(1, 23)] + ["chrX", "chrY", "chrM", "chr1_alt", "chr10_alt", "dupA", "dupA", "swallow"]
EXTRA = ["chrUn_gl000220", "chr1_random", "chr"]   # not @SQ SN: unmatched, but still validated


def _random_files(seed, n_lines=3_000_000):
    rng = np.random.default_rng(seed)
    names = sorted(set(RANDOM_NAMES)) + EXTRA
    weights = rng.random(len(names)) + 0.2
    per = np.maximum(1, (weights / weights.sum() * n_lines).astype(np.int64))
    expect = {}
    rows = []   # (name, starts, ends) blocks
    for name, k in zip(names, per):
        if name == "swallow":
            # one interval over all others, more than ParallelFlatten's grain: the left half swallows the right one (Go panics there)
            s = rng.integers(0, 100_000, size=6000)
            e = s + rng.integers(0, 30, size=6000)
            s[17], e[17] = -5, 10_000_000
        else:
            s = rng.integers(0, 5_000_000, size=k)
            ln = rng.integers(-3, 60, size=k)                      # end < start, touching and overlapping intervals
            e = s + ln
            dup = np.flatnonzero(rng.random(k) < 0.05)             # duplicates of the previous line
            s[dup], e[dup] = s[dup - 1], e[dup - 1]
        if name == "chrM":
            s[:4] = [-2**31, 2**31 - 1, -2**31, 0]
            e[:4] = [2**31 - 1, 2**31 - 1, -2**31, -2**31]
        # split every chromosome into a few blocks, spread over the three files in shuffled order
        cuts = np.sort(rng.integers(0, len(s), size=3))
        for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(s)]):
            if b > a:
                rows.append((name, s[a:b], e[a:b]))
    order = rng.permutation(len(rows))
    files = [[], [], []]
    for j, r in enumerate(order):
        files[j % 3].append(rows[r])
    # the intervals of a chromosome in file order: with end < start among equal starts, the stable sort keeps that order and it matters
    for blocks in files:
        for name, s, e in blocks:
            if name not in EXTRA:
                expect.setdefault(name, []).append(np.stack([s, e], 1))
    out = []
    for fi, blocks in enumerate(files):
        lines = []
        for name, s, e in blocks:
            nb = name.encode()
            lines += [b"%s\t%d\t%d" % (nb, a, b) for a, b in zip(s.tolist(), e.tolist())]
        if fi == 1:   # CRLF lines in the middle file
            body = b"".join(x + (b"\r\n" if i % 3 == 0 else b"\n") for i, x in enumerate(lines))
        elif fi == 2:  # no final '\n'
            body = b"\n".join(lines)
        else:
            body = b"\n".join(lines) + b"\n"
        out.append(er.HEADER + body)
    unmatched = int(sum(per[names.index(x)] for x in EXTRA))
    tables = [er.sort_flatten_fast(np.concatenate(expect[n])) if n in expect else np.zeros((0, 2), np.int32) for n in RANDOM_NAMES]
    return out, tables, unmatched


def test_random_files(tmp_path):
    files, want, wu = _random_files(seed=5)
    paths = _write(tmp_path, files, "rnd")
    total = sum(len(f) for f in files)
    assert sum(len(w) for w in want) > 0 and max(len(w) for w in want) > 4096
    ctx = device.Context(_header(RANDOM_NAMES), profile=True)
    try:
        for chunk in (0, total // 50 + 1):
            ctx.debug_set_sites_chunk(chunk)
            assert ctx.load_known_sites(paths) == wu
            _assert_tables(_tables(ctx, len(RANDOM_NAMES)), want)
        st = ctx.kernel_stats()
        for k in ("sites_lines", "sites_parse", "sites_sort", "sites_flatten"):
            assert k in st and st[k]["launches"] > 0, sorted(st)
    finally:
        ctx.close()


def test_same_as_array_path(tmp_path):
    """the same intervals through a file and through elp_set_known_sites(already_flat = 0) give the same table and the same BQSR run"""
    w, _ = kc.build(kc.handoff_cases(60) + kc.overflow_cases(60), (2, 11, 25, 37, 40), n_rg=2, seed=3)
    flat = w.sites[0]
    rng = np.random.default_rng(1)
    part = flat[rng.permutation(len(flat))[: len(flat) // 2]]
    raw = np.concatenate([flat, part, np.stack([part[:, 0], np.maximum(part[:, 0], part[:, 1] - 1)], 1)])   # duplicates and contained pieces
    raw = raw[rng.permutation(len(raw))]
    name = w.header.SQ[0]["SN"]
    path = _write(tmp_path, [er.write([(name, int(s), int(e)) for s, e in raw])], "bq")
    res = []
    for mode in ("file", "array"):
        ctx = device.Context(w.header)
        try:
            for ci in range(len(w.header.SQ)):
                ctx.set_reference(ci, w.contig_bases[ci])
            if mode == "file":
                assert ctx.load_known_sites(path) == 0
            else:
                ctx.set_known_sites(0, raw, already_flat=False)
            t = ctx.known_sites(0)
            ctx.append(w.batch)
            r = gpu_phases(ctx)
            r["sites"] = t
            res.append(r)
        finally:
            ctx.close()
    a, b = res
    assert np.array_equal(a["sites"], b["sites"]) and np.array_equal(a["sites"], flat)
    assert np.array_equal(a["tables"], b["tables"]) and a["report"] == b["report"]
    assert np.array_equal(a["emp"], b["emp"]) and np.array_equal(a["qual"], b["qual"]) and np.array_equal(a["perm"], b["perm"])


def test_lifetime(tmp_path):
    names = ["c0", "c1", "c2"]
    f1 = _write(tmp_path, [er.write([("c0", 1, 5), ("c1", 10, 20), ("c2", 3, 3)])], "l1")
    f2 = _write(tmp_path, [er.write([("c1", 7, 8)])], "l2")
    ctx = device.Context(_header(names))
    try:
        ctx.set_known_sites(2, [[100, 200]])
        ctx.load_known_sites(f1)                        # replaces every contig
        assert [t.tolist() for t in _tables(ctx, 3)] == [[[1, 5]], [[10, 20]], [[3, 3]]]
        ctx.set_known_sites(1, [[50, 60], [55, 70]], already_flat=False)   # one contig, inside the loaded block
        ctx.set_known_sites(0, [])
        assert [t.tolist() for t in _tables(ctx, 3)] == [[], [[50, 70]], [[3, 3]]]
        ctx.reset()                                     # the table survives elp_reset
        assert [t.tolist() for t in _tables(ctx, 3)] == [[], [[50, 70]], [[3, 3]]]
        ctx.load_known_sites(f2)                        # load -> load: contigs without sites are emptied
        assert [t.tolist() for t in _tables(ctx, 3)] == [[], [[7, 8]], []]
        ctx.load_known_sites([])                        # clears all
        assert [t.tolist() for t in _tables(ctx, 3)] == [[], [], []]
        ctx.load_known_sites(f1)
    finally:
        ctx.close()                                     # load -> destroy
    ctx = device.Context(_header(names))
    ctx.load_known_sites(f1)
    ctx.close()
    with pytest.raises(device.ElprepError):
        device.Context(_header(names)).known_sites(3)
