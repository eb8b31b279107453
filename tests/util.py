"""Shared helpers for the parity tests: run the same workload through the oracle (CPU restatement of the
reference) and through the CUDA library (C ABI via ctypes), and return comparable results."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_check(name, directory):
    """tests/c/<name>.cpp built with -O2 against the library's headers and zlib -> the executable's path"""
    exe = os.path.join(str(directory), name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "elprep_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "c", name + ".cpp"), "-lz"])
    return exe


@pytest.fixture(scope="module")
def host_encoder(tmp_path_factory):
    """run(data, eof, tmp) -> the BGZF bytes of the host build of deflate.cuh (deflate_check deflate); run.exe is the binary"""
    exe = build_check("deflate_check", tmp_path_factory.mktemp("deflate"))

    def run(data, eof, tmp):
        src, dst = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bgzf")
        with open(src, "wb") as f:
            f.write(data)
        subprocess.check_call([exe, "deflate", src, dst, "1" if eof else "0"])
        return open(dst, "rb").read()
    run.exe = exe
    return run


def oracle_pipeline(w, bqsr=True, threads=4, max_cycle=500, quantize_levels=0, sqq=None, sort=True, markdup=True):
    import oracle
    b = w.batch.copy()
    if markdup:
        oracle.mark_duplicates(b, w.header, n_threads=1)
    perm = oracle.coordinate_sort(b, n_threads=threads) if sort else np.arange(b.n, dtype=np.int64)
    srt = b.take(perm)
    res = dict(perm=perm.astype(np.uint64), flag=srt.flag.copy(), qual=srt.qual.copy(), qual_off=srt.qual_off.copy())
    if bqsr:
        ref = oracle.Reference(w.header, w.contig_bases, w.sites)
        t = oracle.bqsr_gather(srt, w.header, ref, max_cycle=max_cycle, n_threads=threads)
        oracle.bqsr_finalize(t)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "o.recal")
            oracle.bqsr_report(t, oracle.OracleHeader(w.header).cov_names, p)
            res["report"] = open(p).read()
        oracle.bqsr_apply(srt, w.header, t, quantize_levels=quantize_levels, sqq=sqq, n_threads=threads)
        res["qual"] = srt.qual.copy()
        res["tables"] = t
    return res


def compare_bqsr(g, o, max_cycle=500):
    """gpu_pipeline vs oracle_pipeline results, bit for bit: order, FLAG, table counters, EmpiricalQuality, report text, QUAL bytes"""
    assert np.array_equal(g["perm"], o["perm"]), "output order differs"
    assert np.array_equal(g["flag"], o["flag"]), "FLAG differs"
    assert np.array_equal(g["qual_off"], o["qual_off"])
    d, e = oracle_tables_dense(o["tables"], max_cycle)
    assert np.array_equal(g["tables"], d), "BQSR table counters differ"
    assert np.array_equal(g["emp"], e), "EmpiricalQuality differs"
    assert g["report"] == o["report"], "recalibration report text differs"
    assert np.array_equal(g["qual"], o["qual"]), "QUAL bytes differ"


def oracle_tables_dense(t, max_cycle=500):
    """oracle tables -> the C ABI's dense layout [n_cov][94][1+(2mc+1)+16][2] (+ empirical [..][..][..])"""
    n_cov = t.n_cov
    ncol = 1 + (2 * max_cycle + 1) + 16
    d = np.zeros((n_cov, 94, ncol, 2), dtype=np.int64)
    e = np.zeros((n_cov, 94, ncol), dtype=np.uint8)
    d[:, :, 0, 0] = t.q_obs[:, :94]; d[:, :, 0, 1] = t.q_mis[:, :94]; e[:, :, 0] = t.q_emp[:, :94]
    d[:, :, 1:1 + 2 * max_cycle + 1, 0] = t.c_obs[:, :94]; d[:, :, 1:1 + 2 * max_cycle + 1, 1] = t.c_mis[:, :94]; e[:, :, 1:1 + 2 * max_cycle + 1] = t.c_emp[:, :94]
    d[:, :, 1 + 2 * max_cycle + 1:, 0] = t.x_obs[:, :94]; d[:, :, 1 + 2 * max_cycle + 1:, 1] = t.x_mis[:, :94]; e[:, :, 1 + 2 * max_cycle + 1:] = t.x_emp[:, :94]
    assert t.q_obs[:, 94:].sum() == 0 and t.c_obs[:, 94:].sum() == 0
    return d, e


SYNTH_QUALS = (2, 12, 23, 37)      # the four QUAL levels of the synthetic generator (Q4 in synth.cpp)


def with_qual_alphabet(w, values, seed=0):
    """A copy of workload ``w`` whose QUAL arena uses exactly ``values``: the generator's four levels map monotonically onto the sorted
    targets; with more targets than levels, each level is split between neighbouring targets by a seeded RNG.  Duplicate scores and
    BQSR both follow from QUAL, so the oracle simply runs on the remapped batch."""
    from elprep_b200 import synth
    vals = sorted(set(int(v) for v in values))
    k = len(vals)
    assert k >= 1 and 0 <= vals[0] and vals[-1] <= 93
    q = w.batch.qual
    assert set(np.nonzero(np.bincount(q, minlength=256))[0].tolist()) <= set(SYNTH_QUALS), "with_qual_alphabet starts from the generator's four levels"
    groups = []
    for i in range(4):
        lo = i * k // 4
        groups.append(np.array(vals[lo:max(lo + 1, (i + 1) * k // 4)], dtype=np.uint8))
    rng = np.random.default_rng(seed)
    out = np.empty_like(q)
    step = 1 << 24                                    # chunks keep the temporaries small on C1-sized arenas
    for s in range(0, q.size, step):
        qs, os_ = q[s:s + step], out[s:s + step]
        r = rng.integers(0, 1 << 16, size=qs.size, dtype=np.uint16)
        for lv, g in zip(SYNTH_QUALS, groups):
            m = qs == lv
            os_[m] = g[r[m] % g.size]
    b = w.batch.copy()
    b.qual = out
    assert np.nonzero(np.bincount(out, minlength=256))[0].tolist() == vals, "the remapped workload does not use exactly the requested QUAL alphabet"
    return synth.Workload(w.header, b, w.contig_bases, w.sites, dict(w.params, quals=tuple(vals)))


def fast_plan(values, n_cov, lseq_max):
    """Restatement of plan_fast (csrc/bqsr_gather.cu): (S, sh) of the bqsr_count_kernel instance the library picks for a QUAL alphabet,
    or None when the general kernels gather."""
    vals = sorted(set(int(v) for v in values))
    slots = [q for q in vals if q >= 6]
    if max(vals) > 93 or not slots or len(slots) > 4 or len(vals) > 8:
        return None
    if n_cov < 1 or 2 * n_cov > 64 or not 1 <= lseq_max <= 1024:
        return None
    for sh in range(5):
        if len({(q >> sh) & 7 for q in vals}) == len(vals):
            return len(slots), sh
    return None


def apply_plan(values, n_cov, lseq_max, max_cycle=500):
    """Which apply kernel elp_bqsr_apply picks (run_apply_kernel / build_compact_lut): "v2" (bqsr_apply2_kernel, compact table in
    shared memory) when the table of the QUAL values >= 6 present fits 80 KB, else "gmem" (bqsr_apply_kernel, global table).  Values 6..93
    have a slot each; all values above 93 share one more."""
    S = sum(1 for q in set(values) if 6 <= q <= 93) + (1 if any(q > 93 for q in values) else 0)
    Lc = max(1, min(max_cycle, lseq_max))
    blk = n_cov * S * 17
    blk += 1 - (blk & 1)
    nbytes = ((2 * Lc + 1 + 64) * blk + 15) // 16 * 16
    return "v2" if S and n_cov and nbytes <= 80 * 1024 and lseq_max <= min(Lc, 1024) else "gmem"


def bqsr_paths(stats):
    """(gather, apply) kernels a profiled context ran, from kernel_stats(): gather "fast" (bqsr_count_kernel, with bqsr_g_prep only for the
    reads it hands to the general kernels) or "general" (bqsr_prep + bqsr_chunk over every read); apply "v2" or "gmem"."""
    fast, general = "bqsr_g_count" in stats, "bqsr_g_chunk" in stats
    assert not (fast and general), sorted(stats)
    if fast:
        assert "bqsr_g_count_indel" in stats and "bqsr_g_prep2" in stats, sorted(stats)
    v2, gmem = "bqsr_apply" in stats, "bqsr_apply_gmem" in stats
    assert not (v2 and gmem), sorted(stats)
    return ("fast" if fast else "general" if general else None), ("v2" if v2 else "gmem" if gmem else None)


def gpu_pipeline(w, bqsr=True, n_batches=1, max_cycle=500, quantize_levels=0, sqq=None, sort=True, markdup=True, profile=False, keep_ctx=False):
    from elprep_b200 import device
    ctx = device.Context(w.header, max_cycle=max_cycle, quantize_levels=quantize_levels, sqq=sqq, profile=profile)
    try:
        if bqsr:
            set_side_inputs(ctx, w)
        n = w.batch.n
        if n_batches <= 1 or n < n_batches:
            ctx.append(w.batch)
        else:
            bounds = [n * i // n_batches for i in range(n_batches + 1)]
            for a, b in zip(bounds[:-1], bounds[1:]):
                ctx.append(w.batch.take(np.arange(a, b)))
        res = gpu_phases(ctx, bqsr=bqsr, sort=sort, markdup=markdup, profile=profile)
        if keep_ctx:
            res["ctx"] = ctx
        return res
    finally:
        if not keep_ctx:
            ctx.close()


def set_side_inputs(ctx, w):
    for ci in range(len(w.header.SQ)):
        ctx.set_reference(ci, w.contig_bases[ci])
        ctx.set_known_sites(ci, w.sites[ci], already_flat=True)


def gpu_phases(ctx, bqsr=True, sort=True, markdup=True, profile=False):
    """sort + duplicate marking (+ BQSR gather, finalize, apply) over the reads already appended to ``ctx``, then fetch"""
    from elprep_b200 import device
    ctx.sort_markdup(device.SO_COORDINATE if sort else device.SO_KEEP, markdup)
    res = {}
    if bqsr:
        ctx.bqsr_gather()
        res["tables"] = ctx.tables_get()
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "g.recal")
            ctx.bqsr_finalize(p)
            res["report"] = open(p).read()
        res["emp"] = ctx.empirical_get()
        ctx.bqsr_apply()
    idx, flag, qoff, qual = ctx.fetch()
    res.update(perm=idx, flag=flag, qual=qual[:int(qoff[-1])] if ctx.n else qual[:0], qual_off=qoff)
    if profile:
        res["stats"] = ctx.kernel_stats()
    res["launches"] = ctx.launch_count()
    return res


# ---- BAM alignment records (sam/bam-files.go:300-400) for the device ingest tests ----
def encode_bam(batch, header, rng=None, with_aux=True, extra_tags=None):
    """AlignmentBatch -> (uint8 record bytes, uint64 record offsets [n+1]).  Each record carries its block_size, the fixed
    fields of parseBamAlignment, NUL-terminated name, CIGAR words, SEQ nibbles, QUAL bytes and typed optional fields
    (RG:Z plus a mix of the other value types, so that the tag walk is exercised)."""
    import struct
    rng = rng or np.random.default_rng(0)
    ids = [r["ID"] for r in header.RG]
    out, offs = bytearray(), [0]
    qo, co = batch.qname_off.astype(np.int64), batch.cigar_off.astype(np.int64)
    so, uo = batch.seq_off.astype(np.int64), batch.qual_off.astype(np.int64)
    for i in range(batch.n):
        name = bytes(batch.qname[qo[i]:qo[i + 1]]) + b"\0"
        cig = batch.cigar[co[i]:co[i + 1]].astype("<u4").tobytes()
        L = int(batch.lseq[i])
        seq = bytes(batch.seq[so[i]:so[i] + (L + 1) // 2]); qual = bytes(batch.qual[uo[i]:uo[i] + L])
        aux = b""
        if with_aux:
            k = int(rng.integers(0, 4))
            if k >= 1: aux += b"NMC" + struct.pack("<B", int(rng.integers(0, 9)))
            if k >= 2: aux += b"MDZ" + b"75A74\0"
            if int(batch.rg[i]) >= 0: aux += b"RGZ" + ids[int(batch.rg[i])].encode() + b"\0"
            if k >= 3: aux += b"ASi" + struct.pack("<i", -5) + b"XSf" + struct.pack("<f", 1.5) + b"ZBBs" + struct.pack("<I", 3) + struct.pack("<3h", 1, -2, 3) + b"XAA" + b"q"
        elif int(batch.rg[i]) >= 0:
            aux += b"RGZ" + ids[int(batch.rg[i])].encode() + b"\0"
        if extra_tags is not None:
            aux += extra_tags[i]
        body = struct.pack("<iiBBHHHiiii", int(batch.refid[i]), int(batch.pos[i]) - 1, len(name), int(batch.mapq[i]), 4680, (co[i + 1] - co[i]) & 0xffff,
                           int(batch.flag[i]), L, int(batch.nref[i]), int(batch.pnext[i]) - 1, int(batch.tlen[i])) + name + cig + seq + qual + aux
        out += struct.pack("<I", len(body)) + body
        offs.append(len(out))
    return np.frombuffer(bytes(out), dtype=np.uint8).copy(), np.array(offs, dtype=np.uint64)


def decode_bam(raw, offs, header):
    """restatement of parseBamAlignment (sam/bam-files.go:314-400) for the fields of the path -> AlignmentBatch"""
    import struct
    from elprep_b200 import sam
    ids = {r["ID"]: k for k, r in enumerate(header.RG)}
    cols = {k: [] for k in ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg", "lseq")}
    qn, cg, sq, ql, qoff, coff = bytearray(), [], bytearray(), bytearray(), [0], [0]
    b = raw.tobytes()
    sizes = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}
    for i in range(len(offs) - 1):
        r = b[int(offs[i]):int(offs[i + 1])]
        bs, refid, pos, lname, mapq, _bin, ncig, flag, lseq, nref, pnext, tlen = struct.unpack_from("<IiiBBHHHiiii", r, 0)
        assert bs + 4 == len(r)
        x = 36
        qn += r[x:x + lname - 1]; qoff.append(len(qn)); x += lname
        cg += list(struct.unpack_from("<%dI" % ncig, r, x)); coff.append(len(cg)); x += 4 * ncig
        sq += r[x:x + (lseq + 1) // 2]; x += (lseq + 1) // 2
        ql += r[x:x + lseq]; x += lseq
        rg = -1
        while x < len(r):
            tag, ty = r[x:x + 2], chr(r[x + 2]); x += 3
            if ty in sizes: x += sizes[ty]
            elif ty in "ZH":
                e = r.index(b"\0", x)
                if tag == b"RG" and ty == "Z": rg = ids[r[x:e].decode()]
                x = e + 1
            elif ty == "B":
                sub, cnt = chr(r[x]), struct.unpack_from("<I", r, x + 1)[0]; x += 5 + cnt * sizes[sub]
            else: raise ValueError("bad type")
        for k, v in zip(cols, (refid, pos + 1, flag, mapq, nref, pnext + 1, tlen, rg, lseq)):
            cols[k].append(v)
    return sam.AlignmentBatch(qname_off=np.array(qoff, np.uint64), qname=np.frombuffer(bytes(qn), np.uint8), cigar_off=np.array(coff, np.uint64),
                              cigar=np.array(cg, np.uint32), seq=np.frombuffer(bytes(sq), np.uint8), qual=np.frombuffer(bytes(ql), np.uint8).copy(),
                              **{k: np.array(v) for k, v in cols.items()})
