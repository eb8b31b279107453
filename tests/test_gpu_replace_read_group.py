"""--replace-read-group on the device (elp_set_replace_read_group): ingest accepts every RG state of a record and puts every read in @RG 0;
the byte outputs equal the restatement (tests/readgroup_ref.py) of SetRG followed by the field filters; a run with the replacement equals a
run whose records were rewritten on the host first; with the replacement off nothing changes."""
import struct

import numpy as np
import pytest

from elprep_b200 import _lib, bgzf, device, sam, synth
from outfilter import split_records
from readgroup_ref import set_rg_record, set_rg_sam
from samformat import bam_to_sam
from test_gpu_bgzf_egress import header_bytes, inflate_all
from util import encode_bam, set_side_inputs

pytestmark = pytest.mark.gpu

SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]
REPL = {"ID": "grp", "LB": "libR", "PU": "unitR"}
SR_TAG = b"sri\x01\x00\x00\x00"


def rg_state(k, two_z):
    """the RG fields of a record, by state k: none, the new ID, an ID of no @RG, non-Z types (i, f, B:f, H, A), two RG fields"""
    return [b"", b"RGZgrp\0", b"RGZnot_a_group\0", b"RGi" + struct.pack("<i", 5), b"RGf" + struct.pack("<f", 2.5),
            b"RGBf" + struct.pack("<I", 2) + struct.pack("<2f", 0.5, -1.25), b"RGH1AE3\0",
            b"RGAx" + (b"RGZother\0" if two_z else b"RGi" + struct.pack("<i", 9))][k % 8]


def workload(n_pairs, seed, two_z=True, with_aux=True):
    """synthetic reads whose records carry every RG state, the mixed optional fields of util.encode_bam (f and B fields among them) and,
    on every 13th record, the sr tag; -> (workload, one-@RG header of the replacement, records, offsets).  (Without with_aux the records
    are also valid SAM: the B:s field of util.encode_bam holds -2, which parseSamAlignment refuses.)"""
    w = synth.make_workload(n_pairs, SMALL, seed=seed)
    w.batch.rg[:] = -1
    extra = [rg_state(i, two_z) + (SR_TAG if i % 13 == 5 else b"") for i in range(w.batch.n)]
    w.batch.opt_flags[:] = [1 if i % 13 == 5 else 0 for i in range(w.batch.n)]
    raw, off = encode_bam(w.batch, w.header, np.random.default_rng(seed), extra_tags=extra, with_aux=with_aux)
    h = sam.Header(sq=w.header.SQ, rg=[REPL])
    return w, h, raw, off


def rewritten(raw, off, rg_id=b"grp"):
    """run B's input: every record rewritten by the restatement of SetRG"""
    recs = [set_rg_record(r, rg_id) for r in split_records(raw, off)]
    o = np.zeros(len(recs) + 1, np.uint64)
    o[1:] = np.cumsum([len(r) for r in recs])
    return np.frombuffer(b"".join(recs), np.uint8).copy(), o


def bgzf_file(w, raw):
    return bgzf.deflate(np.concatenate([np.frombuffer(header_bytes(w), np.uint8), raw]), level=1, write_eof=True).tobytes()


def ingest(ctx, how, w, raw, off):
    if how == "bam":
        ctx.append_bam(raw, off)
    elif how == "sam":
        names = [s["SN"].encode() for s in w.header.SQ]
        ctx.append_sam(b"".join(bam_to_sam(r, names) for r in split_records(raw, off)))
    else:
        f = bgzf_file(w, raw)
        for a in range(0, len(f), 65_537):
            ctx.append_bgzf(f[a:a + 65_537])
        ctx.append_bgzf_end()


def run(w, h, raw, off, replace, how="bam", ingest_mask=0, out_filter=None, profile=False, report=None):
    ctx = device.Context(h, profile=profile)
    set_side_inputs(ctx, w)
    if replace:
        ctx.set_replace_read_group(True)
    if ingest_mask:
        ctx.set_ingest_filter(ingest_mask, 10)
    if out_filter:
        ctx.set_output_filter(**out_filter)
    ingest(ctx, how, w, raw, off)
    ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
    ctx.bqsr_gather()
    ctx.bqsr_finalize(report)
    ctx.bqsr_apply()                                                      # ELP_ENORG if any read had no read group
    return ctx


@pytest.fixture(scope="module")
def wl():
    return workload(1500, 31)


@pytest.fixture(scope="module")
def wl_one_z():
    """the same reads without a second RG:Z field (run B's ingest must accept its records: the device resolves every RG:Z value)"""
    return workload(1500, 31, two_z=False)


@pytest.fixture(scope="module")
def wl_plain():
    return workload(1500, 37, with_aux=False)


@pytest.mark.parametrize("how", ["bam", "sam", "bgzf"])
@pytest.mark.parametrize("mask", [0, _lib.FILTER_UNMAPPED | _lib.FILTER_DUPLICATES])
def test_ingest_accepts_every_rg_state(wl, wl_plain, how, mask):
    w, h, raw, off = wl_plain if how == "sam" else wl
    ctx = run(w, h, raw, off, True, how=how, ingest_mask=mask)
    assert ctx.n > 0 and ctx.cov_names() == ["unitR"]
    assert ctx.n + ctx.n_filtered() == w.batch.n
    ctx.close()
    ctx = device.Context(h)                                               # without the replacement the unknown RG:Z values are refused, as before
    ctx.set_ingest_filter(mask, 10)
    with pytest.raises(device.ElprepError) as ei:
        ingest(ctx, how, w, raw, off)
    assert ei.value.code == _lib.EBAM and "not an @RG ID" in str(ei.value)
    ctx.close()


def test_malformed_rg_still_refused(wl):
    """structure is still checked: an RG:Z without its NUL fails the call whatever the filters"""
    w, h, raw, off = wl
    bad = split_records(raw, off)[:3]
    body = bad[0][4:] + b"RGZnul"
    bad[0] = struct.pack("<I", len(body)) + body
    for mask in (0, _lib.FILTER_UNMAPPED):
        ctx = device.Context(h)
        ctx.set_replace_read_group(True)
        ctx.set_ingest_filter(mask, 0)
        with pytest.raises(device.ElprepError) as ei:
            ctx.append_bam(np.frombuffer(b"".join(bad), np.uint8))
        assert ei.value.code == _lib.EBAM
        ctx.close()


def _outputs(ctx, n, ranges):
    b, s = ctx.fetch_bam(), ctx.fetch_sam()
    z = inflate_all(ctx.fetch_bgzf(eof=True).tobytes())
    parts = [(ctx.fetch_bam(a, m)[0].tobytes(), ctx.fetch_sam(a, m)[0].tobytes(), inflate_all(ctx.fetch_bgzf(a, m, eof=False).tobytes())) for a, m in ranges]
    return b[0].tobytes(), b[1], s[0].tobytes(), s[1], z, parts


def test_equivalent_to_host_rewrite(wl_one_z, tmp_path):
    """run A (replacement on) and run B (records rewritten on the host, replacement off) give the same result everywhere"""
    w, h, raw, off = wl_one_z
    rb, ob = rewritten(raw, off)
    a = run(w, h, raw, off, True, report=str(tmp_path / "a.recal"))
    b = run(w, h, rb, ob, False, report=str(tmp_path / "b.recal"))
    fa, fb = a.fetch(), b.fetch()
    for x, y in zip(fa, fb):
        assert np.array_equal(x, y)
    assert np.array_equal(a.tables_get(), b.tables_get())
    assert open(tmp_path / "a.recal").read() == open(tmp_path / "b.recal").read()
    assert a.optical_libraries() == b.optical_libraries() == ["Unknown Library", "libR"]
    assert str(a.optical_metrics()) == str(b.optical_metrics())          # (percent_duplication may be NaN)
    n = a.n_output()
    ranges = [(0, 1), (n - 1, 1), (n // 3, n // 2 + 7), (5, n - 11)]
    oa, ob_ = _outputs(a, n, ranges), _outputs(b, n, ranges)
    for x, y in zip(oa[:5], ob_[:5]):
        assert (x == y) if isinstance(x, bytes) else np.array_equal(x, y)
    assert oa[5] == ob_[5]
    a.close(); b.close()


def _patch(rec, flag, qual):
    r = bytearray(rec)
    r[18:20] = struct.pack("<H", int(flag))
    lname, ncig, lseq = r[12], struct.unpack_from("<H", r, 16)[0], struct.unpack_from("<i", r, 20)[0]
    q0 = 36 + lname + 4 * ncig + (lseq + 1) // 2
    r[q0:q0 + lseq] = bytes(qual)
    return bytes(r)


OUT = {
    "none": dict(),
    "dups_sr": dict(mask=_lib.OUT_REMOVE_DUPLICATES | _lib.OUT_REMOVE_OPTIONAL_READS),
    "remove_rg": dict(remove=("RG",)),
    "remove_xs": dict(remove=("XS", "NM")),
    "keep_rg": dict(keep=("RG", "XS", "ZB")),
    "keep_no_rg": dict(keep=("NM", "XS")),
    "keep_none": dict(keep=[]),
    "dups_remove_rg_keep": dict(mask=_lib.OUT_REMOVE_DUPLICATES, remove=("MD",), keep=("RG", "MD", "XS")),
}


@pytest.mark.parametrize("name", sorted(OUT))
def test_egress_equals_restatement(wl, name):
    w, h, raw, off = wl
    flt = OUT[name]
    ctx = run(w, h, raw, off, True, out_filter=flt)
    stored = split_records(raw, off)
    idx, flag, qoff, qual = ctx.fetch()
    optf = ctx.fetch_opt_flags()
    keep = np.ones(len(idx), bool)
    if flt.get("mask", 0) & _lib.OUT_REMOVE_DUPLICATES:
        keep &= (flag & 0x400) == 0
    if flt.get("mask", 0) & _lib.OUT_REMOVE_OPTIONAL_READS:
        keep &= optf == 0
    sel = np.nonzero(keep)[0]
    assert ctx.n_output() == len(sel) > 0
    rm, kp = flt.get("remove", ()), flt.get("keep")
    names = [s["SN"].encode() for s in h.SQ]
    want_bam = [_patch(set_rg_record(stored[int(idx[k])], b"grp", rm, kp), flag[k], qual[int(qoff[k]):int(qoff[k + 1])]) for k in sel]
    want_sam = [set_rg_sam(stored[int(idx[k])], b"grp", names, rm, kp, flag=flag[k], qual=qual[int(qoff[k]):int(qoff[k + 1])]) for k in sel]
    got_bam = split_records(*ctx.fetch_bam())
    got_sam = split_records(*ctx.fetch_sam())
    assert got_bam == want_bam
    assert got_sam == want_sam
    assert inflate_all(ctx.fetch_bgzf().tobytes()) == b"".join(want_bam)
    ctx.close()


def test_off_means_unchanged(wl_one_z):
    """never set, or set and turned off: the same kernels and the same bytes; on without a field filter: the field kernels run"""
    w, h, raw, off = wl_one_z
    rb, ob = rewritten(raw, off)
    res = []
    for mode in ("never", "on_off", "on"):
        ctx = device.Context(h, profile=True)
        set_side_inputs(ctx, w)
        if mode != "never":
            ctx.set_replace_read_group(True)
        if mode == "on_off":
            ctx.set_replace_read_group(False)
        ctx.append_bam(rb, ob)
        ctx.sort_markdup(device.SO_COORDINATE, True)
        ctx.reset_stats()
        out = (ctx.fetch_bam()[0].tobytes(), ctx.fetch_sam()[0].tobytes(), ctx.fetch_bgzf().tobytes())
        res.append((out, set(ctx.kernel_stats())))
        ctx.close()
    assert res[0] == res[1]
    assert "bam_format" in res[0][1] and not {"bam_out_fields_measure", "bam_out_fields_emit"} & res[0][1]
    assert {"bam_out_fields_measure", "bam_out_fields_emit"} <= res[2][1]
    assert res[2][0] == res[0][0]                                         # (these records already hold RG:Z:grp first)


def test_state_rules(wl):
    w, h, raw, off = wl
    for rg in ([], [REPL, {"ID": "x"}]):
        ctx = device.Context(sam.Header(sq=h.SQ, rg=rg))
        with pytest.raises(device.ElprepError) as ei:
            ctx.set_replace_read_group(True)
        assert ei.value.code == _lib.EINVAL
        ctx.close()
    ctx = device.Context(h)
    set_side_inputs(ctx, w)
    ctx.set_replace_read_group(True)
    ctx.append_bam(raw, off)
    for on in (True, False):
        with pytest.raises(device.ElprepError) as ei:
            ctx.set_replace_read_group(on)
        assert ei.value.code == _lib.ESTATE
    ctx.sort_markdup(device.SO_COORDINATE, True)
    first = ctx.fetch_sam()[0].tobytes()
    ctx.reset()                                                           # the setting survives
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_COORDINATE, True)
    assert ctx.fetch_sam()[0].tobytes() == first and b"\tRG:Z:grp" in first
    ctx.close()


def test_replacement_without_id(wl, tmp_path):
    """"PU:x" without ID: reads get RG:Z: (empty) and the covariate is "" (no @RG has ID "", so readGroupCovariate returns the read's value)"""
    w, _, raw, off = wl
    h = sam.Header(sq=w.header.SQ, rg=[sam.ParseHeaderLineFromString("PU:unitX SM:s")])
    a = run(w, h, raw, off, True, report=str(tmp_path / "a.recal"))
    assert a.cov_names() == [""]
    lines = split_records(*a.fetch_sam())
    assert all(b"\tRG:Z:\t" in ln or ln.endswith(b"\tRG:Z:\n") for ln in lines)
    _, _, raw2, off2 = workload(1500, 31, two_z=False)                   # (run B resolves every RG:Z value of its records)
    rb, ob = rewritten(raw2, off2, b"")
    b = run(w, sam.Header(sq=w.header.SQ, rg=[{"ID": ""}]), rb, ob, False, report=str(tmp_path / "b.recal"))
    a2 = run(w, h, raw2, off2, True, report=str(tmp_path / "a2.recal"))
    assert open(tmp_path / "a2.recal").read() == open(tmp_path / "b.recal").read()
    assert np.array_equal(a2.fetch()[3], b.fetch()[3])
    assert a2.fetch_bam()[0].tobytes() == b.fetch_bam()[0].tobytes()
    a.close(); a2.close(); b.close()


def test_at_size():
    """two million reads through BGZF in and out: the inflated output equals that of the records rewritten by the restatement"""
    w = synth.make_workload(1_000_000, [("chr1", 60_000_000), ("chr2", 30_000_000)], seed=2026, threads=16, want_reference=False)
    w.batch.rg[::7] = -1                                                  # some reads without RG
    raw, off = synth.encode_bam(w.batch, w.header, threads=16)
    h = sam.Header(sq=w.header.SQ, rg=[REPL])
    b_batch_rg = np.where(w.batch.rg < 0, 0, w.batch.rg).astype(np.int32)
    rg_a = w.batch.rg.copy()
    w.batch.rg[:] = b_batch_rg
    hb = sam.Header(sq=w.header.SQ, rg=[{"ID": "grp"}] * len(w.header.RG))
    rb, ob = synth.encode_bam(w.batch, hb, threads=16)                    # RG:Z:grp where the RG field was, or behind the last field
    w.batch.rg[:] = rg_a
    sa, sb = split_records(raw, off[:201]), split_records(rb, ob[:201])
    assert [set_rg_record(r, b"grp") for r in sa] == sb                   # (the host rewrite is the restatement's)
    outs = []
    for data, o, replace in ((raw, off, True), (rb, ob, False)):
        ctx = device.Context(h)
        if replace:
            ctx.set_replace_read_group(True)
        f = bgzf_file(w, data)
        for a in range(0, len(f), 64 << 20):
            ctx.append_bgzf(f[a:a + (64 << 20)])
        ctx.append_bgzf_end()
        assert ctx.n == w.batch.n
        ctx.sort_markdup(device.SO_COORDINATE, True)
        outs.append(bgzf.inflate(ctx.fetch_bgzf(prefix=header_bytes(w))).tobytes())   # (gzip.decompress is quadratic in the number of members)
        ctx.close()
    assert outs[0] == outs[1]
