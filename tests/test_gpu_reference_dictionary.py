"""--rename-chromosomes and --replace-reference-sequences on the device (elp_set_input_dictionary): ingest remaps and drops as the
reference's filters and AddREFID do, the byte outputs equal the restatement (tests/refdict_ref.py), a run with the setting equals a run
over records rewritten on the host into a context without it, CleanSam reads the input LN, and with the setting off nothing changes."""
import struct

import numpy as np
import pytest

from elprep_b200 import _lib, bgzf, device, sam, synth
from outfilter import split_records
from readgroup_ref import set_rg_record, set_rg_sam
from refdict_ref import refdict_record, refdict_sam, renamed
from samformat import bam_to_sam
from test_gpu_bgzf_egress import inflate_all
from util import encode_bam

pytestmark = pytest.mark.gpu

SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]
R, P = _lib.DICT_RENAME_CHROMOSOMES, _lib.DICT_REPLACE
OUT_REV = ["chrM", "chr20"]                                               # reversed and a subset: chr21 is dropped
REPL_RG = {"ID": "grp", "LB": "libR", "PU": "unitR"}


def setup(mode, w):
    """-> (input names as in the file, output header) of a mode over a workload whose contigs are chr20, chr21, chrM"""
    names = [s["SN"] for s in w.header.SQ]
    inp = [n[3:] for n in names] if mode & R else names
    out = OUT_REV if mode & P else names
    ln = {s["SN"]: int(s["LN"]) for s in w.header.SQ}
    return inp, sam.Header(sq=[{"SN": n, "LN": ln[n]} for n in out], rg=w.header.RG)


def side_inputs(ctx, w, h):
    wi = {s["SN"]: i for i, s in enumerate(w.header.SQ)}
    for j, s in enumerate(h.SQ):
        ctx.set_reference(j, w.contig_bases[wi[s["SN"]]])
        ctx.set_known_sites(j, w.sites[wi[s["SN"]]], already_flat=True)


def bam_header(names, lens, text=b"@HD\tVN:1.6\tSO:coordinate\n"):
    return b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(names)) + b"".join(
        struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", int(l)) for n, l in zip(names, lens))


def ingest(ctx, how, raw, off, inp, lens):
    if how == "bam":
        ctx.append_bam(raw, off)
    elif how == "sam":
        ctx.append_sam(b"".join(bam_to_sam(r, [n.encode() for n in inp]) for r in split_records(raw, off)))
    else:
        f = bgzf.deflate(np.concatenate([np.frombuffer(bam_header(inp, lens), np.uint8), raw]), level=1, write_eof=True).tobytes()
        for a in range(0, len(f), 65_537):
            ctx.append_bgzf(f[a:a + 65_537])
        ctx.append_bgzf_end()


REGIONS = {"chr20": [[1000, 200_000], [350_000, 590_000]], "chr21": [[0, 300_000]], "chrM": [[0, 16_000]]}


def run(w, h, raw, off, mode, inp, how="bam", mask=0, out_filter=None, rg_replace=False, report=None, profile=False, lens=None):
    ctx = device.Context(h, profile=profile)
    side_inputs(ctx, w, h)
    if mode:
        ctx.set_input_dictionary(mode, inp, lens if lens is not None else w.header.contig_lengths())
    if rg_replace:
        ctx.set_replace_read_group(True)
    if mask:
        for j, s in enumerate(h.SQ):
            ctx.set_target_regions(j, np.array(REGIONS[s["SN"]], np.int32))
        ctx.set_ingest_filter(mask, 0)
    if out_filter:
        ctx.set_output_filter(**out_filter)
    ingest(ctx, how, raw, off, inp, lens if lens is not None else w.header.contig_lengths())
    ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
    ctx.bqsr_gather()
    ctx.bqsr_finalize(report)
    ctx.bqsr_apply()
    return ctx


def rewritten(raw, off, inp, mode, out_names):
    """run B's input: the records the restatement keeps, as it writes them"""
    recs = [refdict_record(r, [n.encode() for n in inp], mode, [n.encode() for n in out_names]) for r in split_records(raw, off)]
    recs = [r for r in recs if r is not None]
    o = np.zeros(len(recs) + 1, np.uint64)
    o[1:] = np.cumsum([len(r) for r in recs])
    return np.frombuffer(b"".join(recs), np.uint8).copy(), o


@pytest.fixture(scope="module")
def wl():
    w = synth.make_workload(1500, SMALL, seed=41, cross_contig_frac=0.05)
    raw, off = encode_bam(w.batch, w.header, np.random.default_rng(41), with_aux=False)   # (valid SAM as well)
    return w, raw, off


MODES = [R, P, R | P]


def _bam_wo_bin(recs):
    return [r[:14] + r[16:] for r in recs]                                # (SAM ingest computes bin; encode_bam writes a constant)


@pytest.mark.parametrize("how", ["bam", "sam", "bgzf"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("mask", [0, _lib.FILTER_UNMAPPED | _lib.FILTER_TARGET_REGIONS])
def test_modes(wl, mode, how, mask):
    """kept count, FLAG, QUAL and outputs of every mode and ingest path equal those of a context fed the host-rewritten records"""
    w, raw, off = wl
    inp, h = setup(mode, w)
    out_names = [s["SN"] for s in h.SQ]
    rb, ob = rewritten(raw, off, inp, mode, out_names)
    a = run(w, h, raw, off, mode, inp, how=how, mask=mask)
    b = run(w, h, rb, ob, 0, inp, mask=mask)
    assert a.n == b.n > 0
    assert a.n + a.n_filtered() == w.batch.n and b.n + b.n_filtered() == len(ob) - 1
    if mode & P:
        assert len(ob) - 1 < w.batch.n                                    # (the replacement dropped the chr21 reads)
    for x, y in zip(a.fetch(), b.fetch()):
        assert np.array_equal(x, y)
    ba, bb = split_records(*a.fetch_bam()), split_records(*b.fetch_bam())
    assert (_bam_wo_bin(ba) == _bam_wo_bin(bb)) if how == "sam" else (ba == bb)
    # SAM: A prints the renamed input strings, B the output names of the rewritten ids; the lines differ only where RNEXT names a dropped
    # contig: A keeps the name, B writes "*"
    got, want = split_records(*a.fetch_sam()), split_records(*b.fetch_sam())
    assert len(got) == len(want) == a.n
    for g, x in zip(got, want):
        gf, xf = g.split(b"\t"), x.split(b"\t")
        assert gf[:6] + gf[7:] == xf[:6] + xf[7:]
        assert gf[6] == xf[6] or (xf[6] == b"*" and gf[6] in (b"chr21", b"21"))
    a.close(); b.close()


def _outputs(ctx, ranges):
    z = inflate_all(ctx.fetch_bgzf(eof=True).tobytes())
    parts = [(ctx.fetch_bam(a, m)[0].tobytes(), inflate_all(ctx.fetch_bgzf(a, m, eof=False).tobytes())) for a, m in ranges]
    return ctx.fetch_bam()[0].tobytes(), z, parts


def test_equivalent_to_host_rewrite(wl, tmp_path):
    """run A (rename + reversed subset replacement) and run B (records rewritten on the host, setting off) agree everywhere"""
    w, raw, off = wl
    mode = R | P
    inp, h = setup(mode, w)
    rb, ob = rewritten(raw, off, inp, mode, OUT_REV)
    a = run(w, h, raw, off, mode, inp, report=str(tmp_path / "a.recal"))
    b = run(w, h, rb, ob, 0, inp, report=str(tmp_path / "b.recal"))
    for x, y in zip(a.fetch(), b.fetch()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.tables_get(), b.tables_get())
    assert open(tmp_path / "a.recal").read() == open(tmp_path / "b.recal").read()
    assert a.optical_libraries() == b.optical_libraries()
    assert str(a.optical_metrics()) == str(b.optical_metrics())
    n = a.n_output()
    ranges = [(0, 1), (n - 1, 1), (n // 3, n // 2 + 7), (5, n - 11)]
    assert _outputs(a, ranges) == _outputs(b, ranges)
    a.close(); b.close()


def _patch(rec, flag, qual):
    r = bytearray(rec)
    r[18:20] = struct.pack("<H", int(flag))
    lname, ncig, lseq = r[12], struct.unpack_from("<H", r, 16)[0], struct.unpack_from("<i", r, 20)[0]
    q0 = 36 + lname + 4 * ncig + (lseq + 1) // 2
    r[q0:q0 + lseq] = bytes(qual)
    return bytes(r)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("flt", [dict(), dict(mask=_lib.OUT_REMOVE_DUPLICATES, remove=("RG",)), dict(keep=("RG", "NM"))])
def test_egress_equals_restatement(wl, mode, flt):
    """BAM, BGZF and SAM output against the restatement, with the output filters and --replace-read-group on"""
    w, raw, off = wl
    inp, h0 = setup(mode, w)
    h = sam.Header(sq=h0.SQ, rg=[REPL_RG])
    out_names = [s["SN"].encode() for s in h.SQ]
    in_b = [n.encode() for n in inp]
    ctx = run(w, h, raw, off, mode, inp, out_filter=flt, rg_replace=True)
    stored = [r for r in split_records(raw, off) if refdict_record(r, in_b, mode, out_names) is not None]
    idx, flag, qoff, qual = ctx.fetch()
    keep = np.ones(len(idx), bool)
    if flt.get("mask", 0) & _lib.OUT_REMOVE_DUPLICATES:
        keep &= (flag & 0x400) == 0
    sel = np.nonzero(keep)[0]
    rm, kp = flt.get("remove", ()), flt.get("keep")
    want_bam = [_patch(set_rg_record(refdict_record(stored[int(idx[k])], in_b, mode, out_names), b"grp", rm, kp), flag[k], qual[int(qoff[k]):int(qoff[k + 1])]) for k in sel]
    want_sam = [set_rg_sam(stored[int(idx[k])], b"grp", renamed(in_b, mode), rm, kp, flag=flag[k], qual=qual[int(qoff[k]):int(qoff[k + 1])]) for k in sel]
    assert refdict_sam(stored[0], in_b, mode, out_names) is not None
    assert split_records(*ctx.fetch_bam()) == want_bam
    assert split_records(*ctx.fetch_sam()) == want_sam
    assert inflate_all(ctx.fetch_bgzf().tobytes()) == b"".join(want_bam)
    ctx.close()


def test_clean_sam_reads_input_ln(wl):
    """CleanSam runs before the replacement: a context whose input chr20 is 590 000 long clips there although the output says 600 000"""
    w, raw, off = wl
    mode = P
    inp, h = setup(mode, w)                                               # output chrM, chr20 (600 000)
    lens = np.array([590_000, 300_000, 16_569], np.int32)                 # the input's LN of chr20, chr21, chrM
    rb, ob = rewritten(raw, off, inp, mode, OUT_REV)
    res = []
    for hh, data, o, m in ((h, raw, off, mode), (sam.Header(sq=[{"SN": "chrM", "LN": 16_569}, {"SN": "chr20", "LN": 590_000}], rg=w.header.RG), rb, ob, 0),
                           (h, rb, ob, 0)):
        ctx = device.Context(hh)
        if m:
            ctx.set_input_dictionary(m, inp, lens)
        ctx.append_bam(data, o)
        k = ctx.clean_sam()
        res.append((k, [x.copy() for x in ctx.debug_cigar()]))
        ctx.close()
    assert res[0][0] == res[1][0] > 0 and res[2][0] < res[0][0]
    for x, y in zip(res[0][1], res[1][1]):
        assert np.array_equal(x, y)


def _sam_line(qname, rname, pos, rnext, pnext=5):
    return b"\t".join([qname, b"0", rname, b"%d" % pos, b"30", b"4M", rnext, b"%d" % pnext, b"0", b"ACGT", b"IIII"]) + b"\n"


@pytest.mark.parametrize("mode", [P, R | P])
def test_sam_names(mode):
    """SAM RNAME / RNEXT that name only the replacement, neither dictionary, "=" or "*" """
    rn = (lambda s: b"chr" + s) if mode & R else (lambda s: s)
    inp = ["1", "2"]
    out = [rn(b"3").decode(), rn(b"1").decode()]
    h = sam.Header(sq=[{"SN": out[0], "LN": 1000}, {"SN": out[1], "LN": 1000}], rg=[])
    text = (_sam_line(b"a", b"3", 10, b"=") + _sam_line(b"b", b"1", 20, b"3") + _sam_line(b"c", b"2", 30, b"1") + _sam_line(b"d", b"zz", 40, b"1")
            + _sam_line(b"e", b"*", 0, b"*") + _sam_line(b"f", b"1", 50, b"2") + _sam_line(b"g", b"chr3", 60, b"=") + _sam_line(b"h", b"1", 70, b"="))
    ctx = device.Context(h)
    ctx.set_input_dictionary(mode, inp, [1000, 1000])
    ctx.append_sam(text)
    assert ctx.n == 5 and ctx.n_filtered() == 3                           # c (RNAME "2"), d (neither) and g ("chr3" / "chrchr3") are dropped
    ctx.sort_markdup(device.SO_KEEP, 0)
    lines = split_records(*ctx.fetch_sam())
    got = [ln.split(b"\t")[:7] for ln in lines]
    assert got == [[b"a", b"0", rn(b"3"), b"10", b"30", b"4M", b"="], [b"b", b"0", rn(b"1"), b"20", b"30", b"4M", rn(b"3")],
                   [b"e", b"0", b"*", b"0", b"30", b"4M", b"*"], [b"f", b"0", rn(b"1"), b"50", b"30", b"4M", rn(b"2")],
                   [b"h", b"0", rn(b"1"), b"70", b"30", b"4M", b"="]]
    bam = split_records(*ctx.fetch_bam())
    assert [struct.unpack_from("<ii", r, 4)[0] for r in bam] == [0, 1, -1, 1, 1]
    assert [struct.unpack_from("<i", r, 24)[0] for r in bam] == [0, 0, -1, -1, 1]
    ctx.close()
    ctx = device.Context(h)                                               # an RNEXT that reaches nothing is lost, as before
    ctx.set_input_dictionary(mode, inp, [1000, 1000])
    ctx.append_sam(_sam_line(b"x", b"1", 5, b"zz"))
    ctx.sort_markdup(device.SO_KEEP, 0)
    assert struct.unpack_from("<i", ctx.fetch_bam()[0].tobytes(), 24)[0] == -1
    with pytest.raises(device.ElprepError) as ei:
        ctx.fetch_sam()
    assert ei.value.code == _lib.ESTATE
    ctx.close()


def test_off_means_unchanged(wl):
    w, raw, off = wl
    res = []
    for state in ("never", "on_off"):
        ctx = device.Context(w.header, profile=True)
        side_inputs(ctx, w, w.header)
        if state == "on_off":
            ctx.set_input_dictionary(R | P, ["20", "21", "M"], w.header.contig_lengths())
            ctx.set_input_dictionary(0)
        ctx.set_ingest_filter(_lib.FILTER_UNMAPPED, 0)
        ctx.append_bam(raw, off)
        ctx.append_sam(b"".join(bam_to_sam(r, [s["SN"].encode() for s in w.header.SQ]) for r in split_records(raw, off)[:300]))
        ctx.sort_markdup(device.SO_COORDINATE, True)
        out = (ctx.fetch()[1].tobytes(), ctx.fetch_bam()[0].tobytes(), ctx.fetch_bgzf().tobytes())
        res.append((out, set(ctx.kernel_stats())))
        ctx.close()
    assert res[0] == res[1]


def test_state_rules(wl):
    w, raw, off = wl
    names = [s["SN"] for s in w.header.SQ]
    lens = w.header.contig_lengths()
    ctx = device.Context(w.header)
    L = ctx.L
    for bad in (4, 8 | P):
        assert L.elp_set_input_dictionary(ctx.h, bad, None, None, 0) == _lib.EINVAL
    assert L.elp_set_input_dictionary(ctx.h, P, None, None, -1) == _lib.EINVAL
    with pytest.raises(device.ElprepError) as ei:
        ctx.set_input_dictionary(R, names[:2], lens[:2])                  # RENAME alone: the counts differ
    assert ei.value.code == _lib.EINVAL
    with pytest.raises(device.ElprepError) as ei:
        ctx.set_input_dictionary(R, names, lens)                          # "chr" + "chr20" is not "chr20"
    assert ei.value.code == _lib.EINVAL
    ctx.set_input_dictionary(R, [n[3:] for n in names], lens)
    ctx.append_bam(raw, off)
    for m in (0, P):
        with pytest.raises(device.ElprepError) as ei:
            ctx.set_input_dictionary(m, names, lens)
        assert ei.value.code == _lib.ESTATE
    ctx.sort_markdup(device.SO_COORDINATE, True)
    first = ctx.fetch_sam()[0].tobytes()
    ctx.reset()                                                           # the setting survives
    ctx.append_bam(raw, off)
    ctx.sort_markdup(device.SO_COORDINATE, True)
    assert ctx.fetch_sam()[0].tobytes() == first
    ctx.close()
    # BGZF: the header's reference list is checked against the input dictionary; an open file refuses the call
    inp, h = setup(R | P, w)
    f = bgzf.deflate(np.concatenate([np.frombuffer(bam_header(inp, lens), np.uint8), raw]), level=1, write_eof=True).tobytes()
    ctx = device.Context(h)
    ctx.append_bgzf(f[:1000])
    with pytest.raises(device.ElprepError) as ei:
        ctx.set_input_dictionary(R | P, inp, lens)
    assert ei.value.code == _lib.ESTATE
    ctx.close()
    for bad_names, bad_lens in ((["20", "21", "X"], lens), (inp, lens + 1), (inp[:2], lens[:2])):
        ctx = device.Context(h)
        ctx.set_input_dictionary(R | P, bad_names, bad_lens)
        with pytest.raises(device.ElprepError) as ei:
            ctx.append_bgzf(f)
            ctx.append_bgzf_end()
        assert ei.value.code == _lib.EINVAL and "input dictionary" in str(ei.value)
        ctx.close()


def test_at_size():
    """two million reads through BGZF in and out, rename plus a reversed replacement: the output equals that of the rewritten records"""
    w = synth.make_workload(1_000_000, [("chr1", 60_000_000), ("chr2", 30_000_000)], seed=2027, threads=16, want_reference=False)
    raw, off = synth.encode_bam(w.batch, w.header, threads=16)
    inp, lens = ["1", "2"], w.header.contig_lengths()
    h = sam.Header(sq=[{"SN": "chr2", "LN": 30_000_000}, {"SN": "chr1", "LN": 60_000_000}], rg=w.header.RG)
    rm = np.array([1, 0, -1], np.int32)                                   # (index -1: "*")
    b = w.batch
    b.refid, b.nref = rm[b.refid], rm[b.nref]
    rb, ob = synth.encode_bam(b, h, threads=16)                           # every read kept: both contigs are in the new dictionary
    sa, sb = split_records(raw, off[:201]), split_records(rb, ob[:201])
    assert [refdict_record(r, [b"1", b"2"], R | P, [b"chr2", b"chr1"]) for r in sa] == sb
    outs = []
    for data, o, mode in ((raw, off, R | P), (rb, ob, 0)):
        ctx = device.Context(h)
        if mode:
            ctx.set_input_dictionary(mode, inp, lens)
        hdr = bam_header(inp, lens) if mode else bam_header(["chr2", "chr1"], [30_000_000, 60_000_000])
        f = bgzf.deflate(np.concatenate([np.frombuffer(hdr, np.uint8), data]), level=1, write_eof=True).tobytes()
        for a in range(0, len(f), 64 << 20):
            ctx.append_bgzf(f[a:a + (64 << 20)])
        ctx.append_bgzf_end()
        assert ctx.n == w.batch.n
        ctx.sort_markdup(device.SO_COORDINATE, True)
        outs.append(bgzf.inflate(ctx.fetch_bgzf(prefix=bam_header(["chr2", "chr1"], [30_000_000, 60_000_000]))).tobytes())
        ctx.close()
    assert outs[0] == outs[1]
