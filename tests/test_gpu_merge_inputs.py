"""Several input files in one context (elp_add_input, elp_select_input, elp_set_tag_rename): three lane files with different @SQ orders
and colliding @RG / @PG IDs, merged by sam.MergeInputs, go through BAM, SAM and BGZF ingest (run A).  Run B ingests the same records,
rewritten on the host into the merged header, into a plain context.  Everything the two runs compute and write must be equal."""
import struct

import numpy as np
import pytest

from elprep_b200 import _lib, bgzf, device, sam, synth
from outfilter import fields, split_records
from samformat import bam_to_sam
from test_gpu_bgzf_egress import inflate_all
from util import encode_bam

pytestmark = pytest.mark.gpu

BASE = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]
EXTRA = {"chrX": 5_000, "chrY": 4_000}
# lane @SQ orders: mergeable, each a different map to the merged [chrX, chr20, chrY, chr21, chrM]
LANE_SQ = [["chr20", "chr21", "chrM"], ["chrX", "chr20", "chr21", "chrM"], ["chr20", "chrY", "chr21", "chrM"]]
LANE_RG = [["1", "2"], ["1", "1S"], ["1S", "2"]]
LANE_PG = [["bwa"], ["bwa"], ["bwa", "samtools"]]
SUFFIX = "S"


def lane_header(k):
    ln = dict(BASE, **EXTRA)
    h = sam.Header(sq=[{"SN": s, "LN": ln[s]} for s in LANE_SQ[k]],
                   rg=[{"ID": i, "LB": "lib" + "AB"[j], "PU": f"u{k}{j}"} for j, i in enumerate(LANE_RG[k])])
    h.PG = [{"ID": p} for p in LANE_PG[k]]
    return h


def tag_fields(i, k):
    """RG and PG fields of record i of lane k, in either order; PG sometimes missing (BQSR needs every read in a read group)"""
    rg = b"RGZ" + LANE_RG[k][i % 2].encode() + b"\0"
    pg = b"PGZ" + LANE_PG[k][i % len(LANE_PG[k])].encode() + b"\0" if i % 3 else b""
    return rg + pg if i % 2 else pg + rg


def host_rewrite(rec, sq_map, rg_map, pg_map):
    """run B's record: refID / next_refID through the input's map, the first RG and PG value through the maps (SetRG / SetPG)"""
    r = bytearray(rec)
    for at in (4, 24):
        v = struct.unpack_from("<i", r, at)[0]
        if v >= 0:
            struct.pack_into("<i", r, at, sq_map[v])
    t0, fl = fields(bytes(r))
    parts, seen = [bytes(r[4:t0])], set()
    for tag, s, e in fl:
        f = bytes(r[s:e])
        if tag in (b"RG", b"PG") and tag not in seen:
            seen.add(tag)
            m = rg_map if tag == b"RG" else pg_map
            v = f[3:-1].decode()
            if v in m:
                f = f[:3] + m[v].encode() + b"\0"
        parts.append(f)
    body = b"".join(parts)
    return struct.pack("<I", len(body)) + body


def pack(recs):
    o = np.zeros(len(recs) + 1, np.uint64)
    o[1:] = np.cumsum([len(x) for x in recs])
    return np.frombuffer(b"".join(recs), np.uint8).copy(), o


def bam_file(h, raw):
    text = b"@HD\tVN:1.6\n"
    hb = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(h.SQ)) + b"".join(
        struct.pack("<i", len(s["SN"]) + 1) + s["SN"].encode() + b"\0" + struct.pack("<i", int(s["LN"])) for s in h.SQ)
    return bgzf.deflate(np.concatenate([np.frombuffer(hb, np.uint8), raw]), level=1, write_eof=True).tobytes()


def make_lanes(n_pairs, seed, with_aux=True):
    w = synth.make_workload(n_pairs, BASE, seed=seed)
    heads = [lane_header(k) for k in range(3)]
    merged, sq_maps, rg_map, pg_map = sam.MergeInputs(heads, SUFFIX)
    assert rg_map == {"1": "1SS", "1S": "1SS", "2": "2S"} and pg_map == {"bwa": "bwaS"}
    b = w.batch
    lane = np.arange(b.n) % 3                                  # mates land in different files
    b.rg[:] = -1
    recs = []
    for k in range(3):                                         # the base contig c of read i is entry LANE_SQ[k].index(name) of lane k
        idx = np.nonzero(lane == k)[0]
        lb = b.take(idx)
        to_lane = np.array([LANE_SQ[k].index(n) for n, _ in BASE], np.int32)
        lb.refid[:] = np.where(lb.refid >= 0, to_lane[np.maximum(lb.refid, 0)], lb.refid)
        lb.nref[:] = np.where(lb.nref >= 0, to_lane[np.maximum(lb.nref, 0)], lb.nref)
        raw, off = encode_bam(lb, heads[k], np.random.default_rng(seed + k), with_aux=with_aux, extra_tags=[tag_fields(int(i), k) for i in idx])
        recs.append(split_records(raw, off))
    b_recs = [host_rewrite(r, sq_maps[k], rg_map, pg_map) for k in range(3) for r in recs[k]]
    base_to_merged = [merged.contig_names().index(n) for n, _ in BASE]
    return dict(w=w, heads=heads, merged=merged, maps=(sq_maps, rg_map, pg_map), lanes=recs, b=b_recs, base_to_merged=base_to_merged)


def side_inputs(ctx, L):
    for c, m in enumerate(L["base_to_merged"]):
        ctx.set_reference(m, L["w"].contig_bases[c])
        ctx.set_known_sites(m, L["w"].sites[c], already_flat=True)


def ingest(ctx, how, header, recs):
    raw, off = pack(recs)
    if how == "bam":
        ctx.append_bam(raw, off)
    elif how == "sam":
        names = [s["SN"].encode() for s in header.SQ]
        ctx.append_sam(b"".join(bam_to_sam(r, names) for r in recs))
    else:
        f = bam_file(header, raw)
        for a in range(0, len(f), 65_537):
            ctx.append_bgzf(f[a:a + 65_537])
        ctx.append_bgzf_end()


REPL = {"ID": "grp", "LB": "libR", "PU": "unitR"}


def ctx_header(L, replace):
    h = sam.Header(sq=L["merged"].SQ, rg=[REPL] if replace else L["merged"].RG)
    return h


def run_a(L, how, replace=False, out_filter=None, mask=0, report=None):
    ctx = device.Context(ctx_header(L, replace))
    side_inputs(ctx, L)
    sq_maps, rg_map, pg_map = L["maps"]
    ids = [ctx.add_input([s["SN"] for s in h.SQ], [int(s["LN"]) for s in h.SQ]) for h in L["heads"]]
    assert ids == [0, 1, 2]
    ctx.set_tag_rename("RG", rg_map)
    ctx.set_tag_rename("PG", pg_map)
    return finish(ctx, replace, out_filter, mask, report, lambda: [(ctx.select_input(k), ingest(ctx, how, L["heads"][k], L["lanes"][k])) for k in range(3)])


def run_b(L, how, replace=False, out_filter=None, mask=0, report=None):
    ctx = device.Context(ctx_header(L, replace))
    side_inputs(ctx, L)
    return finish(ctx, replace, out_filter, mask, report, lambda: ingest(ctx, how, L["merged"], L["b"]))


def finish(ctx, replace, out_filter, mask, report, do_ingest):
    if replace:
        ctx.set_replace_read_group(True)
    if mask:
        ctx.set_ingest_filter(mask, 10)
    if out_filter:
        ctx.set_output_filter(**out_filter)
    do_ingest()
    ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
    ctx.bqsr_gather()
    ctx.bqsr_finalize(report)
    ctx.bqsr_apply()
    return ctx


@pytest.fixture(scope="module")
def lanes():
    return make_lanes(1200, 41)


@pytest.fixture(scope="module")
def lanes_sam():
    return make_lanes(1200, 43, with_aux=False)      # (util.encode_bam's B:s field holds -2, which parseSamAlignment refuses)


OUT = {"none": None, "remove_rg_pg": dict(remove=("RG", "PG")), "keep": dict(mask=_lib.OUT_REMOVE_DUPLICATES, keep=("RG", "PG", "NM"))}


def outputs(ctx):
    n = ctx.n_output()
    ranges = [(0, 1), (n - 1, 1), (n // 3, n // 2 + 7)]
    b, s = ctx.fetch_bam(), ctx.fetch_sam()
    return [b[0].tobytes(), b[1], s[0].tobytes(), s[1], inflate_all(ctx.fetch_bgzf(eof=True).tobytes())] + \
           [(ctx.fetch_bam(a, m)[0].tobytes(), inflate_all(ctx.fetch_bgzf(a, m, eof=False).tobytes())) for a, m in ranges]


@pytest.mark.parametrize("how", ["bam", "sam", "bgzf"])
@pytest.mark.parametrize("out", sorted(OUT))
@pytest.mark.parametrize("replace", [False, True])
def test_equals_host_rewrite(lanes, lanes_sam, how, out, replace, tmp_path):
    L = lanes_sam if how == "sam" else lanes
    mask = _lib.FILTER_UNMAPPED if out == "keep" else 0
    a = run_a(L, how, replace, OUT[out], mask, str(tmp_path / "a.recal"))
    b = run_b(L, how, replace, OUT[out], mask, str(tmp_path / "b.recal"))
    assert a.n == b.n > 0 and a.n_filtered() == b.n_filtered()
    for x, y in zip(a.fetch(), b.fetch()):                    # order, FLAG after marking, recalibrated QUAL
        assert np.array_equal(x, y)
    assert np.array_equal(a.tables_get(), b.tables_get())
    assert open(tmp_path / "a.recal").read() == open(tmp_path / "b.recal").read()
    assert str(a.optical_metrics()) == str(b.optical_metrics())
    if not replace:
        assert a.cov_names() == b.cov_names() and len(a.cov_names()) == 6
    for x, y in zip(outputs(a), outputs(b)):
        assert (x == y) if not isinstance(x, np.ndarray) else np.array_equal(x, y)
    a.close(); b.close()


def test_renamed_values_in_output(lanes):
    """the stored records carry the merged refIDs and the renamed values, which every RG / PG value of the file reaches"""
    a = run_a(lanes, "bam")
    text = a.fetch_sam()[0].tobytes()
    assert b"RG:Z:1SS" in text and b"RG:Z:2S" in text
    assert b"PG:Z:bwaS" in text and b"PG:Z:samtools" in text
    for bad in (b"RG:Z:1\t", b"RG:Z:1\n", b"RG:Z:1S\t", b"RG:Z:2\t", b"PG:Z:bwa\t", b"PG:Z:bwa\n"):
        assert bad not in text
    assert b"\tchrX\t" not in text and b"\tchr20\t" in text
    a.close()


def _refused(ctx, fn, code, text=None):
    with pytest.raises(device.ElprepError) as ei:
        fn()
    assert ei.value.code == code, str(ei.value)
    if text:
        assert text in str(ei.value)


def test_refusals(lanes):
    L = lanes
    h = L["heads"]
    sqn = lambda k: ([s["SN"] for s in h[k].SQ], [int(s["LN"]) for s in h[k].SQ])
    ctx = device.Context(ctx_header(L, False))
    _refused(ctx, lambda: ctx.add_input(["chrQ"], [5]), _lib.EINVAL, "not in the merged dictionary")
    _refused(ctx, lambda: ctx.set_tag_rename("XX", {}), _lib.EINVAL)
    _refused(ctx, lambda: ctx.select_input(0), _lib.EINVAL)
    ctx.add_input(*sqn(0)); ctx.add_input(*sqn(1))
    raw, off = pack(L["lanes"][1])
    _refused(ctx, lambda: ctx.append_bam(raw, off), _lib.ESTATE, "elp_select_input")            # nothing selected
    _refused(ctx, lambda: ctx.set_input_dictionary(_lib.DICT_REPLACE, *sqn(0)), _lib.EINVAL)   # does not combine
    ctx.select_input(0)
    f = bam_file(h[1], raw)                                    # lane 1's file while lane 0 is selected
    _refused(ctx, lambda: ctx.append_bgzf(f), _lib.EINVAL, "selected input")
    ctx.reset()
    ctx.select_input(1)
    ctx.append_bgzf(f[:70_000])
    _refused(ctx, lambda: ctx.select_input(0), _lib.ESTATE)   # a BGZF file is open
    ctx.append_bgzf(f[70_000:]); ctx.append_bgzf_end()
    _refused(ctx, lambda: ctx.add_input(*sqn(2)), _lib.ESTATE)                                   # the context holds reads
    _refused(ctx, lambda: ctx.set_tag_rename("RG", {"1": "1S"}), _lib.ESTATE)
    ctx.reset()                                               # the inputs survive the reset
    ctx.select_input(0)
    raw0, off0 = pack(L["lanes"][0])
    ctx.append_bam(raw0, off0)
    assert ctx.n == len(L["lanes"][0])
    ctx.close()
    ctx = device.Context(ctx_header(L, False))
    ctx.set_input_dictionary(_lib.DICT_REPLACE, *sqn(0))
    _refused(ctx, lambda: ctx.add_input(*sqn(0)), _lib.EINVAL)
    _refused(ctx, lambda: ctx.set_tag_rename("RG", {"1": "1S"}), _lib.EINVAL)
    ctx.close()


@pytest.mark.parametrize("tag", ["RG", "PG"])
def test_non_z_value_and_bad_refid_refused(lanes, tag):
    L = lanes
    recs = L["lanes"][0][:50]
    r = recs[7]
    t0, _ = fields(r)
    body = r[4:t0] + tag.encode() + b"i" + struct.pack("<i", 3)  # the record's first field of the tag is not a string
    bad = recs[:7] + [struct.pack("<I", len(body)) + body] + recs[8:]
    for rename in (True, False):
        ctx = device.Context(ctx_header(L, False))
        ctx.add_input([s["SN"] for s in L["heads"][0].SQ], [int(s["LN"]) for s in L["heads"][0].SQ])
        ctx.select_input(0)
        if rename:
            ctx.set_tag_rename(tag, L["maps"][1 if tag == "RG" else 2])
            _refused(ctx, lambda: ctx.append_bam(*pack(bad)), _lib.EBAM, "not a string")
        elif tag == "PG":
            ctx.append_bam(*pack(bad))                          # without a rename of the tag the reference never converts it
        ctx.close()
    # a refID past the input's three @SQ lines, though inside the merged five
    r = bytearray(recs[3]); struct.pack_into("<i", r, 4, 3)
    ctx = device.Context(ctx_header(L, False))
    ctx.add_input([s["SN"] for s in L["heads"][0].SQ], [int(s["LN"]) for s in L["heads"][0].SQ])
    ctx.select_input(0)
    _refused(ctx, lambda: ctx.append_bam(*pack(recs[:3] + [bytes(r)])), _lib.EBAM, "beyond the @SQ lines of its input")
    ctx.close()


def test_millions_of_reads_bgzf():
    """about 2 M reads in three lane BGZF files, @SQ remapped and RG renamed, against one file encoded with the merged header"""
    w = synth.make_workload(1_000_000, BASE, seed=47)
    heads = [lane_header(k) for k in range(3)]
    merged, sq_maps, rg_map, pg_map = sam.MergeInputs(heads, SUFFIX)
    b = w.batch
    lane = (np.arange(b.n) * 7 // 1000) % 3                   # runs of reads per lane
    sel = b.rg % 2
    order, lane_files = [], []
    for k in range(3):
        idx = np.nonzero(lane == k)[0]
        lb = b.take(idx)
        to_lane = np.array([LANE_SQ[k].index(n) for n, _ in BASE], np.int32)
        lb.refid[:] = np.where(lb.refid >= 0, to_lane[np.maximum(lb.refid, 0)], lb.refid)
        lb.nref[:] = np.where(lb.nref >= 0, to_lane[np.maximum(lb.nref, 0)], lb.nref)
        lb.rg[:] = sel[idx]
        raw, _ = synth.encode_bam(lb, heads[k])
        lane_files.append(bam_file(heads[k], raw))
        order.append(idx)
    order = np.concatenate(order)
    mb = b.take(order)                                        # run B: the same reads in the same order, encoded with the merged header
    to_m = np.array([merged.contig_names().index(n) for n, _ in BASE], np.int32)
    mb.refid[:] = np.where(mb.refid >= 0, to_m[np.maximum(mb.refid, 0)], mb.refid)
    mb.nref[:] = np.where(mb.nref >= 0, to_m[np.maximum(mb.nref, 0)], mb.nref)
    ids = [r["ID"] for r in merged.RG]
    lane_of = lane[order]
    mb.rg[:] = [ids.index(rg_map.get(LANE_RG[k][s], LANE_RG[k][s])) for k, s in zip(lane_of, sel[order])]
    mraw, _ = synth.encode_bam(mb, merged)
    L = dict(w=w, base_to_merged=list(to_m))
    a = device.Context(sam.Header(sq=merged.SQ, rg=merged.RG))
    side_inputs(a, L)
    for h in heads:
        a.add_input([s["SN"] for s in h.SQ], [int(s["LN"]) for s in h.SQ])
    a.set_tag_rename("RG", rg_map)
    for k in range(3):
        a.select_input(k)
        f = lane_files[k]
        for x in range(0, len(f), 8 << 20):
            a.append_bgzf(f[x:x + (8 << 20)])
        a.append_bgzf_end()
    bctx = device.Context(sam.Header(sq=merged.SQ, rg=merged.RG))
    side_inputs(bctx, L)
    fb = bam_file(merged, mraw)
    for x in range(0, len(fb), 8 << 20):
        bctx.append_bgzf(fb[x:x + (8 << 20)])
    bctx.append_bgzf_end()
    assert a.n == bctx.n == b.n > 1_900_000
    for c in (a, bctx):
        c.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
        c.bqsr_gather(); c.bqsr_finalize(None); c.bqsr_apply()
    for x, y in zip(a.fetch(), bctx.fetch()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.tables_get(), bctx.tables_get())
    assert inflate_all(a.fetch_bgzf(eof=True).tobytes()) == inflate_all(bctx.fetch_bgzf(eof=True).tobytes())
    a.close(); bctx.close()
