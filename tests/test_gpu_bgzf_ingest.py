"""elp_append_bgzf / elp_append_bgzf_end / elp_debug_inflate: a BGZF-compressed BAM file inflated, framed and ingested on the device,
against the host path (elp_bgzf_inflate + elp_bam_header_size + elp_append_bam) and the oracle."""
import struct
import zlib

import numpy as np
import pytest

from elprep_b200 import _lib, bgzf, synth
from util import encode_bam, oracle_pipeline

pytestmark = pytest.mark.gpu

SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]
EOF_BLOCK = bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0])


def bgzf_block(payload, level=6, extra=b""):
    """one BGZF member as the reference's writer makes it (any ISIZE up to 65536), optionally with a foreign extra subfield before BC"""
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    cdata = co.compress(payload) + co.flush()
    xtra = extra + b"BC" + struct.pack("<HH", 2, 0)
    bsize = 12 + len(xtra) + len(cdata) + 8
    xtra = extra + b"BC" + struct.pack("<HH", 2, bsize - 1)
    return bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff]) + struct.pack("<H", len(xtra)) + xtra + cdata + struct.pack("<II", zlib.crc32(payload), len(payload))


def bam_header(w, text=b"@HD\tVN:1.6\tSO:unsorted\n"):
    return b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(w.header.SQ)) + b"".join(
        struct.pack("<i", len(sq["SN"]) + 1) + sq["SN"].encode() + b"\0" + struct.pack("<i", int(sq["LN"])) for sq in w.header.SQ)


def bam_file(w, raw, text=b"@HD\tVN:1.6\tSO:unsorted\n", level=-1):
    return bytes(bgzf.deflate(np.concatenate([np.frombuffer(bam_header(w, text), np.uint8), raw]), level=level))


def context(w, **kw):
    from elprep_b200 import device
    ctx = device.Context(w.header, **kw)
    for ci in range(len(w.header.SQ)):
        if ci < len(w.contig_bases):
            ctx.set_reference(ci, w.contig_bases[ci]); ctx.set_known_sites(ci, w.sites[ci], already_flat=True)
    return ctx


def finish(ctx, bqsr=True):
    """the path after ingest -> everything a caller reads back"""
    ctx.sort_markdup()
    r = {"n": ctx.n, "filtered": ctx.n_filtered()}
    if bqsr:
        ctx.bqsr_gather(); r["tables"] = ctx.tables_get(); ctx.bqsr_finalize(None); ctx.bqsr_apply()
    idx, flag, qoff, qual = ctx.fetch()
    r.update(idx=idx.copy(), flag=flag.copy(), qual=qual[:int(qoff[-1])].copy())
    r["bam"] = ctx.fetch_bam()[0].tobytes()
    r["sam"] = ctx.fetch_sam()[0].tobytes()
    ctx.close()
    return r


def host_path(w, raw, bqsr=True, mask=0, mq=0):
    ctx = context(w)
    ctx.set_ingest_filter(mask, mq)
    ctx.append_bam(raw, None)
    return finish(ctx, bqsr)


def device_path(w, data, cuts, bqsr=True, mask=0, mq=0, profile=False, stats=None):
    ctx = context(w, profile=profile)
    ctx.set_ingest_filter(mask, mq)
    prev = 0
    for c in list(cuts) + [len(data)]:
        ctx.append_bgzf(data[prev:c]); prev = c
    ctx.append_bgzf_end()
    if stats is not None:
        stats.update(ctx.kernel_stats())
    return finish(ctx, bqsr)


def same(a, b):
    assert a["n"] == b["n"] and a["filtered"] == b["filtered"]
    for k in ("idx", "flag", "qual"):
        assert np.array_equal(a[k], b[k]), k
    if "tables" in a:
        assert np.array_equal(a["tables"], b["tables"])
    assert a["bam"] == b["bam"] and a["sam"] == b["sam"]


@pytest.fixture(scope="module")
def wl():
    w = synth.make_workload(3_000, SMALL, seed=23)
    raw, _ = encode_bam(w.batch, w.header)
    return w, raw


def test_debug_inflate_matches_host_inflate(wl):
    from elprep_b200 import device
    w, raw = wl
    ctx = context(w)
    rng = np.random.default_rng(5)
    payloads = [raw[:65536].tobytes(), rng.integers(0, 256, 0xff00, dtype=np.uint8).tobytes(), b"A" * 65536, b"", b"x",
                bytes(raw[:0xff00]), bytes((np.arange(40000) % 37).astype(np.uint8))]
    corpus = [bytes(bgzf.deflate(raw, level=lv)) for lv in (0, 1, 6, 9)]
    corpus.append(b"".join(bgzf_block(p, lv) for p in payloads for lv in (0, 1, 9) if lv or len(p) <= 0xff00))                 # 65536-byte blocks, as the reference writes them
    corpus.append(bgzf_block(payloads[0], 6, extra=b"XY" + struct.pack("<H", 3) + b"abc") + EOF_BLOCK + bgzf_block(payloads[2]))   # foreign subfield, EOF mid-stream
    for data in corpus:
        assert np.array_equal(ctx.debug_inflate(data), bgzf.inflate(data))
    good = bgzf_block(payloads[0])
    crc_flip = bytearray(good); crc_flip[-8] ^= 1
    isize = bytearray(good); isize[-4] ^= 1
    no_bc = bytearray(good); no_bc[12:14] = b"XC"
    deflate_bad = bytearray(good); deflate_bad[18] ^= 0x06                                            # block type 3 or a broken header
    bad = [bytes(crc_flip), bytes(isize), good[:-3], bytes(no_bc), bytes(deflate_bad), good + good[:30]]
    for data in bad:
        with pytest.raises(bgzf.BgzfError):
            bgzf.inflate(data)
        with pytest.raises(device.ElprepError) as ei:
            ctx.debug_inflate(data)
        assert ei.value.code == _lib.EBGZF
        assert np.array_equal(ctx.debug_inflate(good), bgzf.inflate(good))                           # no sticky error
    ctx.close()


def test_whole_bgzf_file_on_the_device(wl):
    """test_whole_bam_file_in_memory with elp_append_bgzf in place of host inflate + elp_append_bam"""
    w, raw = wl
    data = bam_file(w, raw)
    h = host_path(w, raw)
    d = device_path(w, data, [])
    same(d, h)
    o = oracle_pipeline(w)
    assert np.array_equal(d["flag"], o["flag"]) and np.array_equal(d["qual"], o["qual"])
    assert np.array_equal(d["idx"].astype(np.uint32), o["perm"].astype(np.uint32))


def block_bounds(data):
    b, x = [], 0
    while x < len(data):
        b.append(x); x += struct.unpack_from("<H", data, x + 16)[0] + 1                  # (bgzf.deflate writes BC as the only subfield)
    return b


def test_cuts_anywhere(wl):
    w, raw = wl
    data = bam_file(w, raw, level=1)
    h = host_path(w, raw, bqsr=False)
    bounds = block_bounds(data)
    rng = np.random.default_rng(7)
    cut_sets = [bounds[1:],                                                      # exactly on block boundaries
                [b + 5 for b in bounds[1:]],                                     # inside gzip headers
                [b - 3 for b in bounds[1:]],                                     # inside trailers
                list(range(1, 3000)),                                            # 1-byte calls over the first 3 KiB
                sorted(set(int(v) for v in rng.integers(1, len(data), 40)))]     # random
    for cuts in cut_sets:
        same(device_path(w, data, cuts, bqsr=False), h)


def test_header_over_several_blocks_and_long_record():
    w = synth.make_workload(400, SMALL, seed=31)
    b = w.batch
    extra = [b""] * b.n
    extra[b.n // 2] = b"ZZBC" + struct.pack("<I", 100_000) + bytes(np.random.default_rng(1).integers(0, 256, 100_000, dtype=np.uint8))   # a 100 kb record
    extra[b.n // 3] = b"ZYZ" + b"q" * 150_000 + b"\0"                                                   # straddles three blocks
    raw, _ = encode_bam(b, w.header, extra_tags=extra)
    text = b"@HD\tVN:1.6\tSO:unsorted\n" + b"".join(b"@CO\t" + (b"comment %d " % i) * 40 + b"\n" for i in range(1000))   # ~400 KB of header text
    data = bam_file(w, raw, text=text)
    h = host_path(w, raw, bqsr=False)
    same(device_path(w, data, [], bqsr=False), h)
    same(device_path(w, data, list(range(1000, len(data), 50_000)), bqsr=False), h)


def test_many_contigs_header():
    contigs = [(f"ctg{i}", 20_000) for i in range(3000)]
    w = synth.make_workload(300, contigs, seed=3)
    raw, _ = encode_bam(w.batch, w.header)
    data = bam_file(w, raw)
    same(device_path(w, data, [17, 5000, 30000], bqsr=False), host_path(w, raw, bqsr=False))


def test_framing_with_false_record_starts(wl):
    """optional fields that carry plausible record headers at false offsets: the framing guesses wrong and re-walks, and still finds
    the serial walk's records"""
    w, _ = wl
    b = w.batch
    fake = struct.pack("<iiiBBHHHiiii", 35, 0, 1000, 3, 60, 4680, 0, 0, 0, 0, 900, 0) + b"ab\0"          # 39 bytes: six of them chain
    extra = [b"ZFBC" + struct.pack("<I", len(fake) * 6) + fake * 6 for _ in range(b.n)]
    raw, _ = encode_bam(b, w.header, extra_tags=extra)
    stats = {}
    d = device_path(w, bam_file(w, raw), [], bqsr=False, profile=True, stats=stats)
    same(d, host_path(w, raw, bqsr=False))
    assert stats["bam_frame"]["launches"] > 4                       # guess, a repair round that changed something, the last round, count, emit


def test_many_tiny_records():
    w = synth.make_workload(50, SMALL, seed=2)
    recs = bytearray()
    for i in range(200_000):
        name = b"t%d\0" % i
        body = struct.pack("<iiBBHHHiiii", -1, -1, len(name), 0, 4680, 0, 4, 0, -1, -1, 0) + name
        recs += struct.pack("<I", len(body)) + body
    raw = np.frombuffer(bytes(recs), np.uint8)
    data = bam_file(w, raw)
    h = host_path(w, raw, bqsr=False)
    assert h["n"] == 200_000
    same(device_path(w, data, [70_001], bqsr=False), h)


def test_ingest_filters_and_unknown_rg():
    from elprep_b200 import device
    w0 = synth.make_workload(2_000, SMALL, seed=29, unmapped_frac=0.1)
    w0.batch.flag[::17] |= 0x400
    raw, _ = encode_bam(w0.batch, w0.header)
    data = bam_file(w0, raw)
    for mask, mq in [(_lib.FILTER_UNMAPPED, 0), (_lib.FILTER_UNMAPPED_STRICT, 0), (_lib.FILTER_NON_EXACT, 0), (_lib.FILTER_DUPLICATES, 0),
                     (_lib.FILTER_NON_EXACT_STRICT, 0), (_lib.FILTER_CLEAR_DUPLICATE_FLAG, 0), (0, 30), (_lib.FILTER_UNMAPPED | _lib.FILTER_DUPLICATES, 20)]:
        same(device_path(w0, data, [], bqsr=False, mask=mask, mq=mq), host_path(w0, raw, bqsr=False, mask=mask, mq=mq))
    ctx = context(w0)
    for ci in range(len(w0.header.SQ)):
        ctx.set_target_regions(ci, [(1, 100_000), (200_000, 250_000)])
    ctx.set_ingest_filter(_lib.FILTER_TARGET_REGIONS)
    ctx.append_bgzf(data); ctx.append_bgzf_end()
    ref = context(w0)
    for ci in range(len(w0.header.SQ)):
        ref.set_target_regions(ci, [(1, 100_000), (200_000, 250_000)])
    ref.set_ingest_filter(_lib.FILTER_TARGET_REGIONS)
    ref.append_bam(raw, None)
    same(finish(ctx, False), finish(ref, False))
    # an RG:Z value that is no @RG ID
    b2 = w0.batch.copy(); b2.rg[7] = -1
    raw2, _ = encode_bam(b2, w0.header, extra_tags=[b"RGZnope\0" if i == 7 else b"" for i in range(b2.n)], with_aux=False)
    ctx = context(w0)
    with pytest.raises(device.ElprepError) as ei:
        ctx.append_bgzf(bam_file(w0, raw2))
    assert ei.value.code == _lib.EBAM
    ctx.close()


def test_stream_errors(wl):
    from elprep_b200 import device
    w, raw = wl
    data = bam_file(w, raw)

    def code(f, *a):
        with pytest.raises(device.ElprepError) as ei:
            f(*a)
        return ei.value.code

    ctx = context(w)
    ctx.append_bgzf(data[:-len(EOF_BLOCK)])
    assert code(ctx.append_bgzf_end) == _lib.EBGZF                                # no EOF marker
    assert code(ctx.append_bgzf, EOF_BLOCK) == _lib.ESTATE                        # poisoned
    ctx.reset()
    trunc = bam_file(w, raw[:-10])
    ctx.append_bgzf(trunc)
    assert code(ctx.append_bgzf_end) == _lib.EBAM                                 # truncated last record
    ctx.reset()
    ctx.append_bgzf(data[:100])                                                   # a file is open
    assert code(ctx.append_bam, raw, None) == _lib.ESTATE
    assert code(ctx.sort_markdup) == _lib.ESTATE
    ctx.reset()
    ctx.append_bgzf(data)                                                         # after reset: a new file ingests correctly
    ctx.append_bgzf_end()
    same(finish(ctx, False), host_path(w, raw, bqsr=False))
    # a header that disagrees with elp_config
    w2 = synth.make_workload(100, [("chr20", 600_000), ("chr21", 300_001), ("chrM", 16_569)], seed=4)
    ctx = context(w)
    assert code(ctx.append_bgzf, bam_file(w2, encode_bam(w2.batch, w2.header)[0])) == _lib.EINVAL
    ctx.close()
    w3 = synth.make_workload(100, [("chr20", 600_000), ("chrX", 300_000), ("chrM", 16_569)], seed=4)
    ctx = context(w)
    assert code(ctx.append_bgzf, bam_file(w3, encode_bam(w3.batch, w3.header)[0])) == _lib.EINVAL
    ctx.close()
    w4 = synth.make_workload(100, SMALL[:2], seed=4)
    ctx = context(w)
    assert code(ctx.append_bgzf, bam_file(w4, encode_bam(w4.batch, w4.header)[0])) == _lib.EINVAL
    ctx.close()


def test_two_files_in_one_context(wl):
    w, raw = wl
    x, offs = 0, [0]
    while x < raw.size:
        x += 4 + int(struct.unpack_from("<I", raw.tobytes(), x)[0]); offs.append(x)
    half = offs[len(offs) // 2]
    a, b = raw[:half], raw[half:]
    ctx = context(w)
    ctx.append_bgzf(bam_file(w, a)); ctx.append_bgzf_end()
    ctx.append_bgzf(bam_file(w, b, level=1)); ctx.append_bgzf_end()
    d = finish(ctx)
    ref = context(w)
    ref.append_bam(a, None); ref.append_bam(b, None)
    same(d, finish(ref))
