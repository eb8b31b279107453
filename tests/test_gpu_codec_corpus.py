"""The CPU corpora of the DEFLATE decoder and encoder through the device kernels.

Decoder: every stream of `inflate_check dump` (zlib's streams, the crafted invalid ones, the CRC lane-slice edges and a sample of mutated
ones) as one BGZF member through elp_debug_inflate (bgzf_inflate: inflate.cuh as one warp per block; bgzf_crc).  The verdict must be the
host inflater's; accepted bytes must be zlib's; a rejected stream must fail with ELP_EBGZF and the text of the status the team of one gave
it, never as a CRC-32 mismatch (the CRC check runs only on blocks that decoded, so a decoder that wrongly accepts would show up as one).

Encoder: every input of `deflate_check dump` through elp_debug_deflate (bgzf_deflate: deflate.cuh as one CTA per block; bgzf_deflate_crc):
byte for byte the host build of deflate.cuh, inflating back with zlib, CRC-32 and ISIZE right."""
import collections
import struct
import subprocess
import zlib

import numpy as np
import pytest

from elprep_b200 import _lib, bgzf, device, sam
from util import build_check, host_encoder  # noqa: F401 (host_encoder: a fixture)

pytestmark = pytest.mark.gpu

# dfl::status_text (inflate.cuh), by status
STATUS_TEXT = {1: "DEFLATE stream runs past the end of the block", 2: "invalid block type", 3: "invalid stored block lengths",
               4: "too many length or distance symbols", 5: "invalid code lengths set", 6: "invalid bit length repeat",
               7: "invalid literal/lengths set", 8: "invalid distances set", 9: "invalid code -- missing end-of-block",
               10: "invalid literal/length code", 11: "invalid distance code", 12: "invalid distance too far back",
               13: "more output than ISIZE", 14: "less output than ISIZE", 15: "CRC-32 mismatch"}
HEADER = sam.Header(sq=[{"SN": "chr1", "LN": 1000}])
KIND = {0: "zlib", 1: "mutated", 2: "crafted", 3: "edge"}


def read_dump(path):
    """inflate_check's dump -> [(kind, name, isize, status, zlib_ok, stream)]"""
    d, x, out = open(path, "rb").read(), 0, []
    while x < len(d):
        kind, ln = struct.unpack_from("<BH", d, x); x += 3
        name = d[x:x + ln].decode(); x += ln
        isize, st, zok, n = struct.unpack_from("<IIBI", d, x); x += 13
        out.append((KIND[kind], name, isize, st, bool(zok), d[x:x + n])); x += n
    return out


def member(cdata, crc, isize):
    """one BGZF member around a raw DEFLATE stream"""
    bsize = 18 + len(cdata) + 8
    return (bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0]) + struct.pack("<H", bsize - 1) + cdata +
            struct.pack("<II", crc, isize))


def device_error(ctx, data):
    with pytest.raises(device.ElprepError) as ei:
        ctx.debug_inflate(data)
    return ei.value.code, str(ei.value)


def test_decoder_corpus_on_the_device(tmp_path):
    exe = build_check("inflate_check", tmp_path)
    out = subprocess.run([exe, "dump", str(tmp_path / "streams.bin")], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-2000:]
    recs = read_dump(tmp_path / "streams.bin")
    accepted, rejected, skipped = [], [], 0
    for kind, name, isize, st, zok, s in recs:
        if 18 + len(s) + 8 > 65536 or isize > 65536:              # (no BGZF member holds it)
            skipped += 1
            continue
        want = zlib.decompressobj(-15).decompress(s, isize) if zok and isize else b""
        m = member(s, zlib.crc32(want) if zok else 0, isize)
        try:
            host = bgzf.inflate(m).tobytes()
        except bgzf.BgzfError:
            host = None
        assert (host is not None) == (zok or isize == 0), name        # zlib's verdict, and an ISIZE of 0 is not decoded
        if host is not None:
            assert host == want, name
            accepted.append((kind, name, m, host, s[0] >> 1 & 3 if s else 0))
        else:
            assert st != 0, name
            rejected.append((kind, name, m, st))
    ctx = device.Context(HEADER)
    # accepted streams, 12 per call, the first block's type taken in turn, so that the four warps of a CTA decode different block types
    by_type = collections.defaultdict(list)
    for a in accepted:
        by_type[a[4]].append(a)
    order, queues = [], [by_type[k] for k in sorted(by_type)]
    while any(queues):
        for q in queues:
            if q:
                order.append(q.pop())
    n_calls = 0
    for i in range(0, len(order), 12):
        part = order[i:i + 12]
        got = ctx.debug_inflate(b"".join(a[2] for a in part)).tobytes()
        assert got == b"".join(a[3] for a in part), [a[1] for a in part]
        n_calls += 1
    # rejected streams alone, then behind k accepted ones
    seen, sent = collections.Counter(), collections.Counter()
    for kind, name, m, st in rejected:
        code, msg = device_error(ctx, m)
        assert code == _lib.EBGZF, (name, msg)
        assert "CRC-32 mismatch" not in msg, (name, msg)
        assert msg.endswith(STATUS_TEXT[st]), (name, msg, STATUS_TEXT[st])
        assert "BGZF block 0 of the call" in msg, (name, msg)
        seen[st] += 1; sent[(kind, st)] += 1
    for j, (kind, name, m, st) in enumerate(rejected[::max(1, len(rejected) // 60)]):
        k = j % 9
        lead = [order[(7 * j + t) % len(order)] for t in range(k)]
        code, msg = device_error(ctx, b"".join(a[2] for a in lead) + m + order[j % len(order)][2])
        assert code == _lib.EBGZF and f"BGZF block {k} of the call" in msg and msg.endswith(STATUS_TEXT[st]), (name, k, msg)
    assert ctx.debug_inflate(order[0][2]).tobytes() == order[0][3]                 # no sticky error
    ctx.close()
    host_statuses = {st for _, _, _, st in rejected}
    assert set(seen) == host_statuses
    print(f"\ndecoder: {len(recs)} dumped streams, {len(accepted) + len(rejected)} sent ({skipped} larger than a BGZF member); "
          f"{len(accepted)} accepted in {n_calls} calls, {len(rejected)} rejected: " +
          ", ".join(f"{STATUS_TEXT[s]} {c}" for s, c in sorted(seen.items())))
    print("rejected by kind: " + ", ".join(f"{k}/{STATUS_TEXT[s]} {c}" for (k, s), c in sorted(sent.items())))


def bgzf_members(z):
    """-> [(crc, isize, cdata)] of a BGZF byte string, checking each header"""
    out, x = [], 0
    while x < len(z):
        assert z[x:x + 4] == b"\x1f\x8b\x08\x04" and z[x + 10:x + 16] == b"\x06\x00BC\x02\x00"
        bsize = struct.unpack_from("<H", z, x + 16)[0] + 1
        crc, isize = struct.unpack_from("<II", z, x + bsize - 8)
        out.append((crc, isize, z[x + 18:x + bsize - 8]))
        x += bsize
    assert x == len(z)
    return out


def test_encoder_corpus_on_the_device(host_encoder, tmp_path):
    d = tmp_path / "inputs"
    d.mkdir()
    out = subprocess.run([host_encoder.exe, "dump", str(d)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout[-2000:]
    names = [line.split("\t", 1) for line in (d / "names.txt").read_text().splitlines()]
    ctx = device.Context(HEADER)
    n_blocks = 0
    for file, name in names:
        data = (d / file).read_bytes()
        z = ctx.debug_deflate(data, eof=False).tobytes()
        assert z == host_encoder(data, False, str(tmp_path)), name                     # byte for byte the host build of deflate.cuh
        blocks = bgzf_members(z)
        assert [b[1] for b in blocks] == [min(0xff00, len(data) - k) for k in range(0, len(data), 0xff00)], name
        for k, (crc, isize, cdata) in enumerate(blocks):
            part = data[k * 0xff00:k * 0xff00 + isize]
            zo = zlib.decompressobj(-15)
            assert zo.decompress(cdata) == part and zo.eof and not zo.unused_data, name
            assert crc == zlib.crc32(part), name                                       # bgzf_deflate_crc
        assert bgzf.inflate(np.frombuffer(z, np.uint8)).tobytes() == data if z else data == b""
        n_blocks += len(blocks)
    ctx.close()
    print(f"\nencoder: {len(names)} inputs, {n_blocks} BGZF blocks")
