"""SAM text output restatement (tests/samformat.py) and the host float formatter of elp_fetch_sam (elprep_b200/csrc/gofloat.hpp), without a
GPU.  The lines below are derived by hand from FormatAlignment / formatSamTag / cigarToString (sam/sam-files.go:485-598) and
parseBamAlignment (sam/bam-files.go:317-400); tests/test_gpu_sam_output.py sends the same records through elp_fetch_sam."""
import functools
import os
import struct
import subprocess

import numpy as np
import pytest

from samformat import bam_to_sam, format_f32, parse_sam_alignment, sam_to_sam, shortest_digits
from samtext import f32_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = [b"chr1", b"chr2", b"chr1"]                                     # a duplicate @SQ name, as in test_sam_text.HEADER


def fbits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


KNOWN = [(fbits(1.5), b"1.5"), (fbits(0.1), b"0.1"), (fbits(np.float32(1) / np.float32(3)), b"0.33333334"), (fbits(16777216), b"1.6777216e+07"),
         (fbits(1e6), b"1e+06"), (fbits(999999), b"999999"), (fbits(123456.7), b"123456.7"), (fbits(0.0001), b"0.0001"), (fbits(0.00001), b"1e-05"),
         (0x7F7FFFFF, b"3.4028235e+38"), (0x00800000, b"1.1754944e-38"), (0x00000001, b"1e-45"), (fbits(100), b"100"),
         (0x7FC00000, b"NaN"), (0xFFC00001, b"NaN"), (0x7F800001, b"NaN"), (0x7F800000, b"+Inf"), (0xFF800000, b"-Inf"), (0, b"0"), (0x80000000, b"-0"),
         (fbits(-2.5), b"-2.5"), (fbits(1e-4) ^ 0x80000000, b"-0.0001"), (fbits(100000), b"100000"), (fbits(1234567), b"1.234567e+06")]
EDGE = [b for b, _ in KNOWN] + [e << 23 for e in range(1, 255)] + [1 << k for k in range(23)]   # every power of two 2^-149 .. 2^127


@functools.lru_cache(maxsize=None)
def random_patterns():
    bits = np.random.default_rng(20261015).integers(0, 1 << 32, 200_000, dtype=np.uint64).astype(np.uint32)
    return bits, [format_f32(int(b)) for b in bits]


@pytest.mark.parametrize("bits,text", KNOWN, ids=[t.decode() for _, t in KNOWN])
def test_float_known_answers(bits, text):
    assert format_f32(bits) == text


def test_float_powers_of_two():
    for k in range(-149, 128):
        b = fbits(2.0 ** k)
        t = format_f32(b)
        assert f32_bits(t) == b, (k, t)
        assert format_f32(b | 0x80000000) == b"-" + t
    assert format_f32(fbits(2.0 ** 10)) == b"1024" and format_f32(fbits(2.0 ** 20)) == b"1.048576e+06" and format_f32(fbits(2.0 ** -14)) == b"6.1035156e-05"


def test_float_random_round_trip_and_minimal():
    """200 000 seeded bit patterns: the text reads back as the same float32 and no decimal with one digit fewer does"""
    bits, texts = random_patterns()
    for b, t in zip(bits.tolist(), texts):
        if (b & 0x7FFFFFFF) > 0x7F800000:
            assert t == b"NaN"
            continue
        if (b & 0x7FFFFFFF) == 0x7F800000:
            continue
        assert f32_bits(t) == b, (hex(b), t)
        if b & 0x7FFFFFFF:
            d, dp = shortest_digits(b & 0x7FFFFFFF)
            p = len(d)
            if p > 1:                                                   # the two (p-1)-digit neighbours of the value do not round-trip
                v = f32_bits(t) & 0x7FFFFFFF
                e = dp - (p - 1)
                lo = int(d[:p - 1])
                for c in (lo, lo + 1):
                    try:
                        assert f32_bits(b"%de%d" % (c, e)) != v, (hex(b), t, c, e)
                    except ValueError:
                        pass


def test_gofloat_hpp_matches_restatement(tmp_path):
    """gofloat.hpp compiled into a host client gives the restatement's text on the edge values and the 200 000 random patterns"""
    exe = str(tmp_path / "gofloat_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "elprep_b200", "csrc"), "-o", exe, os.path.join(ROOT, "tests", "c", "gofloat_check.cpp")])
    bits, texts = random_patterns()
    allbits = np.concatenate([np.array(EDGE, np.uint32), np.array(EDGE, np.uint32) | np.uint32(0x80000000), bits])
    want = [format_f32(int(b)) for b in allbits[:2 * len(EDGE)]] + texts
    (tmp_path / "bits").write_bytes(allbits.astype("<u4").tobytes())
    out = subprocess.run([exe, str(tmp_path / "bits")], capture_output=True, check=True).stdout.split(b"\n")[:-1]
    assert len(out) == len(want)
    bad = [(hex(int(b)), o, w) for b, o, w in zip(allbits, out, want) if o != w]
    assert not bad, bad[:10]


# ---- hand-built BAM records -> the line FormatAlignment writes ----
def bam_record(qname=b"r1", flag=0, refid=1, pos=99, mapq=60, cigar=((4, 0),), nref=1, pnext=299, tlen=250, seq=b"\x12\x48", lseq=4,
               qual=b"\x28\x28\x28\x28", tags=b""):
    """BAM record bytes (block_size included); cigar: (length, op code) pairs; seq: packed nibbles"""
    body = struct.pack("<iiBBHHHiiii", refid, pos, len(qname) + 1, mapq, 4680, len(cigar), flag, lseq, nref, pnext, tlen)
    body += qname + b"\0" + b"".join(struct.pack("<I", (ln << 4) | op) for ln, op in cigar) + seq + qual + tags
    return struct.pack("<I", len(body)) + body


BASE_TEXT = b"r1\t0\tchr2\t100\t60\t4M\t=\t300\t250\tACGT\tIIII"
LINES = [
    ("base", bam_record(), BASE_TEXT + b"\n"),
    # FLAG / MAPQ unsigned, POS / PNEXT int32(x) + 1 wrapping, TLEN signed
    ("fixed_bounds", bam_record(flag=65535, mapq=255, pos=0x7FFFFFFF, pnext=-1, tlen=-2147483648),
     b"r1\t65535\tchr2\t-2147483648\t255\t4M\t=\t0\t-2147483648\tACGT\tIIII\n"),
    ("pos_minus_one", bam_record(pos=-1, pnext=-2), b"r1\t0\tchr2\t0\t60\t4M\t=\t-1\t250\tACGT\tIIII\n"),
    # RNAME / RNEXT: "*" below 0; "=" when the NAMES are equal (duplicate @SQ chr1 at 0 and 2); else the name
    ("refid_star", bam_record(refid=-1, nref=-1), b"r1\t0\t*\t100\t60\t4M\t*\t300\t250\tACGT\tIIII\n"),
    ("rnext_other", bam_record(refid=1, nref=0), b"r1\t0\tchr2\t100\t60\t4M\tchr1\t300\t250\tACGT\tIIII\n"),
    ("rnext_dup_name", bam_record(refid=0, nref=2), b"r1\t0\tchr1\t100\t60\t4M\t=\t300\t250\tACGT\tIIII\n"),
    ("rname_star_rnext_set", bam_record(refid=-1, nref=1), b"r1\t0\t*\t100\t60\t4M\tchr2\t300\t250\tACGT\tIIII\n"),
    # CIGAR: "*" for none, every op, multi-digit lengths
    ("cigar_none", bam_record(cigar=()), b"r1\t0\tchr2\t100\t60\t*\t=\t300\t250\tACGT\tIIII\n"),
    ("cigar_all_ops", bam_record(cigar=tuple((i + 1, i) for i in range(9)) + ((268435455, 0),)),
     b"r1\t0\tchr2\t100\t60\t1M2I3D4N5S6H7P8=9X268435455M\t=\t300\t250\tACGT\tIIII\n"),
    # SEQ: every nibble; odd length; l_seq 0 gives empty SEQ and QUAL; QUAL 0xff prints as a space (+33 mod 256)
    ("seq_nibbles", bam_record(seq=bytes([0x01, 0x23, 0x45, 0x67, 0x89, 0xAB, 0xCD, 0xEF]), lseq=16, qual=bytes(range(16)), cigar=((16, 0),)),
     b"r1\t0\tchr2\t100\t60\t16M\t=\t300\t250\t=ACMGRSVTWYHKDBN\t!\"#$%&'()*+,-./0\n"),
    ("seq_odd", bam_record(seq=b"\x12\x40", lseq=3, qual=b"\x00\x5d\x09", cigar=((3, 0),)), b"r1\t0\tchr2\t100\t60\t3M\t=\t300\t250\tACG\t!~*\n"),
    ("seq_empty", bam_record(seq=b"", lseq=0, qual=b"", cigar=()), b"r1\t0\tchr2\t100\t60\t*\t=\t300\t250\t\t\n"),
    ("qual_ff", bam_record(qual=b"\xff\xff\xff\xff"), b"r1\t0\tchr2\t100\t60\t4M\t=\t300\t250\tACGT\t    \n"),
    ("qname_254", bam_record(qname=b"q" * 254), b"q" * 254 + BASE_TEXT[2:] + b"\n"),
    # tags: A; every integer width at its boundaries prints as i
    ("tag_A", bam_record(tags=b"XAAq"), BASE_TEXT + b"\tXA:A:q\n"),
    ("tag_ints", bam_record(tags=b"a1c\x80" + b"a2C\xff" + b"a3s\x00\x80" + b"a4S\xff\xff" + b"a5i\x00\x00\x00\x80" + b"a6I\xff\xff\xff\xff" + b"a7c\x7f" + b"a8i\xff\xff\xff\x7f"),
     BASE_TEXT + b"\ta1:i:-128\ta2:i:255\ta3:i:-32768\ta4:i:65535\ta5:i:-2147483648\ta6:i:4294967295\ta7:i:127\ta8:i:2147483647\n"),
    ("tag_f", bam_record(tags=b"XSf" + struct.pack("<f", 1.5) + b"XTf\x00\x00\xc0\x7f" + b"XUf\x01\x00\x00\x00" + b"XVf\x00\x00\x00\x80"),
     BASE_TEXT + b"\tXS:f:1.5\tXT:f:NaN\tXU:f:1e-45\tXV:f:-0\n"),
    ("tag_Z", bam_record(tags=b"MDZ75A74\0XEZ\0XCZa:b c\0"), BASE_TEXT + b"\tMD:Z:75A74\tXE:Z:\tXC:Z:a:b c\n"),
    ("tag_H", bam_record(tags=b"XHH1AFF00\0XIH\0"), BASE_TEXT + b"\tXH:H:1aff00\tXI:H:\n"),
    ("tag_B", bam_record(tags=b"B1Bc\x02\x00\x00\x00\x80\x7f" + b"B2BC\x01\x00\x00\x00\xff" + b"B3Bs\x02\x00\x00\x00\xff\xff\x00\x80" + b"B4BS\x01\x00\x00\x00\xff\xff"
                               + b"B5Bi\x01\x00\x00\x00\x00\x00\x00\x80" + b"B6BI\x01\x00\x00\x00\xff\xff\xff\xff" + b"B7Bf\x03\x00\x00\x00" + struct.pack("<3f", 1.5, 0.1, -1e10)),
     BASE_TEXT + b"\tB1:B:c,-128,127\tB2:B:C,255\tB3:B:s,-1,-32768\tB4:B:S,65535\tB5:B:i,-2147483648\tB6:B:I,4294967295\tB7:B:f,1.5,0.1,-1e+10\n"),
    ("tag_B_empty", bam_record(tags=b"E1Bc\x00\x00\x00\x00" + b"E2Bf\x00\x00\x00\x00"), BASE_TEXT + b"\tE1:B:c\tE2:B:f\n"),
]


@pytest.mark.parametrize("name,rec,text", LINES, ids=[x[0] for x in LINES])
def test_bam_record_lines(name, rec, text):
    assert bam_to_sam(rec, NAMES) == text


def test_flag_and_qual_replaced():
    assert bam_to_sam(bam_record(), NAMES, flag=1024, qual=b"\x00\x01\x02\x03") == b"r1\t1024\tchr2\t100\t60\t4M\t=\t300\t250\tACGT\t!\"#$\n"


@pytest.mark.parametrize("line,text", [
    (BASE_TEXT, BASE_TEXT + b"\n"),
    (b"r1\t0\tchr2\t100\t60\t2M2m\tchr2\t300\t250\tacgX\tIIII\tXH:H:aBcD\tNM:i:1\tNM:i:300", b"r1\t0\tchr2\t100\t60\t4M\t=\t300\t250\tNNNN\tIIII\tXH:H:abcd\tNM:i:300\n"),
    (b"r1\t0\tchrZ\t100\t60\t4M\t=\t300\t250\t*\t*\tZB:B:s,65535,0\tXF:f:16777217", b"r1\t0\tchrZ\t100\t60\t4M\t=\t300\t250\tN\t*\tZB:B:s,-1,0\tXF:f:1.6777216e+07\n"),
])
def test_sam_line_restatement(line, text):
    """FormatAlignment(parseSamAlignment(line)): CIGAR merged and upper case, SEQ through the nibble table, RNEXT '=' for RNAME's name,
    a repeated tag at its first position with the last value, B:s through int16"""
    assert sam_to_sam(line) == text
    assert parse_sam_alignment(line)["RNAME"] == line.split(b"\t")[2]
