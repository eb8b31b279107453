"""SAM text -> BAM record restatement (tests/samtext.py) and parse_sam_header, without a GPU.  The known answers below are derived
by hand from the reference source; tests/test_gpu_sam_ingest.py sends the same lines through elp_append_sam."""
import struct

import numpy as np
import pytest

from elprep_b200 import sam, synth
from samtext import SamError, f32_bits, format_sam, sam_line_to_bam, sam_lines_to_bam, sam_text
from util import decode_bam

HEADER = sam.Header(sq=[{"SN": "chr1", "LN": 1000}, {"SN": "chr2", "LN": 1000}, {"SN": "chr1", "LN": 500}], rg=[{"ID": "g1"}, {"ID": "g2"}])
BASE = b"r1\t0\tchr2\t100\t60\t4M\t=\t300\t250\tACGT\tIIII"


def line(**kw):
    """BASE with some mandatory fields replaced and optional fields appended (tags=[...])"""
    f = BASE.split(b"\t")
    for i, k in enumerate(("QNAME", "FLAG", "RNAME", "POS", "MAPQ", "CIGAR", "RNEXT", "PNEXT", "TLEN", "SEQ", "QUAL")):
        if k in kw:
            f[i] = kw[k]
    return b"\t".join(f + list(kw.get("tags", [])))


def fields(rec):
    """(refid, pos, l_read_name, mapq, bin, n_cigar, flag, l_seq, next_refid, pnext, tlen), cigar words, seq, qual, tag bytes"""
    fx = struct.unpack_from("<iiBBHHHiiii", rec, 4)
    x = 36 + fx[2]
    cig = list(struct.unpack_from("<%dI" % fx[5], rec, x)); x += 4 * fx[5]
    seq = rec[x:x + (fx[7] + 1) // 2]; x += (fx[7] + 1) // 2
    qual = rec[x:x + fx[7]]; x += fx[7]
    return fx, cig, seq, qual, rec[x:]


def tag_bytes(*tags):
    return fields(sam_line_to_bam(line(tags=[t.encode() for t in tags]), HEADER))[4]


# ---- known answers: (line, what the record must hold) -- every one is also run on the device ----
KAT = [
    # FLAG / MAPQ: ParseUint 16 / 8 (sam-files.go:378-393); POS / PNEXT / TLEN: ParseInt 32 with an optional sign (:374-376)
    ("flag_max", line(FLAG=b"65535"), lambda r: fields(r)[0][6] == 65535),
    ("flag_leading_zeros", line(FLAG=b"0016"), lambda r: fields(r)[0][6] == 16),
    ("mapq_255", line(MAPQ=b"255"), lambda r: fields(r)[0][3] == 255),
    ("pos_plus", line(POS=b"+100", PNEXT=b"-5", TLEN=b"-2147483648"), lambda r: fields(r)[0][1] == 99 and fields(r)[0][9] == -6 and fields(r)[0][10] == -2147483648),
    # CIGAR (sam-types.go:661-724): case-insensitive, adjacent equal operations merge, '*' -> none
    ("cigar_merge", line(CIGAR=b"2M2m", SEQ=b"ACGT"), lambda r: fields(r)[1] == [(4 << 4) | 0]),
    ("cigar_merge_split", line(CIGAR=b"1S1M1m1I", SEQ=b"ACGT"), lambda r: fields(r)[1] == [(1 << 4) | 4, (2 << 4) | 0, (1 << 4) | 1]),
    ("cigar_lower_all", line(CIGAR=b"1h1s1x1=1p1n1d1i1m", SEQ=b"ACGT"), lambda r: fields(r)[1] == [(1 << 4) | o for o in (5, 4, 8, 7, 6, 3, 2, 1, 0)]),
    ("cigar_star", line(CIGAR=b"*"), lambda r: fields(r)[0][5] == 0 and fields(r)[1] == []),
    ("cigar_empty", line(CIGAR=b""), lambda r: fields(r)[0][5] == 0),
    # SEQ: baseToNibble (sam-types.go:227-236); lower case and others -> 15; '*' is one base of nibble 15 (sam-files.go:356-372)
    ("seq_nibbles", line(SEQ=b"=ACMGRSVTWYHKDBN", QUAL=b"I" * 16, CIGAR=b"16M"), lambda r: fields(r)[2] == bytes([0x01, 0x23, 0x45, 0x67, 0x89, 0xAB, 0xCD, 0xEF])),
    ("seq_lower", line(SEQ=b"acgX"), lambda r: fields(r)[2] == b"\xff\xff" and fields(r)[0][7] == 4),
    ("seq_odd", line(SEQ=b"ACG", QUAL=b"III", CIGAR=b"3M"), lambda r: fields(r)[2] == b"\x12\x40"),
    # QUAL: each byte - 33, so '*' -> 9 (sam-files.go:400-403)
    ("seq_qual_star", line(SEQ=b"*", QUAL=b"*", CIGAR=b"*"), lambda r: fields(r)[0][7] == 1 and fields(r)[2] == b"\xf0" and fields(r)[3] == b"\x09"),
    ("qual_low", line(QUAL=b"!\"#~"), lambda r: fields(r)[3] == bytes([0, 1, 2, 93])),
    # RNAME / RNEXT (simple-filters.go:208-231, bam-files.go:642-681): '*' or unknown -> -1, '=' -> RNAME's refid, duplicate @SQ: last wins
    ("rname_dup_last", line(RNAME=b"chr1", RNEXT=b"chr2"), lambda r: fields(r)[0][0] == 2 and fields(r)[0][8] == 1),
    ("rname_unknown", line(RNAME=b"chrZ", RNEXT=b"="), lambda r: fields(r)[0][0] == -1 and fields(r)[0][8] == -1),
    ("rname_star", line(RNAME=b"*", RNEXT=b"*"), lambda r: fields(r)[0][0] == -1 and fields(r)[0][8] == -1),
    # bin (bam-files.go:443-468): unmapped -> end = beg; POS 0 -> 4680
    ("bin_unmapped_pos0", line(FLAG=b"4", POS=b"0", CIGAR=b"*"), lambda r: fields(r)[0][4] == 4680),
    ("bin_level0", line(POS=b"16380", CIGAR=b"10M", SEQ=b"A" * 10, QUAL=b"I" * 10), lambda r: fields(r)[0][4] == 585),    # [16379, 16388] crosses 2^14: level 1
    ("bin_leaf", line(POS=b"1", CIGAR=b"4M"), lambda r: fields(r)[0][4] == 4681),
    ("bin_second", line(POS=b"16385", CIGAR=b"4M"), lambda r: fields(r)[0][4] == 4682),
    ("bin_negative_pos", line(POS=b"-5", FLAG=b"4"), lambda r: fields(r)[0][4] == 4680),
    # tags: A, i boundaries, f, Z, H, B (sam-files.go:186-317, bam-files.go:481-630)
    ("tag_A", line(tags=[b"XA:A:q"]), lambda r: fields(r)[4] == b"XAAq"),
    ("tag_i_bounds", line(tags=[b"a1:i:-129", b"a2:i:-128", b"a3:i:255", b"a4:i:256", b"a5:i:65535", b"a6:i:65536", b"a7:i:4294967295", b"a8:i:-2147483648"]),
     lambda r: fields(r)[4] == b"a1s\x7f\xff" + b"a2c\x80" + b"a3C\xff" + b"a4S\x00\x01" + b"a5S\xff\xff" + b"a6I\x00\x00\x01\x00" + b"a7I\xff\xff\xff\xff" + b"a8i\x00\x00\x00\x80"),
    ("tag_i_signs", line(tags=[b"b1:i:+7", b"b2:i:-0", b"b3:i:-32768", b"b4:i:-32769"]),
     lambda r: fields(r)[4] == b"b1C\x07" + b"b2C\x00" + b"b3s\x00\x80" + b"b4i" + struct.pack("<i", -32769)),
    ("tag_f_fast", line(tags=[b"f1:f:0.1", b"f2:f:1.5", b"f3:f:-2.5e-3", b"f4:f:1e10", b"f5:f:.5", b"f6:f:7."]),
     lambda r: fields(r)[4] == b"".join(k + b"f" + struct.pack("<I", v) for k, v in
                                        ((b"f1", 0x3DCCCCCD), (b"f2", 0x3FC00000), (b"f3", 0xBB23D70A), (b"f4", 0x501502F9), (b"f5", 0x3F000000), (b"f6", 0x40E00000)))),
    ("tag_f_host", line(tags=[b"g1:f:16777217", b"g2:f:3.4028235e38", b"g3:f:1e-45", b"g4:f:16777219", b"g5:f:1e11", b"g6:f:0.000000000001", b"g7:f:1.0000001788139343"]),
     lambda r: fields(r)[4] == b"".join(k + b"f" + struct.pack("<I", v) for k, v in
                                        ((b"g1", 0x4B800000), (b"g2", 0x7F7FFFFF), (b"g3", 0x00000001), (b"g4", 0x4B800002), (b"g5", 0x51BA43B7), (b"g6", 0x2B8CBCCC), (b"g7", 0x3F800001)))),
    ("tag_f_special", line(tags=[b"h1:f:inf", b"h2:f:-Infinity", b"h3:f:NaN", b"h4:f:-0", b"h5:f:0e99999"]),
     lambda r: fields(r)[4] == b"h1f\x00\x00\x80\x7f" + b"h2f\x00\x00\x80\xff" + b"h3f\x00\x00\xc0\x7f" + b"h4f\x00\x00\x00\x80" + b"h5f\x00\x00\x00\x00"),
    ("tag_Z", line(tags=[b"MD:Z:75A74", b"XE:Z:", b"XC:Z:a:b c"]), lambda r: fields(r)[4] == b"MDZ75A74\x00XEZ\x00XCZa:b c\x00"),
    ("tag_H", line(tags=[b"XH:H:1aFf00"]), lambda r: fields(r)[4] == b"XHH1AFF00\x00"),
    ("tag_B", line(tags=[b"B1:B:c,-128,127", b"B2:B:C,255", b"B3:B:s,65535,0", b"B4:B:S,1", b"B5:B:i,-1", b"B6:B:I,4294967295", b"B7:B:f,1.5,0.1"]),
     lambda r: fields(r)[4] == b"B1Bc\x02\x00\x00\x00\x80\x7f" + b"B2BC\x01\x00\x00\x00\xff" + b"B3Bs\x02\x00\x00\x00\xff\xff\x00\x00" + b"B4BS\x01\x00\x00\x00\x01\x00"
     + b"B5Bi\x01\x00\x00\x00\xff\xff\xff\xff" + b"B6BI\x01\x00\x00\x00\xff\xff\xff\xff" + b"B7Bf\x02\x00\x00\x00\x00\x00\xc0\x3f\xcd\xcc\xcc\x3d"),
    # SmallMap.Set (utils/small-map.go:59-67): a repeated tag keeps its first position and takes the last value
    ("tag_repeat", line(tags=[b"NM:i:1", b"XA:Z:x", b"NM:Z:two", b"XB:A:c", b"NM:i:300"]), lambda r: fields(r)[4] == b"NMS\x2c\x01XAZx\x00XBAc"),
    ("trailing_tab", line(tags=[b"NM:i:1", b""]), lambda r: fields(r)[4] == b"NMC\x01"),
    ("rg_tag", line(tags=[b"RG:Z:g2"]), lambda r: fields(r)[4] == b"RGZg2\x00"),
    ("qname_254", line(QNAME=b"q" * 254), lambda r: fields(r)[0][2] == 255),
]

# lines elp_append_sam refuses: (name, line, kind)
ERRORS = [
    ("missing_tab", b"r1\t0\tchr1\t1\t60\t4M\t=\t1\t0\tACGT", "ESAM"),
    ("flag_sign", line(FLAG=b"+1"), "ESAM"),
    ("flag_range", line(FLAG=b"65536"), "ESAM"),
    ("mapq_range", line(MAPQ=b"256"), "ESAM"),
    ("pos_range", line(POS=b"2147483648"), "ESAM"),
    ("pos_empty", line(POS=b""), "ESAM"),
    ("tlen_junk", line(TLEN=b"1x"), "ESAM"),
    ("cigar_op", line(CIGAR=b"4Q"), "ESAM"),
    ("cigar_no_len", line(CIGAR=b"M"), "ESAM"),
    ("cigar_no_op", line(CIGAR=b"4M3"), "ESAM"),
    ("cigar_len_2p28", line(CIGAR=b"268435455M1M"), "ESAM"),
    ("tag_3_letters", line(tags=[b"NMX:i:1"]), "ESAM"),
    ("tag_1_letter", line(tags=[b"N:i:1"]), "ESAM"),
    ("tag_type", line(tags=[b"NM:q:1"]), "ESAM"),
    ("tag_type_sep", line(tags=[b"NM:ii:1"]), "ESAM"),
    ("tag_A_two", line(tags=[b"XA:A:ab"]), "ESAM"),
    ("tag_A_empty", line(tags=[b"XA:A:"]), "ESAM"),
    ("tag_H_odd", line(tags=[b"XH:H:abc"]), "ESAM"),
    ("tag_H_digit", line(tags=[b"XH:H:zz"]), "ESAM"),
    ("tag_B_neg_s", line(tags=[b"ZB:B:s,1,-2"]), "ESAM"),
    ("tag_B_empty_entry", line(tags=[b"ZB:B:c,1,"]), "ESAM"),
    ("tag_B_type", line(tags=[b"ZB:B:q,1"]), "ESAM"),
    ("tag_B_nocomma", line(tags=[b"ZB:B:c"]), "ESAM"),
    ("tag_i_low", line(tags=[b"XI:i:-2147483649"]), "ESAM"),
    ("tag_i_high", line(tags=[b"XI:i:4294967296"]), "ESAM"),
    ("tag_f_overflow", line(tags=[b"XF:f:3.4028236e38"]), "ESAM"),
    ("tag_f_syntax", line(tags=[b"XF:f:1e"]), "ESAM"),
    ("tag_f_hex", line(tags=[b"XF:f:0x1p3"]), "ESAM"),
    ("tag_f_nan_sign", line(tags=[b"XF:f:+nan"]), "ESAM"),
    ("tag_repeat_bad_first", line(tags=[b"NM:i:x", b"NM:i:1"]), "ESAM"),
    ("empty_segment", line(tags=[b"NM:i:1", b"", b"XA:A:c"]), "ESAM"),
    ("qname_255", line(QNAME=b"q" * 255), "ESAM"),
    ("qual_len", line(QUAL=b"III"), "ESAM"),
    ("empty_line", b"", "ESAM"),
    ("cigar_65536", line(CIGAR=b"1M1I" * 32768, SEQ=b"A" * 65536, QUAL=b"I" * 65536), "ELIMIT"),
]


@pytest.mark.parametrize("name,text,check", KAT, ids=[k[0] for k in KAT])
def test_kat(name, text, check):
    rec = sam_line_to_bam(text, HEADER)
    assert struct.unpack_from("<I", rec)[0] + 4 == len(rec)
    assert check(rec), (name, rec)


@pytest.mark.parametrize("name,text,kind", ERRORS, ids=[e[0] for e in ERRORS])
def test_errors(name, text, kind):
    with pytest.raises(SamError) as ei:
        sam_line_to_bam(text, HEADER)
    assert ei.value.kind == kind


def test_f32_halfway_and_denormals():
    """correct rounding from the exact decimal, not through float64: 1 + 2^-24 is half-way between two float32 values (ties to even)"""
    assert f32_bits(b"1.000000059604644775390625") == 0x3F800000
    assert f32_bits(b"1.000000059604644775390626") == 0x3F800001
    # just below 1 + 3 * 2^-24 (a half-way point): rounds down; float64 first would round it onto the half-way point and then up to ...02
    assert f32_bits(b"1.0000001788139343") == 0x3F800001
    assert f32_bits(b"7e-46") == 0x00000000 and f32_bits(b"7.1e-46") == 0x00000001
    assert f32_bits(b"3.40282356779733661637539395458142568447e38") == 0x7F7FFFFF   # just below the overflow threshold
    with pytest.raises(SamError):
        f32_bits(b"3.40282356779733661637539395458142568448e38")


def test_round_trip_synthetic_batch():
    """synthetic batch -> format_sam -> sam_line_to_bam -> decode_bam equals the batch on every path field"""
    w = synth.make_workload(300, [("chr20", 200_000), ("chr21", 100_000)], seed=5)
    b = w.batch
    lines = format_sam(b, w.header)
    raw, off = sam_lines_to_bam(lines, w.header)
    d = decode_bam(raw, off, w.header)
    for f in ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg", "qname_off", "qname", "cigar_off", "cigar", "lseq", "seq", "qual"):
        assert np.array_equal(getattr(d, f), getattr(b, f).astype(getattr(d, f).dtype)), f
    # the vectorised writer produces the same text
    assert sam_text(b, w.header).tobytes() == b"".join(x + b"\n" for x in lines)
    tags = b"NM:i:0\tXS:f:1.5"
    assert sam_text(b, w.header, const_tags=tags).tobytes().split(b"\n")[0].split(b"\t")[11:13] == tags.split(b"\t")


def test_parse_sam_header():
    text = (b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:1000\tM5:abc\n@SQ\tSN:chr2\tLN:500\n@RG\tID:g1\tLB:lib\tPU:u1\tSM:s\n"
            b"@PG\tID:bwa\tPN:bwa\tCL:bwa mem x y\n@CO\tfree text: anything\n@xy\tAB:1\n")
    h, n = sam.parse_sam_header(text + b"r1\t0\tchr1\t1\t60\t*\t*\t0\t0\t*\t*\n")
    assert n == len(text)
    assert h.HD == {"VN": "1.6", "SO": "coordinate"} and h.HDSO() == "coordinate"
    assert h.SQ == [{"SN": "chr1", "LN": "1000", "M5": "abc"}, {"SN": "chr2", "LN": "500"}]
    assert h.RG == [{"ID": "g1", "LB": "lib", "PU": "u1", "SM": "s"}]
    assert list(h.contig_lengths()) == [1000, 500]
    h2, n2 = sam.parse_sam_header(b"@SQ\tSN:c\tLN:5")          # header only, last line without '\n'
    assert n2 == 13 and h2.SQ == [{"SN": "c", "LN": "5"}]
    assert sam.parse_sam_header(b"") [1] == 0


@pytest.mark.parametrize("bad", [b"@SQ\tSN:c\tLN:5\n@HD\tVN:1.6\n", b"@XX\tAB:1\n", b"@SQ\tSN:c\tSN:d\n", b"@SQ\tSNN:c\n", b"@xy AB:1\n", b"@R\n", b"@CO\n",
                                 b"@PG\tIDbwa\n"])
def test_parse_sam_header_errors(bad):
    with pytest.raises(ValueError):
        sam.parse_sam_header(bad)
