"""`--replace-read-group` without a GPU: the flag's parser (sam.ParseHeaderLineFromString and elprep::ParseHeaderLineFromString against
hand-derived answers and against each other), filters.AddOrReplaceReadGroup on the header and the columns, and the restatement of SetRG
on BAM record bytes (tests/readgroup_ref.py) with the field filters after it and the SAM text of the result."""
import os
import struct
import subprocess

import numpy as np
import pytest

from elprep_b200 import filters, sam
from readgroup_ref import set_rg_record, set_rg_sam
from samformat import bam_to_sam

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (input bytes, expected dict of bytes or the start of the refusal)
PARSE = [
    (b"ID:g1 LB:lib1 PU:u1", {b"ID": b"g1", b"LB": b"lib1", b"PU": b"u1"}),
    (b"ID:a\tLB:b\nPU:c\vSM:d\fPL:e\rCN:f", {b"ID": b"a", b"LB": b"b", b"PU": b"c", b"SM": b"d", b"PL": b"e", b"CN": b"f"}),
    (b"  ID:a \t\n LB:b  \r\n", {b"ID": b"a", b"LB": b"b"}),
    (b"ID:a\xc2\x85LB:b", {b"ID": b"a", b"LB": b"b"}),                         # U+0085
    (b"ID:a\xc2\xa0LB:b", {b"ID": b"a", b"LB": b"b"}),                         # U+00A0
    (b"ID:a\xe2\x80\x80LB:b", {b"ID": b"a", b"LB": b"b"}),                     # U+2000
    (b"ID:a\xe2\x80\x8aLB:b", {b"ID": b"a", b"LB": b"b"}),                     # U+200A
    (b"ID:a\xe3\x80\x80LB:b", {b"ID": b"a", b"LB": b"b"}),                     # U+3000
    (b"ID:a\xe2\x80\x8bLB:b", {b"ID": b"a\xe2\x80\x8bLB:b"}),                   # U+200B is no space
    (b"ID:a\x1cLB:b", {b"ID": b"a\x1cLB:b"}),                                   # \x1c .. \x1f: Python's str.split splits there, Go does not
    (b"ID:a\x1dLB:b\x1eSM:c\x1fPL:d", {b"ID": b"a\x1dLB:b\x1eSM:c\x1fPL:d"}),
    (b"ID:a\x85LB:b", {b"ID": b"a\x85LB:b"}),                                   # the Latin-1 NEL byte alone is not valid UTF-8
    (b"ID:a\xa0LB:b", {b"ID": b"a\xa0LB:b"}),
    (b"ID:a\xc0\x85LB:b", {b"ID": b"a\xc0\x85LB:b"}),                           # overlong encoding of U+0005 / bad lead byte
    (b"ID:a\xe0\x82\x85LB:b", {b"ID": b"a\xe0\x82\x85LB:b"}),                   # overlong U+0085
    (b"ID:a\xc2 LB:b", {b"ID": b"a\xc2", b"LB": b"b"}),                         # a truncated sequence, then a space
    (b"ID:a\xe3\x80", {b"ID": b"a\xe3\x80"}),                                   # truncated U+3000 at the end
    (b"ID:\xc3\xa9t\xc3\xa9 LB:x", {b"ID": b"\xc3\xa9t\xc3\xa9", b"LB": b"x"}),
    (b"\xc3\xa9:x", {b"\xc3\xa9": b"x"}),                                       # a 2-byte tag that is one rune
    (b"ID:", {b"ID": b""}),
    (b"ID: LB:", {b"ID": b"", b"LB": b""}),
    (b"ID:a:b", {b"ID": b"a:b"}),
    (b"", {}),
    (b" \t\n", {}),
    (b"IDx:a", "incorrectly formatted SAM file field IDx:a"),
    (b"ID:a LBx", "incorrectly formatted SAM file field LBx"),
    (b"ID", "incorrectly formatted SAM file field ID"),
    (b"I:", "incorrectly formatted SAM file field I:"),
    (b"ID:a x", "incorrectly formatted SAM file field x"),
    (b"ID:a ID:b", "duplicate field tag ID in a SAM header line"),
    (b"ID:a LB:x ID:a", "duplicate field tag ID in a SAM header line"),
]


@pytest.mark.parametrize("line,want", PARSE, ids=[repr(x) for x, _ in PARSE])
def test_parse_header_line_bytes(line, want):
    if isinstance(want, str):
        with pytest.raises(ValueError) as ei:
            sam.ParseHeaderLineFromString(line)
        assert str(ei.value) == want
    else:
        assert sam.ParseHeaderLineFromString(line) == want


def test_parse_header_line_str():
    """a str is parsed as its UTF-8 bytes; the result is str, bytes that are no UTF-8 kept as surrogate escapes"""
    assert sam.ParseHeaderLineFromString("ID:grp\u3000LB:lib\u00a0PU:x\u0085SM:é") == {"ID": "grp", "LB": "lib", "PU": "x", "SM": "é"}
    assert sam.ParseHeaderLineFromString("ID:a\x1cb") == {"ID": "a\x1cb"}
    raw = b"ID:a\xff LB:b"
    assert sam.ParseHeaderLineFromString(raw.decode("utf-8", "surrogateescape")) == {"ID": "a\udcff", "LB": "b"}
    with pytest.raises(ValueError, match="duplicate field tag LB"):
        sam.ParseHeaderLineFromString("LB:x\u2003LB:y")


def test_cpp_parser_agrees(tmp_path):
    exe = str(tmp_path / "parse_rg_check")
    libdir = os.path.join(ROOT, "elprep_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "c", "parse_rg_check.cpp"),
                           "-o", exe, "-L", libdir, "-lelprep_b200", "-Wl,-rpath," + libdir])
    rng = np.random.default_rng(7)
    alphabet = [b"I", b"D", b":", b"L", b"B", b" ", b"\t", b"\x1c", b"\x85", b"\xc2", b"\xa0", b"\xe3\x80\x80", b"\xe3\x80", b"a", b"\xff", b"\xe2\x80\x80"]
    extra = [b"".join(alphabet[int(k)] for k in rng.integers(0, len(alphabet), int(rng.integers(0, 12)))) for _ in range(2000)]
    cases = [x for x, _ in PARSE] + extra
    out = subprocess.run([exe], input="".join(c.hex() + "\n" for c in cases), capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.split("\n")[:-1]
    assert len(lines) == len(cases)
    for c, got in zip(cases, lines):
        try:
            d = sam.ParseHeaderLineFromString(c)
            want = "ok" + "".join(f" {k.hex()}={v.hex()}" for k, v in sorted(d.items()))
        except ValueError as e:
            want = "panic " + str(e).encode("utf-8", "surrogateescape").hex()
        assert got == want, c


def test_add_or_replace_read_group_filter():
    """the Filter replaces header.RG; its AlignmentFilter puts every read in @RG 0; MarkDuplicates after it refuses LB without ID"""
    h = sam.Header(sq=[{"SN": "c", "LN": 100}], rg=[{"ID": "a", "LB": "x"}, {"ID": "b"}])
    rg = sam.ParseHeaderLineFromString("ID:new LB:lib PU:unit")
    b = sam.AlignmentBatch.from_records(h, [dict(QNAME="r1", RG="a"), dict(QNAME="r2", RG=None), dict(QNAME="r3", RG="b")])
    alns = filters.compose_filters(h, [filters.AddOrReplaceReadGroup(rg)])
    assert h.RG == [{"ID": "new", "LB": "lib", "PU": "unit"}]
    assert alns[0](b).rg.tolist() == [0, 0, 0]
    h2 = sam.Header(sq=[{"SN": "c", "LN": 100}], rg=[{"ID": "a"}])
    md, _, _ = filters.MarkDuplicates(False)
    with pytest.raises(ValueError, match="Missing mandatory ID entry in an @RG line in a SAM file header."):
        filters.compose_filters(h2, [filters.AddOrReplaceReadGroup({"LB": "lib"}), md])
    h3 = sam.Header(sq=[{"SN": "c", "LN": 100}], rg=[{"ID": "a"}])
    assert len(filters.compose_filters(h3, [filters.AddOrReplaceReadGroup({"PU": "p"}), md])) == 2   # no LB: no refusal


# ---- SetRG on BAM record bytes ----
NAMES = [b"chr1", b"chr2"]


def record(tags, name=b"q1"):
    """a mapped 4-base read on chr1 with the given optional-field bytes"""
    body = struct.pack("<iiBBHHHiiii", 0, 99, len(name) + 1, 60, 4680, 1, 99, 4, -1, -1, 0) + name + b"\0" + struct.pack("<I", (4 << 4) | 0)
    body += bytes([0x12, 0x48]) + bytes([30, 31, 32, 33]) + tags
    return struct.pack("<I", len(body)) + body


NM, XA, MD = b"NMC\x01", b"XAAq", b"MDZ10\0"
NEW = b"RGZgrp\0"
SETRG = [   # (stored fields, fields after SetRG("grp")), derived by hand from SmallMap.Set
    ("first", b"RGZold\0" + NM, NEW + NM),
    ("middle", NM + b"RGZold\0" + XA, NM + NEW + XA),
    ("last", NM + MD + b"RGZold\0", NM + MD + NEW),
    ("type_A", NM + b"RGAx" + XA, NM + NEW + XA),
    ("type_i", b"RGi" + struct.pack("<i", -7) + NM, NEW + NM),
    ("type_f", NM + b"RGf" + struct.pack("<f", 2.5) + b"XSf" + struct.pack("<f", 1.5), NM + NEW + b"XSf" + struct.pack("<f", 1.5)),
    ("type_H", b"RGH1AE3\0" + NM, NEW + NM),
    ("type_Bf", b"RGBf" + struct.pack("<I", 2) + struct.pack("<2f", 0.5, -1.25) + NM, NEW + NM),
    ("two_rg", b"RGi" + struct.pack("<i", 3) + XA + b"RGZold\0", NEW + XA + b"RGZold\0"),
    ("two_rg_z", b"RGZa\0RGZb\0", NEW + b"RGZb\0"),
    ("no_rg", NM + XA, NM + XA + NEW),
    ("no_fields", b"", NEW),
    ("same_value", b"RGZgrp\0" + NM, NEW + NM),
]


@pytest.mark.parametrize("name,stored,want", SETRG, ids=[c[0] for c in SETRG])
def test_set_rg_record(name, stored, want):
    assert set_rg_record(record(stored), b"grp") == record(want)


FILTERS = [   # (field filter, fields written for the "two_rg" record, for a record with NM only), by hand: SetRG first, then
              # RemoveOptionalFields, then KeepOptionalFields; the appended field is filtered as RG too
    (dict(remove=("RG",)), XA, NM),
    (dict(remove=("XA",)), NEW + b"RGZold\0", NM + NEW),
    (dict(remove=("XA", "RG")), b"", NM),
    (dict(keep=("XA",)), XA, b""),
    (dict(keep=("RG",)), NEW + b"RGZold\0", NEW),
    (dict(keep=("RG", "XA")), NEW + XA + b"RGZold\0", NEW),
    (dict(keep=("NM", "RG")), NEW + b"RGZold\0", NM + NEW),
    (dict(keep=()), b"", b""),
    (dict(remove=("RG",), keep=("RG", "XA")), XA, b""),
]


@pytest.mark.parametrize("flt,want,want_nm", FILTERS, ids=[repr(f[0]) for f in FILTERS])
def test_set_rg_then_field_filters(flt, want, want_nm):
    assert set_rg_record(record(b"RGi" + struct.pack("<i", 3) + XA + b"RGZold\0"), b"grp", **flt) == record(want)
    assert set_rg_record(record(NM), b"grp", **flt) == record(want_nm)


def test_set_rg_empty_id():
    assert set_rg_record(record(NM), b"") == record(NM + b"RGZ\0")
    assert set_rg_record(record(b"RGZx\0"), b"") == record(b"RGZ\0")


def test_sam_text():
    """the SAM line of the rewritten record: RG:Z:id where the first RG field was, behind the last field without one"""
    prefix = bam_to_sam(record(b""), NAMES)[:-1]
    assert prefix == b"q1\t99\tchr1\t100\t60\t4M\t*\t0\t0\tACGT\t?@AB"
    cases = [(b"RGZold\0" + NM, b"\tRG:Z:grp\tNM:i:1"), (NM + XA, b"\tNM:i:1\tXA:A:q\tRG:Z:grp"),
             (NM + b"RGf" + struct.pack("<f", 2.5) + b"XSf" + struct.pack("<f", 1.5), b"\tNM:i:1\tRG:Z:grp\tXS:f:1.5"),
             (b"RGBf" + struct.pack("<I", 2) + struct.pack("<2f", 0.5, -1.25) + b"XSBf" + struct.pack("<I", 1) + struct.pack("<f", 0.25), b"\tRG:Z:grp\tXS:B:f,0.25"),
             (b"RGi" + struct.pack("<i", 3) + XA + b"RGZold\0", b"\tRG:Z:grp\tXA:A:q\tRG:Z:old"),
             (b"RGH1AE3\0", b"\tRG:Z:grp")]
    for stored, tail in cases:
        assert set_rg_sam(record(stored), b"grp", NAMES) == prefix + tail + b"\n"
    assert set_rg_sam(record(NM + XA), b"grp", NAMES, remove=("RG",)) == prefix + b"\tNM:i:1\tXA:A:q\n"
    assert set_rg_sam(record(NM + XA), b"grp", NAMES, keep=("RG",)) == prefix + b"\tRG:Z:grp\n"
    assert set_rg_sam(record(NM), b"", NAMES) == prefix + b"\tNM:i:1\tRG:Z:\n"
