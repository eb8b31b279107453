"""The write-phase filters on the host side: the restatement of RemoveOptionalFields / KeepOptionalFields over BAM record bytes
(tests/outfilter.py) against hand-derived answers, its agreement with FormatAlignment of the filtered TAGS list, the translation of the
`elprep filter` flags into elp_set_output_filter arguments (cmd/filter.go:803-902) and ClearDuplicateFlag on a batch."""
import struct

import numpy as np
import pytest

from elprep_b200 import _lib, filters, sam
from outfilter import fields, filter_record, filter_tags
from samformat import bam_to_sam, format_alignment, parse_bam_alignment
from test_sam_format import LINES, NAMES, bam_record

# one field of every type; the Z value holds text that looks like a tag; NM comes twice
A_ = b"XAAq"
c_ = b"c1c\x80"
C_ = b"C1C\xff"
s_ = b"s1s\x00\x80"
S_ = b"S1S\xff\xff"
i_ = b"i1i\x00\x00\x00\x80"
I_ = b"I1I\xff\xff\xff\xff"
f_ = b"f1f" + struct.pack("<f", 1.5)
Z_ = b"MDZNM:i:5\0"
H_ = b"H1H1AFF\0"
Bc = b"BcBc\x02\x00\x00\x00\x80\x7f"
BC = b"BCBC\x01\x00\x00\x00\xff"
Bs = b"BsBs\x02\x00\x00\x00\xff\xff\x00\x80"
BS = b"BSBS\x01\x00\x00\x00\xff\xff"
Bi = b"BiBi\x01\x00\x00\x00\x00\x00\x00\x80"
BI = b"BIBI\x01\x00\x00\x00\xff\xff\xff\xff"
Bf = b"BfBf\x02\x00\x00\x00" + struct.pack("<2f", 1.5, -2.0)
NM1 = b"NMC\x01"
NM2 = b"NMi\x02\x00\x00\x00"
ALL = [A_, c_, C_, s_, S_, i_, I_, f_, Z_, H_, Bc, BC, Bs, BS, Bi, BI, Bf, NM1, NM2]

KNOWN = [
    ("none", (), None, ALL),
    ("remove_only", ("c1", "S1", "f1", "H1", "Bs", "Bf", "NM"), None, [A_, C_, s_, i_, I_, Z_, Bc, BC, BS, Bi, BI]),
    ("keep_only", None, ("MD", "NM", "BI"), [Z_, BI, NM1, NM2]),
    ("keep_none", None, (), []),
    ("remove_then_keep", ("NM", "XA"), ("NM", "MD", "XA", "i1"), [i_, Z_]),
    ("remove_case_and_lengths", ("nm", "", "N", "NMX", "md"), None, ALL),
    ("keep_case", None, ("nm",), []),
    ("keep_lengths", None, ("MD", "", "N", "MDX"), [Z_]),
    ("remove_Z_text", ("NM",), None, [x for x in ALL if x not in (NM1, NM2)]),
]


@pytest.mark.parametrize("name,remove,keep,want", KNOWN, ids=[k[0] for k in KNOWN])
def test_known_answers(name, remove, keep, want):
    rec = bam_record(tags=b"".join(ALL))
    got = filter_record(rec, remove or (), keep)
    assert got == bam_record(tags=b"".join(want))
    assert struct.unpack_from("<I", got)[0] == len(got) - 4


def test_field_walk():
    rec = bam_record(tags=b"".join(ALL))
    t0, fl = fields(rec)
    assert rec[t0:] == b"".join(ALL)
    assert [rec[s:e] for _, s, e in fl] == ALL
    assert [t for t, _, _ in fl][-2:] == [b"NM", b"NM"]


@pytest.mark.parametrize("remove,keep", [((), None), (("NM",), None), ((), ()), (("XA",), ("XA", "MD"))])
def test_record_without_fields(remove, keep):
    rec = bam_record()
    assert fields(rec)[1] == []
    assert filter_record(rec, remove, keep) == rec


SHAPES = [(("XA", "a3", "B7", "MD", "XH", "XS"), None), ((), ("a1", "a6", "B3", "XC", "XT", "E2")), ((), ()), (("a1", "XE", "B2"), ("a1", "a2", "XE", "XI", "B2", "B4", "XV"))]


@pytest.mark.parametrize("name,rec,text", LINES, ids=[x[0] for x in LINES])
def test_sam_of_filtered_record(name, rec, text):
    """FormatAlignment of the filtered record equals FormatAlignment with the same filters applied to the parsed TAGS list"""
    for remove, keep in SHAPES:
        a = parse_bam_alignment(rec, NAMES)
        a["TAGS"] = filter_tags(a["TAGS"], remove, keep)
        assert bam_to_sam(filter_record(rec, remove, keep), NAMES) == format_alignment(a), (remove, keep)


K, R, D, S = _lib.OUT_KEEP_FIELDS, _lib.OUT_REMOVE_OPTIONAL_READS, _lib.OUT_REMOVE_DUPLICATES, None


@pytest.mark.parametrize("args,want", [
    ((False, "", "", False), (0, [], None)),
    ((True, "", "", False), (D, [], None)),
    ((False, "", "", True), (R, [], None)),
    ((True, "", "", True), (D | R, [], None)),
    ((False, "all", "", False), (K, [], [])),                             # KeepOptionalFields(nil)
    ((False, "", "none", False), (K, [], [])),
    ((False, "XA, MD", "", False), (0, ["XA", "MD"], None)),              # comma split, TrimSpace
    ((False, ",", "", False), (0, ["", ""], None)),                       # two empty strings: match nothing
    ((False, " all", "", False), (0, ["all"], None)),                     # "all" is compared before trimming
    ((False, "", " RG ,NM", False), (K, [], ["RG", "NM"])),
    ((False, "", ",", False), (K, [], ["", ""])),                         # keeps nothing
    ((True, "XA", "RG,XA", True), (D | R | K, ["XA"], ["RG", "XA"])),     # both flags: remove, then keep
    ((False, "all", "RG", False), (K, [], [])),                           # KeepOptionalFields(nil), then KeepOptionalFields(RG): nothing left
    ((False, "XA", "none", False), (K, ["XA"], [])),
])
def test_write_phase_flags(args, want):
    assert filters.write_phase_filters(*args) == want


@pytest.mark.parametrize("rof,kof", [("all", ""), ("", "none"), ("XA, MD", ""), (",", ""), ("", "RG, XA"), ("XA", "RG,XA"), ("all", "RG"), ("NM", ",")])
def test_write_phase_flags_act_as_filters2(rof, kof):
    """the translated arguments drop exactly the fields the filters2 chain of cmd/filter.go drops"""
    rec = bam_record(tags=b"".join(ALL) + b"RGZrg1\0" + b"XAAz")
    chain = []                                                           # filters2, in the order cmd/filter.go appends them
    if rof:
        chain.append(("keep", []) if rof == "all" else ("remove", [t.strip() for t in rof.split(",")]))
    if kof:
        chain.append(("keep", [] if kof == "none" else [t.strip() for t in kof.split(",")]))
    want = rec
    for kind, tags in chain:
        want = filter_record(want, tags, None) if kind == "remove" else filter_record(want, (), tags)
    _, remove, keep = filters.write_phase_filters(False, rof, kof, False)
    assert filter_record(rec, remove, keep) == want


def test_clear_duplicate_flag():
    n = 4
    b = sam.AlignmentBatch(refid=[0] * n, pos=[1] * n, flag=[0x400, 0x401, 0x10, 0xffff], mapq=[60] * n, nref=[-1] * n, pnext=[0] * n, tlen=[0] * n,
                           rg=[-1] * n, qname_off=np.arange(n + 1), qname=np.frombuffer(b"abcd", np.uint8), cigar_off=np.zeros(n + 1), cigar=[],
                           lseq=[0] * n, seq=[], qual=[])
    before = b.flag.copy()
    out = filters.ClearDuplicateFlag(None)(b)
    assert out.flag.dtype == np.uint16 and list(out.flag) == [0, 0x1, 0x10, 0xfbff]
    assert list(before) == [0x400, 0x401, 0x10, 0xffff]
