"""`--rename-chromosomes` and `--replace-reference-sequences` without a GPU: the header transforms of filters.RenameChromosomes and
filters.ReplaceReferenceSequenceDictionary (the SO rule with utils.Find's first match) against hand-derived answers and against their C++
counterparts, the columnar AlignmentFilter, and the restatement of the filters plus AddREFID on BAM record bytes (tests/refdict_ref.py) with
the SAM text of the result."""
import os
import struct
import subprocess

import numpy as np
import pytest

from elprep_b200 import filters, sam
from refdict_ref import RENAME, REPLACE, refdict_record, refdict_sam

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header(names, so=sam.Coordinate):
    return sam.Header(sq=[{"SN": n, "LN": 100 + i} for i, n in enumerate(names)], so=so)


def replaced(old, new, so=sam.Coordinate):
    h = header(old, so)
    filters.ReplaceReferenceSequenceDictionary([{"SN": n, "LN": 1} for n in new])(h)
    return h.HDSO(), h.contig_names()


# (old names, new names, SO after the replacement of an SO:coordinate header)
SO_CASES = [
    (["a", "b", "c"], ["a", "b", "c"], sam.Coordinate),
    (["a", "b", "c"], ["c", "b", "a"], sam.Unknown),                      # reordered
    (["a", "b", "c"], ["a", "c"], sam.Coordinate),                        # subset, in order
    (["a", "b", "c"], ["b", "a"], sam.Unknown),                           # subset, out of order
    (["a", "b"], ["x", "a", "y", "b", "z"], sam.Coordinate),              # superset: the new names are not looked at
    (["a", "b"], ["b", "x", "a"], sam.Unknown),
    (["a", "b", "a"], ["b", "a"], sam.Unknown),                           # Find: "a" is found at 0 (first match), after "b" at 1
    (["a", "b", "a"], ["a", "b"], sam.Coordinate),
    (["a", "b"], ["a", "a"], sam.Unknown),                                # a name twice in the new dictionary: 0, then 0 again
    (["a", "b"], [], sam.Coordinate),                                     # an empty replacement
]


@pytest.mark.parametrize("old,new,so", SO_CASES)
def test_so_rule(old, new, so):
    got_so, got_names = replaced(old, new)
    assert got_so == so and got_names == new


@pytest.mark.parametrize("so", [sam.Queryname, sam.Unknown, sam.Unsorted])
def test_so_rule_only_for_coordinate(so):
    assert replaced(["a", "b"], ["b", "a"], so)[0] == so


def test_rename_header():
    h = header(["1", "chr1", "X"])
    h.SQ.append({"LN": 5})                                                # an @SQ without SN stays without one
    assert filters.RenameChromosomes(h) is None
    assert [e.get("SN") for e in h.SQ] == ["chr1", "chrchr1", "chrX", None]


def test_dictionary_remap():
    assert filters.dictionary_remap(["a", "b", "c"], ["c", "a"]).tolist() == [1, -1, 0]
    assert filters.dictionary_remap(["a", "a", "b"], ["b", "a", "a"]).tolist() == [2, 2, 0]   # the last of equal new names wins
    assert filters.dictionary_remap(["a"], []).tolist() == [-1]
    assert filters.dictionary_remap([], ["a"]).tolist() == []


def test_columnar_filter():
    h = header(["a", "b", "c"])
    z = np.zeros(5, np.int32)
    b = sam.AlignmentBatch(refid=np.array([0, 1, 2, -1, 2], np.int32), nref=np.array([1, 0, -1, 2, 1], np.int32), pos=np.arange(1, 6, dtype=np.int32),
                           flag=z, mapq=z, pnext=z, tlen=z, rg=z - 1, qname_off=np.arange(6, dtype=np.uint64), qname=np.frombuffer(b"abcde", np.uint8),
                           cigar_off=np.zeros(6, np.uint64), cigar=np.zeros(0, np.uint32), lseq=z, seq=np.zeros(0, np.uint8), qual=np.zeros(0, np.uint8),
                           opt_flags=np.zeros(5, np.uint8))
    flt = filters.ReplaceReferenceSequenceDictionary([{"SN": "c", "LN": 1}, {"SN": "a", "LN": 1}])(h)
    out = flt(b)
    assert out.pos.tolist() == [1, 3, 4, 5]                               # refid 1 ("b") has no new entry: dropped; "*" kept
    assert out.refid.tolist() == [1, 0, -1, 0]
    assert out.nref.tolist() == [-1, -1, 0, -1]                           # RNEXT "b" on a dropped contig: -1


def rec(refid, nref, pnext=7, tail=b"XYZhello\0"):
    """a minimal BAM record: name "r", no CIGAR, one base"""
    body = struct.pack("<iiBBHHHiiii", refid, 99, 2, 30, 4680, 0, 0, 1, nref, pnext, 0) + b"r\0" + b"\x10" + b"\x1e" + tail
    return struct.pack("<I", len(body)) + body


def ids(r):
    return struct.unpack_from("<i", r, 4)[0], struct.unpack_from("<i", r, 24)[0]


IN = [b"1", b"chr1", b"2", b"2"]


def test_record_rename_only():
    for rid, nid in [(0, 1), (1, 0), (3, 2), (-1, -1), (2, -1)]:
        r = rec(rid, nid)
        assert refdict_record(r, IN, RENAME, [b"chr1", b"chrchr1", b"chr2", b"chr2"]) == r   # ids as read
    assert refdict_sam(rec(0, 1), IN, RENAME, None).split(b"\t")[2:7] == [b"chr1", b"100", b"30", b"*", b"chrchr1"]
    assert refdict_sam(rec(2, 3), IN, RENAME, None).split(b"\t")[6] == b"="             # equal names: "="


def test_record_replace():
    out = [b"chr2", b"chr1", b"chrX", b"chr2"]                                        # duplicate SN in the new dictionary
    mode = RENAME | REPLACE
    assert ids(refdict_record(rec(0, 2), IN, mode, out)) == (1, 3)                     # "chr1" -> 1, "chr2" -> the last, 3
    assert ids(refdict_record(rec(3, 0), IN, mode, out)) == (3, 1)                     # a duplicate old name ("2" twice) -> 3
    assert refdict_record(rec(1, 0), IN, mode, out) is None                            # "chrchr1" is not in the new dictionary
    r = refdict_record(rec(0, 1, pnext=55), IN, mode, out)
    assert ids(r) == (1, -1) and struct.unpack_from("<i", r, 28)[0] == 55                # RNEXT on a dropped contig: -1, PNEXT kept
    assert ids(refdict_record(rec(-1, -1), IN, mode, out)) == (-1, -1)                 # RNAME "*": kept
    assert ids(refdict_record(rec(-1, 0), IN, mode, out)) == (-1, 1)
    line = refdict_sam(rec(0, 1), IN, mode, out)
    assert line.split(b"\t")[2] == b"chr1" and line.split(b"\t")[6] == b"chrchr1"      # SAM keeps the RNEXT name
    assert ids(refdict_record(rec(0, 2), IN, REPLACE, [b"2", b"1"])) == (1, 0)        # replace without rename
    assert refdict_record(rec(0, 2), IN, REPLACE, [b"chr1"]) is None


def test_record_empty_replacement():
    for rid, nid in [(0, 0), (2, -1), (3, 1)]:
        assert refdict_record(rec(rid, nid), IN, REPLACE, []) is None
    assert ids(refdict_record(rec(-1, 2), IN, REPLACE, [])) == (-1, -1)


def test_record_bytes_untouched():
    """only bytes 4-7 and 24-27 change"""
    r = rec(0, 2)
    o = refdict_record(r, IN, RENAME | REPLACE, [b"chr2", b"chr1"])
    assert len(o) == len(r) and o[:4] == r[:4] and o[8:24] == r[8:24] and o[28:] == r[28:]


def _cpp_cases(rng, n):
    pool = ["1", "2", "chr1", "chr2", "X", "chrX", "a"]
    cases = []
    for _ in range(n):
        so = [sam.Coordinate, sam.Queryname, sam.Unknown, ""][int(rng.integers(0, 4))]
        mode = int(rng.integers(1, 4))
        old = [pool[int(k)] for k in rng.integers(0, len(pool), int(rng.integers(0, 6)))]
        new = [pool[int(k)] for k in rng.integers(0, len(pool), int(rng.integers(0, 6)))]
        cases.append((so, mode, old, new))
    return cases


def test_cpp_header_transforms_agree(tmp_path):
    exe = str(tmp_path / "refdict_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "refdict_check.cpp"), "-o", exe])
    cases = [(sam.Coordinate, REPLACE, o, n) for o, n, _ in SO_CASES] + [(sam.Coordinate, RENAME | REPLACE, ["1", "2"], ["chr2", "chr1"])]
    cases += _cpp_cases(np.random.default_rng(11), 2000)
    enc = lambda xs: ",".join(x.encode().hex() for x in xs)
    inp = "".join(f"{so.encode().hex()}\t{mode}\t{enc(old)}\t{enc(new)}\n" for so, mode, old, new in cases)
    out = subprocess.run([exe], input=inp, capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.split("\n")[:-1]
    assert len(lines) == len(cases)
    for (so, mode, old, new), got in zip(cases, lines):
        h = header(old, so)
        if mode & RENAME:
            filters.RenameChromosomes(h)
        if mode & REPLACE:
            filters.ReplaceReferenceSequenceDictionary([{"SN": n, "LN": 1} for n in new])(h)
        assert got == f"{h.HDSO().encode().hex()}\t{enc(h.contig_names())}", (so, mode, old, new)


def test_from_sam_file(tmp_path):
    p = tmp_path / "ref.dict"
    p.write_bytes(b"@HD\tVN:1.6\n@SQ\tSN:chr2\tLN:20\tM5:x\n@SQ\tSN:chr1\tLN:10\n")
    h = header(["chr1", "chr2"])
    flt = filters.ReplaceReferenceSequenceDictionaryFromSamFile(str(p))(h)
    assert h.contig_names() == ["chr2", "chr1"] and h.contig_lengths().tolist() == [20, 10] and h.HDSO() == sam.Unknown
    assert flt is not None
