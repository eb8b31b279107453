"""The --reference restatement (fasta_ref) against hand-derived known answers: ParseFasta and contigFromHeader
(fasta/fasta-files.go:75-89,159-229), OpenElfasta (:286-336), bufio.ScanLines, binary.Varint, the ToElfasta layout and the BGZF rules
of utils.HandleBGZF.  Each case in fasta_cases cites the Go line it follows."""
import pytest

import fasta_cases as fc
import fasta_ref as fr


@pytest.mark.parametrize("cid,text,want", fc.FASTA_VALID, ids=[c[0] for c in fc.FASTA_VALID])
def test_fasta_valid(cid, text, want):
    assert fr.parse_fasta(text) == want


@pytest.mark.parametrize("cid,text,where", fc.FASTA_INVALID, ids=[c[0] for c in fc.FASTA_INVALID])
def test_fasta_invalid(cid, text, where):
    with pytest.raises(fr.FastaError) as ei:
        fr.parse_fasta(text)
    assert (ei.value.line, ei.value.reason) == where


@pytest.mark.parametrize("cid,data,want", fc.ELFASTA_VALID, ids=[c[0] for c in fc.ELFASTA_VALID])
def test_elfasta_valid(cid, data, want):
    assert fr.open_elfasta(data) == want


@pytest.mark.parametrize("cid,data,where", fc.ELFASTA_INVALID, ids=[c[0] for c in fc.ELFASTA_INVALID])
def test_elfasta_invalid(cid, data, where):
    with pytest.raises(fr.ElfastaError) as ei:
        fr.open_elfasta(data)
    assert (ei.value.offset, ei.value.reason) == where


def test_scan_lines():
    """bufio.ScanLines: '\\n' ends a line, dropCR removes one '\\r', the final segment is a line only when non-empty; the byte after
    each token is what Go's b[len(b):len(b)+1] reads"""
    assert fr.scan_lines(b"a\nb\r\n\r\nc") == [(1, b"a", b"\n"), (2, b"b", b"\r"), (1, b"", b"\r"), (1, b"c", b"\x00")]
    assert fr.scan_lines(b"") == []
    assert fr.scan_lines(b"x\r\r\n") == [(3, b"x\r", b"\r")]


@pytest.mark.parametrize("v", [0, 1, -1, 63, -64, 64, 200, 1 << 40, -(1 << 62), (1 << 63) - 1, -(1 << 63)])
def test_varint_round_trip(v):
    """binary.PutVarint / Varint: zig-zag, 7 bits per byte"""
    b = fr.put_varint(v)
    assert fr.varint(b.ljust(10, b"\0")) == (v, len(b))


def test_varint_rejects():
    """binary.Uvarint: no terminating byte in the buffer -> n == 0; a 10th byte above 1 -> n < 0"""
    assert fr.varint(b"\x80" * 10)[1] == 0
    assert fr.varint(b"\xff" * 9 + b"\x02")[1] < 0
    assert fr.varint(b"\xff" * 9 + b"\x01") == (-(1 << 63), 10)


def test_elfasta_layout_round_trip():
    """ToElfasta's layout (any data order) reads back with OpenElfasta"""
    fa = {b"chr1": b"ACGT" * 10, b"chr2": b"", b"chrM": b"nN*"}
    for order in (None, [b"chrM", b"chr1", b"chr2"]):
        assert fr.open_elfasta(fr.to_elfasta(fa, order)) == fa


def test_bgzf_rules():
    """utils.HandleBGZF: the blocks read back; a plain gzip file (no BC subfield), a bad CRC32 and a missing EOF marker are refused"""
    import gzip
    text = b">chr1\n" + b"ACGTACGTAC\n" * 20000
    z = fr.bgzf_blocks(text, level=1)
    assert fr.inflate_bgzf(z) == text and fr.read_reference(z) == {b"chr1": b"ACGTACGTAC" * 20000}
    with pytest.raises(fr.BgzfError):
        fr.inflate_bgzf(gzip.compress(text))
    bad = bytearray(z)
    bad[-28 - 6] ^= 1                                 # the CRC32 of the last data block
    with pytest.raises(fr.BgzfError):
        fr.inflate_bgzf(bytes(bad))
    with pytest.raises(fr.BgzfError, match="EOF"):
        fr.inflate_bgzf(fr.bgzf_blocks(text, eof=False))


def test_load_counts():
    """unmatched: the file's names that are no SN (a nameless header always); missing: contigs without a sequence (each SN of a
    duplicate pair counts)"""
    text = b">chr1\nAC\n>other\nG\n>\nT\n>dup\nA\n>chr1\nTT\n"
    seqs, nu, nm = fr.load(text, ["chr1", "dup", "dup", "chrM", "\n"])
    assert seqs == [b"TT", b"A", b"A", None, None] and nu == 2 and nm == 2
    seqs, nu, nm = fr.load(fr.to_elfasta({b"chr1": b"AC", b"\x01": b"G"}), ["chr1", "\x01"])
    assert seqs == [b"AC", b"G"] and nu == 0 and nm == 0   # .elfasta names are byte strings without the header rule


def test_hot_nibbles():
    """the packing of elp_set_reference, low nibble first"""
    assert fr.hot_nibbles(b"ACGT") == bytes([0x21, 0x84])
    assert fr.hot_nibbles(b"a*cgtNx") == bytes([0x11, 0x42, 0x08, 0x00])
