"""--reference known answers, derived by hand from fasta/fasta-files.go (ParseFasta :159-229, contigFromHeader :75-89, OpenElfasta
:286-336), bufio.ScanLines and binary.Varint.

FASTA_VALID:    (id, text, {name: sequence}) -- the whole map ParseFasta returns
FASTA_INVALID:  (id, text, (1-based line, reason))
ELFASTA_VALID:  (id, bytes, {name: sequence})
ELFASTA_INVALID: (id, bytes, (byte offset, reason))
NAMES: the @SQ names the GPU test loads the cases against."""
from fasta_ref import (BAD_OFFSET, BAD_SIZE, EMPTY_FILE, EMPTY_LINE, FIRST_HEADER, LONG, MAGIC, NAME_END, OFFSET_END, RANGE, SIZE_END,
                       TABLE_END, put_varint)

NAMES = ["chr1", "chr2", "chrM", "dup", "dup", "x", "never"]   # "dup": two @SQ lines share one SN; "never" is in no file


def field(v):
    return put_varint(v).ljust(10, b"\0")


def entry(name, off, size):
    return name + b"\t" + field(off) + field(size)


FASTA_VALID = [
    # :170-186: the first header, then sequence lines appended verbatim (toUpper and toN false)
    ("basic", b">chr1\nACGT\nTTAA\n>chr2\nGG\n", {b"chr1": b"ACGTTTAA", b"chr2": b"GG"}),
    # bufio.ScanLines: the last line may lack its '\n'; one '\r' before '\n' is dropped
    ("no_final_newline_crlf", b">chr1\r\nAC\r\nGT", {b"chr1": b"ACGT"}),
    # :174-180: empty lines (and "\r" lines, which ScanLines makes empty) before the first header are skipped
    ("leading_empty", b"\n\r\n\n>chr1\nA\n", {b"chr1": b"A"}),
    # :192-197: after empty lines, a header continues the parse; :194-196: after empty lines, the end of the file ends it
    ("empty_between_and_after", b">chr1\nAC\n\n\n>chr2\nG\n\n\n", {b"chr1": b"AC", b"chr2": b"G"}),
    # :75-89: the name is the first run of '!'..'~' after index 1: leading blanks and control bytes are skipped, the run ends at a blank
    ("name_rule", b">  \tchr1 description here\nA\n>chr2|x:1-5\tmore\nC\n", {b"chr1": b"A", b"chr2|x:1-5": b"C"}),
    # :83: the name starts at index 1 even without blanks; a '>' inside the name stays
    ("name_gt", b">>x\nA\n>x>y\nC\n", {b">x": b"A", b"x>y": b"C"}),
    # :207-221: every other line is appended verbatim: lower case, IUPAC, blanks, ';', '>' not at byte 0, bytes 0x80-0xff, a lone '\r'
    ("verbatim", b">chr1\nacgtNRYKM\n A;C\tG\nT>G\n\x80\xff\x00\nA\rC\n", {b"chr1": b"acgtNRYKM A;C\tGT>G\x80\xff\x00A\rC"}),
    # :187-192: a header with no sequence lines gives an empty sequence
    ("empty_sequence", b">chr1\n>chr2\nAC\n>chrM\n", {b"chr1": b"", b"chr2": b"AC", b"chrM": b""}),
    # :192: map assignment -- the later of equal names wins, even when it is empty
    ("duplicate_later_wins", b">chr1\nAAAA\n>chr2\nC\n>chr1\nGG\n>chr2\n", {b"chr1": b"GG", b"chr2": b""}),
    # :88 with no byte in '!'..'~': Go slices one byte past the token -- the '\n' (or the dropped '\r'); such a name matches nothing
    ("nameless_header", b">\nAC\n> \t\r\nGT\n>chr1\nA\n", {b"\n": b"AC", b"\r": b"GT", b"chr1": b"A"}),
    # ... and at the end of the file, where Go reads a stale buffer byte, the restatement takes 0
    ("nameless_last", b">chr1\nA\n>", {b"chr1": b"A", b"\x00": b""}),
    # the longest line the scanner accepts: 65535 bytes before '\n'
    ("line_65535", b">chr1\n" + b"A" * 65535 + b"\nC\n", {b"chr1": b"A" * 65535 + b"C"}),
    # a header only, without '\n'
    ("header_only", b">chrM", {b"chrM": b""}),
    # two SNs share "dup"; "x" is a one-letter name
    ("dup_sn", b">dup\nACGTN*\n>x\nt\n", {b"dup": b"ACGTN*", b"x": b"t"}),
]

FASTA_INVALID = [
    # :164-173: no first line, or only empty lines: "empty fasta file"
    ("empty_file", b"", (1, EMPTY_FILE)),
    ("only_empty_lines", b"\n\r\n\n", (4, EMPTY_FILE)),
    # :181-183: the first non-empty line must start with '>'
    ("missing_first_header", b"ACGT\n>chr1\nA\n", (1, FIRST_HEADER)),
    ("missing_first_header_after_empty", b"\n\nAC\n", (3, FIRST_HEADER)),
    ("space_before_gt", b" >chr1\nA\n", (1, FIRST_HEADER)),
    # :197-199: after empty lines, anything but a header is refused -- inside a sequence, or between a header and its first line
    ("empty_inside_sequence", b">chr1\nAC\n\nGT\n", (4, EMPTY_LINE)),
    ("empty_after_header", b">chr1\n\nAC\n", (3, EMPTY_LINE)),
    ("crlf_empty_inside", b">chr1\r\nAC\r\n\r\n\r\nGT\r\n", (5, EMPTY_LINE)),
    # bufio.Scanner: a line of 65536 bytes or more stops the scanner; the reference then panics (scanner.Err, or "empty fasta file")
    ("line_65536", b">chr1\nA\n" + b"C" * 65536 + b"\n", (3, LONG)),
    ("line_65536_unterminated", b">chr1\n" + b"C" * 65536, (2, LONG)),
    ("line_65535_cr", b">chr1\n" + b"C" * 65535 + b"\r\n", (2, LONG)),
    ("first_line_long", b">" + b"n" * 70000 + b"\n", (1, LONG)),
    # the first failure in file order wins: an empty-line refusal before a long line
    ("empty_before_long", b">c\n\nA\n" + b"C" * 70000 + b"\n", (3, EMPTY_LINE)),
]


def _elfasta(entries, data, tail=b"\n"):
    """magic + the table (names with (offset, size) relative to the data start) + tail + data; the offsets made absolute"""
    size = len(MAGIC) + sum(len(n) + 21 for n, _, _ in entries) + len(tail)
    out = bytearray(MAGIC)
    for n, o, s in entries:
        out += entry(n, size + o, s)
    return bytes(out) + tail + data


ELFASTA_VALID = [
    # :301-326: entries until one begins with '\n'; sequences are slices of the file
    ("basic", _elfasta([(b"chr1", 0, 4), (b"chr2", 4, 2)], b"ACGTGG"), {b"chr1": b"ACGT", b"chr2": b"GG"}),
    # :323: the last of equal names wins
    ("duplicate_last_wins", _elfasta([(b"chr1", 0, 2), (b"chr1", 2, 3)], b"AAGGG"), {b"chr1": b"GGG"}),
    # sequences may overlap, alias and come in any order; an empty one is fine
    ("overlap_alias", _elfasta([(b"chr2", 2, 4), (b"chr1", 0, 4), (b"x", 0, 4), (b"chrM", 6, 0)], b"ACGTNN"),
     {b"chr2": b"GTNN", b"chr1": b"ACGT", b"x": b"ACGT", b"chrM": b""}),
    # no entries at all
    ("empty_table", MAGIC + b"\n", {}),
    # names are any bytes up to '\t' (even blanks); the data may hold any byte
    ("odd_names", _elfasta([(b"chr 1", 0, 3), (b"dup", 3, 3)], bytes([0, 0x41, 0xff, 0x61, 0x63, 0x2a])),
     {b"chr 1": bytes([0, 0x41, 0xff]), b"dup": b"ac*"}),
    # a varint of more than one byte, with trailing garbage after it in the 10-byte field ignored by binary.Varint
    ("long_varint", MAGIC + b"chr1\t" + put_varint(200).ljust(10, b"\xee") + field(3) + b"\n" + b"N" * (200 - 30) + b"ACG",
     {b"chr1": b"ACG"}),
]

ELFASTA_INVALID = [
    # :305-306: data[index] past the end of the file: no '\n' closes the table
    ("table_no_end", MAGIC, (4, TABLE_END)),
    ("table_no_end_after_entry", MAGIC + entry(b"chr1", 0, 0), (4 + 25, TABLE_END)),
    # :307-308: the name runs past the end of the file
    ("name_runs_off", MAGIC + b"chr1", (4, NAME_END)),
    # :311: data[index : index+10] past the end of the file
    ("offset_field_short", MAGIC + b"chr1\t" + b"\x00" * 9, (9, OFFSET_END)),
    ("size_field_short", MAGIC + b"chr1\t" + field(0) + b"\x00" * 9, (19, SIZE_END)),
    # :312-316: binary.Varint n <= 0 -- no terminating byte within 10 bytes, or an overflow in the 10th byte
    ("offset_no_terminator", MAGIC + b"chr1\t" + b"\x80" * 10 + field(0) + b"\n", (9, BAD_OFFSET)),
    ("size_overflow", MAGIC + b"chr1\t" + field(0) + b"\xff" * 9 + b"\x02" + b"\n", (19, BAD_SIZE)),
    # :323: data[offset : offset+size] out of range -- a negative offset, a negative size, past the end
    ("negative_offset", MAGIC + entry(b"chr1", -1, 1) + b"\n", (9, RANGE)),
    ("negative_size", MAGIC + entry(b"chr1", 30, -1) + b"\nA", (9, RANGE)),
    ("past_end", MAGIC + entry(b"chr1", 30, 2) + b"\nA", (9, RANGE)),
    # a bad entry after good ones refuses the whole file
    ("bad_second_entry", MAGIC + entry(b"chr1", 55, 1) + entry(b"chr2", 55, 5) + b"\nA", (34, RANGE)),
]
