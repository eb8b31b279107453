""".elsites known answers, derived by hand from intervals/intervals.go:199-254, bufio.ScanLines and strconv.ParseInt.

VALID:   (id, files, {contig name: flattened [(start, end)]}, unmatched lines) over the header NAMES
INVALID: (id, files, (file index, line, reason)); lines are 0-based with the header as line 0

The CPU test pins elsites_ref against these answers; the GPU test loads every case through elp_load_known_sites."""
from elsites_ref import END, FIELDS, HEADER, HEADER_BAD, LONG, START

H = HEADER
NAMES = ["chr1", "chr10", "chr1_alt", "chrX", "dup", "dup", "*"]   # "dup": two @SQ lines share one SN; a contig literally named "*"

VALID = [
    # intervals.go:221-247: chromosome before the first tab, start between the tabs, end the rest of the line
    ("basic", [H + b"chr1\t10\t20\nchr1\t30\t40\n"], {"chr1": [(10, 20), (30, 40)]}, 0),
    # bufio.ScanLines: the last line may lack its '\n'
    ("no_final_newline", [H + b"chr1\t10\t20\nchr10\t5\t6"], {"chr1": [(10, 20)], "chr10": [(5, 6)]}, 0),
    # ScanLines drops one '\r' before '\n' (dropCR), also on an unterminated last line
    ("crlf", [H + b"chr1\t1\t2\r\nchr1\t5\t9\r"], {"chr1": [(1, 2), (5, 9)]}, 0),
    # header only, and an empty segment after the last '\n' is no line
    ("header_only", [H], {}, 0),
    # ParseInt(s, 10, 32): an optional sign and leading zeros are accepted
    ("signs_zeros", [H + b"chrX\t+5\t007\nchrX\t-0\t-0\n"], {"chrX": [(0, 0), (5, 7)]}, 0),
    # int32 extremes
    ("int32_extremes", [H + b"chrX\t-2147483648\t2147483647\n"], {"chrX": [(-2147483648, 2147483647)]}, 0),
    # Extend: touching (start == end) merges, start == end + 1 does not
    ("touching", [H + b"chr1\t1\t5\nchr1\t5\t8\nchr1\t9\t9\n"], {"chr1": [(1, 8), (9, 9)]}, 0),
    # contained intervals vanish; end < start stays as it is and never extends a group
    ("contained_and_reversed", [H + b"chr1\t1\t100\nchr1\t10\t20\nchr1\t200\t150\nchr1\t180\t190\n"], {"chr1": [(1, 100), (180, 190), (200, 150)]}, 0),
    # a reversed interval heading a group: the next start lies above its end, so it opens a new group
    ("reversed_head", [H + b"chr1\t0\t10\nchr1\t20\t5\nchr1\t21\t8\n"], {"chr1": [(0, 10), (20, 5), (21, 8)]}, 0),
    # unsorted starts and duplicates; the sort is by start only
    ("unsorted_dups", [H + b"chr10\t50\t60\nchr10\t1\t2\nchr10\t50\t55\nchr10\t1\t2\n"], {"chr10": [(1, 2), (50, 60)]}, 0),
    # names that share prefixes resolve byte for byte; unknown names count as unmatched but are kept out of every contig
    ("prefixes_unknown", [H + b"chr1\t1\t1\nchr10\t2\t2\nchr1_alt\t3\t3\nchr\t4\t4\nchr100\t5\t5\nchr1 \t6\t6\n"],
     {"chr1": [(1, 1)], "chr10": [(2, 2)], "chr1_alt": [(3, 3)]}, 3),
    # "*" is never a chromosome a read is looked up by: unmatched, even with a contig named "*"
    ("star", [H + b"*\t1\t2\n"], {}, 1),
    # two @SQ lines with one SN: both get the interval
    ("dup_name", [H + b"dup\t7\t9\n"], {"dup": [(7, 9)]}, 0),
    # several files append per chromosome (NewBaseRecalibrator), then one sort and flatten
    ("two_files", [H + b"chr1\t10\t20\n", H + b"chr1\t15\t30\nchrX\t1\t1\n"], {"chr1": [(10, 30)], "chrX": [(1, 1)]}, 0),
    # an empty file in between is invalid, but a header-only one is fine
    ("header_only_between", [H + b"chr1\t1\t1\n", H, H + b"chr1\t3\t3"], {"chr1": [(1, 1), (3, 3)]}, 0),
    # a '\r' that is not right before '\n' stays in the field: here it ends the chromosome name
    ("cr_in_name", [H + b"chr1\r\t1\t1\n"], {}, 1),
    # the longest line the scanner accepts: 65535 bytes before '\n' (a long chromosome name)
    ("line_65535", [H + b"Q" * (65535 - 4) + b"\t1\t1\n"], {}, 1),
]

INVALID = [
    # ReadString('\n') must return exactly ElsitesHeader (intervals.go:204-210)
    ("empty_file", [b""], (0, 0, HEADER_BAD)),
    ("header_crlf", [b"# elsites format version 1.0\r\nchr1\t1\t1\n"], (0, 0, HEADER_BAD)),
    ("header_no_newline", [b"# elsites format version 1.0"], (0, 0, HEADER_BAD)),
    ("header_other", [b"# elsites format version 1.1\n"], (0, 0, HEADER_BAD)),
    ("no_header", [b"chr1\t1\t1\n"], (0, 0, HEADER_BAD)),
    # i == 0 || i == len(str): a leading tab, no tab at all, an empty line
    ("leading_tab", [H + b"chr1\t1\t1\n\t1\t1\n"], (0, 2, FIELDS)),
    ("no_tab", [H + b"chr1\n"], (0, 1, FIELDS)),
    ("empty_line", [H + b"chr1\t1\t1\n\nchr1\t2\t2\n"], (0, 2, FIELDS)),
    ("cr_only_line", [H + b"chr1\t1\t1\n\r\n"], (0, 2, FIELDS)),
    # no second tab
    ("one_tab", [H + b"chr1\t1\n"], (0, 1, FIELDS)),
    # ParseInt failures: empty, space, underscore, out of int32, a third tab inside the end
    ("empty_start", [H + b"chr1\t\t5\n"], (0, 1, START)),
    ("space_start", [H + b"chr1\t 5\t5\n"], (0, 1, START)),
    ("underscore_start", [H + b"chr1\t1_000\t5\n"], (0, 1, START)),
    ("sign_only_start", [H + b"chr1\t-\t5\n"], (0, 1, START)),
    ("double_sign_start", [H + b"chr1\t+-5\t5\n"], (0, 1, START)),
    ("start_2p31", [H + b"chr1\t2147483648\t5\n"], (0, 1, START)),
    ("start_below", [H + b"chr1\t-2147483649\t5\n"], (0, 1, START)),
    ("empty_end", [H + b"chr1\t5\t\n"], (0, 1, END)),
    ("third_tab", [H + b"chr1\t5\t6\t7\n"], (0, 1, END)),
    ("end_hex", [H + b"chr1\t5\t0x6\n"], (0, 1, END)),
    ("end_cr_cr", [H + b"chr1\t5\t6\r\r\n"], (0, 1, END)),
    # lines on unknown chromosomes are validated as well
    ("unknown_chrom_bad", [H + b"nope\t1\tx\n"], (0, 1, END)),
    # bufio.Scanner: a line of 65536 bytes or more before its '\n'
    ("line_65536", [H + b"chr1\t1\t1\n" + b"Q" * 65532 + b"\t1\t1\n"], (0, 2, LONG)),
    ("line_65536_unterminated", [H + b"Q" * 65532 + b"\t1\t1"], (0, 1, LONG)),
    # the smallest (file, line) wins: the first file's error, although the second file fails earlier in its own lines
    ("smallest_file", [H + b"chr1\t1\t1\nchr1\t1\n", H + b"x\n"], (0, 2, FIELDS)),
    ("second_file", [H + b"chr1\t1\t1\n", H + b"chr1\t1\t1\nchr1\t2\t2\nchr1\t3\n"], (1, 3, FIELDS)),
    ("second_file_header", [H + b"chr1\t1\t1\n", b"#\n"], (1, 0, HEADER_BAD)),
]
