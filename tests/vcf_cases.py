"""VCF known-sites answers, derived by hand from vcf/vcf-files.go, vcf/string-scanner.go, vcf/vcf-types.go and strconv (see vcf_ref for
the line ranges), one or more per rule.

VALID:   (id, files, {contig name: flattened [(start, end)]}, lines on no @SQ SN) over the header NAMES
INVALID: (id, files, (file index, line, reason)); lines are 1-based and count the header lines

Files are plain VCF text unless a case says otherwise; the GPU test also loads every all-VCF case as BGZF.  H is an 11-line header, so
the first data line is line 12."""
from elsites_ref import HEADER as ELSITES
from vcf_ref import CHROM, END, HEADER, INFO, LONG, POS, QUAL, QUAL_RANGE, TAB, bgzf

NAMES = ["chr1", "chr10", "chrX", "dup", "dup", "*", "."]   # "dup": two @SQ lines share one SN; contigs literally named "*" and "."

H0 = b"##fileformat=VCFv4.2\n"
COLS = b"#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n"
H = (H0 + b'##INFO=<ID=DP,Number=1,Type=Integer,Description="depth">\n'
     + b'##INFO=<ID=DB,Number=0,Type=Flag,Description="dbSNP membership">\n'
     + b'##INFO=<ID=CH,Number=1,Type=Character,Description="one character">\n'
     + b'##INFO=<ID=CN,Number=.,Type=Character,Description="characters">\n'
     + b'##INFO=<ID=ST,Number=1,Type=String,Description="a string">\n'
     + b'##INFO=<ID=FL,Number=A,Type=Float,Description="floats">\n'
     + b'##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">\n'
     + b"##contig=<ID=chr1,length=1000>\n"
     + b"##source=hand\n"
     + COLS)
L1 = 12   # the first data line after H


def row(chrom=b"chr1", pos=b"5", id_=b".", ref=b"A", alt=b"G", qual=b".", filt=b".", info=b"."):
    return b"\t".join([chrom, pos, id_, ref, alt, qual, filt, info])


VALID = [
    # ParseVariant: the interval is [POS, POS - 1 + len(REF)] (vcf-types.go:141-161); dbSNP-style INFO is one undeclared key
    ("basic", [H + row(pos=b"100", id_=b"rs1", info=b"RS=1;VC=SNV;FREQ=1000Genomes:0.99,0.01") + b"\n"], {"chr1": [(100, 100)]}, 0),
    # len(REF) sets the end; ID and ALT are lists (';' and ','); FILTER with ';'; QUAL a number
    ("ref_len", [H + row(pos=b"10", id_=b"rs1;rs2", ref=b"ACGT", alt=b"A,AC", qual=b"50", filt=b"q10;s50", info=b"DP=5") + b"\n"], {"chr1": [(10, 13)]}, 0),
    # missingEntry: a '.' at the end of the line; the index lands past the end and every later field is missing (REF "." has length 1)
    ("dot_at_end", [H + b"chr1\t7\t.\n"], {"chr1": [(7, 7)]}, 0),
    # the line ends after a field's tab: later fields are missing too
    ("ends_after_tab", [H + b"chr1\t8\t\n"], {"chr1": [(8, 8)]}, 0),
    # a missing POS is -1: end = -1 - 1 + len("AC") = 0
    ("pos_missing", [H + row(pos=b".", ref=b"AC") + b"\n"], {"chr1": [(-1, 0)]}, 0),
    # an empty line is a line: CHROM "." (the missing entry), POS -1, REF "." -> (-1, -1) on a contig named "."
    ("empty_line", [H + row(pos=b"5") + b"\n\n" + row(pos=b"6") + b"\n"], {"chr1": [(5, 5), (6, 6)], ".": [(-1, -1)]}, 0),
    # CRLF everywhere: getLine drops the '\r' of header lines, bufio.ScanLines that of data lines (also without a final '\n')
    ("crlf", [H.replace(b"\n", b"\r\n") + row(pos=b"1") + b"\r\n" + row(pos=b"3", ref=b"AA") + b"\r"], {"chr1": [(1, 1), (3, 4)]}, 0),
    ("no_final_newline", [H + row(pos=b"9")], {"chr1": [(9, 9)]}, 0),
    ("header_only", [H], {}, 0),
    # the #column line may end the file without its '\n'
    ("column_line_at_eof", [H[:-1]], {}, 0),
    # the shortest header: the first line and a '#' line
    ("minimal_header", [H0 + b"#\n" + row(pos=b"4") + b"\n"], {"chr1": [(4, 4)]}, 0),
    # POS - 1 + len(REF) wraps in int32
    ("int32_wrap", [H + row(chrom=b"chrX", pos=b"2147483647", ref=b"AA") + b"\n"], {"chrX": [(2147483647, -2147483648)]}, 0),
    ("int32_low", [H + row(chrom=b"chrX", pos=b"-2147483648", ref=b"") + b"\n"], {"chrX": [(-2147483648, 2147483647)]}, 0),
    # strconv.ParseFloat's syntax: underscores between digits, hex with a 'p' exponent, inf / infinity / nan, underflow to zero,
    # and values right below the overflow bound
    ("qual_forms", [H + b"".join(row(pos=b"%d" % (i + 1), qual=q) + b"\n" for i, q in enumerate(
        [b"1_000.5", b"0x1p-2", b"0X1.8P+1", b"inf", b"-Infinity", b"+INF", b"nan", b"NaN", b"1e-400", b".5", b"5.", b"1e+5", b"+.5e1_0",
         b"0x_1p0", b"1.7976931348623157e308", b"0x1.fffffffffffff7p1023", b"179769313486231580793728971405303415079934132710037826936173778980444968292764750946649017977587207096330286416692887910946555547851940402630657488671505820681908902000708383676273854845817711531764475730270069855571366959622842914819860834936475292719074168444365510704342711559699508093042880177904174497791e0",
         b"0.0001797693134862315708e312", b"-1e308", b"0e99999", b"0x0p99999", b"1e-99999999"])) ],
     {"chr1": [(i + 1, i + 1) for i in range(22)]}, 0),
    # FILTER "." at the end of the line is missing: "...\t.\t." is accepted (the INFO column is missing too)
    ("filter_dot_at_end", [H + b"chr1\t5\t.\tA\tG\t.\t.\n"], {"chr1": [(5, 5)]}, 0),
    # INFO keys run to ' ', ':' or tab.  Declared: a Flag never fails and consumes nothing; Character (Number=1) returns '=';
    # String keeps the '='; Character lists decode UTF-8 runes; undeclared keys take any value
    ("info_declared", [H + b"".join(row(pos=b"%d" % (i + 1), info=v) + b"\n" for i, v in enumerate(
        [b"DB", b"DB:DB", b"DB =5", b"CH =", b"CH  =x", b"ST =abc", b"ST =a,b;c", b"CN =,a,\xc3\xa9 , \xe2\x82\xac,\xf0\x9f\x98\x80", b"CN =x",
         b"X Y", b"A:B=1:C", b"A = 1 , 2 ,3", b"DP=5:DB", b"END=5", b"END=5;DP", b"FL=1.0", b" DB", b"DB\tGT\t0/1"]))],
     {"chr1": [(i + 1, i + 1) for i in range(18)]}, 0),
    # the first of two INFO lines with one ID is the one SmallMap.Get finds (String here; Integer would refuse "DQ =x")
    ("info_first_declaration", [H0 + b"##INFO=<ID=DQ,Number=1,Type=String>\n##INFO=<ID=DQ,Number=1,Type=Integer>\n" + COLS + row(info=b"DQ =x") + b"\n"],
     {"chr1": [(5, 5)]}, 0),
    # ParseFormatInformation: a Number of InvalidNumber (-5) counts as no Number, so a second Number is accepted
    ("number_minus5", [H0 + b"##INFO=<ID=NN,Number=-5,Number=1,Type=String>\n" + COLS + row(info=b"NN =1") + b"\n"], {"chr1": [(5, 5)]}, 0),
    # meta-information values: quotes with escapes, a plain value, a second Description after an empty one, an empty ID
    ("meta_forms", [H0 + b'##a=<ID=x,Description="q \\" y, z>">\n##b=plain value\n##c=<ID=x,Description=,Description=y>\n'
                   + b"##d=<ID=,k=v,  m = n >trailing\n##e=<ID=\"\">\n" + COLS + row() + b"\n"], {"chr1": [(5, 5)]}, 0),
    # an INFO declared with the empty ID: the key of an empty INFO column (a Flag: fine)
    ("empty_id_flag", [H0 + b"##INFO=<ID=,Number=0,Type=Flag>\n" + COLS + b"chr1\t5\t\n" + row(pos=b"6", info=b"") + b"\n"],
     {"chr1": [(5, 5), (6, 6)]}, 0),
    # "*" and names that are no @SQ SN count as unmatched; a name shared by two @SQ lines gives both the interval
    ("unmatched", [H + row(chrom=b"*") + b"\n" + row(chrom=b"chrZ") + b"\n" + row(chrom=b"chr1 ") + b"\n" + row(chrom=b"dup", pos=b"3") + b"\n"],
     {"dup": [(3, 3)]}, 3),
    # Flatten over the VCF's intervals: touching merges, contained vanish
    ("flatten", [H + row(pos=b"1", ref=b"AAAAA") + b"\n" + row(pos=b"5", ref=b"AAAA") + b"\n" + row(pos=b"9") + b"\n" + row(pos=b"20", ref=b"AAAAAAAAAA") + b"\n"
                 + row(pos=b"22") + b"\n"], {"chr1": [(1, 8), (9, 9), (20, 29)]}, 0),
    # a list mixing .elsites and VCF files, flattened together
    ("mixed", [ELSITES + b"chr1\t1\t5\nchr10\t7\t7\n", H + row(pos=b"3", ref=b"ACGTACGT") + b"\n", ELSITES + b"chr1\t40\t50\n"],
     {"chr1": [(1, 10), (40, 50)], "chr10": [(7, 7)]}, 0),
    # a data line of 65535 bytes (bufio.MaxScanTokenSize - 1) is accepted
    ("line_65535", [H + row(info=b"") + b"X" * (65535 - len(row(info=b""))) + b"\n" + row(pos=b"6") + b"\n"], {"chr1": [(5, 5), (6, 6)]}, 0),
    # a BGZF file (vcf.Open sniffs the first byte)
    ("bgzf", [bgzf(H + row(pos=b"11") + b"\n", block=17)], {"chr1": [(11, 11)]}, 0),
]


def _q(q):
    return [H + row(qual=q) + b"\n"]


def _i(v):
    return [H + row(info=v) + b"\n"]


def _h(lines):
    return [H0 + lines + COLS + row() + b"\n"]


INVALID = [
    # ---- the header (ParseHeader and NewVariantParser) ----
    # line[:len(prefix)] panics on a shorter first line; a BGZF file is a VCF whatever it holds
    ("first_line_short", [bgzf(b"##fileformat=VCFv4\n#C\n")], (0, 1, HEADER)),
    ("first_line_other", [bgzf(b"##fileformat=VCFv3.3\n#C\n")], (0, 1, HEADER)),
    ("bgzf_empty", [bgzf(b"")], (0, 1, HEADER)),
    # readUntilByte('=') must find a '='; a second fileformat line panics
    ("meta_no_eq", _h(b"##foo\n"), (0, 2, HEADER)),
    ("second_fileformat", _h(b"##fileformat=VCFv4.2\n"), (0, 2, HEADER)),
    # sc.data[sc.index] on an empty value
    ("meta_empty", _h(b"##foo=\n"), (0, 2, HEADER)),
    ("info_empty", _h(b"##INFO=\n"), (0, 2, HEADER)),
    ("info_no_bracket", _h(b"##INFO=ID\n"), (0, 2, HEADER)),
    # ParseMetaField: a key without '=', an unterminated value, an unterminated quote, a '\' ending the line inside quotes
    ("field_no_eq", _h(b"##x=<ID>\n"), (0, 2, HEADER)),
    ("field_no_close", _h(b"##x=<ID=a\n"), (0, 2, HEADER)),
    ("field_value_at_end", _h(b"##x=<ID=\n"), (0, 2, HEADER)),
    ("quote_unterminated", _h(b'##x=<ID=a,Description="abc>\n'), (0, 2, HEADER)),
    ("quote_backslash_end", _h(b'##x=<ID=a,Description="abc\\\n'), (0, 2, HEADER)),
    # after a field only ',' or '>' may follow; the line may not end there
    ("after_field_junk", _h(b'##x=<ID="a"b>\n'), (0, 2, HEADER)),
    ("after_field_end", _h(b'##x=<ID="a"\n'), (0, 2, HEADER)),
    # duplicates and missing entries
    ("meta_dup_id", _h(b"##x=<ID=a,ID=b>\n"), (0, 2, HEADER)),
    ("meta_dup_description", _h(b"##x=<ID=a,Description=d,Description=e>\n"), (0, 2, HEADER)),
    ("meta_dup_key", _h(b"##x=<ID=a,k=1,k=2>\n"), (0, 2, HEADER)),
    ("meta_no_id", _h(b"##x=<k=1>\n"), (0, 2, HEADER)),
    ("info_dup_number", _h(b"##INFO=<ID=a,Number=1,Number=2,Type=String>\n"), (0, 2, HEADER)),
    ("info_dup_type", _h(b"##INFO=<ID=a,Number=1,Type=String,Type=String>\n"), (0, 2, HEADER)),
    ("info_no_number", _h(b"##INFO=<ID=a,Type=String>\n"), (0, 2, HEADER)),
    ("info_no_type", _h(b"##INFO=<ID=a,Number=1>\n"), (0, 2, HEADER)),
    ("info_no_id", _h(b"##INFO=<Number=1,Type=String>\n"), (0, 2, HEADER)),
    ("info_bad_type", _h(b"##INFO=<ID=a,Number=1,Type=Str>\n"), (0, 2, HEADER)),
    ("info_bad_number", _h(b"##INFO=<ID=a,Number=x,Type=String>\n"), (0, 2, HEADER)),
    ("info_number_minus7", _h(b"##INFO=<ID=a,Number=-7,Type=String>\n"), (0, 2, HEADER)),
    # CreateInfoParser: a Flag with Number != 0; CreateFormatParser: any Flag.  Unused declarations still refuse the file, and they
    # are named even before a later malformed header line
    ("info_flag_number", _h(b"##INFO=<ID=F,Number=1,Type=Flag>\n"), (0, 2, HEADER)),
    ("format_flag", _h(b"##FORMAT=<ID=F,Number=0,Type=Flag>\n"), (0, 2, HEADER)),
    ("flag_before_syntax", _h(b"##INFO=<ID=F,Number=.,Type=Flag>\n##bad\n"), (0, 2, HEADER)),
    # the header must continue with '#' lines up to the column line
    ("no_column_line", [H0 + b"##a=b\n"], (0, 3, HEADER)),
    ("hash_at_eof", [H0 + b"#"], (0, 2, HEADER)),
    ("data_after_meta", [H0 + row() + b"\n"], (0, 2, HEADER)),
    ("meta_at_eof", [H0 + b"##a=b"], (0, 3, HEADER)),
    # ---- data lines (ParseVariant, NSamples = 0) ----
    ("tab_chrom", [H + b"chr1\n"], (0, L1, TAB)),
    ("tab_pos", [H + b"chr1\t5\n"], (0, L1, TAB)),
    ("tab_ref", [H + b"chr1\t5\t.\tA\n"], (0, L1, TAB)),
    ("tab_alt", [H + b"chr1\t5\t.\tA\tG\n"], (0, L1, TAB)),
    ("tab_id_list", [H + b"chr1\t5\trs1;rs2\n"], (0, L1, TAB)),
    ("tab_qual", [H + b"chr1\t5\t.\tA\tG\t50\n"], (0, L1, TAB)),
    # FILTER must be followed by a tab unless it is missing; after "PASS" that tab cannot be a ';'
    ("filter_no_tab", [H + b"chr1\t5\t.\tA\tG\t.\tPASS\n"], (0, L1, TAB)),
    ("filter_pass_semicolon", [H + row(filt=b"PASS;q10") + b"\n"], (0, L1, TAB)),
    ("filter_list_no_tab", [H + b"chr1\t5\t.\tA\tG\t.\tq10;s50\n"], (0, L1, TAB)),
    # POS: strconv.ParseInt(s, 10, 32)
    ("pos_letters", [H + row(pos=b"x") + b"\n"], (0, L1, POS)),
    ("pos_empty", [H + row(pos=b"") + b"\n"], (0, L1, POS)),
    ("pos_range", [H + row(pos=b"2147483648") + b"\n"], (0, L1, POS)),
    ("pos_underscore", [H + row(pos=b"1_0") + b"\n"], (0, L1, POS)),
    # QUAL: strconv.ParseFloat(s, 64) syntax
    ("qual_word", _q(b"abc"), (0, L1, QUAL)),
    ("qual_empty", _q(b""), (0, L1, QUAL)),
    ("qual_exp_empty", _q(b"1e"), (0, L1, QUAL)),
    ("qual_exp_sign_only", _q(b"1e+"), (0, L1, QUAL)),
    ("qual_hex_no_p", _q(b"0x1.8"), (0, L1, QUAL)),
    ("qual_hex_bare", _q(b"0x"), (0, L1, QUAL)),
    ("qual_double_underscore", _q(b"1__0"), (0, L1, QUAL)),
    ("qual_leading_underscore", _q(b"_1"), (0, L1, QUAL)),
    ("qual_trailing_underscore", _q(b"1_"), (0, L1, QUAL)),
    ("qual_underscore_dot", _q(b"1_.5"), (0, L1, QUAL)),
    ("qual_exp_underscore_first", _q(b"1e_5"), (0, L1, QUAL)),
    ("qual_signed_nan", _q(b"+nan"), (0, L1, QUAL)),
    ("qual_infx", _q(b"infx"), (0, L1, QUAL)),
    ("qual_infin", _q(b"infin"), (0, L1, QUAL)),
    ("qual_two_dots", _q(b"1.5."), (0, L1, QUAL)),
    ("qual_space", _q(b" 1"), (0, L1, QUAL)),
    ("qual_dot_dot", _q(b".."), (0, L1, QUAL)),
    # QUAL: a value that rounds to +-Inf is a range error; at the bound the host decides
    ("qual_1e309", _q(b"1e309"), (0, L1, QUAL_RANGE)),
    ("qual_neg_1e400", _q(b"-1e400"), (0, L1, QUAL_RANGE)),
    ("qual_above_max", _q(b"1.7976931348623159e308"), (0, L1, QUAL_RANGE)),
    ("qual_halfway_dec", _q(b"179769313486231580793728971405303415079934132710037826936173778980444968292764750946649017977587207096330286416692887910946555547851940402630657488671505820681908902000708383676273854845817711531764475730270069855571366959622842914819860834936475292719074168444365510704342711559699508093042880177904174497792"), (0, L1, QUAL_RANGE)),
    ("qual_halfway_hex", _q(b"0x1.fffffffffffff8p1023"), (0, L1, QUAL_RANGE)),
    ("qual_hex_1024", _q(b"0x1p1024"), (0, L1, QUAL_RANGE)),
    ("qual_saturated_exp", _q(b"1e99999999"), (0, L1, QUAL_RANGE)),
    # INFO: a declared key goes through its parser.  '=' must follow (after spaces); Integer and Float then read "=..." and fail
    ("info_int_no_eq", _i(b"DP"), (0, L1, INFO)),
    ("info_int_colon", _i(b"DP:DB"), (0, L1, INFO)),
    ("info_int_value", _i(b"DP =5"), (0, L1, INFO)),
    ("info_float_value", _i(b"FL =1.0"), (0, L1, INFO)),
    ("info_string_no_eq", _i(b"ST"), (0, L1, INFO)),
    ("info_char_list_end", _i(b"CN =,"), (0, L1, INFO)),
    ("info_char_bad_utf8", _i(b"CN =,\xff"), (0, L1, INFO)),
    ("info_char_fffd", _i(b"CN =,\xef\xbf\xbd"), (0, L1, INFO)),
    ("info_char_truncated", _i(b"CN =,\xe2\x82"), (0, L1, INFO)),
    ("info_char_overlong", _i(b"CN =,\xc0\x80"), (0, L1, INFO)),
    ("info_char_surrogate", _i(b"CN =,\xed\xa0\x80"), (0, L1, INFO)),
    ("info_second_key", _i(b"X=1:DP"), (0, L1, INFO)),
    # End(): a key equal to END has no value of type int, so the line is refused; "END=5" is a key of its own
    ("info_end_bare", _i(b"END"), (0, L1, END)),
    ("info_end_value", _i(b"END =100"), (0, L1, END)),
    ("info_end_second", _i(b"DB:END"), (0, L1, END)),
    ("info_end_declared_string", [H0 + b"##INFO=<ID=END,Number=1,Type=String>\n" + COLS + row(info=b"END =7") + b"\n"], (0, 4, END)),
    # an empty CHROM converts, but vcf-to-elsites writes a line its .elsites loader refuses
    ("chrom_empty", [H + row(chrom=b"") + b"\n"], (0, L1, CHROM)),
    # bufio.Scanner: a line of 65536 bytes or more
    ("line_65536", [H + row(info=b"") + b"X" * (65536 - len(row(info=b""))) + b"\n"], (0, L1, LONG)),
    ("line_65536_cr", [H + row(info=b"") + b"X" * (65535 - len(row(info=b""))) + b"\r\n"], (0, L1, LONG)),
    # the first failing field of a line; the smallest line of a file; the first failing file
    ("pos_before_tab", [H + b"chr1\tx\t.\tA\n"], (0, L1, POS)),
    ("smallest_line", [H + row() + b"\n" + row(pos=b"x") + b"\n" + b"chr1\n"], (0, L1 + 1, POS)),
    ("second_file", [H + row() + b"\n", ELSITES + b"chr1\t1\t1\n", H + row() + b"\n" + row(qual=b"q") + b"\n"], (2, L1 + 1, QUAL)),
]
