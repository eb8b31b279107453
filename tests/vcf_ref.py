"""Plain restatement of a VCF in the --known-sites list, written from the reference's Go source:

  vcf.Open                         vcf/vcf-files.go:1285-1312   a first byte 0x1f is BGZF, anything else plain text
  getLine                          vcf/vcf-files.go:245-258     ReadString('\\n'), one '\\r' before the '\\n' dropped, no length limit
  ParseHeader                      vcf/vcf-files.go:261-305     the first line, the ##key=value lines, the #column line
  ParseMetaField                   vcf/vcf-files.go:73-113
  ParseMetaInformation             vcf/vcf-files.go:116-158
  ParseFormatInformation           vcf/vcf-files.go:161-243
  NewVariantParser                 vcf/vcf-files.go:749-765     CreateInfoParser (:442-477) and CreateFormatParser (:569-598) on every
                                                                declaration
  ParseVariant, NSamples = 0       vcf/vcf-files.go:600-738,773-782, string-scanner.go
  Variant.Start / End              vcf/vcf-types.go:141-161
  FromVcfFile                      intervals/intervals.go:306-338 (the data lines through bufio.Scanner, as elsites_ref.scan_lines)
  vcf-to-elsites                   cmd/convert.go:34-52 (sort + ParallelFlatten per chromosome, then ToElsitesFile, intervals.go:179-196)
  strconv.ParseFloat(s, 64)        Go's atof.go (special, readFloat, underscoreOK) and the n == len(s) check; the value is rounded here
                                   with Python's correctly rounded float(), and a result of +-Inf is the range error

A refusal is VcfError(file, line, reason): lines are 1-based and count the header lines.  Where Go's panics would come in another order
(the parser checks of NewVariantParser run after the whole header; vcf-to-elsites converts every line before its .elsites is read back),
the smallest line is reported, as elp_load_known_sites does.  Nothing here imports the CUDA library."""
from __future__ import annotations

import gzip
import struct
import zlib

import numpy as np

import elsites_ref as er

PREFIX = b"##fileformat=VCFv4."               # fileFormatVersionLinePrefix (vcf-types.go:32)
INVALID_NUMBER = -5                           # vcf-types.go:53-58: NumberA -1, NumberR -2, NumberG -3, NumberDot -4, InvalidNumber -5
INTEGER, FLOAT, FLAG, CHARACTER, STRING = 1, 2, 3, 4, 5   # vcf-types.go:43-48
TYPES = {b"Integer": INTEGER, b"Float": FLOAT, b"Flag": FLAG, b"Character": CHARACTER, b"String": STRING}

# reasons
HEADER = "header"
LONG, TAB, POS, QUAL, QUAL_RANGE, INFO, END, CHROM = "long", "tab", "pos", "qual", "qual range", "info", "end", "chrom"


class VcfError(ValueError):
    def __init__(self, file, line, reason):
        super().__init__(f"file {file}, line {line}: {reason}")
        self.file, self.line, self.reason = file, line, reason


class Panic(Exception):
    """a log.Panic (or an index / slice out of range) of the Go code; .reason as above"""
    def __init__(self, reason):
        super().__init__(reason)
        self.reason = reason


# ---------------------------------------------------------------- strconv
def _lower(c):   # strconv's lower(): c | ('x' - 'X')
    return c | 0x20


def _underscore_ok(s: bytes) -> bool:
    """underscoreOK (strconv/atoi.go)"""
    saw, i = "^", 0
    if len(s) >= 1 and s[0] in b"+-":
        s = s[1:]
    hexa = False
    if len(s) >= 2 and s[0] == 0x30 and _lower(s[1]) in b"box":
        i, saw, hexa = 2, "0", _lower(s[1]) == ord("x")
    while i < len(s):
        c = s[i]
        if 0x30 <= c <= 0x39 or (hexa and ord("a") <= _lower(c) <= ord("f")):
            saw = "0"
        elif c == ord("_"):
            if saw != "0":
                return False
            saw = "_"
        else:
            if saw == "_":
                return False
            saw = "!"
        i += 1
    return saw != "_"


def _prefix_ci(s: bytes, p: bytes) -> int:
    """commonPrefixLenIgnoreCase"""
    n = 0
    while n < len(s) and n < len(p) and s[n:n + 1].lower() == p[n:n + 1]:
        n += 1
    return n


def parse_float(s: bytes) -> float:
    """strconv.ParseFloat(s, 64); ValueError for a syntax error, OverflowError for a range error"""
    # special (atof.go): optional sign + "inf" / "infinity", or "nan"; then ParseFloat wants n == len(s)
    if s:
        if s[0] in b"+-iI":
            ns = 1 if s[0] in b"+-" else 0
            n = _prefix_ci(s[ns:], b"infinity")
            if 3 < n < 8:
                n = 3
            if n in (3, 8):
                if ns + n != len(s):
                    raise ValueError(s)
                return float("-inf") if s[:1] == b"-" else float("inf")
        elif s[0] in b"nN" and _prefix_ci(s, b"nan") == 3:
            if len(s) != 3:
                raise ValueError(s)
            return float("nan")
    # readFloat
    i, underscores, neg = 0, False, False
    if i >= len(s):
        raise ValueError(s)
    if s[i] in b"+-":
        neg = s[i] == ord("-")
        i += 1
    hexa, exp_char = False, ord("e")
    if i + 2 < len(s) and s[i] == 0x30 and _lower(s[i + 1]) == ord("x"):
        hexa, exp_char = True, ord("p")
        i += 2
    digits, before, sawdot, sawdigits = [], 0, False, False
    while i < len(s):
        c = s[i]
        if c == ord("_"):
            underscores = True
        elif c == ord("."):
            if sawdot:
                break
            sawdot = True
        elif 0x30 <= c <= 0x39 or (hexa and ord("a") <= _lower(c) <= ord("f")):
            sawdigits = True
            digits.append(chr(c))
            if not sawdot:
                before += 1
        else:
            break
        i += 1
    if not sawdigits:
        raise ValueError(s)
    e, esign = 0, 1
    if i < len(s) and _lower(s[i]) == exp_char:
        i += 1
        if i >= len(s):
            raise ValueError(s)
        if s[i] == ord("+"):
            i += 1
        elif s[i] == ord("-"):
            i, esign = i + 1, -1
        if i >= len(s) or not 0x30 <= s[i] <= 0x39:
            raise ValueError(s)
        while i < len(s) and (0x30 <= s[i] <= 0x39 or s[i] == ord("_")):
            if s[i] == ord("_"):
                underscores = True
            elif e < 10000:                      # "if e < 10000": a very long exponent saturates
                e = e * 10 + s[i] - 0x30
            i += 1
    elif hexa:
        raise ValueError(s)                      # a hex mantissa must have a 'p' exponent
    if underscores and not _underscore_ok(s[:i]):
        raise ValueError(s)
    if i != len(s):
        raise ValueError(s)
    m = "".join(digits)
    sign = "-" if neg else ""
    if hexa:
        try:
            v = float.fromhex(f"{sign}0x0.{m}p{4 * before + esign * e}")
        except OverflowError:
            raise OverflowError(s) from None
    else:
        v = float(f"{sign}0.{m}e{before + esign * e}")
        if v in (float("inf"), float("-inf")):
            raise OverflowError(s)
    return v


def parse_int32(s: bytes) -> int:
    return er.parse_int32(s)


# ---------------------------------------------------------------- StringScanner (string-scanner.go)
class Scanner:
    def __init__(self, data: bytes):
        self.d, self.i = data, 0

    def at(self, i):
        if i >= len(self.d):
            raise Panic("index out of range")
        return self.d[i]

    def skip_space(self):
        while self.i < len(self.d) and self.d[self.i] == 0x20:
            self.i += 1
        if self.i > len(self.d):                 # SkipSpace: past the end it lands on len(data)
            self.i = len(self.d)

    def read_until_byte(self, c):
        start = self.i
        j = self.d.find(bytes([c]), start) if start <= len(self.d) else -1
        if j >= 0:
            self.i = j + 1
            return self.d[start:j], True
        if start > len(self.d):
            raise Panic("slice out of range")
        self.i = len(self.d)
        return self.d[start:], False

    def read_until_bytes(self, cs: bytes):
        start = self.i
        if start > len(self.d):
            raise Panic("slice out of range")
        for j in range(start, len(self.d)):
            if self.d[j] in cs:
                self.i = j
                return self.d[start:j]
        self.i = len(self.d)
        return self.d[start:]


# ---------------------------------------------------------------- header (vcf-files.go:73-305)
def _meta_field(sc: Scanner):
    sc.skip_space()
    start = sc.i
    while sc.i < len(sc.d) and sc.d[sc.i] not in b" =":
        sc.i += 1
    key = sc.d[start:sc.i]
    sc.skip_space()
    if sc.i >= len(sc.d) or sc.d[sc.i] != ord("="):
        raise Panic("invalid key=pair pair")
    sc.i += 1
    sc.skip_space()
    if sc.at(sc.i) == ord('"'):
        sc.i += 1
        buf = bytearray()
        while sc.i < len(sc.d):
            c = sc.d[sc.i]
            if c == ord('"'):
                sc.i += 1
                return key, bytes(buf)
            if c == ord("\\"):
                sc.i += 1
            buf.append(sc.at(sc.i))
            sc.i += 1
        raise Panic('missing closing "')
    start = sc.i
    while sc.i < len(sc.d):
        if sc.d[sc.i] in b" ,>":
            return key, sc.d[start:sc.i]
        sc.i += 1
    raise Panic("missing closing >")


def _after_field(sc: Scanner):
    """True when '>' closed the entry"""
    sc.skip_space()
    c = sc.at(sc.i)
    if c == ord(","):
        sc.i += 1
        return False
    if c == ord(">"):
        sc.i += 1
        return True
    raise Panic("invalid syntax in a meta-information line")


def _meta_information(sc: Scanner):
    if sc.at(sc.i) != ord("<"):
        sc.i = len(sc.d)
        return
    sc.i += 1
    has_id, desc, fields = False, b"", set()
    while True:
        key, value = _meta_field(sc)
        if key == b"ID":
            if has_id:
                raise Panic("multiple IDs")
            has_id = True                        # utils.Intern(""): not nil either
        elif key == b"Description":
            if desc != b"":
                raise Panic("multiple Descriptions")
            desc = value
        else:
            if key in fields:
                raise Panic("duplicate field key")
            fields.add(key)
        if _after_field(sc):
            break
    if not has_id:
        raise Panic("missing ID")


def _format_information(sc: Scanner):
    """-> (ID, Number, Type)"""
    if sc.at(sc.i) != ord("<"):
        raise Panic("missing open angle bracket")
    sc.i += 1
    fid, desc, number, typ, fields = None, b"", INVALID_NUMBER, 0, set()
    while True:
        key, value = _meta_field(sc)
        if key == b"ID":
            if fid is not None:
                raise Panic("multiple IDs")
            fid = value
        elif key == b"Description":
            if desc != b"":
                raise Panic("multiple Descriptions")
            desc = value
        elif key == b"Number":
            if number > INVALID_NUMBER:
                raise Panic("multiple Number entries")
            special = {b"a": -1, b"A": -1, b"r": -2, b"R": -2, b"g": -3, b"G": -3, b".": -4}
            if value in special:
                number = special[value]
            else:
                try:
                    number = parse_int32(value)
                except ValueError:
                    raise Panic("Number: ParseInt") from None
        elif key == b"Type":
            if typ != 0:
                raise Panic("multiple types")
            if value not in TYPES:
                raise Panic("unknown type")
            typ = TYPES[value]
        else:
            if key in fields:
                raise Panic("duplicate field key")
            fields.add(key)
        if _after_field(sc):
            break
    if fid is None:
        raise Panic("missing ID")
    if number <= INVALID_NUMBER:
        raise Panic("missing number entry")
    if typ == 0:
        raise Panic("missing type")
    return fid, number, typ


def parse_header(data: bytes, file=0):
    """ParseHeader, then NewVariantParser's CreateInfoParser / CreateFormatParser -> (header lines, header bytes, [(ID, Number, Type)]
    of the INFO lines in order); VcfError at the smallest failing line"""
    pos = 0

    def get_line():
        nonlocal pos
        j = data.find(b"\n", pos)
        if j < 0:                                # io.EOF: the rest, unchanged
            line, pos = data[pos:], len(data)
            return line
        line, pos = data[pos:j + 1], j + 1
        return line[:-2] if len(line) > 1 and line[-2] == 0x0D else line[:-1]

    infos, checks = [], []                       # checks: (line, ok) of CreateInfoParser / CreateFormatParser, run after the header
    fail = None
    lines = 0
    try:
        line = get_line()
        lines += 1
        if len(line) < len(PREFIX):
            raise Panic("slice out of range")
        if line[:len(PREFIX)] != PREFIX:
            raise Panic("invalid first line")
        while True:
            if pos >= len(data) or data[pos] != ord("#"):
                lines += 1
                raise Panic("unexpected end of VCF header")
            pos += 1
            if pos >= len(data):
                lines += 1
                raise Panic("unexpected end of VCF header")
            if data[pos] != ord("#"):
                break
            pos += 1
            line = get_line()
            lines += 1
            sc = Scanner(line)
            key, found = sc.read_until_byte(ord("="))
            if not found:
                raise Panic("invalid syntax in a VCF header")
            if key == b"fileformat":
                raise Panic("multiple file format lines")
            if key in (b"INFO", b"FORMAT"):
                fid, number, typ = _format_information(sc)
                if key == b"INFO":
                    infos.append((fid, number, typ))
                    checks.append((lines, not (typ == FLAG and number != 0)))      # CreateInfoParser
                else:
                    checks.append((lines, typ != FLAG))                            # CreateFormatParser
            else:
                _meta_information(sc)
        get_line()                               # the #column line
        lines += 1
    except Panic:
        fail = lines
    bad = [ln for ln, ok in checks if not ok]
    if bad and (fail is None or bad[0] < fail):
        fail = bad[0]
    if fail is not None:
        raise VcfError(file, fail, HEADER)
    return lines, pos, infos


# ---------------------------------------------------------------- data lines (vcf-files.go:600-738,773-782)
def _missing_entry(sc: Scanner) -> bool:
    if sc.i >= len(sc.d):
        return True
    if sc.d[sc.i] == ord("."):
        nxt = sc.i + 1
        if nxt >= len(sc.d) or sc.d[nxt] == 0x09:
            sc.i = nxt + 1
            return True
    return False


def _scan_tab(sc: Scanner):
    if sc.i >= len(sc.d) or sc.d[sc.i] != 0x09:
        raise Panic(TAB)
    sc.i += 1


def _do_string(sc):
    if _missing_entry(sc):
        return b"."
    v, ok = sc.read_until_byte(0x09)
    if not ok:
        raise Panic(TAB)
    return v


def _do_int32(sc):
    if _missing_entry(sc):
        return -1
    v, ok = sc.read_until_byte(0x09)
    if not ok:
        raise Panic(TAB)
    try:
        return parse_int32(v)
    except ValueError:
        raise Panic(POS) from None


def _do_float(sc):
    if _missing_entry(sc):
        return None
    v, ok = sc.read_until_byte(0x09)
    if not ok:
        raise Panic(TAB)
    try:
        return parse_float(v)
    except OverflowError:
        raise Panic(QUAL_RANGE) from None
    except ValueError:
        raise Panic(QUAL) from None


def _do_string_list(sc, sep: bytes):
    if _missing_entry(sc):
        return None
    out = []
    while True:
        out.append(sc.read_until_bytes(sep))
        if sc.i >= len(sc.d) or sc.d[sc.i] != sep[0]:
            break
        sc.i += 1
    _scan_tab(sc)
    return out


def _do_filter(sc):
    if _missing_entry(sc):
        return None
    s = sc.read_until_bytes(b";\t")
    if s == b"PASS":
        _scan_tab(sc)
        return [s]
    out = [s]
    while sc.i < len(sc.d) and sc.d[sc.i] == ord(";"):
        sc.i += 1
        out.append(sc.read_until_bytes(b";\t"))
    _scan_tab(sc)
    return out


END_OF_INFO_ENTRY = b" ,;\t"


def _decode_rune(b: bytes):
    """utf8.DecodeRune -> (rune, size); (0xFFFD, 1) for an invalid encoding"""
    for size in (2, 3, 4):
        if len(b) >= size:
            try:
                ch = b[:size].decode("utf-8")        # Python's strict decoder rejects what DecodeRune does: overlong forms, surrogates,
            except UnicodeDecodeError:               # > U+10FFFF, bad continuation bytes
                continue
            if len(ch) == 1:
                return ord(ch), size
    return 0xFFFD, 1


def _info_entry(sc: Scanner, typ):
    """ParseInfoInteger / Float / Character / String -> (kind, value)"""
    if typ == INTEGER:
        try:
            return "int", parse_int32(sc.read_until_bytes(END_OF_INFO_ENTRY))
        except ValueError:
            raise Panic(INFO) from None
    if typ == FLOAT:
        try:
            return "float", parse_float(sc.read_until_bytes(END_OF_INFO_ENTRY))
        except (ValueError, OverflowError):
            raise Panic(INFO) from None
    if typ == CHARACTER:
        if sc.i >= len(sc.d):
            raise Panic(INFO)
        c = sc.d[sc.i]
        if c < 0x80:
            sc.i += 1
            return "rune", c
        r, size = _decode_rune(sc.d[sc.i:])
        if r == 0xFFFD:
            raise Panic(INFO)
        sc.i += size
        return "rune", r
    return "str", sc.read_until_bytes(END_OF_INFO_ENTRY)


def _info_parser(sc: Scanner, number, typ):
    """CreateInfoParser's parser (make1InfoParser / makeNInfoParser / ParseInfoFlag)"""
    if typ == FLAG:
        sc.skip_space()
        return "bool", True
    sc.skip_space()
    if sc.i >= len(sc.d) or sc.d[sc.i] != ord("="):
        raise Panic(INFO)
    sc.skip_space()
    if number == 1:
        v = _info_entry(sc, typ)
        sc.skip_space()
        return v
    out = []
    while True:
        out.append(_info_entry(sc, typ))
        sc.skip_space()
        if sc.i >= len(sc.d) or sc.d[sc.i] != ord(","):
            break
        sc.i += 1
    return "list", out


def _generic_info(sc: Scanner):
    sc.skip_space()
    if sc.i < len(sc.d) and sc.d[sc.i] == ord("="):
        out = []
        sc.i += 1
        sc.skip_space()
        while True:
            out.append(sc.read_until_bytes(END_OF_INFO_ENTRY))
            sc.skip_space()
            if sc.i >= len(sc.d) or sc.d[sc.i] != ord(","):
                break
            sc.i += 1
        return "list", out
    return "bool", True


def _do_info(sc: Scanner, parsers: dict):
    out = []
    while True:
        sc.skip_space()
        key = sc.read_until_bytes(b" :\t")
        if key in parsers:
            value = _info_parser(sc, *parsers[key])
        else:
            value = _generic_info(sc)
        out.append((key, value))
        sc.skip_space()
        if sc.i >= len(sc.d) or sc.d[sc.i] != ord(":"):
            return out
        sc.i += 1


def _wrap32(v):
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def parse_line(tok: bytes, parsers: dict):
    """ParseVariant(NSamples = 0), then Start() and End() -> (CHROM, start, end); Panic(reason)"""
    sc = Scanner(tok)
    chrom = _do_string(sc)
    pos = _do_int32(sc)
    _do_string_list(sc, b";\t")
    ref = _do_string(sc)
    _do_string_list(sc, b",\t")
    _do_float(sc)
    _do_filter(sc)
    info = _do_info(sc, parsers)
    end = _wrap32(pos - 1 + len(ref))
    for key, (kind, value) in info:                 # Variant.End: Info.Get(END), the first entry with that key
        if key == b"END":
            if kind == "int":
                end = value
            elif kind == "str":
                try:
                    end = parse_int32(value)
                except ValueError:
                    raise Panic(END) from None
            else:
                raise Panic(END)
            break
    return chrom, pos, end


def parser_table(infos):
    """NewVariantParser's InfoParsers: the first declaration of an ID is the one SmallMap.Get finds"""
    t = {}
    for fid, number, typ in infos:
        t.setdefault(fid, (number, typ))
    return t


def from_vcf(data: bytes, file=0):
    """FromVcfFile over a VCF's (inflated) bytes -> [(CHROM, start, end)] in file order; VcfError at the first refused line.  A CHROM
    that is empty is refused: vcf-to-elsites would write a line its .elsites loader refuses."""
    lines, nbytes, infos = parse_header(data, file)
    parsers = parser_table(infos)
    out = []
    for k, (raw, tok) in enumerate(er.scan_lines(data[nbytes:])):
        line = lines + 1 + k
        if raw >= er.MAX_TOKEN:
            raise VcfError(file, line, LONG)
        try:
            chrom, st, en = parse_line(tok, parsers)
        except Panic as p:
            raise VcfError(file, line, p.reason) from None
        if chrom == b"":
            raise VcfError(file, line, CHROM)
        out.append((chrom, st, en))
    return out


def is_vcf(data: bytes) -> bool:
    return not data.startswith(er.HEADER) and (data[:1] == b"\x1f" or data.startswith(PREFIX))


def rows(data: bytes, file=0):
    """one --known-sites file by its content -> [(CHROM, start, end)]"""
    if data.startswith(er.HEADER):
        return er.from_elsites(data, file)
    if data[:1] == b"\x1f":
        return from_vcf(gzip.decompress(data), file)
    if data.startswith(PREFIX):
        return from_vcf(data, file)
    raise er.ElsitesError(file, 0, er.HEADER_BAD)


def load(files, contig_names, fast=False):
    """elp_load_known_sites over a list of .elsites and VCF contents -> (per-contig (k, 2) int32 lists, lines on no @SQ SN): one stable
    sort and one flatten over every file's intervals in list order"""
    names = [n.encode() if isinstance(n, str) else n for n in contig_names]
    known = set(names) - {b"*"}
    per_name, unmatched = {}, 0
    for f, data in enumerate(files):
        for chrom, st, en in rows(data, f):
            if chrom not in known:
                unmatched += 1
            else:
                per_name.setdefault(chrom, []).append((st, en))
    flat = er.sort_flatten_fast if fast else er.sort_flatten
    tables = [flat(np.array(per_name.get(n, []) if n in known else [], dtype=np.int64).reshape(-1, 2)) for n in names]
    return tables, unmatched


def vcf_to_elsites(data: bytes) -> bytes:
    """elprep vcf-to-elsites: FromVcfFile, ParallelSortByStart + ParallelFlatten per chromosome, ToElsitesFile"""
    per = {}
    for chrom, st, en in from_vcf(gzip.decompress(data) if data[:1] == b"\x1f" else data):
        per.setdefault(chrom, []).append((st, en))
    out = []
    for chrom, iv in per.items():
        for s, e in er.sort_flatten(np.array(iv, dtype=np.int64).reshape(-1, 2)).tolist():
            out.append((chrom, s, e))
    return er.write(out)


def bgzf(data: bytes, block=65280, level=6) -> bytes:
    """BGZF blocks of at most `block` input bytes each, and the EOF marker"""
    out = bytearray()
    for i in range(0, len(data), block):
        piece = data[i:i + block]
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        cdata = co.compress(piece) + co.flush()
        bsize = 18 + len(cdata) + 8
        out += b"\x1f\x8b\x08\x04" + b"\x00" * 4 + b"\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize - 1)
        out += cdata + struct.pack("<II", zlib.crc32(piece) & 0xFFFFFFFF, len(piece))
    out += bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
    return bytes(out)
