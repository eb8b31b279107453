"""SAM text output restated from the reference for the elp_fetch_sam tests: FormatAlignment (sam/sam-files.go:563-598) with
formatSamTag (:485-546) and cigarToString (:548-557), over either parseBamAlignment (sam/bam-files.go:317-400) of a BAM record or
parseSamAlignment (sam/sam-files.go:386-410) of a SAM line.

An alignment here is a dict with the reference's fields: QNAME / RNAME / RNEXT bytes, FLAG / POS / MAPQ / PNEXT / TLEN ints, CIGAR
[(length, op char)], SEQ bytes (the bases SEQ.Base gives back), QUAL bytes (phred, no +33), TAGS [(tag, Go type, value)] with Go type one
of "byte", "int64", "float32" (value: IEEE bits), "string", "ByteArray" and "[]int8" ... "[]float32" (list of ints, or of bits for floats).

``format_f32`` is strconv.AppendFloat(b, float64(v), 'g', -1, 32) computed from exact rationals: the shortest digit string that reads
back as the same float32 (through samtext.f32_bits), the closest of those to the exact value (a tie to the even digit), laid out as
Go's %e / %f.
"""
import functools
import struct
from fractions import Fraction

from samtext import _Scanner, _esam, _scan_cigar, f32_bits, parse_dec

SEQ_BASES = b"=ACMGRSVTWYHKDBN"
CIGAR_OPS = b"MIDNSHP=X"
_BASE_TO_NIBBLE = {c: i for i, c in enumerate(SEQ_BASES)}


# ---- strconv 'g', -1, 32 ----
def _exact(bits):
    """float32 bits of a finite non-zero magnitude -> exact Fraction"""
    e, m = (bits >> 23) & 0xFF, bits & 0x7FFFFF
    return Fraction(m, 1 << 149) if e == 0 else Fraction((1 << 23) | m) * Fraction(2) ** (e - 150)


@functools.lru_cache(maxsize=None)
def shortest_digits(bits):
    """(digit string d1...dn, dp) with value 0.d1...dn x 10^dp: the shortest decimal that f32_bits maps back to these bits (of a
    positive finite float32), the closest to the exact value among those of that length"""
    v = _exact(bits)
    E = len(str(v.numerator)) - len(str(v.denominator))            # 10^E <= v < 10^(E+1), after the correction below
    if Fraction(10) ** E > v:
        E -= 1
    elif Fraction(10) ** (E + 1) <= v:
        E += 1
    def closest(p):
        """the closest p-digit candidate that round-trips, or None: floor or ceil of v at p significant digits"""
        scale = Fraction(10) ** (E - p + 1)
        lo = v.numerator * scale.denominator // (v.denominator * scale.numerator)
        best = None
        for d in (lo, lo + 1):
            try:
                ok = f32_bits(b"%de%d" % (d, E - p + 1)) == bits
            except ValueError:                                          # rounds to +Inf
                ok = False
            if ok and (best is None or abs(d * scale - v) < abs(best * scale - v) or (abs(d * scale - v) == abs(best * scale - v) and d % 2 == 0)):
                best = d                                                # a tie goes to the even digit, as Go's and C++'s shortest forms do
        return best
    # a round-tripping p-digit candidate implies one with p + 1 digits, so the shortest p is found by bisection over 1..9
    lo_p, hi_p, best = 1, 9, None
    while lo_p < hi_p:
        mid = (lo_p + hi_p) // 2
        if closest(mid) is not None:
            hi_p = mid
        else:
            lo_p = mid + 1
    best = closest(lo_p)
    assert best is not None, "every float32 round-trips with 9 digits"
    s = str(best)
    return s.rstrip("0"), E + 1 + (len(s) - lo_p)                       # lo + 1 may be 10^p: one more integer digit


def format_f32(bits):
    """strconv.AppendFloat(nil, float64(math.Float32frombits(bits)), 'g', -1, 32) as bytes"""
    neg, mag = bits >> 31, bits & 0x7FFFFFFF
    if mag > 0x7F800000:
        return b"NaN"
    if mag == 0x7F800000:
        return b"-Inf" if neg else b"+Inf"
    sign = "-" if neg else ""
    if mag == 0:
        return (sign + "0").encode()
    d, dp = shortest_digits(mag)
    x = dp - 1
    if x < -4 or x >= 6:                                                # %e, eprec = 6 for shortest
        s = d[0] + ("." + d[1:] if len(d) > 1 else "") + "e" + ("-" if x < 0 else "+") + "%02d" % abs(x)
    else:                                                               # %f, precision max(n - dp, 0)
        ip = (d[:dp] + "0" * (dp - len(d))) if dp > 0 else "0"
        fr = ("0" * -dp + d) if dp <= 0 else d[dp:]
        s = ip + ("." + fr if fr else "")
    return (sign + s).encode()


# ---- parseBamAlignment ----
def _u32(b, i):
    return struct.unpack_from("<I", b, i)[0]


def _i32(b, i):
    return struct.unpack_from("<i", b, i)[0]


def _wrap32(x):
    return ((x + (1 << 31)) % (1 << 32)) - (1 << 31)


_ARRAY = {ord("c"): ("[]int8", "<b", 1), ord("C"): ("[]uint8", "<B", 1), ord("s"): ("[]int16", "<h", 2), ord("S"): ("[]uint16", "<H", 2),
          ord("i"): ("[]int32", "<i", 4), ord("I"): ("[]uint32", "<I", 4), ord("f"): ("[]float32", "<I", 4)}


def parse_bam_alignment(rec, names):
    """one BAM record (block_size included) -> alignment; names: the @SQ names as bytes (BAM refID order).  The H field is read up to
    its NUL (the reference looks for the character '0', a bug; see DESIGN.md)"""
    rec = bytes(rec)
    r = rec[4:]
    refid, pos = _i32(r, 0), _i32(r, 4)
    l_name, mapq, ncig, flag, lseq = r[8], r[9], struct.unpack_from("<H", r, 12)[0], struct.unpack_from("<H", r, 14)[0], _i32(r, 16)
    nref, pnext, tlen = _i32(r, 20), _i32(r, 24), _i32(r, 28)
    a = {"RNAME": b"*" if refid < 0 else names[refid]}
    a["POS"] = _wrap32(pos + 1)
    if nref < 0:
        a["RNEXT"] = b"*"
    else:
        a["RNEXT"] = b"=" if names[nref] == a["RNAME"] else names[nref]
    a.update(PNEXT=_wrap32(pnext + 1), TLEN=tlen, FLAG=flag, MAPQ=mapq, QNAME=r[32:32 + l_name - 1])
    i = 32 + l_name
    a["CIGAR"] = []
    for _ in range(ncig):
        w = _u32(r, i)
        if w & 15 > 8:
            raise _esam("CIGAR operation code above 8 (index out of range)")
        a["CIGAR"].append((w >> 4, CIGAR_OPS[w & 15]))
        i += 4
    nb = (lseq + 1) >> 1
    a["SEQ"] = bytes(SEQ_BASES[(r[i + (k >> 1)] >> (0 if k & 1 else 4)) & 15] for k in range(lseq))
    i += nb
    a["QUAL"] = r[i:i + lseq]
    i += lseq
    tags = []
    while i < len(r):
        tag, ty = r[i:i + 2], r[i + 2]
        i += 3
        if ty == ord("A"):
            tags.append((tag, "byte", r[i])); i += 1
        elif ty in b"cCsSiI":
            fmt, sz = {ord("c"): ("<b", 1), ord("C"): ("<B", 1), ord("s"): ("<h", 2), ord("S"): ("<H", 2), ord("i"): ("<i", 4), ord("I"): ("<I", 4)}[ty]
            tags.append((tag, "int64", struct.unpack_from(fmt, r, i)[0])); i += sz
        elif ty == ord("f"):
            tags.append((tag, "float32", _u32(r, i))); i += 4
        elif ty in b"ZH":
            e = r.index(b"\0", i)
            if ty == ord("Z"):
                tags.append((tag, "string", r[i:e]))
            else:
                tags.append((tag, "ByteArray", bytes(int(r[j:j + 2], 16) for j in range(i, e, 2))))
            i = e + 1
        elif ty == ord("B"):
            gt, fmt, es = _ARRAY[r[i]]
            cnt = _u32(r, i + 1)
            i += 5
            tags.append((tag, gt, [struct.unpack_from(fmt, r, i + es * k)[0] for k in range(cnt)])); i += es * cnt
        else:
            raise _esam(f"unknown BAM tag type {ty}")
    a["TAGS"] = tags
    return a


# ---- parseSamAlignment ----
def _sam_tag(sc):
    """parseSamOptionalField -> (tag, Go type, value), the Go conversions of parseSam* (sam/sam-files.go:186-317)"""
    name, ok = sc.read_until(ord(":"))
    if not ok or len(name) != 2:
        raise _esam(f"invalid field tag {name!r}")
    ty, ok = sc.read_byte_until(ord(":"))
    if not ok:
        raise _esam("invalid field type")
    ty = chr(ty)
    if ty == "A":
        v, _ = sc.read_byte_until(9)
        return name, "byte", v
    if ty in "ifZH":
        v, _ = sc.read_until(9)
        if ty == "i":
            return name, "int64", parse_dec(v, -(1 << 63), (1 << 63) - 1, True)
        if ty == "f":
            return name, "float32", f32_bits(v)
        if ty == "Z":
            return name, "string", v
        return name, "ByteArray", bytes(int(v[j:j + 2], 16) for j in range(0, len(v), 2))
    if ty == "B":
        nt, ok = sc.read_byte_until(ord(","))
        if not ok:
            raise _esam("missing entry in numeric array")
        gt = _ARRAY[nt][0]
        vals = []
        while True:
            e, sep = sc.read_until2(ord(","), 9)
            if nt == ord("c"):
                vals.append(parse_dec(e, -128, 127, True))
            elif nt == ord("C"):
                vals.append(parse_dec(e, 0, 255, False))
            elif nt == ord("s"):
                vals.append(_wrap16(parse_dec(e, 0, 65535, False)))     # int16(ParseUint(s, 10, 16))
            elif nt == ord("S"):
                vals.append(parse_dec(e, 0, 65535, False))
            elif nt == ord("i"):
                vals.append(parse_dec(e, -(1 << 31), (1 << 31) - 1, True))
            elif nt == ord("I"):
                vals.append(parse_dec(e, 0, (1 << 32) - 1, False))
            else:
                vals.append(f32_bits(e))
            if sep != ord(","):
                break
        return name, gt, vals
    raise _esam(f"unknown optional field type {ty!r}")


def _wrap16(x):
    return ((x + (1 << 15)) % (1 << 16)) - (1 << 15)


def parse_sam_alignment(line):
    """one SAM alignment line (bytes, no '\\n') -> alignment; RNAME / RNEXT stay the text of the line"""
    sc = _Scanner(bytes(line))
    a = {"QNAME": sc.do_string(), "FLAG": parse_dec(sc.do_string(), 0, 65535, False), "RNAME": sc.do_string(),
         "POS": parse_dec(sc.do_string(), -(1 << 31), (1 << 31) - 1, True), "MAPQ": parse_dec(sc.do_string(), 0, 255, False)}
    a["CIGAR"] = [(ln, CIGAR_OPS[op]) for op, ln in _scan_cigar(sc.do_string())]
    a["RNEXT"] = sc.do_string()
    a["PNEXT"] = parse_dec(sc.do_string(), -(1 << 31), (1 << 31) - 1, True)
    a["TLEN"] = parse_dec(sc.do_string(), -(1 << 31), (1 << 31) - 1, True)
    seq, ok = sc.read_until(9)                                          # doSeq: baseToNibble, anything else 15
    if not ok:
        raise _esam("missing tabulator in SAM alignment line")
    a["SEQ"] = bytes(SEQ_BASES[_BASE_TO_NIBBLE.get(c, 15)] for c in seq)
    qual, _ = sc.read_until(9)
    a["QUAL"] = bytes((q - 33) & 0xFF for q in qual)
    tags = []                                                           # TAGS.Set: a repeated tag keeps its position, takes the last value
    while sc.len() > 0:
        t = _sam_tag(sc)
        for j, u in enumerate(tags):
            if u[0] == t[0]:
                tags[j] = t
                break
        else:
            tags.append(t)
    a["TAGS"] = tags
    return a


# ---- FormatAlignment ----
def format_tag(tag, gt, v):
    out = b"\t" + tag
    if gt == "byte":
        return out + b":A:" + bytes([v])
    if gt == "int64":
        return out + b":i:%d" % v
    if gt == "float32":
        return out + b":f:" + format_f32(v)
    if gt == "string":
        return out + b":Z:" + v
    if gt == "ByteArray":
        return out + b":H:" + b"".join(b"%02x" % x for x in v)
    sub = {"[]int8": b"c", "[]uint8": b"C", "[]int16": b"s", "[]uint16": b"S", "[]int32": b"i", "[]uint32": b"I", "[]float32": b"f"}[gt]
    out += b":B:" + sub
    for x in v:
        out += b"," + (format_f32(x) if sub == b"f" else b"%d" % x)
    return out


def format_alignment(a):
    """FormatAlignment(aln, nil): one line with its '\\n'"""
    cig = b"".join(b"%d" % ln + bytes([op]) for ln, op in a["CIGAR"]) if a["CIGAR"] else b"*"
    rnext = a["RNEXT"]
    if rnext not in (b"=", b"*") and rnext == a["RNAME"]:
        rnext = b"="
    f = [a["QNAME"], b"%d" % a["FLAG"], a["RNAME"], b"%d" % a["POS"], b"%d" % a["MAPQ"], cig, rnext, b"%d" % a["PNEXT"], b"%d" % a["TLEN"],
         a["SEQ"], bytes((q + 33) & 0xFF for q in a["QUAL"])]
    return b"\t".join(f) + b"".join(format_tag(*t) for t in a["TAGS"]) + b"\n"


def bam_to_sam(rec, names, flag=None, qual=None):
    """FormatAlignment(parseBamAlignment(rec)) with FLAG / QUAL replaced when given (what elp_fetch_sam writes for the record)"""
    a = parse_bam_alignment(rec, names)
    if flag is not None:
        a["FLAG"] = int(flag)
    if qual is not None:
        a["QUAL"] = bytes(qual)
    return format_alignment(a)


def sam_to_sam(line, flag=None):
    """FormatAlignment(parseSamAlignment(line)), the reference's own SAM -> SAM text"""
    a = parse_sam_alignment(line)
    if flag is not None:
        a["FLAG"] = int(flag)
    return format_alignment(a)
