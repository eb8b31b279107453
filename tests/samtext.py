"""SAM text for the device SAM ingest tests: a restatement of the reference's SAM alignment-line parser and BAM record
writer, and two ways to produce SAM text from a batch.

* ``sam_line_to_bam(line, header)`` -- parseSamAlignment (sam/sam-files.go:386-410, scanner sam/string-scanner.go) followed by
  formatBamAlignment (sam/bam-files.go:635-737), written from the Go source.  Raises ``SamError`` where the reference panics, and
  where elp_append_sam refuses a line the reference would write as a malformed record (QNAME > 254 bytes, a merged CIGAR
  operation >= 2^28, QUAL / SEQ length mismatch), a hexadecimal float, a tab as an A value, a tag name with a tab
  (kind "ESAM"), or more than 65535 CIGAR operations (kind "ELIMIT").
* ``format_sam(batch, header, tags)`` -- FormatAlignment-style text, one read at a time, with any optional fields.
* ``sam_text(batch, header, const_tags)`` -- the same text built with vectorised NumPy for millions of reads (RG:Z plus a
  constant tag string per line).
"""
import re
import struct
from fractions import Fraction

import numpy as np

from elprep_b200 import sam

CIGAR_TEXT = "MIDNSHP=X"
_CIGAR_OP = {c: "MIDNSHP=X".index(c.upper()) for c in "MmIiDdNnSsHhPpXx="}
_REF_CONSUMING = {0, 2, 3, 7, 8}


class SamError(ValueError):
    def __init__(self, kind, msg):
        super().__init__(f"{kind}: {msg}")
        self.kind = kind


def _esam(msg):
    return SamError("ESAM", msg)


# ---- strconv ----
def parse_dec(s, lo, hi, signed):
    """strconv.ParseInt (signed) / ParseUint, base 10, plus a range [lo, hi]"""
    body = s[1:] if signed and s[:1] in (b"+", b"-") else s
    if not body or not body.isdigit():
        raise _esam(f"invalid integer {s!r}")
    v = int(s)
    if not lo <= v <= hi:
        raise _esam(f"integer {s!r} out of range")
    return v


_DEC = re.compile(rb"[+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?")


def f32_bits(s):
    """float32(strconv.ParseFloat(s, 32)) as IEEE bits, correctly rounded from the exact decimal value"""
    low = s.lower()
    if low in (b"inf", b"+inf", b"infinity", b"+infinity"):
        return 0x7F800000
    if low in (b"-inf", b"-infinity"):
        return 0xFF800000
    if low == b"nan":
        return 0x7FC00000
    if not _DEC.fullmatch(s):
        raise _esam(f"invalid float {s!r}")
    neg = s[:1] == b"-"
    a = abs(Fraction(s.decode()))
    sign = 0x80000000 if neg else 0
    if a == 0:
        return sign
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)
    q = Fraction(2) ** (e - 23)                         # the float32 quantum at this exponent (denormals: 2^-149)
    m = a / q
    n = m.numerator // m.denominator
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n & 1):
        n += 1
    v = n * q
    if v >= Fraction(2) ** 128:
        raise _esam(f"float {s!r} out of range")
    return sign | struct.unpack("<I", struct.pack("<f", float(v)))[0]


# ---- stringScanner (sam/string-scanner.go) ----
class _Scanner:
    def __init__(self, data):
        self.d, self.i = data, 0

    def len(self):
        return len(self.d) - self.i

    def read_byte_until(self, c):
        start, nxt = self.i, self.i + 1
        if start >= len(self.d):
            raise _esam("index out of range")
        if nxt >= len(self.d):
            self.i = len(self.d)
            return self.d[start], False
        if self.d[nxt] != c:
            raise _esam(f"unexpected character {self.d[nxt]} in stringScanner.ReadByteUntil")
        self.i = nxt + 1
        return self.d[start], True

    def read_until(self, c):
        j = self.d.find(bytes([c]), self.i)
        if j < 0:
            s, self.i = self.d[self.i:], len(self.d)
            return s, False
        s, self.i = self.d[self.i:j], j + 1
        return s, True

    def read_until2(self, c1, c2):
        for j in range(self.i, len(self.d)):
            if self.d[j] in (c1, c2):
                s, self.i = self.d[self.i:j], j + 1
                return s, self.d[j]
        s, self.i = self.d[self.i:], len(self.d)
        return s, 0

    def do_string(self):
        s, ok = self.read_until(9)
        if not ok:
            raise _esam("missing tabulator in SAM alignment line")
        return s


def _scan_cigar(s):
    """ScanCigarString (sam/sam-types.go:672-740): [(op, length)], adjacent equal operations merged"""
    if s == b"*" or s == b"":
        return []
    out, i = [], 0
    while i < len(s):
        j = i
        while j < len(s) and 48 <= s[j] <= 57:
            j += 1
        if j == len(s):
            raise _esam("CIGAR: index out of range")
        ln = parse_dec(s[i:j], -(1 << 31), (1 << 31) - 1, True)
        op = _CIGAR_OP.get(chr(s[j]))
        if op is None:
            raise _esam(f"invalid CIGAR operation {chr(s[j])!r}")
        if out and out[-1][0] == op:
            out[-1][1] += ln
        else:
            out.append([op, ln])
        i = j + 1
    return out


def _tag_value(sc):
    """parseSamOptionalField (sam/sam-files.go:335-346) -> (tag, (BAM type byte(s), payload))"""
    name, ok = sc.read_until(ord(":"))
    if not ok or len(name) != 2:
        raise _esam(f"invalid field tag {name!r}")
    if 9 in name:
        raise _esam("tag name with a tab (refused by elp_append_sam)")
    ty, ok = sc.read_byte_until(ord(":"))
    if not ok:
        raise _esam("invalid field type")
    ty = chr(ty)
    if ty == "A":
        v, _ = sc.read_byte_until(9)
        if v == 9:
            raise _esam("a tab as the value of an A field (refused by elp_append_sam)")
        return name, b"A" + bytes([v])
    if ty == "i":
        v, _ = sc.read_until(9)
        x = parse_dec(v, -(1 << 63), (1 << 63) - 1, True)
        if x < 0:
            for t, lo, fmt in (("c", -128, "<b"), ("s", -32768, "<h"), ("i", -(1 << 31), "<i")):
                if x >= lo:
                    return name, t.encode() + struct.pack(fmt, x)
            raise _esam("integer value too small in BAM alignment tag")
        for t, hi, fmt in (("C", 255, "<B"), ("S", 65535, "<H"), ("I", (1 << 32) - 1, "<I")):
            if x <= hi:
                return name, t.encode() + struct.pack(fmt, x)
        raise _esam("integer value too large in BAM alignment tag")
    if ty == "f":
        v, _ = sc.read_until(9)
        return name, b"f" + struct.pack("<I", f32_bits(v))
    if ty == "Z":
        v, _ = sc.read_until(9)
        return name, b"Z" + v + b"\0"
    if ty == "H":
        v, _ = sc.read_until(9)
        out = bytearray()
        for i in range(0, len(v), 2):
            pair = v[i:i + 2]
            if len(pair) != 2 or not all(chr(ch) in "0123456789abcdefABCDEF" for ch in pair):
                raise _esam("invalid hex pair")
            out.append(int(pair, 16))
        return name, b"H" + out.hex().upper().encode() + b"\0"
    if ty == "B":
        nt, ok = sc.read_byte_until(ord(","))
        if not ok:
            raise _esam("missing entry in numeric array")
        nt = chr(nt)
        spec = {"c": (-128, 127, True, "<b"), "C": (0, 255, False, "<B"), "s": (0, 65535, False, "<H"), "S": (0, 65535, False, "<H"),
                "i": (-(1 << 31), (1 << 31) - 1, True, "<i"), "I": (0, (1 << 32) - 1, False, "<I"), "f": None}
        if nt not in spec:
            raise _esam(f"invalid numeric array type {nt}")
        vals = bytearray()
        cnt = 0
        while True:
            e, sep = sc.read_until2(ord(","), 9)
            if nt == "f":
                vals += struct.pack("<I", f32_bits(e))
            else:
                lo, hi, sg, fmt = spec[nt]
                vals += struct.pack(fmt, parse_dec(e, lo, hi, sg))   # B:s: ParseUint(s, 10, 16), stored as int16 bits
            cnt += 1
            if sep != ord(","):
                break
        return name, b"B" + nt.encode() + struct.pack("<I", cnt) + bytes(vals)
    raise _esam(f"unknown optional field type {ty!r}")


def _bin(beg, end):
    """bin() (sam/bam-files.go:443-468): beg / end are int32 values"""
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return (base + (beg >> shift)) & 0xFFFF
    return 0


def _i32(x):
    return ((x + (1 << 31)) % (1 << 32)) - (1 << 31)


def sam_line_to_bam(line, header):
    """one SAM alignment line (bytes, without '\\n') -> the BAM record bytes formatBamAlignment writes, block_size included"""
    sc = _Scanner(bytes(line))
    qname = sc.do_string()
    flag = parse_dec(sc.do_string(), 0, 65535, False)
    rname = sc.do_string()
    pos = parse_dec(sc.do_string(), -(1 << 31), (1 << 31) - 1, True)
    mapq = parse_dec(sc.do_string(), 0, 255, False)
    cigar = _scan_cigar(sc.do_string())
    rnext = sc.do_string()
    pnext = parse_dec(sc.do_string(), -(1 << 31), (1 << 31) - 1, True)
    tlen = parse_dec(sc.do_string(), -(1 << 31), (1 << 31) - 1, True)
    seq, ok = sc.read_until(9)                         # doSeq: the SEQ field must end with a tab
    if not ok:
        raise _esam("missing tabulator in SAM alignment line")
    qual, _ = sc.read_until(9)
    tags = []                                          # SmallMap: a repeated tag replaces the value at its first position
    while sc.len() > 0:
        k, v = _tag_value(sc)
        for t in tags:
            if t[0] == k:
                t[1] = v
                break
        else:
            tags.append([k, v])
    if len(qname) > 254:
        raise _esam("QNAME longer than 254 bytes")
    if any(ln >= 1 << 28 for _, ln in cigar):
        raise _esam("CIGAR operation length of 2^28 or more")
    if len(qual) != len(seq):
        raise _esam("QUAL and SEQ differ in length")
    if len(cigar) > 65535:
        raise SamError("ELIMIT", "more than 65535 CIGAR operations")
    dict_ = {"*": -1}
    for i, s in enumerate(header.SQ):
        dict_[s["SN"]] = i
    refid = dict_.get(rname.decode("latin-1"), -1)
    nref = refid if rnext == b"=" else dict_.get(rnext.decode("latin-1"), -1)
    beg = _i32(pos - 1)
    end = beg
    if not flag & 4:
        for op, ln in cigar:
            if op in _REF_CONSUMING:
                end = _i32(end + ln)
        end = _i32(end - 1)
    nib = bytearray((len(seq) + 1) // 2)
    for i, ch in enumerate(seq):
        v = sam.NIBBLE_TO_BASE.find(chr(ch)) if chr(ch) in sam.NIBBLE_TO_BASE else 15
        nib[i >> 1] |= v << (0 if i & 1 else 4)
    body = struct.pack("<iiBBHHHIiii", refid, beg, len(qname) + 1, mapq, _bin(beg, end), len(cigar), flag, len(seq), nref, _i32(pnext - 1), tlen)
    body += qname + b"\0" + b"".join(struct.pack("<I", (ln << 4) | op) for op, ln in cigar) + bytes(nib) + bytes((q - 33) & 0xFF for q in qual)
    body += b"".join(k + v for k, v in tags)
    return struct.pack("<I", len(body)) + body


def sam_lines_to_bam(lines, header):
    """-> (uint8 records, uint64 offsets [n+1]) of sam_line_to_bam over every line"""
    recs = [sam_line_to_bam(x, header) for x in lines]
    off = np.zeros(len(recs) + 1, np.uint64)
    np.cumsum([len(r) for r in recs], out=off[1:])
    return np.frombuffer(b"".join(recs), np.uint8).copy(), off


# ---- SAM text from a batch ----
def format_sam(batch, header, tags=None):
    """FormatAlignment-style SAM lines (bytes each, no '\\n') of every read of ``batch``: RNEXT is '=' when it equals a mapped
    RNAME; RG:Z from batch.rg first, then tags[i] (a list of "TG:T:value" strings) if given"""
    names = [s["SN"] for s in header.SQ]
    ids = [r["ID"] for r in header.RG]
    qo, co = batch.qname_off.astype(np.int64), batch.cigar_off.astype(np.int64)
    so, uo = batch.seq_off.astype(np.int64), batch.qual_off.astype(np.int64)
    out = []
    for i in range(batch.n):
        L = int(batch.lseq[i])
        rid, nid = int(batch.refid[i]), int(batch.nref[i])
        rname = names[rid] if rid >= 0 else "*"
        rnext = "=" if nid >= 0 and nid == rid else (names[nid] if nid >= 0 else "*")
        seq = sam.decode_seq(batch.seq[so[i]:so[i] + (L + 1) // 2], L) if L else "*"
        qual = bytes(batch.qual[uo[i]:uo[i] + L] + 33).decode() if L else "*"
        f = [bytes(batch.qname[qo[i]:qo[i + 1]]).decode(), str(int(batch.flag[i])), rname, str(int(batch.pos[i])), str(int(batch.mapq[i])),
             sam.decode_cigar(batch.cigar[co[i]:co[i + 1]]), rnext, str(int(batch.pnext[i])), str(int(batch.tlen[i])), seq, qual]
        if int(batch.rg[i]) >= 0:
            f.append("RG:Z:" + ids[int(batch.rg[i])])
        if tags is not None:
            f += list(tags[i])
        out.append("\t".join(f).encode())
    return out


def _ragged(lens):
    off = np.zeros(lens.size + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return off


def _gather(data, off, idx):
    """the ragged rows idx of (data, off) -> (bytes, lengths)"""
    lens = (off[1:] - off[:-1])[idx]
    no = _ragged(lens)
    src = np.repeat(off[:-1][idx] - no[:-1], lens) + np.arange(int(no[-1]), dtype=np.int64)
    return data[src], lens


def _int_text(v):
    """decimal text of int64 values -> (bytes, lengths)"""
    v = np.asarray(v, np.int64)
    a, neg = np.abs(v), v < 0
    nd = np.ones(v.size, np.int64)
    for k in range(1, 11):
        nd += a >= 10 ** k
    W = 12
    D = np.empty((v.size, W), np.uint8)
    for j in range(11):
        D[:, W - 1 - j] = (a // 10 ** j) % 10 + 48
    L = nd + neg
    D[np.arange(v.size), W - 1 - nd] = np.where(neg, 45, D[np.arange(v.size), W - 1 - nd])
    mask = np.arange(W)[None, :] >= (W - L)[:, None]
    return D[mask], L


def _join(fields):
    """fields: [(bytes, lengths)] per read -> lines "f0\\tf1...\\n" as one uint8 array"""
    K, n = len(fields), fields[0][1].size
    line_len = sum(f[1] for f in fields) + K
    lo = _ragged(line_len)
    out = np.empty(int(lo[-1]), np.uint8)
    start = lo[:-1].copy()
    for k, (data, lens) in enumerate(fields):
        fo = _ragged(lens)
        out[np.repeat(start - fo[:-1], lens) + np.arange(int(fo[-1]), dtype=np.int64)] = data
        start += lens
        out[start] = 10 if k == K - 1 else 9
        start += 1
    return out


def sam_text(batch, header, const_tags=b"", chunk=1 << 20):
    """format_sam's text (tags: const_tags, then RG:Z) for every read, vectorised -> one uint8 array; reads need lseq >= 1"""
    assert np.all(batch.lseq >= 1)
    parts = []
    names = [s["SN"].encode() for s in header.SQ] + [b"*"]
    ndat = np.frombuffer(b"".join(names), np.uint8)
    noff = _ragged(np.array([len(x) for x in names], np.int64))
    ids = [b"RG:Z:" + r["ID"].encode() for r in header.RG] + [b""]
    idat = np.frombuffer(b"".join(ids), np.uint8)
    ioff = _ragged(np.array([len(x) for x in ids], np.int64))
    lut = np.frombuffer(sam.NIBBLE_TO_BASE.encode(), np.uint8)
    ctext = np.frombuffer(CIGAR_TEXT.encode(), np.uint8)
    for a in range(0, batch.n, chunk):
        b = batch.take(np.arange(a, min(batch.n, a + chunk)))
        n = b.n
        qo = b.qname_off.astype(np.int64)
        rid = np.where(b.refid >= 0, b.refid, len(names) - 1).astype(np.int64)
        nid = np.where(b.nref >= 0, b.nref, len(names) - 1).astype(np.int64)
        rname = _gather(ndat, noff, rid)
        same = (b.nref >= 0) & (b.nref == b.refid)
        rn_d, rn_l = _gather(ndat, noff, nid)
        eq_l = np.where(same, 1, rn_l)
        keep = np.repeat(~same, rn_l)
        eq_off = _ragged(eq_l)
        rnext_d = np.empty(int(eq_off[-1]), np.uint8)
        rnext_d[np.repeat(eq_off[:-1] - _ragged(rn_l)[:-1], rn_l)[keep] + np.arange(rn_d.size)[keep]] = rn_d[keep]
        rnext_d[eq_off[:-1][same]] = ord("=")
        # CIGAR: "<len><op>" per operation, "*" for none
        co = b.cigar_off.astype(np.int64)
        nops = co[1:] - co[:-1]
        od, ol = _int_text((b.cigar >> 4).astype(np.int64))
        op_len = ol + 1
        oo = _ragged(op_len)
        opt = np.empty(int(oo[-1]), np.uint8)
        opt[np.repeat(oo[:-1] - _ragged(ol)[:-1], ol) + np.arange(od.size)] = od
        opt[oo[1:] - 1] = ctext[b.cigar & 15]
        per_read = np.add.reduceat(np.append(op_len, 0), co[:-1]) if op_len.size else np.zeros(n, np.int64)
        per_read = np.where(nops > 0, per_read, 0)
        cig_l = np.where(nops > 0, per_read, 1)
        cig_off = _ragged(cig_l)
        cig = np.full(int(cig_off[-1]), ord("*"), np.uint8)
        src_off = _ragged(per_read)
        cig[np.repeat(cig_off[:-1] - src_off[:-1], per_read) + np.arange(int(src_off[-1]))] = opt
        # SEQ / QUAL
        L = b.lseq.astype(np.int64)
        so = b.seq_off.astype(np.int64)
        k = np.arange(int(L.sum()), dtype=np.int64) - np.repeat(_ragged(L)[:-1], L)
        byte = b.seq[np.repeat(so[:-1], L) + (k >> 1)]
        seq = lut[np.where(k & 1, byte & 15, byte >> 4)]
        fields = [(b.qname, qo[1:] - qo[:-1]), _int_text(b.flag), rname, _int_text(b.pos), _int_text(b.mapq), (cig, cig_l),
                  (rnext_d, eq_l), _int_text(b.pnext), _int_text(b.tlen), (seq, L), (b.qual + np.uint8(33), L)]
        if const_tags:
            ct = np.frombuffer(const_tags, np.uint8)
            fields.append((np.tile(ct, n), np.full(n, ct.size, np.int64)))
        has_rg = b.rg >= 0
        if has_rg.any():
            assert has_rg.all(), "sam_text: every read or none carries RG"
            fields.append(_gather(idat, ioff, b.rg.astype(np.int64)))
        parts.append(_join(fields))
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)
