"""Host-side mirror of the reference's record layer for the hot path.

Mirrors (names and meaning) the subset of ``sam/sam-types.go`` the path needs:

* ``Header``   -- ``sam.Header`` (``sam/sam-types.go:60-120``): ``SQ``, ``RG``, ``HD`` ``SO``.
* ``AlignmentBatch`` -- a columnar (SoA) batch of ``sam.Alignment`` records
  (``sam/sam-types.go:289-331``) plus the ``REFID`` / ``NextREFID`` temps that
  ``filters.AddREFID`` (``filters/simple-filters.go:208-231``) fills in.  This is
  exactly the payload of ``elp_batch`` in ``include/elprep_b200.h``.
* FLAG constants (``sam/sam-types.go:485-520``) and ``SortingOrder`` values
  (``sam/sam-types.go:40-58``).

CIGAR uses the BAM encoding ``len<<4 | op`` with ``op`` indexing ``MIDNSHP=X``;
SEQ is 4-bit BAM nibbles, high nibble first, each read byte aligned
(``utils/nibbles/nibbles.go:91-100``); QUAL is phred bytes without +33.
"""
from __future__ import annotations

import numpy as np

# FLAG bits (sam/sam-types.go:485-520)
Multiple, Proper, Unmapped, NextUnmapped = 0x1, 0x2, 0x4, 0x8
Reversed, NextReversed, First, Last = 0x10, 0x20, 0x40, 0x80
Secondary, QCFailed, Duplicate, Supplementary = 0x100, 0x200, 0x400, 0x800

# SortingOrder (sam/sam-types.go:40-58)
Keep, Unknown, Unsorted, Queryname, Coordinate = "keep", "unknown", "unsorted", "queryname", "coordinate"

CIGAR_OPS = "MIDNSHP=X"
NIBBLE_TO_BASE = "=ACMGRSVTWYHKDBN"
_BASE_TO_NIBBLE = {c: i for i, c in enumerate(NIBBLE_TO_BASE)}


class Header:
    """``sam.Header`` subset: @HD SO, @SQ (SN, LN), @RG (ID, LB, PU, ...)."""

    def __init__(self, sq=None, rg=None, so=Unknown):
        self.SQ = [dict(x) for x in (sq or [])]   # [{"SN": name, "LN": int}]
        self.RG = [dict(x) for x in (rg or [])]   # [{"ID":..., "LB":..., "PU":...}]
        self.HD = {"VN": "1.6", "SO": so}
        self.PG = []                              # [{"ID":..., "PP":..., ...}] (MergeInputs)
        self.CO = []                              # comment lines (MergeInputs)
        self.UserRecords = {}

    def HDSO(self):
        return self.HD.get("SO", Unknown)

    def SetHDSO(self, so):
        self.HD["SO"] = so

    # ---- derived tables the C ABI takes (elp_config) ----
    def contig_names(self):
        return [s["SN"] for s in self.SQ]

    def contig_lengths(self):
        return np.array([int(s["LN"]) for s in self.SQ], dtype=np.int32)

    def refid_table(self):
        """RNAME -> refid as ``filters.AddREFID`` builds it (simple-filters.go:208-214)."""
        t = {"*": -1}
        for i, s in enumerate(self.SQ):
            t[s["SN"]] = i
        return t

    def rg_index(self):
        return {r["ID"]: i for i, r in enumerate(self.RG)}

    def rg_lib_ids(self):
        """library id per @RG: equal LB strings share an id, -1 = no LB
        (lbTable, filters/mark-duplicates.go:413-423)."""
        libs, out = {}, []
        for r in self.RG:
            lb = r.get("LB")
            out.append(-1 if lb is None else libs.setdefault(lb, len(libs)))
        return np.array(out, dtype=np.int32).reshape(-1), list(libs.keys())

    def rg_cov_ids(self):
        """read-group covariate per @RG: PU if present else ID (filters/bqsr.go:35-51)."""
        covs, out = {}, []
        for r in self.RG:
            name = r.get("PU", r["ID"])
            out.append(covs.setdefault(name, len(covs)))
        return np.array(out, dtype=np.int32).reshape(-1), list(covs.keys())


def encode_cigar(s):
    """SAM CIGAR text -> BAM u32 ops, merging adjacent identical ops the way
    ``slowScanCigarString`` does (sam/sam-types.go:700-724). '*' -> empty."""
    if s in ("*", ""):
        return []
    ops, num = [], ""
    for ch in s:
        if ch.isdigit():
            num += ch
        else:
            op = CIGAR_OPS.index(ch.upper())
            ln = int(num)
            num = ""
            if ops and (ops[-1] & 15) == op:
                ops[-1] = (((ops[-1] >> 4) + ln) << 4) | op
            else:
                ops.append((ln << 4) | op)
    return ops


def decode_cigar(ops):
    return "".join(f"{int(o) >> 4}{CIGAR_OPS[int(o) & 15]}" for o in ops) or "*"


def encode_seq(s):
    """bases -> BAM nibbles (unknown chars -> 15 'N', sam-types.go:270-277)."""
    n = len(s)
    out = bytearray((n + 1) // 2)
    for i, c in enumerate(s):
        nib = _BASE_TO_NIBBLE.get(c, 15)
        if i & 1:
            out[i >> 1] |= nib
        else:
            out[i >> 1] |= nib << 4
    return bytes(out)


def decode_seq(b, n):
    return "".join(NIBBLE_TO_BASE[(b[i >> 1] >> (0 if i & 1 else 4)) & 15] for i in range(n))


class AlignmentBatch:
    """Columnar batch of alignment records (the ``elp_batch`` payload)."""

    FIELDS = ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg",
              "qname_off", "qname", "cigar_off", "cigar", "lseq", "seq", "qual", "opt_flags")

    def __init__(self, **kw):
        self.refid = np.ascontiguousarray(kw["refid"], dtype=np.int32)
        n = self.refid.shape[0]
        self.pos = np.ascontiguousarray(kw["pos"], dtype=np.int32)
        self.flag = np.ascontiguousarray(kw["flag"], dtype=np.uint16)
        self.mapq = np.ascontiguousarray(kw["mapq"], dtype=np.uint8)
        self.nref = np.ascontiguousarray(kw["nref"], dtype=np.int32)
        self.pnext = np.ascontiguousarray(kw["pnext"], dtype=np.int32)
        self.tlen = np.ascontiguousarray(kw["tlen"], dtype=np.int32)
        self.rg = np.ascontiguousarray(kw["rg"], dtype=np.int32)
        self.qname_off = np.ascontiguousarray(kw["qname_off"], dtype=np.uint64)
        self.qname = np.ascontiguousarray(kw["qname"], dtype=np.uint8)
        self.cigar_off = np.ascontiguousarray(kw["cigar_off"], dtype=np.uint64)
        self.cigar = np.ascontiguousarray(kw["cigar"], dtype=np.uint32)
        self.lseq = np.ascontiguousarray(kw["lseq"], dtype=np.int32)
        self.seq = np.ascontiguousarray(kw["seq"], dtype=np.uint8)
        self.qual = np.ascontiguousarray(kw["qual"], dtype=np.uint8)
        # presence bits of optional fields the path looks at (bit 0: the `sr` tag of `elprep split`, sam/split-merge.go:286-293)
        self.opt_flags = np.ascontiguousarray(kw["opt_flags"], dtype=np.uint8) if kw.get("opt_flags") is not None else np.zeros(n, dtype=np.uint8)
        assert self.qname_off.shape[0] == n + 1 and self.cigar_off.shape[0] == n + 1
        self._seq_off = None
        self._qual_off = None

    def __len__(self):
        return int(self.refid.shape[0])

    @property
    def n(self):
        return len(self)

    @property
    def qual_off(self):
        if self._qual_off is None:
            o = np.zeros(self.n + 1, dtype=np.uint64)
            np.cumsum(self.lseq.astype(np.uint64), out=o[1:])
            self._qual_off = o
        return self._qual_off

    @property
    def seq_off(self):
        if self._seq_off is None:
            o = np.zeros(self.n + 1, dtype=np.uint64)
            np.cumsum((self.lseq.astype(np.uint64) + 1) // 2, out=o[1:])
            self._seq_off = o
        return self._seq_off

    def copy(self):
        return AlignmentBatch(**{f: getattr(self, f).copy() for f in self.FIELDS})

    def qname_str(self, i):
        return bytes(self.qname[int(self.qname_off[i]):int(self.qname_off[i + 1])]).decode()

    def take(self, idx):
        """Gather records ``idx`` (any order) into a new batch."""
        idx = np.asarray(idx, dtype=np.int64)

        def ragged(off, data, scale=None):
            lens = (off[1:] - off[:-1]).astype(np.int64)[idx]
            no = np.zeros(len(idx) + 1, dtype=np.uint64)
            np.cumsum(lens, out=no[1:].view(np.int64))
            tot = int(no[-1])
            starts = off[:-1].astype(np.int64)[idx]
            src = np.repeat(starts - no[:-1].astype(np.int64), lens) + np.arange(tot, dtype=np.int64)
            return no, data[src]
        qo, qn = ragged(self.qname_off, self.qname)
        co, cg = ragged(self.cigar_off, self.cigar)
        _, sq = ragged(self.seq_off, self.seq)
        _, ql = ragged(self.qual_off, self.qual)
        return AlignmentBatch(refid=self.refid[idx], pos=self.pos[idx], flag=self.flag[idx], mapq=self.mapq[idx],
                              nref=self.nref[idx], pnext=self.pnext[idx], tlen=self.tlen[idx], rg=self.rg[idx],
                              qname_off=qo, qname=qn, cigar_off=co, cigar=cg, lseq=self.lseq[idx], seq=sq, qual=ql, opt_flags=self.opt_flags[idx])

    @staticmethod
    def concat(batches):
        def cat_off(name):
            offs, base = [np.zeros(1, dtype=np.uint64)], 0
            for b in batches:
                o = getattr(b, name)
                offs.append(o[1:] + np.uint64(base))
                base += int(o[-1])
            return np.concatenate(offs)
        kw = {f: np.concatenate([getattr(b, f) for b in batches]) for f in AlignmentBatch.FIELDS if not f.endswith("_off")}
        kw["qname_off"] = cat_off("qname_off")
        kw["cigar_off"] = cat_off("cigar_off")
        return AlignmentBatch(**kw)

    @staticmethod
    def from_records(header, recs):
        """Build a batch from dict records with SAM-like text fields:
        QNAME, FLAG, RNAME, POS, MAPQ, CIGAR, RNEXT, PNEXT, TLEN, SEQ, QUAL (list of ints or
        phred+33 string), RG (ID or None).  RNAME/RNEXT -> refid as AddREFID does."""
        ref = header.refid_table()
        rgidx = header.rg_index()
        n = len(recs)
        cols = {k: np.zeros(n, dtype=np.int32) for k in ("refid", "pos", "nref", "pnext", "tlen", "rg", "lseq")}
        flag = np.zeros(n, dtype=np.uint16)
        mapq = np.zeros(n, dtype=np.uint8)
        qoff, coff = [0], [0]
        qn, cg, sq, ql = bytearray(), [], bytearray(), bytearray()
        for i, r in enumerate(recs):
            rname = r.get("RNAME", "*")
            cols["refid"][i] = ref.get(rname, -1)
            rnext = r.get("RNEXT", "*")
            cols["nref"][i] = cols["refid"][i] if rnext == "=" else ref.get(rnext, -1)
            cols["pos"][i] = r.get("POS", 0)
            cols["pnext"][i] = r.get("PNEXT", 0)
            cols["tlen"][i] = r.get("TLEN", 0)
            flag[i] = r.get("FLAG", 0)
            mapq[i] = r.get("MAPQ", 0)
            g = r.get("RG")
            cols["rg"][i] = -1 if g is None else rgidx[g]
            qn += r.get("QNAME", "").encode()
            qoff.append(len(qn))
            cg += encode_cigar(r.get("CIGAR", "*"))
            coff.append(len(cg))
            s = r.get("SEQ", "")
            s = "" if s == "*" else s
            q = r.get("QUAL", [])
            if isinstance(q, str):
                q = [ord(c) - 33 for c in q]
            assert len(q) == len(s), "QUAL must have one byte per base"
            cols["lseq"][i] = len(s)
            sq += encode_seq(s)
            ql += bytes(q)
        return AlignmentBatch(flag=flag, mapq=mapq, qname_off=np.array(qoff, dtype=np.uint64),
                              qname=np.frombuffer(bytes(qn), dtype=np.uint8), cigar_off=np.array(coff, dtype=np.uint64),
                              cigar=np.array(cg, dtype=np.uint32), seq=np.frombuffer(bytes(sq), dtype=np.uint8),
                              qual=np.frombuffer(bytes(ql), dtype=np.uint8).copy(), **cols)


# unicode.IsSpace of Go: the Latin-1 spaces, then the White_Space property above U+00FF
_GO_SPACE = frozenset([0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000] + list(range(0x2000, 0x200B)))


def _go_rune(b, i):
    """utf8.DecodeRuneInString(b[i:]) -> (rune, width); an invalid byte is (U+FFFD, 1)"""
    c = b[i]
    if c < 0x80:
        return c, 1
    if 0xC2 <= c <= 0xDF:
        n, lo, hi = 1, 0x80, 0xBF
    elif 0xE0 <= c <= 0xEF:
        n, lo, hi = 2, (0xA0 if c == 0xE0 else 0x80), (0x9F if c == 0xED else 0xBF)
    elif 0xF0 <= c <= 0xF4:
        n, lo, hi = 3, (0x90 if c == 0xF0 else 0x80), (0x8F if c == 0xF4 else 0xBF)
    else:
        return 0xFFFD, 1
    if i + n >= len(b):
        return 0xFFFD, 1
    if not lo <= b[i + 1] <= hi or any(not 0x80 <= b[i + k] <= 0xBF for k in range(2, n + 1)):
        return 0xFFFD, 1
    r = c & (0x1F if n == 1 else (0x0F if n == 2 else 0x07))
    for k in range(1, n + 1):
        r = (r << 6) | (b[i + k] & 0x3F)
    return r, n + 1


def _go_fields(b):
    """strings.Fields: the runs of bytes between runs of unicode.IsSpace runes"""
    out, start, i = [], None, 0
    while i < len(b):
        r, w = _go_rune(b, i)
        if r in _GO_SPACE:
            if start is not None:
                out.append(b[start:i])
                start = None
        elif start is None:
            start = i
        i += w
    if start is not None:
        out.append(b[start:])
    return out


def ParseHeaderLineFromString(line):
    """sam.ParseHeaderLineFromString (sam/sam-files.go:153-177), the parser of `--replace-read-group`: TG:value fields separated by white
    space as strings.Fields splits them (unicode.IsSpace on the decoded runes; a byte that is not valid UTF-8 is no space).  line: str
    (its UTF-8 bytes, surrogate escapes as the bytes they stand for) or bytes -> dict of the same type.  ValueError where the reference
    panics: a field whose third byte is not ':' ("incorrectly formatted SAM file field"; also a field shorter than 3 bytes, a Go index
    panic there) and a repeated tag ("duplicate field tag")."""
    text = isinstance(line, str)
    b = line.encode("utf-8", "surrogateescape") if text else bytes(line)
    dec = (lambda x: x.decode("utf-8", "surrogateescape")) if text else (lambda x: x)
    txt = lambda x: x.decode("utf-8", "surrogateescape")                 # the message carries the field's bytes, as Go's %v of a string
    rec = {}
    for f in _go_fields(b):
        if len(f) < 3 or f[2] != 0x3A:
            raise ValueError(f"incorrectly formatted SAM file field {txt(f)}")
        tag, value = dec(f[:2]), dec(f[3:])
        if tag in rec:
            raise ValueError(f"duplicate field tag {txt(f[:2])} in a SAM header line")
        rec[tag] = value
    return rec


def _is_user_tag(code):
    """IsHeaderUserTag (sam/sam-types.go:49-56): a record type code with a lower-case letter"""
    return any("a" <= ch <= "z" for ch in code)


def _header_line(line):
    """parseSamHeaderLine (sam/sam-files.go:38-63): TG:value fields separated by tabs, no repeated TG"""
    rec, i = {}, 0
    while i < len(line):
        j = line.find(":", i)
        if j < 0 or j - i != 2:
            raise ValueError(f"invalid field tag {line[i:j if j >= 0 else len(line)]!r}")
        k = line.find("\t", j + 1)
        k = len(line) if k < 0 else k
        tag, value = line[i:j], line[j + 1:k]
        if tag in rec:
            raise ValueError(f"duplicate field tag {tag} in a SAM header line")
        rec[tag] = value
        i = k + 1
    return rec


def parse_sam_header(buf):
    """``ParseSamHeader`` (sam/sam-files.go:70-120) over the start of a SAM file -> (Header, n_header_bytes): the alignment lines
    (for ``Context.append_sam``) start at n_header_bytes.  @HD, @SQ and @RG are kept with all their fields; @PG, @CO and user
    records are checked and skipped.  ValueError where the reference panics: @HD not on the first line, an unknown record type
    code, a malformed field."""
    data = bytes(buf)
    h = Header()
    h.HD = {}
    pos, first = 0, True
    while pos < len(data) and data[pos:pos + 1] == b"@":
        nl = data.find(b"\n", pos)
        end = len(data) if nl < 0 else nl
        raw = data[pos:end].decode("latin-1")
        nxt = len(data) if nl < 0 else nl + 1
        if len(raw) < 4:                                  # (bytes[4:length] panics in the reference)
            raise ValueError(f"SAM header line too short: {raw!r}")
        code, line = raw[:4], raw[4:]
        if code == "@HD\t":
            if not first:
                raise ValueError("@HD line not in first line when parsing a SAM header")
            h.HD = _header_line(line)
        elif code == "@SQ\t":
            h.SQ.append(_header_line(line))
        elif code == "@RG\t":
            h.RG.append(_header_line(line))
        elif code == "@PG\t":
            _header_line(line)
        elif raw[:3] == "@CO":
            pass
        elif _is_user_tag(raw[:3]):
            if raw[3] != "\t":
                raise ValueError(f"header code {raw[:3]} not followed by a tab when parsing a SAM header")
            _header_line(line)
        else:
            raise ValueError(f"unknown SAM record type code {raw[:3]}")
        pos, first = nxt, False
    return h, pos


# ---- several input files: sam.MergeInputs (sam/merge-inputs.go:16-219) ----

MERGE_DICT_PANIC = "Cannot merge sequence dictionaries."


def _member(d, sn):
    """memberOfSequenceDictionary (merge-inputs.go:85-92): the first index whose SN is sn, or -1"""
    for i, sq in enumerate(d):
        if sq["SN"] == sn:
            return i
    return -1


def merge_sequence_dictionaries(to_dict, from_dict):
    """mergeSequenceDictionaries (merge-inputs.go:100-124) as written: order-preserving and recursive.  j is set from an index in
    from_dict after a recursive merge and from an index in the new dictionary after a shared entry, so a later from_dict[j:iFrom] can
    start behind its end; Go panics on that slice, and so does this.  ValueError where the reference panics."""
    new, j = [], 0
    for i_to, sq in enumerate(to_dict):
        sn = sq["SN"]
        i_from = _member(from_dict, sn)
        if i_from >= 0:
            i_new = _member(new, sn)
            if i_new >= 0:
                if i_new != i_to:
                    raise ValueError(MERGE_DICT_PANIC)
                j = i_new + 1
            else:
                if j > i_from:
                    raise ValueError(f"runtime error: slice bounds out of range [{j}:{i_from}]")
                new = merge_sequence_dictionaries(new, from_dict[j:i_from])
                new.append(sq)
                j = i_from + 1
        else:
            new.append(sq)
    new.extend(from_dict[j:])
    return new


def MergeInputs(headers, suffix):
    """sam.MergeInputs / mergeHeaders (sam/merge-inputs.go:16-219) over the parsed headers of the input files, in file order.  suffix
    stands for strconv.FormatInt(time.Now().Unix(), 10), the text a colliding @RG or @PG ID gets appended.  The inputs are not changed.

    Returns (merged, sq_maps, rg_map, pg_map):
      merged  the merged Header: the first header, then each later one merged into it (HD fields and user records overwritten, @SQ
              merged in order, @RG / @PG appended with colliding IDs renamed, comments appended, SO unknown after any merge);
      sq_maps per input, its @SQ index -> the index of that SN in the merged dictionary (first match, memberOfSequenceDictionary);
      rg_map / pg_map  the update filters replaceReadGroupIfExists / replaceProgramIDIfExists, which every record of every file runs in
              list order, composed into one map of old value -> final value (values it leaves alone are not in it).
    ValueError with the reference's text where it panics."""
    import copy
    merged, filters = None, []
    for h in headers:
        if merged is None:
            merged = copy.deepcopy(h)
            for a in ("PG", "CO"):
                setattr(merged, a, [copy.deepcopy(x) for x in getattr(h, a, [])])
            continue
        h = copy.deepcopy(h)
        merged.HD.update(h.HD)                                                     # mergeMetaData
        merged.SQ = merge_sequence_dictionaries(merged.SQ, h.SQ)
        ids = {r["ID"] for r in merged.RG}                                         # mergeReadGroups: the IDs before this file
        for r in h.RG:
            if r["ID"] in ids:
                old = r["ID"]
                r["ID"] = old + suffix
                filters.append(("RG", old, r["ID"]))
            merged.RG.append(r)
        pg_ids, replaced = {r["ID"] for r in merged.PG}, {}                        # mergeProgramLines
        for r in getattr(h, "PG", []):
            if r["ID"] in pg_ids:
                old = r["ID"]
                r["ID"] = old + suffix
                filters.append(("PG", old, r["ID"]))
                replaced[old] = r["ID"]
            merged.PG.append(r)
        for i in range(1, len(h.RG)):                                              # (the PP fix-up walks the RG lines, as written)
            rec = merged.RG[i]
            if "PP" in rec and rec["PP"] in replaced:
                rec["PP"] = replaced[rec["PP"]]
        merged.CO.extend(getattr(h, "CO", []))                                     # mergeCommentLines
        merged.UserRecords.update(getattr(h, "UserRecords", {}))                  # mergeUserRecords
        merged.SetHDSO(Unknown)
    if merged is None:
        raise ValueError("MergeInputs: no input headers")
    sq_maps = [[_member(merged.SQ, s["SN"]) for s in h.SQ] for h in headers]
    maps = {"RG": {}, "PG": {}}
    for tag in maps:
        for start in dict.fromkeys(old for t, old, _ in filters if t == tag):
            v = start
            for t, old, new in filters:
                if t == tag and v == old:
                    v = new
            if v != start:
                maps[tag][start] = v
    return merged, sq_maps, maps["RG"], maps["PG"]
