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
