"""Plain restatement of the --reference input, written from the reference's Go source:

  fasta.ParseFasta(path, nil, false, false)   fasta/fasta-files.go:159-229 (what `elprep fasta-to-elfasta` calls, cmd/convert.go:99)
  contigFromHeader                            fasta-files.go:75-89
  fasta.OpenElfasta                           fasta-files.go:286-336
  fasta.ToElfasta                             fasta-files.go:240-282 (the layout only, for fixtures)
  bufio.ScanLines / MaxScanTokenSize          a line ends at '\\n', one '\\r' before it is dropped, the last line may lack its '\\n'; a line
                                              of 65536 bytes or more stops the scanner (ErrTooLong), and the reference panics
  utils.HandleBGZF                            a first byte 0x1f is BGZF: BC subfield, CRC32, ISIZE, the EOF marker block at the end

Where Go slices one byte past a header without a name (b[len(b):len(b)+1], inside the scanner's buffer) the restatement takes the byte
that follows the token in the file: '\\r' when one was dropped, '\\n' otherwise, and 0 at the end of the file (Go reads a stale buffer
byte there).  Such a name is outside '!'..'~' and matches no @SQ SN.  Nothing here imports the CUDA library."""
from __future__ import annotations

import struct
import zlib

import numpy as np

MAX_TOKEN = 65536                              # bufio.MaxScanTokenSize
MAGIC = bytes([0x31, 0xFA, 0x57, 0xA1])        # fasta.ElfastaMagic
VARINT = 10                                    # binary.MaxVarintLen64
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")

# reasons, as elp_last_error words them
EMPTY_FILE, FIRST_HEADER, EMPTY_LINE, LONG = "empty fasta file", "missing first header", "empty line", "too long"
TABLE_END, NAME_END, OFFSET_END, SIZE_END = "offset table runs past", "name of an offset table entry", "offset field runs past", "size field runs past"
BAD_OFFSET, BAD_SIZE, RANGE = "while parsing offset", "while parsing size", "lies outside the file"


class FastaError(ValueError):
    def __init__(self, line, reason):
        super().__init__(f"line {line}: {reason}")
        self.line, self.reason = line, reason


class ElfastaError(ValueError):
    def __init__(self, offset, reason):
        super().__init__(f"byte offset {offset}: {reason}")
        self.offset, self.reason = offset, reason


class BgzfError(ValueError):
    pass


def scan_lines(data: bytes):
    """bufio.ScanLines -> [(raw length before '\\n', token, the byte after the token in the file or 0 at the end)]"""
    out, i = [], 0
    while i < len(data):
        j = data.find(b"\n", i)
        raw = data[i:] if j < 0 else data[i:j]
        i = len(data) if j < 0 else j + 1
        tok = raw[:-1] if raw.endswith(b"\r") else raw
        after = b"\r" if len(tok) < len(raw) else (b"\n" if j >= 0 else b"\x00")
        out.append((len(raw), tok, after))
    return out


def contig_from_header(b: bytes, after: bytes) -> bytes:
    """contigFromHeader: the first run of bytes in '!'..'~' after index 1; with none, the one byte past the token"""
    i = 1
    while i < len(b) and not 0x21 <= b[i] <= 0x7E:
        i += 1
    if i >= len(b):
        return after
    j = i + 1
    while j < len(b) and 0x21 <= b[j] <= 0x7E:
        j += 1
    return b[i:j]


def parse_fasta(data: bytes) -> dict:
    """ParseFasta(path, nil, false, false) -> {name: sequence bytes}; FastaError(1-based line, reason) where the reference panics"""
    lines = scan_lines(data)
    for k, (raw, _, _) in enumerate(lines):          # the scanner stops at a long line; every earlier line is checked first
        if raw >= MAX_TOKEN:
            lines, long_at = lines[:k], k + 1
            break
    else:
        long_at = None

    def stop(k):                                    # the scanner ran out of lines at index k (0-based)
        if long_at is not None:
            raise FastaError(long_at, LONG)

    k = 0
    while k < len(lines) and not lines[k][1]:         # :174-180
        k += 1
    if k == len(lines):
        stop(k)
        raise FastaError(len(lines) + 1, EMPTY_FILE)
    if lines[k][1][:1] != b">":                       # :181-183
        raise FastaError(k + 1, FIRST_HEADER)
    contig, seq, fasta = contig_from_header(lines[k][1], lines[k][2]), bytearray(), {}
    k += 1
    while k < len(lines):                           # scanLoop, :189-225
        b = lines[k][1]
        if not b:
            while k < len(lines) and not lines[k][1]:
                k += 1
            if k == len(lines):
                break
            b = lines[k][1]
            if b[:1] != b">":
                raise FastaError(k + 1, EMPTY_LINE)
        if b[:1] == b">":
            fasta[contig] = bytes(seq)
            contig, seq = contig_from_header(b, lines[k][2]), bytearray()
        else:
            seq += b
        k += 1
    stop(k)
    fasta[contig] = bytes(seq)
    return fasta


def uvarint(buf: bytes):
    """binary.Uvarint -> (value, n); n == 0: buffer too small, n < 0: overflow"""
    x, s = 0, 0
    for i, b in enumerate(buf):
        if i == VARINT:
            return 0, -(i + 1)
        if b < 0x80:
            if i == VARINT - 1 and b > 1:
                return 0, -(i + 1)
            return x | (b << s), i + 1
        x |= (b & 0x7F) << s
        s += 7
    return 0, 0


def varint(buf: bytes):
    """binary.Varint"""
    ux, n = uvarint(buf)
    x = ux >> 1
    if ux & 1:
        x = ~x
    return x, n


def put_varint(x: int) -> bytes:
    """binary.PutVarint"""
    ux = ((x << 1) ^ (x >> 63)) & ((1 << 64) - 1)
    out = bytearray()
    while ux >= 0x80:
        out.append((ux & 0x7F) | 0x80)
        ux >>= 7
    out.append(ux)
    return bytes(out)


def open_elfasta(data: bytes) -> dict:
    """OpenElfasta -> {name: sequence bytes}; ElfastaError(byte offset, reason) where Go panics (an index or slice out of range, or a
    Varint that returns n <= 0)"""
    if len(data) < len(MAGIC) or data[:4] != MAGIC:
        raise ElfastaError(0, "not an .elfasta file")
    out, i = {}, len(MAGIC)
    while True:
        if i >= len(data):
            raise ElfastaError(i, TABLE_END)
        if data[i] == 0x0A:
            return out
        start = i
        while True:
            if i >= len(data):
                raise ElfastaError(start, NAME_END)
            if data[i] == 0x09:
                break
            i += 1
        name = data[start:i]
        i += 1
        if i + VARINT > len(data):
            raise ElfastaError(i, OFFSET_END)
        off, n = varint(data[i:i + VARINT])
        if n <= 0:
            raise ElfastaError(i, BAD_OFFSET)
        if i + 2 * VARINT > len(data):
            raise ElfastaError(i + VARINT, SIZE_END)
        size, n = varint(data[i + VARINT:i + 2 * VARINT])
        if n <= 0:
            raise ElfastaError(i + VARINT, BAD_SIZE)
        hi = (off + size + (1 << 63)) % (1 << 64) - (1 << 63)   # Go's int arithmetic wraps
        if off < 0 or hi < off or hi > len(data):
            raise ElfastaError(i, RANGE)
        out[name] = data[off:hi]
        i += 2 * VARINT


def to_elfasta(fasta: dict, data_order=None) -> bytes:
    """ToElfasta's layout: the magic, per contig its name, '\\t' and two 10-byte fields (offset, size as PutVarint, zero padded), '\\n',
    then the sequences (in data_order, default the table order)"""
    names = list(fasta)
    data_order = names if data_order is None else list(data_order)
    table_len = len(MAGIC) + sum(len(n) + 1 + 2 * VARINT for n in names) + 1
    offs, at = {}, table_len
    for n in data_order:
        offs[n] = at
        at += len(fasta[n])
    out = bytearray(MAGIC)
    for n in names:
        out += n + b"\t" + put_varint(offs[n]).ljust(VARINT, b"\0") + put_varint(len(fasta[n])).ljust(VARINT, b"\0")
    out += b"\n"
    for n in data_order:
        out += fasta[n]
    return bytes(out)


def bgzf_blocks(data: bytes, level=6, block=0xFF00, eof=True) -> bytes:
    """data as BGZF blocks of `block` input bytes (raw DEFLATE at `level`), the EOF marker block behind when eof"""
    out = bytearray()
    for i in range(0, len(data), block):
        piece = data[i:i + block]
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        cdata = co.compress(piece) + co.flush()
        bsize = 18 + len(cdata) + 8
        out += struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 0xFF, 6, 66, 67, 2, bsize - 1) + cdata
        out += struct.pack("<II", zlib.crc32(piece), len(piece))
    if eof:
        out += EOF_BLOCK
    return bytes(out)


def inflate_bgzf(data: bytes) -> bytes:
    """utils.HandleBGZF's reader: BgzfError for a missing BC subfield (a plain gzip file), a bad CRC32 or ISIZE, a truncated block, or no
    EOF marker block at the end"""
    out, x, last = bytearray(), 0, None
    while x < len(data):
        h = data[x:x + 12]
        if len(h) < 12 or h[:4] != b"\x1f\x8b\x08\x04":
            raise BgzfError("bad gzip member header")
        xlen = struct.unpack("<H", h[10:12])[0]
        extra, bsize, i = data[x + 12:x + 12 + xlen], None, 0
        while i + 4 <= len(extra):
            slen = struct.unpack("<H", extra[i + 2:i + 4])[0]
            if extra[i:i + 2] == b"BC" and slen == 2:
                bsize = struct.unpack("<H", extra[i + 4:i + 6])[0] + 1
                break
            i += 4 + slen
        if bsize is None:
            raise BgzfError("missing BC extra subfield")
        if x + bsize > len(data) or bsize < 12 + xlen + 8:
            raise BgzfError("truncated block")
        cdata = data[x + 12 + xlen:x + bsize - 8]
        crc, isize = struct.unpack("<II", data[x + bsize - 8:x + bsize])
        piece = zlib.decompressobj(-15).decompress(cdata) if isize else b""
        if len(piece) != isize or zlib.crc32(piece) != crc:
            raise BgzfError("CRC32 or ISIZE mismatch")
        out += piece
        last = data[x:x + bsize]
        x += bsize
    if last != EOF_BLOCK:
        raise BgzfError("does not end in proper EOF marker")
    return bytes(out)


def read_reference(data: bytes) -> dict:
    """the format decided from the content, as elp_load_reference does it -> {name: sequence bytes}"""
    if data[:4] == MAGIC:
        return open_elfasta(data)
    if data[:1] == b"\x1f":
        return parse_fasta(inflate_bgzf(data))
    return parse_fasta(data)


def is_nameless(name: bytes) -> bool:
    return len(name) == 1 and not 0x21 <= name[0] <= 0x7E


def load(data: bytes, contig_names, elfasta=None):
    """elp_load_reference over file contents -> (per-contig sequence bytes or None, n_unmatched, n_missing).  A name Go read past a
    header without a name matches nothing."""
    fasta = read_reference(data)
    fa = not (elfasta if elfasta is not None else data[:4] == MAGIC)
    names = [n.encode() if isinstance(n, str) else n for n in contig_names]
    matchable = {k: v for k, v in fasta.items() if not (fa and is_nameless(k))}
    seqs = [matchable.get(n) for n in names]
    unmatched = sum(1 for k in fasta if k not in matchable or k not in names)
    return seqs, unmatched, sum(1 for s in seqs if s is None)


def hot_nibbles(seq: bytes) -> bytes:
    """elp_set_reference's packing: one-hot nibbles, low nibble first (A/a/* 1, C/c 2, G/g 4, T/t 8, anything else 0)"""
    code = np.zeros(256, np.uint8)
    for chars, v in ((b"Aa*", 1), (b"Cc", 2), (b"Gg", 4), (b"Tt", 8)):
        code[list(chars)] = v
    a = code[np.frombuffer(seq, np.uint8)]
    if len(a) % 2:
        a = np.concatenate([a, np.zeros(1, np.uint8)])
    return (a[0::2] | (a[1::2] << 4)).astype(np.uint8).tobytes()
