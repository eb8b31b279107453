"""RemoveOptionalFields / KeepOptionalFields (filters/simple-filters.go:235-288) restated over BAM record bytes, for the write-phase filter
tests.  A record's optional fields are walked as parseBamAlignment reads them (sam/bam-files.go:369-397); each filter is SmallMap.DeleteIf
(utils/small-map.go:89-99) over the field list, with the interned-symbol comparison: the whole user string against the 2-byte tag."""
import struct

_SIZE = {ord("A"): 1, ord("c"): 1, ord("C"): 1, ord("s"): 2, ord("S"): 2, ord("i"): 4, ord("I"): 4, ord("f"): 4}
_ES = {ord("c"): 1, ord("C"): 1, ord("s"): 2, ord("S"): 2, ord("i"): 4, ord("I"): 4, ord("f"): 4}


def fields(rec):
    """-> (start of the optional fields, [(tag, start, end)] in record order) of a BAM record (block_size included)"""
    r = bytes(rec)
    l_name, ncig, lseq = r[12], struct.unpack_from("<H", r, 16)[0], struct.unpack_from("<i", r, 20)[0]
    t0 = 36 + l_name + 4 * ncig + (lseq + 1) // 2 + lseq
    out, t = [], t0
    while t < len(r):
        ty, v = r[t + 2], t + 3
        if ty in _SIZE:
            e = v + _SIZE[ty]
        elif ty in b"ZH":
            e = r.index(b"\0", v) + 1
        elif ty == ord("B"):
            e = v + 5 + _ES[r[v]] * struct.unpack_from("<I", r, v + 1)[0]
        else:
            raise ValueError(f"unknown BAM tag type {ty}")
        out.append((r[t:t + 2], t, e))
        t = e
    return t0, out


def _sym(s):
    return s.encode() if isinstance(s, str) else bytes(s)


def _delete_if(tags, test):
    return [x for x in tags if not test(x[0])]


def remove_optional_fields(tags, names):
    """RemoveOptionalFields(names) on a list whose items start with the tag; an empty list is no filter"""
    if not names:
        return tags
    syms = [_sym(s) for s in names]
    return _delete_if(tags, lambda k: any(s == k for s in syms))


def keep_optional_fields(tags, names):
    """KeepOptionalFields(names); an empty list drops every field (aln.TAGS = nil)"""
    if not names:
        return []
    syms = [_sym(s) for s in names]
    return _delete_if(tags, lambda k: not any(s == k for s in syms))


def filter_tags(tags, remove=(), keep=None):
    """the field filters in filters2 order: remove first, then keep (None: no keep filter)"""
    tags = remove_optional_fields(tags, list(remove))
    return tags if keep is None else keep_optional_fields(tags, list(keep))


def filter_record(rec, remove=(), keep=None):
    """the record with the fields the filters drop taken out, block_size rewritten, everything else byte for byte"""
    r = bytes(rec)
    t0, fl = fields(r)
    body = r[4:t0] + b"".join(r[s:e] for _, s, e in filter_tags(fl, remove, keep))
    return struct.pack("<I", len(body)) + body


def split_records(raw, off):
    return [bytes(raw[int(off[i]):int(off[i + 1])]) for i in range(len(off) - 1)]
