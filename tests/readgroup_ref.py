"""`--replace-read-group` restated from the reference for the tests: filters.AddOrReplaceReadGroup (filters/simple-filters.go:154-162) on BAM
record bytes.  aln.SetRG(id) is TAGS.Set(RG, id) (sam/sam-types.go:357-359), SmallMap.Set (utils/small-map.go:59-67): the first field whose
tag is RG gets the string value in place, whatever its type was; later RG fields stay; a record without one gets RG appended behind its last
field.  A Go string is written as RG Z id NUL in BAM.  The write-phase field filters (tests/outfilter.py) then run on the result, as
filters2 runs after filters1 (cmd/filter.go:742-776, 803-902).  The flag's string parser is sam.ParseHeaderLineFromString of the package."""
import struct

from outfilter import fields, filter_tags
from samformat import bam_to_sam


def set_rg_tags(rec, rg_id):
    """-> (start of the optional fields, [(tag, field bytes)]) of the record after SetRG(rg_id)"""
    r = bytes(rec)
    t0, fl = fields(r)
    tags = [(tag, r[s:e]) for tag, s, e in fl]
    new = b"RGZ" + bytes(rg_id) + b"\0"
    for j, (tag, _) in enumerate(tags):
        if tag == b"RG":
            tags[j] = (b"RG", new)
            break
    else:
        tags.append((b"RG", new))
    return t0, tags


def set_rg_record(rec, rg_id, remove=(), keep=None):
    """the BAM record as elp_fetch_bam writes it with the replacement on: SetRG, then the field filters, block_size rewritten"""
    r = bytes(rec)
    t0, tags = set_rg_tags(r, rg_id)
    body = r[4:t0] + b"".join(f for _, f in filter_tags(tags, remove, keep))
    return struct.pack("<I", len(body)) + body


def set_rg_sam(rec, rg_id, names, remove=(), keep=None, flag=None, qual=None):
    """the SAM line elp_fetch_sam writes for the stored record: FormatAlignment(parseBamAlignment) of set_rg_record"""
    return bam_to_sam(set_rg_record(rec, rg_id, remove, keep), names, flag=flag, qual=qual)
