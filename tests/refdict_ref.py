"""`--rename-chromosomes` and `--replace-reference-sequences` restated from the reference for the tests, on BAM record bytes.

parseBamAlignment (sam/bam-files.go:317-400) turns refID / next_refID into the RNAME / RNEXT strings of the input dictionary; RNEXT is "="
when its name equals RNAME's.  RenameChromosomes (filters/simple-filters.go:189-204) prefixes "chr" to both unless they are "=" or "*".
ReplaceReferenceSequenceDictionary (:34-60) keeps a read iff its RNAME is "*" or an SN of the new dictionary.  AddREFID (:208-231) then
indexes RNAME / RNEXT in the output dictionary, the last of equal names winning and an absent name giving -1 ("=" takes RNAME's value),
and formatBamAlignment (sam/bam-files.go:635-690) writes those ids; every other byte of the record is as read.  SAM output
(FormatAlignment, sam/sam-files.go:563-598) prints the RNAME / RNEXT strings, so an RNEXT outside the new dictionary keeps its name.

Without REPLACE the ids are written as read: the output dictionary is the input's, renamed, so AddREFID reaches every record's own
entry (a duplicate @SQ name would send it to the last one; the device keeps the record's own index there, as with the setting off)."""
import struct

from samformat import bam_to_sam

RENAME, REPLACE = 1, 2


def renamed(names, mode):
    """the input @SQ names after RenameChromosomes (bytes)"""
    return [b"chr" + n for n in names] if mode & RENAME else list(names)


def _rnames(rec, names):
    refid, nref = struct.unpack_from("<i", rec, 4)[0], struct.unpack_from("<i", rec, 24)[0]
    rname = b"*" if refid < 0 else names[refid]
    if nref < 0:
        rnext = b"*"
    else:
        rnext = b"=" if names[nref] == rname else names[nref]
    return rname, rnext


def refdict_record(rec, in_names, mode, out_names):
    """the BAM record written for stored record rec (input refIDs) after the filters and AddREFID; None when REPLACE drops it.
    in_names: the input @SQ names as in the file; out_names: the output dictionary (the replacement under REPLACE)."""
    r = bytes(rec)
    names = renamed(in_names, mode)
    rname, rnext = _rnames(r, names)
    if mode & REPLACE:
        if rname != b"*" and rname not in set(out_names):
            return None
        table = {b"*": -1}
        for j, n in enumerate(out_names):
            table[n] = j
        ref = table.get(rname, -1)
        nxt = ref if rnext == b"=" else table.get(rnext, -1)
        r = r[:4] + struct.pack("<i", ref) + r[8:24] + struct.pack("<i", nxt) + r[28:]
    return r


def refdict_sam(rec, in_names, mode, out_names, flag=None, qual=None):
    """the SAM line written for stored record rec, or None when REPLACE drops it: the renamed input strings, whatever the new ids are"""
    if refdict_record(rec, in_names, mode, out_names) is None:
        return None
    return bam_to_sam(rec, renamed(in_names, mode), flag=flag, qual=qual)
