"""Host-side mirror of the reference's operator interface for the hot path (plumbing above the C ABI).

Same names, argument meaning and error behaviour as the Go API, so that the parity tests read like a port of
``cmd/filter.go:142-211``:

    reads = DeviceSam()
    md, fragments, pairs = filters.MarkDuplicates(False)
    InputBatches(header, batches).RunPipeline(reads, [filters.AddREFID, md], sam.Coordinate)   # phase 1
    recal = filters.NewBaseRecalibrator(known_sites, reference)
    tables = recal.Recalibrate(reads, 500)                                                       # phase 3
    tables.FinalizeBQSRTables(); tables.PrintBQSRTables("out.recal")                             # phase 4
    reads.RunPipeline(reads, [tables.ApplyBQSR(0, [], 500)], sam.Keep)                           # phase 5
    reads.RunPipeline(out, [], sam.Keep)                                                         # phase 6

With `--target-regions` (bedRegions) the reference filters the marked reads before the gather, in the full run
(runBestPracticesPipelineIntermediateSam, cmd/filter.go:171-180) and in the `--bqsr-tables-only` worker (:288-296) alike:

    InputBatches(header, batches).RunPipeline(reads, [filters.AddREFID, md], sam.Coordinate)   # phase 1: mark every read
    metrics = filters.MarkOpticalDuplicates(reads, pairs, 100)                                   # optical duplicates, on every read
    filters.FilterTargetRegions(reads, bedRegions)                                               # RemoveNonOverlappingReads on the device
    tables = recal.Recalibrate(reads, 500)                                                       # the gather sees the kept reads only
    tables.PrintBQSRTablesToIntermediateFile("w.elrecal")   # tables-only worker; the full run finalizes and applies as above

Differences forced by the columnar representation: an ``AlignmentFilter`` here receives a whole ``AlignmentBatch``
(the reference calls it once per ``*sam.Alignment``), and operators that run on the device (MarkDuplicates, ApplyBQSR)
return marker filters -- the work happens in the ``Finalize`` of ``DeviceSam.AddNodes`` / in ``DeviceSam.RunPipeline``,
exactly where the reference sorts (``sam/filter-pipeline.go:113-117``).  Failures the reference reports with
``log.Panic`` surface as ``device.ElprepError`` with the same text.
"""
from __future__ import annotations

import os

import numpy as np

from . import device, sam


# ---- sam.Filter / sam.AlignmentFilter (sam/filter-pipeline.go:33-41) -------------------------------------------------
# Filter:          callable(header) -> AlignmentFilter or None
# AlignmentFilter: callable(batch: AlignmentBatch) -> AlignmentBatch (records kept)

class _DeviceOp:
    """marker AlignmentFilter for an operator that runs on the device"""

    def __init__(self, kind, **kw):
        self.kind, self.kw = kind, kw

    def __call__(self, batch):
        return batch


def AddREFID(header):
    """filters.AddREFID (filters/simple-filters.go:208-231): the refid / nref columns of AlignmentBatch already are the
    REFID / NextREFID temps (AlignmentBatch.from_records resolves RNAME/RNEXT against @SQ the same way)."""
    return None


# ---- per-record filters of phase 1 (filters/simple-filters.go), as column predicates for the elp_append_batch path.
# With elp_append_bam the same predicates run fused into the device ingest (elp_set_ingest_filter). ----
def _keep(batch, mask):
    return batch if bool(mask.all()) else batch.take(np.nonzero(mask)[0])


def RemoveUnmappedReads(header):
    """filters.RemoveUnmappedReads (simple-filters.go:73-75)"""
    return lambda batch: _keep(batch, (batch.flag & sam.Unmapped) == 0)


def RemoveUnmappedReadsStrict(header):
    """filters.RemoveUnmappedReadsStrict (simple-filters.go:79-83): FLAG 0x4, POS 0 or RNAME *"""
    return lambda batch: _keep(batch, ((batch.flag & sam.Unmapped) == 0) & (batch.pos != 0) & (batch.refid >= 0))


def RemoveNonExactMappingReads(header):
    """filters.RemoveNonExactMappingReads (simple-filters.go:90-99): only M and S operations"""
    def flt(batch):
        op = batch.cigar & 15
        bad = ((op != 0) & (op != 4)).astype(np.int64)
        cs = np.concatenate([[0], np.cumsum(bad)])
        off = batch.cigar_off.astype(np.int64)
        return _keep(batch, (cs[off[1:]] - cs[off[:-1]]) == 0)
    return flt


def RemoveOptionalReads(header):
    """filters.RemoveOptionalReads (filters/simple-filters.go:142-150): drops the reads that carry the `sr` tag (opt_flags bit 0) -- the copies
    `elprep split` leaves in a group file for reads whose mate lies in another group; a no-op unless the header has the @sr user record"""
    if "@sr" not in getattr(header, "UserRecords", {}):
        return None
    header.UserRecords.pop("@sr")
    return lambda b: _keep(b, (b.opt_flags & 1) == 0)


def RemoveNonOverlappingReads(regions):
    """filters.RemoveNonOverlappingReads (filters/simple-filters.go:310-328) for the columnar path.  regions: per-contig (k,2) int32 arrays, the
    Start / End of the BED records; sorted by start and flattened here (ParallelSortByStart + ParallelFlatten).  Unmapped reads and reads without
    read bases use [POS, POS]; a contig without regions (or RNAME *) drops the read (intervals.Overlap of an empty slice)."""
    flat = []
    for iv in regions:
        iv = np.asarray(iv, dtype=np.int64).reshape(-1, 2)
        iv = iv[np.argsort(iv[:, 0], kind="stable")]
        out = []
        for s_, e_ in iv:
            if out and s_ <= out[-1][1]:
                out[-1][1] = max(out[-1][1], e_)
            else:
                out.append([int(s_), int(e_)])
        flat.append(np.array(out, dtype=np.int64).reshape(-1, 2))

    def overlap(iv, start, end):       # intervals.Overlap (intervals/intervals.go:146-164)
        left, right = 0, len(iv) - 1
        while left <= right:
            mid = (left + right) // 2
            if iv[mid][0] > end - 1:
                right = mid - 1
            elif iv[mid][1] <= start - 1:
                left = mid + 1
            else:
                return True
        return False

    def make(header):
        def flt(batch):
            keep = np.zeros(batch.n, bool)
            co = batch.cigar_off.astype(np.int64)
            for i in range(batch.n):
                pos = int(batch.pos[i]); end = pos
                if not (int(batch.flag[i]) & 0x4):
                    ops = batch.cigar[co[i]:co[i + 1]]
                    rl = sum(int(o >> 4) for o in ops if int(o & 15) in (0, 1, 4, 7, 8))
                    if rl > 0:
                        end = pos + sum(int(o >> 4) for o in ops if int(o & 15) in (0, 2, 3, 7, 8)) - 1
                r = int(batch.refid[i])
                keep[i] = 0 <= r < len(flat) and overlap(flat[r], pos, end)
            return _keep(batch, keep)
        flt.regions = flat          # DeviceSam.RunPipeline runs the filter on the device instead (elp_filter_target_regions)
        return flt
    return make


def FilterTargetRegions(reads, bedRegions):
    """The `--target-regions` phase, "Filtering out reads not in target regions." (cmd/filter.go:171-180, 288-296): after duplicate
    marking and the duplication metrics, before the gather, filteredReads.RunPipeline(filteredReads, [RemoveNonOverlappingReads(bedRegions)]).
    reads: a DeviceSam after phase 1; bedRegions: per-contig (k,2) Start / End arrays.  Returns the number of reads dropped."""
    return reads.RunPipeline(reads, [RemoveNonOverlappingReads(bedRegions)], sam.Keep)


def CleanSam(header):
    """filters.CleanSam (filters/simple-filters.go:292-306): runs on the device over everything appended (DeviceSam.AddNodes applies it after the
    last batch); MAPQ 0 for unmapped reads, CIGAR soft-clipped at the end of the contig (softClipEndOfRead, filters/utils.go:82-119)."""
    return _DeviceOp("clean_sam")


def RemoveMappingQualityLessThan(mq):
    """filters.RemoveMappingQualityLessThan (simple-filters.go:332-347) -> Filter: nil for 0, every read dropped above 255, else MAPQ
    compared against byte(mq) -- so -1 keeps MAPQ 255 only and -256 keeps every read (elp_set_ingest_filter applies the same rule)"""
    if mq == 0:
        return None
    if mq > 255:
        return lambda header: (lambda batch: _keep(batch, np.zeros(batch.n, bool)))
    mapq = int(mq) & 255
    return lambda header: (lambda batch: _keep(batch, batch.mapq.astype(np.int64) >= mapq))


def RemoveDuplicateReads(header):
    """filters.RemoveDuplicateReads (simple-filters.go:131-133)"""
    return lambda batch: _keep(batch, (batch.flag & sam.Duplicate) == 0)


def ClearDuplicateFlag(header):
    """filters.ClearDuplicateFlag (simple-filters.go:350-355): 0x400 cleared in every read, before marking.  With elp_append_bam /
    elp_append_sam the device does it at ingest (_lib.FILTER_CLEAR_DUPLICATE_FLAG)."""
    def flt(batch):
        batch.flag = (batch.flag & ~np.uint16(sam.Duplicate)).astype(np.uint16)
        return batch
    return flt


def AddOrReplaceReadGroup(readGroup):
    """filters.AddOrReplaceReadGroup (filters/simple-filters.go:154-162), `--replace-read-group`: readGroup is the flag's string parsed by
    sam.ParseHeaderLineFromString.  The Filter sets header.RG = [readGroup], so duplicate marking (LB) and BQSR (PU, else ID) read only
    that @RG; its AlignmentFilter puts every read of the batch in it (rg column 0, aln.SetRG(readGroup["ID"])).  It runs after the phase-1
    filters that drop reads and before MarkDuplicates, which then refuses an LB without ID with the reference's text.  On the byte paths
    the device does the same (Context.set_replace_read_group, with the context created from the header after this filter)."""
    def flt(header):
        header.RG = [dict(readGroup)]

        def set_rg(batch):
            batch.rg = np.zeros(batch.n, np.int32)
            return batch
        return set_rg
    return flt


def RenameChromosomes(header):
    """filters.RenameChromosomes (filters/simple-filters.go:189-204), `--rename-chromosomes`: every @SQ with an SN gets "chr" + SN.  The
    refid / nref columns index the dictionary, so the AlignmentFilter has nothing to change on the columnar path (the RNAME / RNEXT texts
    it prefixes exist only in the byte outputs).  On the byte paths the device does it (Context.set_input_dictionary with
    _lib.DICT_RENAME_CHROMOSOMES, the context created from the header after this filter)."""
    for e in header.SQ:
        if "SN" in e:
            e["SN"] = "chr" + e["SN"]
    return None


def _find_sn(sq, sn):
    """utils.Find (utils/utils.go:26-33) over a dictionary by SN: the first match, or -1"""
    for i, e in enumerate(sq):
        if e.get("SN", "") == sn:
            return i
    return -1


def dictionary_remap(old_names, new_names):
    """old @SQ index -> new @SQ index, as AddREFID reaches it after ReplaceReferenceSequenceDictionary: the last new entry with the old
    entry's name, or -1 (the read is dropped when it is its RNAME, and its RNEXT becomes -1).  The table elp_set_input_dictionary builds
    from the (renamed) input names and the replacement."""
    last = {}
    for j, n in enumerate(new_names):
        last[n] = j
    return np.array([last.get(n, -1) for n in old_names], dtype=np.int32).reshape(-1)


def ReplaceReferenceSequenceDictionary(dict_):
    """filters.ReplaceReferenceSequenceDictionary (filters/simple-filters.go:34-60), `--replace-reference-sequences`: dict_ is the new @SQ
    list.  With SO:coordinate the SO becomes unknown when the new entries found in the old dictionary (utils.Find: the first match) do
    not appear in increasing old position.  header.SQ becomes dict_; a read is kept iff its RNAME is "*" or an SN of dict_.  On the
    columnar path the AlignmentFilter remaps the refid / nref columns as AddREFID does after it (dictionary_remap) and drops the reads
    whose refid has no new entry.  On the byte paths the device does it (Context.set_input_dictionary with _lib.DICT_REPLACE)."""
    new = [dict(e) for e in dict_]

    def flt(header):
        if header.HD.get("SO") == sam.Coordinate:
            prev = -1
            for e in new:
                p = _find_sn(header.SQ, e.get("SN", ""))
                if p >= 0:
                    if p > prev:
                        prev = p
                    else:
                        header.SetHDSO(sam.Unknown)
                        break
        remap = dictionary_remap([e.get("SN", "") for e in header.SQ], [e.get("SN", "") for e in new])
        header.SQ = [dict(e) for e in new]

        tab = np.append(remap, -1).astype(np.int32)     # (refid -1 indexes the appended -1)

        def replace(batch):
            r = batch.refid.astype(np.int64)
            batch.refid, batch.nref = tab[r], tab[batch.nref.astype(np.int64)]
            return _keep(batch, (r < 0) | (batch.refid >= 0))
        return replace
    return flt


def ReplaceReferenceSequenceDictionaryFromSamFile(path):
    """filters.ReplaceReferenceSequenceDictionaryFromSamFile (filters/simple-filters.go:65-69): the @SQ lines of a SAM file or a .dict
    (a SAM header), parsed by sam.parse_sam_header, as the new dictionary"""
    with open(path, "rb") as f:
        header, _ = sam.parse_sam_header(f.read())
    return ReplaceReferenceSequenceDictionary(header.SQ)


def write_phase_filters(removeDuplicates=False, removeOptionalFields="", keepOptionalFields="", header_has_sr=False):
    """the write-phase flags of `elprep filter` as the arguments of Context.set_output_filter / elp_set_output_filter -> (mask, remove, keep),
    as cmd/filter.go:803-902 builds them: RemoveOptionalReads iff the header has @sr (the caller drops @sr from the header it writes);
    --remove-duplicates; --remove-optional-fields "all" is KeepOptionalFields(nil), else RemoveOptionalFields of the comma-split, trimmed list;
    --keep-optional-fields "none" is KeepOptionalFields(nil), else KeepOptionalFields of the list.  "all" / "none" are compared untrimmed, as
    there.  keep is None without a keep filter; mask carries _lib.OUT_KEEP_FIELDS when keep is a list.  Two keep filters in a row keep
    what both keep, so remove "all" with any keep list keeps nothing."""
    from . import _lib
    mask, remove, keep = 0, [], None
    if header_has_sr:
        mask |= _lib.OUT_REMOVE_OPTIONAL_READS
    if removeDuplicates:
        mask |= _lib.OUT_REMOVE_DUPLICATES
    if removeOptionalFields != "":
        if removeOptionalFields == "all":
            keep = []
        else:
            remove = [t.strip() for t in removeOptionalFields.split(",")]
    if keepOptionalFields != "":
        tags = [] if keepOptionalFields == "none" else [t.strip() for t in keepOptionalFields.split(",")]
        keep = tags if keep is None else [t for t in keep if t in tags]
    if keep is not None:
        mask |= _lib.OUT_KEEP_FIELDS
    return mask, remove, keep


def MarkDuplicates(alsoOpticals):
    """filters.MarkDuplicates (filters/mark-duplicates.go:406-445). Returns (filter, fragments, pairs); the two maps live on
    the device and are only handles here."""
    fragments, pairs = {"device": "fragments"}, {"device": "pairs"}

    def flt(header):
        for rg in header.RG:
            if "LB" in rg and "ID" not in rg:
                raise ValueError("Missing mandatory ID entry in an @RG line in a SAM file header.")   # :419
        return _DeviceOp("markdup", alsoOpticals=bool(alsoOpticals))
    return flt, fragments, pairs


def MarkOpticalDuplicates(reads, pairs, opticalPixelDistance):
    """filters.MarkOpticalDuplicates (filters/mark-optical-duplicates.go:468-517) -> map[library]*DuplicatesCtr.
    The counting ran on the device inside the Finalize of phase 1 (MarkDuplicates(True)); this returns its result."""
    if opticalPixelDistance != reads._opts["optical_pixel_distance"]:
        raise ValueError("opticalPixelDistance differs from the context's --optical-duplicates-pixel-distance")
    names = reads.ctx.optical_libraries()
    return dict(zip(names, reads.ctx.optical_metrics()))


def PrintDuplicatesMetrics(reads, metrics, commandLine, startedOn=""):
    """filters.PrintDuplicatesMetrics (filters/mark-optical-duplicates.go:601-699); libraries in ascending name order."""
    reads.ctx.print_duplicates_metrics(metrics, commandLine, startedOn)


def compose_filters(header, hdr_filters):
    """sam.ComposeFilters (sam/filter-pipeline.go:163-198): call each Filter with the header, keep the non-nil results."""
    out = []
    for f in hdr_filters or []:
        if f is not None:
            a = f(header)
            if a is not None:
                out.append(a)
    return out


def effective_sorting_order(sorting_order, header, original):
    """effectiveSortingOrder (sam/filter-pipeline.go:208-225)."""
    if sorting_order == sam.Keep:
        sorting_order = original
    current = header.HDSO()
    if sorting_order in (sam.Coordinate, sam.Queryname):
        if current == sorting_order:
            return sam.Keep
        header.SetHDSO(sorting_order)
    elif sorting_order in (sam.Unknown, sam.Unsorted):
        if current != sorting_order:
            header.SetHDSO(sorting_order)
    return sorting_order


class DeviceSam:
    """The device-resident analogue of ``*sam.Sam``: implements both PipelineOutput (AddNodes) and PipelineInput (RunPipeline)."""

    def __init__(self, device_ordinal=0, max_cycle=500, quantize_levels=0, sqq=None, prefix="GATK", profile=False, optical_pixel_distance=100):
        self.Header = None
        self.ctx = None
        self._opts = dict(device=device_ordinal, max_cycle=max_cycle, quantize_levels=quantize_levels, sqq=sqq, prefix=prefix, profile=profile,
                          optical_pixel_distance=optical_pixel_distance)
        self._markdup = False
        self._batches = []       # host copies in arrival order (the Go side keeps []*Alignment and gets indices back)

    # -- PipelineOutput.AddNodes (sam/filter-pipeline.go:108-128): receive batches, sort in the Finalize
    def AddNodes(self, header, sorting_order, batches, alignment_filters):
        self.Header = header
        self._markdup = any(isinstance(a, _DeviceOp) and a.kind == "markdup" for a in alignment_filters)
        host_filters = [a for a in alignment_filters if not isinstance(a, _DeviceOp)]
        self.ctx = device.Context(header, **self._opts)
        for b in batches:
            for a in host_filters:
                b = a(b)
            self._batches.append(b)
            self.ctx.append(b)
        if any(isinstance(a, _DeviceOp) and a.kind == "clean_sam" for a in alignment_filters):
            self.ctx.clean_sam()
        so = device.SO_COORDINATE if sorting_order == sam.Coordinate else (_lib_const("SO_QUERYNAME") if sorting_order == sam.Queryname else device.SO_KEEP)
        opticals = any(isinstance(a, _DeviceOp) and a.kind == "markdup" and a.kw["alsoOpticals"] for a in alignment_filters)
        self.ctx.sort_markdup(so, (2 if opticals else 1) if self._markdup else 0)           # the Finalize node

    # -- PipelineInput.RunPipeline (sam/filter-pipeline.go:242-279): the Sam is the source of a later phase
    def RunPipeline(self, output, hdr_filters, sorting_order):
        alns = compose_filters(self.Header, hdr_filters)
        removed = 0
        for a in alns:
            if isinstance(a, _DeviceOp) and a.kind == "apply":
                self.ctx.bqsr_apply()
            elif isinstance(a, _DeviceOp):
                raise ValueError(f"operator {a.kind} cannot run in this phase")
            elif getattr(a, "regions", None) is not None:        # RemoveNonOverlappingReads over the reads in output order
                for ci in range(len(self.Header.SQ)):
                    self.ctx.set_bqsr_target_regions(ci, a.regions[ci] if ci < len(a.regions) else np.zeros((0, 2), np.int32), already_flat=True)
                removed += self.ctx.filter_target_regions()
        if output is self:
            return removed
        idx, flag, qoff, qual = self.ctx.fetch()
        output.AddResult(self.Header, self._batches, idx, flag, qoff, qual)

    def NofBatches(self, n):
        pass


class InputBatches:
    """PipelineInput over in-memory batches (stands in for sam.InputFile.RunPipeline, sam/filter-pipeline.go:282-296)."""

    def __init__(self, header, batches):
        self.header, self.batches = header, list(batches)

    def RunPipeline(self, output, hdr_filters, sorting_order):
        original = self.header.HDSO()
        alns = compose_filters(self.header, hdr_filters)
        so = effective_sorting_order(sorting_order, self.header, original)
        output.AddNodes(self.header, so, self.batches, alns)


class HostResult:
    """PipelineOutput collecting the final records on the host (stands in for sam.OutputFile)."""

    def AddResult(self, header, batches, idx, flag, qoff, qual):
        self.Header, self.record_index, self.flag, self.qual_off, self.qual = header, idx, flag, qoff, qual
        self.arrival = sam.AlignmentBatch.concat(batches) if len(batches) > 1 else batches[0]


# ---- BQSR (filters/bqsr.go) ---------------------------------------------------------------------------------------------
class BaseRecalibrator:
    """filters.BaseRecalibrator (filters/bqsr.go:417-443): known sites + reference."""

    def __init__(self, known_sites, reference):
        self.known_sites, self.reference = known_sites, reference   # per contig: (k,2) int32 intervals, or .elsites / VCF paths; uint8 bases, or a path

    def _sites_are_files(self):
        ks = self.known_sites
        return bool(ks) and all(isinstance(p, (str, bytes, os.PathLike)) for p in ks)

    def Recalibrate(self, reads, maxCycle):
        """(*BaseRecalibrator).Recalibrate (filters/bqsr.go:467-551) -> *BaseRecalibratorTables"""
        ctx = reads.ctx
        if ctx.max_cycle != maxCycle:
            raise ValueError("maxCycle differs from the context's --max-cycle")
        files = self._sites_are_files()
        if files:
            ctx.load_known_sites(list(self.known_sites))
        ref_file = isinstance(self.reference, (str, bytes, os.PathLike))
        if ref_file:
            ctx.load_reference(self.reference)
        for ci in range(len(reads.Header.SQ)):
            if not ref_file:
                ctx.set_reference(ci, self.reference[ci])
            if not files:
                ctx.set_known_sites(ci, self.known_sites[ci] if self.known_sites else np.zeros((0, 2), np.int32), already_flat=False)
        ctx.bqsr_gather()
        return BaseRecalibratorTables(reads)


def NewBaseRecalibrator(knownSites, referenceFasta):
    """filters.NewBaseRecalibrator (filters/bqsr.go:424-443). knownSites: per-contig interval arrays (sorted+flattened
    inside, as intervals.ParallelSortByStart/ParallelFlatten do), or a list of .elsites or VCF (plain or BGZF) paths like the
    reference's []string (loaded on the device by Context.load_known_sites); referenceFasta: per-contig base arrays (fasta.Seq), or the path of an .elfasta or
    FASTA file (plain or BGZF) like the reference's --reference (loaded on the device by Context.load_reference)."""
    return BaseRecalibrator(knownSites, referenceFasta)


class BaseRecalibratorTables:
    """filters.BaseRecalibratorTables (filters/bqsr.go:445-459): the three integer tables, resident on the device."""

    def __init__(self, reads):
        self.reads = reads
        self._finalized = False

    def dense(self):
        return self.reads.ctx.tables_get()

    def merge(self, dense):
        """bqsrTable.merge (filters/bqsr.go:210-223) / LoadAndCombineBQSRTables (print-bqsr.go:310-329): add another table."""
        self.reads.ctx.tables_put(self.dense() + np.asarray(dense, dtype=np.int64))

    def PrintBQSRTablesToIntermediateFile(self, name):
        """filters/print-bqsr.go:300-308: the `--bqsr-tables-only` worker's output (cmd/filter.go:454, 955-983), gob of the three tables"""
        self.reads.ctx.write_elrecal(name)

    def FinalizeBQSRTables(self):
        """filters/bqsr.go:677-694"""
        self.reads.ctx.bqsr_finalize(None)
        self._finalized = True

    def PrintBQSRTables(self, name):
        """filters/print-bqsr.go:269-298"""
        self.reads.ctx.bqsr_finalize(name)
        self._finalized = True

    def ApplyBQSR(self, quantizeLevels, sqqList, maxCycle):
        """filters/bqsr.go:936-1006 -> sam.Filter"""
        ctx = self.reads.ctx
        if int(quantizeLevels) != ctx_quantize(ctx) or list(sqqList or []) != ctx_sqq(ctx) or maxCycle != ctx.max_cycle:
            raise ValueError("quantizeLevels / sqqList / maxCycle must equal the values the context was created with")

        def flt(header):
            if not self._finalized:
                self.FinalizeBQSRTables()
            return _DeviceOp("apply")
        return flt


def LoadAndCombineBQSRTables(reads, bqsrPath):
    """filters.LoadAndCombineBQSRTables (filters/print-bqsr.go:310-329): sums every .elrecal file of a directory (or the one file) into the
    tables of ``reads``' context -- the input of the `--bqsr-apply` worker (cmd/filter.go:455, 985-997), which then runs
    FinalizeBQSRTables + PrintBQSRTables(recal file) and the ApplyBQSR filter (runBestPracticesPipelineWithBQSRApplyOnly, cmd/filter.go:213-234)."""
    import os
    files = sorted(os.path.join(bqsrPath, f) for f in os.listdir(bqsrPath)) if os.path.isdir(bqsrPath) else [bqsrPath]
    reads.ctx.tables_clear()
    for f in files:
        reads.ctx.add_elrecal(f)
    return BaseRecalibratorTables(reads)


def PrintDuplicatesMetricsToIntermediateFile(reads, name):
    """filters/mark-optical-duplicates.go:701-709: the worker's counters as gob of map[string]*DuplicatesCtr"""
    reads.ctx.optical_write_gob(name)


def LoadAndCombineDuplicateMetrics(reads, metricsPath):
    """filters/mark-optical-duplicates.go:711-731: adds the counters of every file to the context's metrics (derived values are recomputed on read-out)"""
    import os
    files = sorted(os.path.join(metricsPath, f) for f in os.listdir(metricsPath)) if os.path.isdir(metricsPath) else [metricsPath]
    for f in files:
        reads.ctx.optical_add_gob(f)
    return dict(zip(reads.ctx.optical_libraries(), reads.ctx.optical_metrics()))


def _lib_const(name):
    from . import _lib
    return getattr(_lib, name)


def ctx_quantize(ctx):
    return int(ctx._keep_opts["quantize_levels"]) if hasattr(ctx, "_keep_opts") else 0


def ctx_sqq(ctx):
    v = ctx._keep_opts["sqq"] if hasattr(ctx, "_keep_opts") else None
    return list(v) if v is not None else []
