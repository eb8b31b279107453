/*
 * elprep_b200.h -- C ABI of the H100-native hot path of elPrep 5.1.3:
 * coordinate sort -> mark duplicates -> BQSR gather -> finalize -> apply.
 *
 * Plain C: pointers and sizes only, no CUDA/torch types.  Every entry point names the reference
 * interface it replaces (paths relative to the elPrep 5.1.3 tree).  All functions return 0 on success
 * and a negative ELP_E* code on failure; they never abort.  The message for the last failure is
 * available from elp_last_error() -- the reference panics with the same texts (log.Panic; see
 * INTEGRATION.md for the cgo shim that turns a non-zero return back into log.Panic).
 *
 * Ownership: the caller owns every host buffer; the library copies before returning (cgo pointer
 * rules).  Device memory is owned by the elp_ctx.  Thread-safety: elp_append_batch may be called
 * concurrently (pargo LimitedPar stages call filters from several goroutines,
 * sam/filter-pipeline.go:273,292); every other entry point expects a single caller.
 *
 * There is NO CPU fallback: elp_create fails with ELP_ENODEVICE when no CUDA device is usable.
 */
#ifndef ELPREP_B200_H
#define ELPREP_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ELP_OK 0
#define ELP_EINVAL (-1)      /* bad argument */
#define ELP_ENODEVICE (-2)   /* no usable CUDA device (the product never falls back to the CPU) */
#define ELP_ECUDA (-3)       /* CUDA runtime error, text in elp_last_error */
#define ELP_ENOMEM (-4)
#define ELP_EQUAL (-10)      /* "Invalid QUAL character" (filters/mark-duplicates.go:64-66) */
#define ELP_ENORG (-11)      /* "BQSR requires input with read groups" (filters/bqsr.go:38) */
#define ELP_ECYCLE (-12)     /* "cycle value exceeds maximum cycle value" (filters/bqsr.go:364-369) */
#define ELP_ECLIP (-13)      /* "reference coordinate matches a non-existing base in read" (filters/utils.go:250-265) */
#define ELP_EREFEND (-14)    /* eligible read runs past the end of its contig (Go: index out of range in computeSnpEvents) */
#define ELP_ELIMIT (-15)     /* an implementation limit was exceeded (text says which) */
#define ELP_ESTATE (-16)     /* entry point called in the wrong phase order */
#define ELP_ETILE (-17)      /* a QNAME tile/x/y field that strconv.ParseInt rejects (filters/mark-optical-duplicates.go:57-64) */
#define ELP_EBAM (-18)       /* malformed BAM alignment record, or an RG:Z value that is not an @RG ID */
#define ELP_EBGZF (-19)      /* malformed BGZF block (header, BC subfield, CRC32 or ISIZE), utils/bgzf/bgzf-files.go:95-127 */
#define ELP_ESAM (-20)       /* malformed SAM alignment line; elp_last_error names the line (0-based, within the call) and the field */
#define ELP_ESITES (-21)     /* malformed .elsites file; elp_last_error names the file (index in paths), the line (0-based, header = line 0) and the reason */
#define ELP_EFASTA (-22)     /* malformed reference file: elp_last_error names the file, the line (FASTA, 1-based) or byte offset (.elfasta), and the reason */
#define ELP_EVCF (-23)       /* malformed VCF known-sites file: elp_last_error names the file (index in paths), the line (1-based, header lines counted) and the reason */

/* sam.SortingOrder (sam/sam-types.go:40-58) */
#define ELP_SO_KEEP 0
#define ELP_SO_UNKNOWN 1
#define ELP_SO_UNSORTED 2
#define ELP_SO_QUERYNAME 3
#define ELP_SO_COORDINATE 4

typedef struct elp_ctx elp_ctx;

/* What the filters read from sam.Header: @SQ SN/LN (filters/simple-filters.go:208-214, filters/utils.go:130-138),
 * @RG ID/LB/PU (filters/mark-duplicates.go:413-423, filters/bqsr.go:35-51), plus the `elprep filter` flags of the
 * path (cmd/filter.go:435-481). */
typedef struct {
    int32_t device;                       /* CUDA device ordinal */
    int32_t n_contigs;
    const char *const *contig_names;      /* @SQ SN (only used for messages) */
    const int32_t *contig_lengths;        /* @SQ LN */
    int32_t n_read_groups;
    const char *const *rg_id;             /* @RG ID */
    const char *const *rg_lb;             /* @RG LB or NULL */
    const char *const *rg_pu;             /* @RG PU or NULL */
    int32_t max_cycle;                    /* --max-cycle, default 500 */
    int32_t quantize_levels;              /* --quantize-levels, default 0 */
    const uint8_t *sqq; int32_t n_sqq;    /* --sqq list, may be empty */
    const char *tablename_prefix;         /* --bqsr-tablename-prefix, default "GATK" */
    int32_t optical_pixel_distance;       /* --optical-duplicates-pixel-distance, default 100 */
    int32_t profile;                      /* 1: record a CUDA-event pair around every kernel launch (elp_kernel_stats) */
} elp_config;

/* One batch of sam.Alignment records in columnar form (sam/sam-types.go:289-331) -- what a
 * pipeline stage marshals from []*sam.Alignment (sam/filter-pipeline.go:92-104).
 * refid/nref are the REFID/NextREFID temps of filters.AddREFID (simple-filters.go:208-231), each in [-1, n_contigs): a batch
 * with any other value is refused with ELP_EINVAL and nothing of it is appended;
 * rg is the index of the read's RG:Z tag in elp_config.rg_id, -1 if the read has no RG tag.
 * cigar: BAM encoding len<<4|op, op indexes "MIDNSHP=X" (sam/bam-files.go). seq: BAM nibbles, high nibble
 * first, each read byte-aligned, reads packed back to back ((l_seq+1)/2 bytes each). qual: phred bytes
 * without +33, l_seq bytes per read, packed back to back. */
typedef struct {
    uint64_t n;
    const int32_t *refid; const int32_t *pos; const uint16_t *flag; const uint8_t *mapq;
    const int32_t *nref; const int32_t *pnext; const int32_t *tlen; const int32_t *rg;
    const uint64_t *qname_off; const uint8_t *qname;   /* qname_off[n+1], bytes without NUL */
    const uint64_t *cigar_off; const uint32_t *cigar;  /* cigar_off[n+1] */
    const int32_t *l_seq; const uint8_t *seq; const uint8_t *qual;
    const uint8_t *opt_flags;   /* may be NULL. Per read, presence bits of optional fields the path looks at: ELP_OPT_SR = the read carries the `sr`
                                 * tag `elprep split` puts on the group-file copy of a read whose mate lies in another group (sam/split-merge.go:286-293):
                                 * such a read is never recalibrated (recalibrateAln, filters/bqsr.go:225-229) and RemoveOptionalReads drops it at the end
                                 * (filters/simple-filters.go:142-150).  elp_append_bam sets the bit from the record's optional fields. */
} elp_batch;
#define ELP_OPT_SR 1u

/* per-kernel device timing (CUDA events on the launching stream), for bench.py's roofline object */
typedef struct {
    char name[48];
    uint64_t launches;
    double ms;            /* sum over launches */
    double alg_bytes;     /* sum over launches of the ALGORITHMIC bytes (DESIGN.md section "kernels") */
} elp_kernel_stat;

/* ---- lifecycle ---- */
int elp_create(const elp_config *cfg, elp_ctx **out);
void elp_destroy(elp_ctx *ctx);
const char *elp_last_error(const elp_ctx *ctx);          /* ctx may be NULL: error of the last failed elp_create */
/* tests: device and page-locked allocations that the library holds, over every context of the process (back to its earlier value
 * once every context created since has been destroyed) */
int64_t elp_debug_live_allocations(void);
/* optional capacity hint so that appends never reallocate */
int elp_reserve(elp_ctx *ctx, uint64_t n_reads, uint64_t n_bases, uint64_t n_cigar_ops, uint64_t n_qname_bytes);
/* forget all reads/tables but keep device allocations, reference and known sites (bench steps) */
int elp_reset(elp_ctx *ctx);

/* ---- side inputs: fasta.MappedFasta.Seq(contig) (fasta/fasta-files.go:355) and the known-sites intervals
 * of NewBaseRecalibrator (filters/bqsr.go:424-443). start/end pairs; flattened inside unless already_flat. ---- */
int elp_set_reference(elp_ctx *ctx, int32_t contig, const uint8_t *bases, uint64_t n);
int elp_set_known_sites(elp_ctx *ctx, int32_t contig, const int32_t *start_end_pairs, uint64_t n_intervals, int already_flat);
/* --known-sites a.elsites,b.vcf.gz (cmd/filter.go:459,530-538): NewBaseRecalibrator's loop over the files (filters/bqsr.go:424-443)
 * with intervals.FromElsitesFile (intervals/intervals.go:199-254), then ParallelSortByStart + ParallelFlatten per contig, all on the
 * device.  Replaces the known-sites list of EVERY contig (a contig without sites gets an empty list); n_paths == 0 clears them all.
 *  - Header: each file starts with exactly "# elsites format version 1.0\n" (ReadString('\n'), intervals.go:204-210); a "\r\n" header,
 *    a missing header and an empty file are ELP_ESITES at line 0.
 *  - Lines follow bufio.ScanLines: they end at '\n', one '\r' before it is dropped, the last line may lack its '\n'; an empty segment
 *    after the last '\n' is no line.  A line is CHROM '\t' START '\t' END (intervals.go:221-247): CHROM is everything before the first
 *    tab (empty, or no tab at all, is invalid, and so is a missing second tab; an empty line is invalid); START and END go through
 *    strconv.ParseInt(s, 10, 32) (an optional sign, decimal digits, inside int32; "+5", "-0" and "007" are accepted).  A line of 65536
 *    bytes or more (before its '\n') is ELP_ESITES: bufio.Scanner's default token limit stops the reference's scanner there (the pargo
 *    scanner is not part of the reference tree; this assumes it keeps bufio's default buffer).  Lines on unknown chromosomes are
 *    validated as well.  Any rejected line fails the whole call; the smallest (file, line) is reported.
 *  - CHROM resolves against elp_config.contig_names byte for byte; a context with @SQ lines created without names is ELP_EINVAL.  A line
 *    whose CHROM is "*" or no @SQ SN counts in *n_unmatched (may be NULL; the reference keeps such intervals but never looks them up).
 *    When several @SQ lines share one SN, each of those contigs gets the line's interval (the gather looks sites up by RNAME, bqsr.go:496).
 *  - Each contig's list equals what elp_set_known_sites(already_flat = 0) makes of the same intervals: a stable sort by start, then the
 *    serial Flatten (also where ParallelFlatten would panic, see DESIGN.md).
 *  - A missing or unreadable file is ELP_EINVAL (the message names the path); 2^30 or more intervals in total are ELP_ELIMIT.
 *  - Atomic: on any error the previous table is unchanged.  The table survives elp_reset; elp_set_known_sites afterwards replaces one
 *    contig's list, and the two calls mix in either order.
 *  - VCF files: the format of each file comes from its content.  The exact .elsites header is an .elsites file; a first byte 0x1f is a
 *    BGZF VCF (vcf.Open, vcf/vcf-files.go:1285-1312; the BGZF rules of elp_append_bgzf apply, a plain gzip file is ELP_EBGZF); text that
 *    starts with "##fileformat=VCFv4." is a plain VCF; anything else is ELP_ESITES at line 0.  A list may mix both kinds.  A VCF gives
 *    the table that `elprep vcf-to-elsites` on it, followed by loading the .elsites it writes in the same position of the list, gives:
 *    intervals.FromVcfFile (intervals/intervals.go:306-338) with ParseHeader, NewVariantParser and ParseVariant(NSamples = 0)
 *    (vcf-files.go:73-305,600-782).  The header: the first line starts with "##fileformat=VCFv4."; "##key=value" lines follow (a line
 *    without '=', a second fileformat, and every panic of ParseFormatInformation / ParseMetaInformation are refused; an INFO Flag with
 *    Number != 0 and any FORMAT Flag are refused even when unused); then one '#' column line.  Data lines split as .elsites lines do
 *    (65536 bytes or more is refused).  CHROM, POS, REF, QUAL and FILTER must be followed by a tab unless missing ('.' at the end of
 *    the line or before a tab, or the line already ended); ID and ALT are lists followed by a tab; POS is strconv.ParseInt(s, 10, 32)
 *    (-1 when missing); QUAL must pass strconv.ParseFloat(s, 64), overflow to +-Inf included; FILTER "PASS;..." is refused.  INFO keys
 *    run up to ' ', ':' or a tab; a key equal to a declared ID goes through that ID's parser (Integer and Float always fail there), and
 *    a key equal to END refuses the line.  Everything after INFO is ignored.  The interval is [POS, POS - 1 + len(REF)] in wrapping
 *    int32; a missing REF counts as "."; an empty CHROM is refused.  *n_unmatched counts VCF data lines on no @SQ SN.  A refusal is
 *    ELP_EVCF naming the file, the 1-based line (header lines counted) and the reason; the smallest (file, line) is reported. */
int elp_load_known_sites(elp_ctx *ctx, const char *const *paths, int32_t n_paths, uint64_t *n_unmatched);
/* one contig's known sites as the gather uses them: writes up to cap (start, end) pairs and returns the number of pairs (-1 on error);
 * start_end_pairs may be NULL to ask for the count */
int64_t elp_known_sites_get(elp_ctx *ctx, int32_t contig, int32_t *start_end_pairs, uint64_t cap);
/* tests: bytes of the page-locked staging chunks the files are streamed through (0: the default, 32 MiB) */
int elp_debug_set_sites_chunk(elp_ctx *ctx, uint64_t bytes);
/* --reference (cmd/filter.go): the one-hot reference of EVERY contig from one file, read and packed on the device.  The format is decided
 * from the content: the first four bytes 31 FA 57 A1 (ElfastaMagic) make an .elfasta (fasta.OpenElfasta, fasta/fasta-files.go:286-336);
 * a first byte 0x1f makes a BGZF-compressed FASTA, anything else is FASTA text (fasta.ParseFasta(path, nil, false, false) as
 * `elprep fasta-to-elfasta` calls it, fasta-files.go:159-229).
 *  - Contig k afterwards holds what elp_set_reference(k, Seq(SN_k)) gives.  When several @SQ lines share an SN, each gets the sequence.
 *    A contig whose SN has no sequence in the file has none, like a contig never set: a recalibrated read on it is ELP_EREFEND.
 *  - FASTA: lines as bufio.ScanLines splits them (a line of 65536 bytes or more is refused); empty lines before the first header are
 *    skipped and the first other line must start with '>'; after empty lines only a header or the end of the file may follow; a header's
 *    name is its first run of bytes in '!'..'~' after the '>' (contigFromHeader); every other line is appended verbatim; the last of equal
 *    names wins.  An empty file, or one of empty lines only, is refused.  Refusals are ELP_EFASTA naming the 1-based line.
 *  - BGZF: the rules of elp_append_bgzf / elp_append_bgzf_end (BC subfield, CRC32, ISIZE, the EOF marker block at the end); a violation
 *    is ELP_EBGZF naming the file offset; a plain (non-BGZF) gzip file is refused there.
 *  - .elfasta: the offset table (name '\t' then two binary.Varint fields of 10 bytes: offset and size) up to an entry that starts with
 *    '\n'; the last of equal names wins; a table that runs past the end of the file, a field binary.Varint rejects, or a sequence outside
 *    the file is ELP_EFASTA naming the byte offset.  Only the sequences of names that are an @SQ SN are read.
 *  - *n_unmatched (may be NULL): the file's sequences whose name is no SN; *n_missing (may be NULL): the contigs left without a sequence.
 *  - A context with @SQ lines created without names is ELP_EINVAL; so is a missing or unreadable file (the message names the path).
 *  - Atomic: on any error the previous references are unchanged.  They survive elp_reset; elp_set_reference afterwards replaces one
 *    contig, and the two calls mix in either order. */
int elp_load_reference(elp_ctx *ctx, const char *path, uint64_t *n_unmatched, int32_t *n_missing);
/* one contig's reference as the gather reads it: returns its length in bases (-1 on error) and copies its (len + 1) / 2 one-hot nibble
 * bytes (low nibble first: A 1, C 2, G 4, T 8, anything else 0) when nibbles is not NULL and cap allows */
int64_t elp_reference_get(elp_ctx *ctx, int32_t contig, uint8_t *nibbles, uint64_t cap);
/* tests: bytes of the page-locked staging chunks the reference file is streamed through (0: the default, 32 MiB) */
int elp_debug_set_reference_chunk(elp_ctx *ctx, uint64_t bytes);

/* ---- phase 1: (*sam.Sam).AddNodes receiving batches (sam/filter-pipeline.go:108-128) ---- */
int elp_append_batch(elp_ctx *ctx, const elp_batch *batch);
/* Asynchronous form for pipelined callers (one context uploads while another computes and downloads): the copies are queued on the
 * context's ingest stream and the call returns; the caller's buffers -- page-locked, or the copies serialise -- must stay valid and
 * unchanged until elp_append_wait returns.  Every later phase call of the same context orders itself behind the upload. */
int elp_append_batch_async(elp_ctx *ctx, const elp_batch *batch);
int elp_append_wait(elp_ctx *ctx);
/* The same, straight from decompressed BAM alignment records (SURVEY.md 8f row 1): what parseBamAlignment reads on the host
 * (sam/bam-files.go:314-400) is parsed on the device instead, so a Go caller hands over the bytes of a BGZF block without
 * building []*sam.Alignment first.  records: n_bytes of consecutive records, each starting with its 4-byte block_size;
 * record_off[n_records + 1]: byte offset of every record (record_off[n_records] == n_bytes), or NULL to let the library
 * walk the block_size chain.  refID / next_refID index @SQ directly (they ARE the REFID temps); POS and PNEXT become
 * 1-based; the RG:Z tag is matched against elp_config.rg_id (an unknown value is ELP_EBAM, no RG tag is rg = -1).
 * Not supported: the CG:B long-CIGAR convention (ELP_ELIMIT).  Thread-safe like elp_append_batch. */
int elp_append_bam(elp_ctx *ctx, const uint8_t *records, uint64_t n_bytes, const uint64_t *record_off, uint64_t n_records);
/* SAM text alignment lines (no header), whole lines only; the last line may lack its '\n'; a '\r' before '\n' is dropped.
 * Parsed on the device as parseSamAlignment (sam/sam-files.go:386-410) and stored as the record formatBamAlignment
 * (sam/bam-files.go:635-737) writes for it, then ingested as by elp_append_bam (filters, RG:Z, sr, elp_fetch_bam).
 * RNAME/RNEXT are resolved against elp_config.contig_names as AddREFID does (filters/simple-filters.go:208-231), so a context
 * with @SQ lines must have been created with contig_names (else ELP_EINVAL).  Thread-safe like elp_append_bam.
 * On any error nothing of the call is appended: ELP_ESAM for a line the reference rejects (log.Panic) and for three lines it would
 * write as a malformed BAM record -- a QNAME longer than 254 bytes, a merged CIGAR operation of 2^28 or more, QUAL and SEQ of
 * different lengths; ELP_ESAM as well for a hexadecimal float, a tab as the value of an A field and a tag name that contains a tab
 * (the reference accepts these three); ELP_ELIMIT for a CIGAR of more than 65535 operations (the CG:B convention); ELP_EBAM for an
 * RG:Z value that is not an @RG ID. */
int elp_append_sam(elp_ctx *ctx, const char *text, uint64_t n_bytes);
/* Per-record filters fused into elp_append_bam (SURVEY.md 8f row 4): a record that fails a requested predicate never becomes a read
 * of the context (later calls; elp_n_filtered counts them).  filters/simple-filters.go: RemoveUnmappedReads (:73-75),
 * RemoveUnmappedReadsStrict (:79-83: FLAG 0x4, POS 0 or RNAME *), RemoveNonExactMappingReads (:90-99: only M and S operations),
 * RemoveMappingQualityLessThan (:332-347, min_mapq as the reference's `mq int`: 0 keeps every read, more than 255 drops every read,
 * anything else keeps MAPQ >= (min_mapq & 255), so -1 keeps MAPQ 255 only and -256 keeps every read), RemoveDuplicateReads (:131-133, on
 * the FLAG the record comes in with).  Every record of a call is checked for structure whether a filter drops it or not: a malformed
 * record fails the call (ELP_EBAM) with any filter mask, as the reference parses a record before any filter sees it.  The two
 * well-formed records the device cannot hold -- an RG:Z value that is not an @RG ID, the CG:B long-CIGAR convention -- are refused
 * only when they pass the filters; a record a filter drops never needs them, so the call gives the reference's result.  With
 * elp_append_batch the caller's marshaller applies its filters to the []*Alignment before building columns. */
#define ELP_FILTER_UNMAPPED 1u
#define ELP_FILTER_UNMAPPED_STRICT 2u
#define ELP_FILTER_NON_EXACT 4u
#define ELP_FILTER_DUPLICATES 8u
#define ELP_FILTER_NON_EXACT_STRICT 16u   /* RemoveNonExactMappingReadsStrict (:115-136): optional fields X0 = 1, X1 = XM = XO = XG = 0 must all be present */
#define ELP_FILTER_TARGET_REGIONS 32u     /* RemoveNonOverlappingReads (:310-328): keep reads whose [POS, End()] overlaps a region of elp_set_target_regions.
                                           * This is `--filter-non-overlapping-reads` (a phase-1 filter, before duplicate marking).  `--target-regions`
                                           * filters after marking instead: elp_set_bqsr_target_regions + elp_filter_target_regions. */
#define ELP_FILTER_CLEAR_DUPLICATE_FLAG 64u   /* ClearDuplicateFlag (:350-355): 0x400 cleared in the FLAG column at ingest, before marking; drops no record.
                                               * ELP_FILTER_DUPLICATES still tests the FLAG the record comes in with.  With elp_append_batch the
                                               * marshaller clears the bit in the batch's FLAG column (filters.ClearDuplicateFlag), as for the other filters. */
/* regions of one contig as (start, end) pairs, the Start / End of the BED records as the reference's bed parser stores them; sorted by
 * start and flattened inside unless already_flat (intervals.FromBed + ParallelSortByStart + ParallelFlatten, filters/simple-filters.go:311-315) */
int elp_set_target_regions(elp_ctx *ctx, int32_t contig, const int32_t *start_end_pairs, uint64_t n_intervals, int already_flat);
int elp_set_ingest_filter(elp_ctx *ctx, uint32_t mask, int32_t min_mapq);
uint64_t elp_n_filtered(const elp_ctx *ctx);
uint64_t elp_n_reads(const elp_ctx *ctx);
/* filters.CleanSam (filters/simple-filters.go:292-306, softClipEndOfRead filters/utils.go:82-119) over the reads appended so far (either ingest
 * path; call before elp_sort_markdup): MAPQ of unmapped reads becomes 0; a read that runs past the end of its contig gets its CIGAR soft-clipped
 * there.  Returns the number of rewritten CIGARs in *n_rewritten (may be NULL).  The new MAPQ reaches both byte outputs (elp_fetch_bam and
 * elp_fetch_sam write the MAPQ column); only a CIGAR rewrite makes them refuse (the stored records still carry the old CIGAR); the columnar
 * elp_fetch is unaffected. */
int elp_clean_sam(elp_ctx *ctx, uint64_t *n_rewritten);

/* filters.MarkDuplicates (filters/mark-duplicates.go:406-445) + By(CoordinateLess).ParallelStableSort in the
 * Finalize of (*sam.Sam).AddNodes (sam/filter-pipeline.go:113-117, sam/sam-types.go:425-473,639-641).
 * sorting_order: ELP_SO_COORDINATE sorts by CoordinateLess; ELP_SO_QUERYNAME by QNAMELess (sam-types.go:479-481, stable);
 * KEEP/UNKNOWN/UNSORTED leave arrival order.
 * mark_duplicates: 0 none, ELP_MARKDUP = MarkDuplicates(false), ELP_MARKDUP_OPTICAL = MarkDuplicates(true) followed by
 * filters.MarkOpticalDuplicates(reads, pairs, optical_pixel_distance) (filters/mark-optical-duplicates.go:468-517,
 * cmd/filter.go:782) -- the metrics are read with the elp_optical_* calls below. */
#define ELP_MARKDUP 1
#define ELP_MARKDUP_OPTICAL 2
int elp_sort_markdup(elp_ctx *ctx, int sorting_order, int mark_duplicates);

/* ---- phase 2: duplication metrics, map[string]*DuplicatesCtr (filters/mark-optical-duplicates.go:95-110).
 * Libraries are addressed by slot: 0 = "Unknown Library" (reads without LB), 1.. = distinct @RG LB values in header order. */
typedef struct {
    int64_t unpaired_reads_examined, read_pairs_examined, secondary_or_supplementary_reads, unmapped_reads,
            unpaired_read_duplicates, read_pair_duplicates, read_pair_optical_duplicates;
    int64_t estimated_library_size;       /* estimateLibrarySize (:533-562); 0 unless read_pairs_examined > 0 */
    double percent_duplication;           /* NaN when nothing was examined, as in the reference (:524) */
    double roi[100]; int32_t has_roi;     /* histogramRoi (:574-581) */
    int64_t paired_reads_examined;        /* reads behind read_pairs_examined (= 2x + an unmatched mate, :488,503-505) */
} elp_dup_metrics;
int32_t elp_optical_n_libraries(const elp_ctx *ctx);                    /* number of slots */
const char *elp_optical_library_name(const elp_ctx *ctx, int32_t slot);
int elp_optical_metrics(elp_ctx *ctx, int32_t slot, elp_dup_metrics *out);
/* which: 0 duplicatesCountHistogram, 1 nonOpticalDuplicatesCountHistogram, 2 opticalDuplicatesCountHistogram;
 * writes up to cap (key, count) pairs in ascending key order, returns the number of entries (-1 on error) */
int64_t elp_optical_histogram(elp_ctx *ctx, int32_t slot, int32_t which, int64_t *keys, int64_t *counts, int64_t cap);
/* mergeDuplicatesCtrMaps / LoadAndCombineDuplicateMetrics (:451-466, :711-731): add another worker's counters (7 values in
 * the order of elp_dup_metrics, but counters7[1] = that worker's paired_reads_examined so that the halving happens once,
 * after the sum; may be NULL) and/or one of its histograms; derived metrics are recomputed on the next read-out */
int elp_optical_merge(elp_ctx *ctx, int32_t slot, const int64_t *counters7, int32_t which, const int64_t *keys, const int64_t *counts, int64_t n);
/* PrintDuplicatesMetrics (:601-699). The reference prints libraries in Go map order; here ascending by name.
 * started_on replaces time.Now().Format(...) so that the output is reproducible. */
int elp_print_duplicates_metrics(elp_ctx *ctx, const char *path, const char *command_line, const char *started_on);

/* ---- between phases 2 and 3: `--target-regions` (runBestPracticesPipelineIntermediateSam, cmd/filter.go:171-180, and the tables-only
 * worker, :288-296): RemoveNonOverlappingReads(bedRegions) (filters/simple-filters.go:308-328) over the reads in output order, after
 * duplicate marking and the duplication metrics, before the BQSR gather.  Its regions are a table of their own, so that
 * `--filter-non-overlapping-reads A.bed --target-regions B.bed` works in one context.
 *  - elp_set_bqsr_target_regions: one contig's regions, with the conventions of elp_set_target_regions (BED Start / End as the reference's
 *    parser stores them; sorted by start and flattened inside unless already_flat).  The regions survive elp_reset.
 *  - elp_filter_target_regions: keeps output record k iff intervals.Overlap(regions[RNAME], POS, alnEnd), alnEnd = End() for a mapped read
 *    whose CIGAR has read bases and POS otherwise, on the CIGAR the context holds now (after elp_clean_sam).  RNAME * and contigs without
 *    regions never overlap; without any regions every read is dropped (an empty BED file).  The kept records keep their relative order and
 *    their FLAG, whether or not their mates were dropped; duplication metrics already computed are unchanged.  *n_removed (may be NULL):
 *    the records dropped by this call.  ELP_ESTATE before elp_sort_markdup and after elp_bqsr_gather, elp_bqsr_tables_put or elp_bqsr_apply;
 *    a second call drops what the regions set then drop.  Later phases see only the kept records: the BQSR gather and apply, and every fetch.
 *  - elp_n_sorted: the records in output order -- elp_n_reads until elp_filter_target_regions drops some, the kept count afterwards.
 *    elp_fetch, elp_fetch_async, elp_fetch_qual_bytes, elp_fetch_opt_flags, elp_fetch_bam(_bytes) and elp_fetch_sam(_bytes) index
 *    [0, elp_n_sorted) (through the record filters of elp_set_output_filter for the byte outputs); elp_n_reads stays the number of reads
 *    the context holds. ---- */
int elp_set_bqsr_target_regions(elp_ctx *ctx, int32_t contig, const int32_t *start_end_pairs, uint64_t n_intervals, int already_flat);
int elp_filter_target_regions(elp_ctx *ctx, uint64_t *n_removed);
uint64_t elp_n_sorted(const elp_ctx *ctx);

/* ---- phase 3: (*BaseRecalibrator).Recalibrate (filters/bqsr.go:467-551) ---- */
int elp_bqsr_gather(elp_ctx *ctx);
/* dense integer tables: [n_cov][94][1 + (2*max_cycle+1) + 16][2] int64 = (observations, mismatches);
 * column 0 = QualityScores, then Cycles (index cycle+max_cycle), then Contexts (index key>>4).
 * get/put replace the gob .elrecal exchange of filters/print-bqsr.go:300-329; the device pointer is what a
 * host layer hands to ncclAllReduce(sum, int64) in place of LoadAndCombineBQSRTables' summation. */
uint64_t elp_bqsr_tables_len(const elp_ctx *ctx);        /* number of int64 values */
int32_t elp_bqsr_n_cov(const elp_ctx *ctx);
const char *elp_bqsr_cov_name(const elp_ctx *ctx, int32_t cov);
int elp_bqsr_tables_get(elp_ctx *ctx, int64_t *dense, uint64_t n);
int elp_bqsr_tables_put(elp_ctx *ctx, const int64_t *dense, uint64_t n);
int elp_bqsr_tables_device(elp_ctx *ctx, void **device_ptr, uint64_t *n);

/* The same exchange as Go encoding/gob files, for a GPU worker inside an `elprep sfm` run (cmd/filter.go:454-455, 955-997):
 *   --bqsr-tables-only f :  elp_bqsr_gather, then elp_bqsr_tables_write_elrecal(f)     (PrintBQSRTablesToIntermediateFile, filters/print-bqsr.go:300-308)
 *   --bqsr-apply dir     :  elp_bqsr_tables_clear, elp_bqsr_tables_add_elrecal(each file of dir) (LoadAndCombineBQSRTables, :310-329),
 *                           then elp_bqsr_finalize(recal file) and elp_bqsr_apply       (runBestPracticesPipelineWithBQSRApplyOnly, cmd/filter.go:213-234)
 * The stream is gob of filters.BaseRecalibratorTables{QualityScores, Cycles, Contexts map[bqsrTableKey{Qual,Covariate,ReadGroup}]*bqsrEntry};
 * written per the encoding/gob specification, not checked against a Go binary (none in this image). */
int elp_bqsr_tables_clear(elp_ctx *ctx);
int elp_bqsr_tables_write_elrecal(elp_ctx *ctx, const char *path);
int elp_bqsr_tables_add_elrecal(elp_ctx *ctx, const char *path);
/* duplication metrics of a worker as gob of map[string]*DuplicatesCtr (the seven exported counters;
 * PrintDuplicatesMetricsToIntermediateFile / LoadAndCombineDuplicateMetrics, filters/mark-optical-duplicates.go:701-731) */
int elp_optical_write_gob(elp_ctx *ctx, const char *path);
int elp_optical_add_gob(elp_ctx *ctx, const char *path);

/* ---- several GPUs of one box (SURVEY.md 8e): one context per GPU (one process or thread each), reads partitioned by contig group the way
 * `elprep sfm` splits its input (computeContigGroups, sam/split-merge.go:178-213; cmd/sfm.go:605-805).  NCCL is loaded at run time.
 *   elp_comm_unique_id     rank 0 creates the id and hands it to the other ranks by any means (ncclGetUniqueId)
 *   elp_comm_init          collective: every rank with the same id, its rank and the world size (ncclCommInitRank on the context's device)
 *   elp_comm_set_partition contig_owner[n_contigs]: the rank that holds the reads of each contig (unmapped reads may sit anywhere)
 * With a communicator and a partition set, elp_sort_markdup becomes collective: the mates of pairs that span two ranks -- the reference's
 * "spread" reads (sam/split-merge.go:286-293) -- are exchanged as 128-byte records (grouped ncclSend / ncclRecv), classified on the rank that owns
 * the smaller REFID together with its own pairs, and their 0x400 bits are sent back.  elp_bqsr_tables_allreduce is LoadAndCombineBQSRTables
 * (filters/print-bqsr.go:310-329) as one ncclAllReduce(sum, int64) between elp_bqsr_gather and elp_bqsr_finalize; elp_optical_allreduce is
 * mergeDuplicatesCtrMaps (filters/mark-optical-duplicates.go:451-466) over the ranks.  Output order = the ranks' outputs concatenated in
 * contig-group order (MergeSortedFilesSplitPerChromosome, sam/split-merge.go:465-547).
 * A read of a cross-group pair may have a QNAME of at most 92 bytes (a longer one is ELP_ELIMIT; one context has no such limit).  An error
 * of elp_sort_markdup on one rank before marking (an invalid QUAL, a negative POS, that QNAME limit, a failed allocation for the exchange)
 * is returned by every rank: the others with the same code and "on rank r" in elp_last_error, and no rank changes FLAG.  A device fault
 * (a sticky CUDA error) is not agreed. */
int elp_comm_unique_id(uint8_t id[128]);
int elp_comm_init(elp_ctx *ctx, const uint8_t id[128], int rank, int world);
int elp_comm_set_partition(elp_ctx *ctx, const int32_t *contig_owner);
int elp_comm_destroy(elp_ctx *ctx);
int elp_bqsr_tables_allreduce(elp_ctx *ctx);
int elp_optical_allreduce(elp_ctx *ctx);

/* ---- phase 4: FinalizeBQSRTables + PrintBQSRTables (filters/bqsr.go:677-694, filters/print-bqsr.go:269-298).
 * report_path may be NULL (no report). Also builds the apply look-up table. ---- */
int elp_bqsr_finalize(elp_ctx *ctx, const char *report_path);
/* EmpiricalQuality bytes of the finalized tables, same indexing as the dense tables without the [2] */
int elp_bqsr_empirical_get(elp_ctx *ctx, uint8_t *emp, uint64_t n);

/* ---- phase 5: (*BaseRecalibratorTables).ApplyBQSR (filters/bqsr.go:936-1006) ---- */
int elp_bqsr_apply(elp_ctx *ctx);

/* ---- phase 6: pulling the result back ((*sam.Sam).RunPipeline as PipelineInput, sam/filter-pipeline.go:242-279).
 * Records [first, first+n) of the output order. Any output pointer may be NULL.
 * record_index: arrival index of each output record (the permutation the sort produced);
 * flag: FLAG with the 0x400 bits; qual: recalibrated QUAL bytes packed back to back; qual_off[n+1]: offsets into qual. ---- */
int elp_fetch(elp_ctx *ctx, uint64_t first, uint64_t n, uint64_t *record_index, uint16_t *flag, uint64_t *qual_off, uint8_t *qual, uint64_t qual_capacity);
uint64_t elp_fetch_qual_bytes(elp_ctx *ctx, uint64_t first, uint64_t n);
/* Asynchronous form: the device->host copies are queued on the context's download stream (behind everything the phases computed) and the
 * call returns; the buffers are complete when elp_fetch_wait returns.  record_index32: the permutation as 32-bit indices (a context
 * holds fewer than 2^32 reads). */
int elp_fetch_async(elp_ctx *ctx, uint64_t first, uint64_t n, uint32_t *record_index32, uint16_t *flag, uint64_t *qual_off, uint8_t *qual, uint64_t qual_capacity);
int elp_fetch_wait(elp_ctx *ctx);
/* per-read temps of adaptAlignment (filters/mark-duplicates.go:153-156), arrival order; for parity tests */
/* The same as BAM alignment records (only if every read came in through elp_append_bam or elp_append_sam): output records [first, first+n) are
 * the stored records with FLAG, MAPQ and -- once elp_bqsr_apply has run -- QUAL replaced; names, CIGAR and optional fields are the
 * input bytes.  This stands in for formatting every *sam.Alignment again (sam/bam-files.go:635-735); the caller BGZF-
 * compresses the result.  record_off[n+1] may be NULL. */
uint64_t elp_fetch_bam_bytes(elp_ctx *ctx, uint64_t first, uint64_t n);
int elp_fetch_bam(elp_ctx *ctx, uint64_t first, uint64_t n, uint8_t *out, uint64_t capacity, uint64_t *record_off);
/* The same as SAM text alignment lines (FormatAlignment, sam/sam-files.go:563-598, of parseBamAlignment of the record elp_fetch_bam returns):
 * output records [first, first+n) as lines ending in '\n', with the context's FLAG, MAPQ and -- once elp_bqsr_apply has run -- QUAL; no header
 * lines (the caller writes the header text).  line_off[n+1] (may be NULL): offset of every line in out.  The reference's quirks are kept:
 * every integer tag prints as i, POS / PNEXT wrap in int32, RNEXT is '=' when its @SQ name equals RNAME's, f values print as Go's
 * strconv 'g' shortest float32, H digits in lower case.  Refusals as elp_fetch_bam (ELP_ESTATE before elp_sort_markdup, for reads that did
 * not come through elp_append_bam / elp_append_sam, after elp_clean_sam rewrote a CIGAR; ELP_EINVAL for a range past the reads or a buffer
 * too small, nothing written), plus: ELP_EINVAL when a context with @SQ lines was created without elp_config.contig_names; ELP_ESTATE when
 * elp_append_sam took a line whose RNAME or RNEXT the stored record cannot reproduce (a name that is not an @SQ name, or RNEXT '=' with
 * such an RNAME; elp_last_error gives their number); ELP_EBAM for a CIGAR operation code above 8.  elp_fetch_sam_bytes returns 0 on error. */
uint64_t elp_fetch_sam_bytes(elp_ctx *ctx, uint64_t first, uint64_t n);
int elp_fetch_sam(elp_ctx *ctx, uint64_t first, uint64_t n, char *out, uint64_t capacity, uint64_t *line_off);
/* Write-phase filters (the filters2 of `elprep filter`, cmd/filter.go:803-902, and RemoveOptionalReads): applied by elp_fetch_bam,
 * elp_fetch_bam_bytes, elp_fetch_sam and elp_fetch_sam_bytes only.  elp_fetch, elp_fetch_async, elp_fetch_qual_bytes and elp_fetch_opt_flags
 * are unchanged: a columnar caller owns its *Alignments and runs filters2 itself.
 *  - Record selection.  With a record bit set, [first, first+n) of those four calls indexes the output records that pass, in output order
 *    (elp_n_output of them); record_off / line_off describe the records written.  With no record bit the calls behave as without a filter.
 *  - Field filter.  One decision per tag: remove_tags (RemoveOptionalFields, :235-257; active iff n_remove > 0) first, then keep_tags
 *    (KeepOptionalFields, :261-288; active iff ELP_OUT_KEEP_FIELDS, n_keep == 0 drops every optional field), the order in which filters2
 *    appends them.  A string matches the 2-byte tag when it equals it, case-sensitively; a string that is not 2 bytes long (also "") matches
 *    no field.  Repeated tags are all dropped or all kept (SmallMap.DeleteIf).  The fields that remain keep their bytes and their order;
 *    block_size is rewritten; FLAG, MAPQ and QUAL are patched as without a filter.  "all" / "none" and TrimSpace belong to the caller's flag parsing.
 *  - Lifetime.  The setting survives elp_reset, like the ingest filter; the selection is rebuilt after elp_sort_markdup, elp_set_output_filter
 *    or elp_reset.  Unknown mask bits, and keep_tags without ELP_OUT_KEEP_FIELDS, are ELP_EINVAL.  A range past elp_n_output is ELP_EINVAL and
 *    nothing is written; the other refusals of the fetch calls still apply (before elp_sort_markdup, after elp_clean_sam, ...). */
#define ELP_OUT_REMOVE_DUPLICATES     1u  /* RemoveDuplicateReads (filters/simple-filters.go:138-140) on the FLAG after elp_sort_markdup */
#define ELP_OUT_REMOVE_OPTIONAL_READS 2u  /* RemoveOptionalReads (:146-152): reads with ELP_OPT_SR; the caller sets it iff the header has @sr (and drops @sr from the header it writes) */
#define ELP_OUT_KEEP_FIELDS           4u  /* KeepOptionalFields(keep_tags) (:261-288); n_keep == 0 drops every optional field */
int elp_set_output_filter(elp_ctx *ctx, uint32_t mask, const char *const *remove_tags, int32_t n_remove, const char *const *keep_tags, int32_t n_keep);
/* `--replace-read-group "ID:x LB:y ..."`: filters.AddOrReplaceReadGroup (filters/simple-filters.go:154-162) on the byte paths.  The caller
 * parses the flag's string (sam.ParseHeaderLineFromString, sam/sam-files.go:153-177) and creates the context from the header after the
 * filter: exactly one @RG, the replacement, with its ID, LB and PU (an @RG without ID is passed as ID "" without PU, so that the BQSR
 * covariate is "" as readGroupCovariate returns it, filters/bqsr.go:35-51).  on = 0 turns the setting off.
 *  - When.  Only while the context holds no reads (after elp_create or elp_reset), else ELP_ESTATE; with on != 0 a context whose
 *    n_read_groups is not 1 is ELP_EINVAL.  The setting survives elp_reset, like the ingest filter.
 *  - Ingest (elp_append_bam, elp_append_sam, elp_append_bgzf).  Every read that passes the ingest filters is in read group 0, whatever RG
 *    field its record has: no RG, an RG:Z value that is no @RG ID (otherwise ELP_EBAM), an RG of another type, several RG fields.  Every
 *    record is still checked for structure (a malformed RG field is ELP_EBAM with any filter mask, CG:B is still ELP_ELIMIT), and the stored
 *    records keep the input's bytes.  elp_append_batch is unchanged: the caller's marshaller sets the rg column to 0 (the filter runs on the
 *    host there, as the other per-record filters do).
 *  - Egress (elp_fetch_bam, elp_fetch_bam_bytes, elp_fetch_bgzf, elp_fetch_sam, elp_fetch_sam_bytes).  Each record is written as aln.SetRG(id)
 *    (sam/sam-types.go:357-359, SmallMap.Set utils/small-map.go:59-67) leaves it, followed by the field filter of elp_set_output_filter:
 *    the first field whose tag is RG, of whatever type, becomes RG Z id NUL in place (SAM: RG:Z:id at the same position), later RG fields
 *    stay, and a record without an RG field gets the new one behind its last field; block_size is rewritten.  --remove-optional-fields RG
 *    and --keep-optional-fields lists without RG drop the new field too.  The record filters, FLAG / MAPQ / QUAL and the refusals of the
 *    fetch calls (after elp_clean_sam rewrote a CIGAR, ...) are as without the setting.  The header bytes (the new @RG line) are the
 *    caller's, as the prefix of elp_fetch_bgzf.
 *  - The columnar elp_fetch is unchanged: a columnar caller owns its *Alignments and sets RG itself. */
int elp_set_replace_read_group(elp_ctx *ctx, int on);
/* `--rename-chromosomes` and `--replace-reference-sequences dict`: filters.RenameChromosomes (filters/simple-filters.go:189-204) and
 * ReplaceReferenceSequenceDictionary (:34-60), followed by AddREFID (:208-231), on the byte paths.  The context is created from the header
 * after the filters: elp_config's contig_names / contig_lengths are the output @SQ (RENAME alone: the input's with "chr" prefixed; REPLACE:
 * the replacement dictionary as read).  Everything keyed by contig -- the reference, the known sites, both target-region tables, the sort,
 * duplicate marking, BQSR, elp_comm_set_partition -- works on the output contigs.  names / lengths: the input file's @SQ as it stands in the
 * file, unrenamed (BAM / BGZF: its binary reference list).  mode = 0 turns the setting off.
 *  - Refusals.  ELP_EINVAL for unknown mode bits, n < 0, a context without contig_names, and, with RENAME alone, n != n_contigs or a
 *    contig_names[i] other than "chr" + names[i].  ELP_ESTATE while the context holds reads or a BGZF file is open.  The setting survives
 *    elp_reset.
 *  - The remap.  Input entry i goes to the last output entry whose name equals its (renamed) name, or nowhere; without REPLACE to i.
 *  - Ingest (elp_append_bam, elp_append_sam, elp_append_bgzf).  refID / next_refID are bounded by the input's entry count, and
 *    elp_append_bgzf checks the BAM header's reference list against names / lengths.  With REPLACE a read whose refID >= 0 has no output
 *    entry is dropped (counted in elp_n_filtered), after the other ingest filters; ELP_FILTER_TARGET_REGIONS looks up the output contig of
 *    a read's refID (elp_set_target_regions stays indexed by output contig; resolve BED names through the input names).  The refid / nref
 *    columns hold the output contigs (-1 for none); the stored records keep the input's bytes.  elp_append_sam resolves RNAME / RNEXT
 *    against the input names; with REPLACE also against the replacement names no input name reaches (under RENAME spelled without "chr"),
 *    and an RNAME that reaches nothing drops the read, as the reference drops it.
 *  - elp_clean_sam uses per read the input LN of its name (the last input entry with that name, 0 for a name outside the input), as
 *    CleanSam runs before the replacement.  This holds on every ingest path; elp_append_batch is otherwise unchanged (the caller's
 *    marshaller remaps refid / nref and drops reads on the host).
 *  - Egress.  elp_fetch_bam, elp_fetch_bam_bytes and elp_fetch_bgzf write refID and next_refID (bytes 4-7 and 24-27) as the output contig,
 *    -1 where there is none; bin, PNEXT and everything else are as without the setting.  elp_fetch_sam prints RNAME / RNEXT by the input
 *    name table ("chr" prefixed under RENAME), so an RNEXT outside the new dictionary keeps its (renamed) name, as in the reference.  The
 *    header bytes (the new @SQ lines and SO) are the caller's, as the prefix of elp_fetch_bgzf. */
#define ELP_DICT_RENAME_CHROMOSOMES 1u   /* --rename-chromosomes */
#define ELP_DICT_REPLACE            2u   /* --replace-reference-sequences */
int elp_set_input_dictionary(elp_ctx *ctx, uint32_t mode, const char *const *names, const int32_t *lengths, int32_t n);
/* Several input files in one context: a directory of inputs, one BAM per lane, as `elprep filter` and `elprep sfm` take it
 * (sam.MergeInputs, sam/merge-inputs.go:16-219, and its update filters, sam/split-merge.go:230-311).  The caller merges the files' headers
 * on the host (elprep_b200.sam.MergeInputs, elprep::MergeInputs) and creates the context from the merged header: elp_config holds the
 * merged @SQ and the merged @RG lines, colliding IDs renamed.
 *  - elp_add_input: one input's @SQ as it stands in the file (BAM / BGZF: its binary reference list).  Returns the input's id (0, 1, ...),
 *    or a negative error code.  Each name maps to the first entry of elp_config.contig_names with that name (memberOfSequenceDictionary);
 *    a name that is not there is ELP_EINVAL, as is a context without contig_names.  At most ELP_MAX_INPUTS inputs (else ELP_ELIMIT).
 *  - elp_select_input: the input whose records the next appends carry.  Once an input is added, every append needs one selected
 *    (ELP_ESTATE without).  ELP_ESTATE while a BGZF file is open: a new file starts after elp_append_bgzf_end, elp_select_input, then
 *    elp_append_bgzf.
 *  - elp_set_tag_rename: tag "RG" or "PG"; old_ids[i] -> new_ids[i] is the composed map of the merge's replaceReadGroupIfExists /
 *    replaceProgramIDIfExists filters (each value through every filter in order).  It applies to the records of every input.  n = 0
 *    clears the tag's map; an old value given twice is ELP_EINVAL.
 *  - elp_add_input and elp_set_tag_rename are ELP_ESTATE while the context holds reads or a BGZF file is open.  All three settings survive
 *    elp_reset; with none of them made, every path is byte for byte as before.  They do not combine with elp_set_input_dictionary
 *    (ELP_EINVAL either way).
 *  - Ingest (elp_append_bam, elp_append_sam, elp_append_bgzf).  Every record is rewritten on the device, before the ingest filters, into
 *    the record the reference writes with the merged header: BAM refID / next_refID through the selected input's map (a value at or past
 *    the input's entry count is ELP_EBAM); the value of the first RG and the first PG field through the maps (aln.SetRG / SetPG: in place,
 *    block_size rewritten; a first field of such a tag that is not of type Z is ELP_EBAM, as the filter's string conversion panics).
 *    elp_append_sam resolves RNAME / RNEXT by name against the merged dictionary, as the reference looks the names up in the merged
 *    header.  elp_append_bgzf checks the file's reference list against the selected input's names and lengths.
 *  - Everything after ingest sees records of the merged header: the RG column is the renamed value's @RG, elp_clean_sam reads the merged
 *    LN, elp_fetch_bam / _bgzf / _sam write the rewritten records, and --replace-read-group and the output field filter apply to them as
 *    to any record (the replacement wins for RG; the PG rename stays). */
#define ELP_MAX_INPUTS 255
int elp_add_input(elp_ctx *ctx, const char *const *names, const int32_t *lengths, int32_t n_sq);
int elp_select_input(elp_ctx *ctx, int32_t input);
int elp_set_tag_rename(elp_ctx *ctx, const char *tag, const char *const *old_ids, const char *const *new_ids, int32_t n);
/* after elp_sort_markdup: the number of records of the output order (elp_n_sorted) that pass the record filters (elp_n_sorted without them);
 * 0 on error or before the sort */
uint64_t elp_n_output(elp_ctx *ctx);
int elp_debug_adapt(elp_ctx *ctx, int32_t *upos, int32_t *score);
/* per read, the 64-bit (library, QNAME) hash duplicate marking joins mates by (its low 31 bits are the join key); 0 for a read that is
 * not a true pair (unmapped, secondary, supplementary, unpaired or mate unmapped) */
int elp_debug_join_hash(elp_ctx *ctx, uint64_t *qhash);
/* per read in arrival order, chunk `chunk` of the composite key by which the coordinate sort orders runs of more than 32 reads with
 * equal (REFID, POS, strand), as that sort would compute it for the reads appended so far: 0 TLEN, 1 NextREFID|PNEXT (0 if unpaired),
 * 2 modFlag|MAPQ, 3 the number of trailing NUL bytes of the QNAME, 4..3+nq the QNAME in 8-byte big-endian chunks (4 = the last),
 * 4+nq the (REFID, POS, strand) key; nq = ceil(longest QNAME / 8), at least 1.  A chunk outside [0, 5+nq) is ELP_EINVAL. */
int elp_debug_coord_chunk_keys(elp_ctx *ctx, int chunk, uint64_t *keys);
/* opt_flags of output records [first, first+n) (what filters.RemoveOptionalReads looks at when the worker writes its output) */
int elp_fetch_opt_flags(elp_ctx *ctx, uint64_t first, uint64_t n, uint8_t *opt_flags);
/* arrival-order CIGARs as the context holds them (after elp_clean_sam), for parity tests: cigar_off[n+1] relative to the first operation */
int elp_debug_cigar(elp_ctx *ctx, uint64_t *cigar_off, uint32_t *cigar, uint64_t capacity);

/* ---- host utilities for callers that hold BAM files in memory (SURVEY.md 8f row 2): BGZF blocks are independent gzip members,
 * (de)compressed here on n_threads host threads with zlib (utils/bgzf/bgzf-files.go:95-127 reader, :324-431 writer).  No context,
 * no GPU.  inflate: data = whole BGZF blocks back to back (an EOF marker block may be among them); bound = exact output size.
 * deflate: blocks of 0xff00 input bytes, level as zlib (-1 = default), optional EOF marker block (bgzfEOF) at the end.
 * elp_bam_header_size: length of magic + text + reference list at the start of an inflated BAM file -- the alignment
 * records for elp_append_bam start there; the references are in BAM refID order, which must be elp_config's contig order. ---- */
int64_t elp_bgzf_inflate_bound(const uint8_t *data, uint64_t n);                 /* >= 0, or ELP_EBGZF */
int elp_bgzf_inflate(const uint8_t *data, uint64_t n, uint8_t *out, uint64_t capacity, uint64_t *out_n, int n_threads);
uint64_t elp_bgzf_deflate_bound(uint64_t n);
int elp_bgzf_deflate(const uint8_t *data, uint64_t n, uint8_t *out, uint64_t capacity, uint64_t *out_n, int level, int n_threads, int write_eof);
int64_t elp_bam_header_size(const uint8_t *bam, uint64_t n, int32_t *n_ref_out);  /* -1 if malformed or truncated */

/* ---- a BGZF-compressed BAM file straight into a context (SURVEY.md 8f row 2; utils/bgzf/bgzf-files.go:95-127,164-221 and the header part
 * of sam/bam-files.go), inflated on the device:
 *  - elp_append_bgzf: the file's bytes, handed over in order and cut anywhere (mid gzip header, mid block, mid record); the file's first
 *    call starts at byte 0 of the file.  An incomplete trailing BGZF block (host side, < 64 KiB) and an incomplete trailing record (device
 *    side) are carried to the next call.  The BAM header is walked on the device and checked against elp_config: n_ref must equal
 *    n_contigs, every l_ref contig_lengths and, when contig_names were given, every name (ELP_EINVAL otherwise; ELP_EBAM for bytes that are
 *    not a BAM header); a header may span several blocks and calls.  The complete records are ingested exactly as by elp_append_bam:
 *    ingest filters, RG:Z, the sr bit, and the arena of elp_fetch_bam / elp_fetch_sam; CG:B is ELP_ELIMIT.
 *  - Validity.  A block is valid exactly when elp_bgzf_inflate accepts it: magic, FEXTRA, a BC subfield, bsize, ISIZE <= 65536; the DEFLATE
 *    stream ends with exactly ISIZE bytes out; the CRC-32 matches; an empty block has CRC 0.  Anything else is ELP_EBGZF.
 *  - Atomic calls.  Nothing of a failing call is appended; the reads of earlier calls stay.  After an error the stream is poisoned:
 *    elp_append_bgzf and elp_append_bgzf_end return ELP_ESTATE until elp_reset (the reference panics at that point).
 *  - Ordering.  While a file is open (from its first elp_append_bgzf to its elp_append_bgzf_end, or an error) elp_append_bam,
 *    elp_append_sam, elp_append_batch and elp_sort_markdup return ELP_ESTATE.  elp_reset discards the stream.  One caller per stream:
 *    the calls serialise like the other appends, but only the caller knows the byte order.
 *  - elp_append_bgzf_end ends the file: ELP_EBGZF if block bytes remain or the last block was not the EOF marker (bgzf-files.go:111-115),
 *    ELP_EBAM if header or record bytes remain, ELP_ESTATE without an open file; afterwards a new file may start.
 *  - elp_debug_inflate: whole BGZF blocks -> inflated bytes, with the contract of elp_bgzf_inflate but decoded on the device (tests,
 *    micro-benchmark); it does not touch an open stream. ---- */
int elp_append_bgzf(elp_ctx *ctx, const uint8_t *data, uint64_t n_bytes);
int elp_append_bgzf_end(elp_ctx *ctx);
int elp_debug_inflate(elp_ctx *ctx, const uint8_t *data, uint64_t n, uint8_t *out, uint64_t capacity, uint64_t *out_n);

/* ---- the output records as a BGZF-compressed BAM file, deflated on the device (SURVEY.md 8f row 2; the writer of
 * utils/bgzf/bgzf-files.go:324-431): the records never cross to the host uncompressed.
 *  - elp_fetch_bgzf writes the BGZF blocks of prefix || elp_fetch_bam(first, n) to out and their length to *out_n.  prefix (n_prefix
 *    bytes, may be NULL when 0) is typically the BAM header -- magic, text and reference list, which only the caller can format -- on the
 *    first call of a file.  The records are exactly those of elp_fetch_bam: output order, FLAG, MAPQ and QUAL patched, the record and field
 *    filters of elp_set_output_filter, the kept records after elp_filter_target_regions; [first, first+n) indexes elp_n_output.  n == 0
 *    is allowed (prefix only, EOF marker only, or nothing).
 *  - Blocks.  The bytes are cut into blocks of 0xff00 bytes, the last one partial, as elp_bgzf_deflate cuts them (so both writers give the
 *    same ISIZE sequence), each one gzip member with the BC subfield and one final DEFLATE block: dynamic Huffman codes, or stored when
 *    that is smaller, so every block is at most 65536 bytes.  The bytes out depend only on the bytes in.  write_eof != 0 appends the
 *    28-byte EOF marker.  Not byte-identical to zlib or Go's compress/flate; any inflater decodes the same bytes.
 *  - Calls compose.  Every call ends its own last block: the outputs of consecutive ranges, concatenated with write_eof on the last call
 *    only, are a valid BGZF file that inflates to the same bytes as one call over the whole range (the block layouts differ).  Several
 *    ranks' outputs, concatenated in contig-group order, make one file the same way.
 *  - Refusals, with nothing written to out: those of elp_fetch_bam with its codes (ELP_ESTATE before elp_sort_markdup, for reads that did
 *    not all come in as BAM, SAM or BGZF, after elp_clean_sam rewrote a CIGAR; ELP_EINVAL for a range past elp_n_output), and ELP_EINVAL
 *    when capacity < elp_bgzf_deflate_bound(elp_fetch_bam_bytes(ctx, first, n) + n_prefix).
 *  - elp_debug_deflate: host bytes in, the same kernels, BGZF out (capacity >= elp_bgzf_deflate_bound(n)); the counterpart of
 *    elp_debug_inflate, for tests and the micro-benchmark. ---- */
int elp_fetch_bgzf(elp_ctx *ctx, uint64_t first, uint64_t n, const uint8_t *prefix, uint64_t n_prefix, int write_eof,
                   uint8_t *out, uint64_t capacity, uint64_t *out_n);
int elp_debug_deflate(elp_ctx *ctx, const uint8_t *data, uint64_t n, int write_eof,
                      uint8_t *out, uint64_t capacity, uint64_t *out_n);

/* ---- measurement ---- */
uint64_t elp_launch_count(const elp_ctx *ctx);           /* kernels launched by this library since create/reset */
int elp_kernel_stats(elp_ctx *ctx, elp_kernel_stat *out, int cap); /* returns number of entries; profile must be on */
int elp_synchronize(elp_ctx *ctx);
int elp_reset_stats(elp_ctx *ctx);                       /* forget kernel stats and the launch count */
/* device-side stopwatch: CUDA events recorded on the library's own stream (torch.cuda.Event would not see it) */
int elp_timer_start(elp_ctx *ctx);
int elp_timer_stop(elp_ctx *ctx, double *elapsed_ms);    /* synchronizes */

/* ---- stand-alone access to the device radix sort (the graded kernel), for tests and the sort micro-benchmark:
 * stable LSD sort of n 64-bit keys (only the low key_bits are significant) carrying 32-bit values. Host buffers. ---- */
int elp_debug_sort_u64(elp_ctx *ctx, uint64_t *keys, uint32_t *vals, uint64_t n, int key_bits);
int elp_debug_sort_u128(elp_ctx *ctx, uint64_t *keys_hi, uint64_t *keys_lo, uint32_t *vals, uint64_t n, int key_bits);
/* the same sorts over bits [lo_bit, lo_bit + key_bits) only: the bits below lo_bit travel with the key unsorted, and keys equal
 * in the sorted range keep their input order (the fragment-group sort of duplicate marking uses such a range) */
int elp_debug_sort_u64_range(elp_ctx *ctx, uint64_t *keys, uint32_t *vals, uint64_t n, int lo_bit, int key_bits);
int elp_debug_sort_u128_range(elp_ctx *ctx, uint64_t *keys_hi, uint64_t *keys_lo, uint32_t *vals, uint64_t n, int lo_bit, int key_bits);
/* the 32-bit-key sort (the mate join's), over bits [lo_bit, lo_bit + key_bits) with lo_bit + key_bits <= 32 */
int elp_debug_sort_u32_range(elp_ctx *ctx, uint32_t *keys, uint32_t *vals, uint64_t n, int lo_bit, int key_bits);
/* the device prefix sum: out[i] = base + in[0] + ... + in[i-1] for i <= n (out has n + 1 entries, out[n] the total). Host buffers. */
int elp_debug_scan_u32(elp_ctx *ctx, const uint32_t *in, uint64_t *out, uint64_t n, uint64_t base);

#ifdef __cplusplus
}
#endif
#endif
