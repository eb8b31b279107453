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
 * refid/nref are the REFID/NextREFID temps of filters.AddREFID (simple-filters.go:208-231);
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
/* optional capacity hint so that appends never reallocate */
int elp_reserve(elp_ctx *ctx, uint64_t n_reads, uint64_t n_bases, uint64_t n_cigar_ops, uint64_t n_qname_bytes);
/* forget all reads/tables but keep device allocations, reference and known sites (bench steps) */
int elp_reset(elp_ctx *ctx);

/* ---- side inputs: fasta.MappedFasta.Seq(contig) (fasta/fasta-files.go:355) and the known-sites intervals
 * of NewBaseRecalibrator (filters/bqsr.go:424-443). start/end pairs; flattened inside unless already_flat. ---- */
int elp_set_reference(elp_ctx *ctx, int32_t contig, const uint8_t *bases, uint64_t n);
int elp_set_known_sites(elp_ctx *ctx, int32_t contig, const int32_t *start_end_pairs, uint64_t n_intervals, int already_flat);

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
 * RemoveMappingQualityLessThan (:332-347: keeps MAPQ >= min_mapq), RemoveDuplicateReads (:131-133, on the FLAG the record comes
 * in with).  With elp_append_batch the caller's marshaller applies its filters to the []*Alignment before building columns. */
#define ELP_FILTER_UNMAPPED 1u
#define ELP_FILTER_UNMAPPED_STRICT 2u
#define ELP_FILTER_NON_EXACT 4u
#define ELP_FILTER_DUPLICATES 8u
#define ELP_FILTER_NON_EXACT_STRICT 16u   /* RemoveNonExactMappingReadsStrict (:115-136): optional fields X0 = 1, X1 = XM = XO = XG = 0 must all be present */
#define ELP_FILTER_TARGET_REGIONS 32u     /* RemoveNonOverlappingReads (:310-328): keep reads whose [POS, End()] overlaps a region of elp_set_target_regions */
/* regions of one contig as (start, end) pairs, the Start / End of the BED records as the reference's bed parser stores them; sorted by
 * start and flattened inside unless already_flat (intervals.FromBed + ParallelSortByStart + ParallelFlatten, filters/simple-filters.go:311-315) */
int elp_set_target_regions(elp_ctx *ctx, int32_t contig, const int32_t *start_end_pairs, uint64_t n_intervals, int already_flat);
int elp_set_ingest_filter(elp_ctx *ctx, uint32_t mask, int32_t min_mapq);
uint64_t elp_n_filtered(const elp_ctx *ctx);
uint64_t elp_n_reads(const elp_ctx *ctx);
/* filters.CleanSam (filters/simple-filters.go:292-306, softClipEndOfRead filters/utils.go:82-119) over the reads appended so far (either ingest
 * path; call before elp_sort_markdup): MAPQ of unmapped reads becomes 0; a read that runs past the end of its contig gets its CIGAR soft-clipped
 * there.  Returns the number of rewritten CIGARs in *n_rewritten (may be NULL).  After a rewrite elp_fetch_bam is refused (the stored records
 * still carry the old CIGAR); the columnar elp_fetch is unaffected. */
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
 * contig-group order (MergeSortedFilesSplitPerChromosome, sam/split-merge.go:465-547). */
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
 * the stored records with FLAG and -- once elp_bqsr_apply has run -- QUAL replaced; names, CIGAR and optional fields are the
 * input bytes.  This stands in for formatting every *sam.Alignment again (sam/bam-files.go:635-735); the caller BGZF-
 * compresses the result.  record_off[n+1] may be NULL. */
uint64_t elp_fetch_bam_bytes(elp_ctx *ctx, uint64_t first, uint64_t n);
int elp_fetch_bam(elp_ctx *ctx, uint64_t first, uint64_t n, uint8_t *out, uint64_t capacity, uint64_t *record_off);
/* The same as SAM text alignment lines (FormatAlignment, sam/sam-files.go:563-598, of parseBamAlignment of the record elp_fetch_bam returns):
 * output records [first, first+n) as lines ending in '\n', with the context's FLAG and -- once elp_bqsr_apply has run -- QUAL; no header
 * lines (the caller writes the header text).  line_off[n+1] (may be NULL): offset of every line in out.  The reference's quirks are kept:
 * every integer tag prints as i, POS / PNEXT wrap in int32, RNEXT is '=' when its @SQ name equals RNAME's, f values print as Go's
 * strconv 'g' shortest float32, H digits in lower case.  Refusals as elp_fetch_bam (ELP_ESTATE before elp_sort_markdup, for reads that did
 * not come through elp_append_bam / elp_append_sam, after elp_clean_sam rewrote a CIGAR; ELP_EINVAL for a range past the reads or a buffer
 * too small, nothing written), plus: ELP_EINVAL when a context with @SQ lines was created without elp_config.contig_names; ELP_ESTATE when
 * elp_append_sam took a line whose RNAME or RNEXT the stored record cannot reproduce (a name that is not an @SQ name, or RNEXT '=' with
 * such an RNAME; elp_last_error gives their number); ELP_EBAM for a CIGAR operation code above 8.  elp_fetch_sam_bytes returns 0 on error. */
uint64_t elp_fetch_sam_bytes(elp_ctx *ctx, uint64_t first, uint64_t n);
int elp_fetch_sam(elp_ctx *ctx, uint64_t first, uint64_t n, char *out, uint64_t capacity, uint64_t *line_off);
int elp_debug_adapt(elp_ctx *ctx, int32_t *upos, int32_t *score);
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

#ifdef __cplusplus
}
#endif
#endif
