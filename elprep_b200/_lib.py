"""ctypes binding of include/elprep_b200.h (libelprep_b200.so, built in-tree by __graft_entry__.build()).

Fails loudly when the CUDA library is missing or no GPU is usable: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("ELPREP_B200_LIB", os.path.join(_HERE, "lib", "libelprep_b200.so"))   # override: kernel-ablation builds (tools/ablate.sh)

SO_KEEP, SO_UNKNOWN, SO_UNSORTED, SO_QUERYNAME, SO_COORDINATE = 0, 1, 2, 3, 4
MARKDUP, MARKDUP_OPTICAL = 1, 2
EINVAL, ELIMIT, ESTATE, EBAM, ESAM = -1, -15, -16, -18, -20
FILTER_UNMAPPED, FILTER_UNMAPPED_STRICT, FILTER_NON_EXACT, FILTER_DUPLICATES, FILTER_NON_EXACT_STRICT, FILTER_TARGET_REGIONS = 1, 2, 4, 8, 16, 32


class ElpConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("n_contigs", C.c_int32), ("contig_names", C.POINTER(C.c_char_p)), ("contig_lengths", C.c_void_p),
                ("n_read_groups", C.c_int32), ("rg_id", C.POINTER(C.c_char_p)), ("rg_lb", C.POINTER(C.c_char_p)), ("rg_pu", C.POINTER(C.c_char_p)),
                ("max_cycle", C.c_int32), ("quantize_levels", C.c_int32), ("sqq", C.c_void_p), ("n_sqq", C.c_int32),
                ("tablename_prefix", C.c_char_p), ("optical_pixel_distance", C.c_int32), ("profile", C.c_int32)]


class ElpBatch(C.Structure):
    _fields_ = [("n", C.c_uint64)] + [(k, C.c_void_p) for k in
                ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg", "qname_off", "qname", "cigar_off", "cigar", "l_seq", "seq", "qual", "opt_flags")]


class ElpDupMetrics(C.Structure):
    COUNTERS = ("unpaired_reads_examined", "read_pairs_examined", "secondary_or_supplementary_reads", "unmapped_reads",
                "unpaired_read_duplicates", "read_pair_duplicates", "read_pair_optical_duplicates")
    _fields_ = [(k, C.c_int64) for k in COUNTERS] + [("estimated_library_size", C.c_int64), ("percent_duplication", C.c_double),
                                                      ("roi", C.c_double * 100), ("has_roi", C.c_int32), ("paired_reads_examined", C.c_int64)]


class ElpKernelStat(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("launches", C.c_uint64), ("ms", C.c_double), ("alg_bytes", C.c_double)]


EXPORTS = ["elp_create", "elp_destroy", "elp_last_error", "elp_reserve", "elp_reset", "elp_set_reference", "elp_set_known_sites",
           "elp_fetch_opt_flags", "elp_set_target_regions", "elp_clean_sam", "elp_debug_cigar", "elp_comm_unique_id", "elp_comm_init", "elp_comm_set_partition", "elp_comm_destroy", "elp_bqsr_tables_allreduce", "elp_optical_allreduce", "elp_bqsr_tables_clear", "elp_bqsr_tables_write_elrecal", "elp_bqsr_tables_add_elrecal", "elp_optical_write_gob", "elp_optical_add_gob", "elp_append_batch", "elp_append_batch_async", "elp_append_wait", "elp_fetch_async", "elp_fetch_wait", "elp_append_bam", "elp_append_sam", "elp_set_ingest_filter", "elp_n_filtered", "elp_n_reads", "elp_sort_markdup", "elp_bqsr_gather", "elp_bqsr_tables_len", "elp_bqsr_n_cov",
           "elp_bqsr_cov_name", "elp_bqsr_tables_get", "elp_bqsr_tables_put", "elp_bqsr_tables_device", "elp_bqsr_finalize",
           "elp_bqsr_empirical_get", "elp_bqsr_apply", "elp_fetch", "elp_fetch_qual_bytes", "elp_fetch_bam", "elp_fetch_bam_bytes", "elp_fetch_sam", "elp_fetch_sam_bytes", "elp_debug_adapt", "elp_launch_count",
           "elp_kernel_stats", "elp_synchronize", "elp_reset_stats", "elp_timer_start", "elp_timer_stop", "elp_debug_sort_u64", "elp_debug_sort_u128",
           "elp_optical_n_libraries", "elp_optical_library_name", "elp_optical_metrics", "elp_optical_histogram", "elp_optical_merge",
           "elp_print_duplicates_metrics",
           "elp_bgzf_inflate_bound", "elp_bgzf_inflate", "elp_bgzf_deflate_bound", "elp_bgzf_deflate", "elp_bam_header_size"]

_lib = None


def load():
    """Load the shared library (no GPU needed for loading; elp_create needs one)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise RuntimeError(f"elprep_b200: CUDA library {SO_PATH} is missing -- run `python -c 'import __graft_entry__ as g; g.build()'`; "
                           "there is no CPU fallback")
    L = C.CDLL(SO_PATH)
    L.elp_last_error.restype = C.c_char_p
    L.elp_last_error.argtypes = [C.c_void_p]
    L.elp_create.argtypes = [C.POINTER(ElpConfig), C.POINTER(C.c_void_p)]
    L.elp_destroy.argtypes = [C.c_void_p]
    L.elp_destroy.restype = None
    L.elp_n_reads.restype = C.c_uint64
    L.elp_n_reads.argtypes = [C.c_void_p]
    L.elp_bqsr_tables_len.restype = C.c_uint64
    L.elp_bqsr_tables_len.argtypes = [C.c_void_p]
    L.elp_bqsr_n_cov.argtypes = [C.c_void_p]
    L.elp_bqsr_cov_name.restype = C.c_char_p
    L.elp_bqsr_cov_name.argtypes = [C.c_void_p, C.c_int32]
    L.elp_launch_count.restype = C.c_uint64
    L.elp_launch_count.argtypes = [C.c_void_p]
    L.elp_fetch_qual_bytes.restype = C.c_uint64
    L.elp_fetch_qual_bytes.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    L.elp_reserve.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64]
    L.elp_reset.argtypes = [C.c_void_p]
    L.elp_set_reference.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64]
    L.elp_set_known_sites.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_int]
    L.elp_append_batch.argtypes = [C.c_void_p, C.POINTER(ElpBatch)]
    for f in ("elp_bqsr_tables_write_elrecal", "elp_bqsr_tables_add_elrecal", "elp_optical_write_gob", "elp_optical_add_gob"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_char_p]
    L.elp_bqsr_tables_clear.argtypes = [C.c_void_p]
    L.elp_fetch_opt_flags.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
    L.elp_set_target_regions.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_int]
    L.elp_clean_sam.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.elp_debug_cigar.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.elp_comm_unique_id.argtypes = [C.c_void_p]
    L.elp_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.elp_comm_set_partition.argtypes = [C.c_void_p, C.c_void_p]
    L.elp_comm_destroy.argtypes = [C.c_void_p]
    L.elp_bqsr_tables_allreduce.argtypes = [C.c_void_p]
    L.elp_optical_allreduce.argtypes = [C.c_void_p]
    L.elp_append_batch_async.argtypes = [C.c_void_p, C.POINTER(ElpBatch)]
    L.elp_append_wait.argtypes = [C.c_void_p]
    L.elp_fetch_async.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.elp_fetch_wait.argtypes = [C.c_void_p]
    L.elp_sort_markdup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.elp_fetch_bam_bytes.restype = C.c_uint64
    L.elp_fetch_bam_bytes.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    L.elp_fetch_bam.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
    L.elp_fetch_sam_bytes.restype = C.c_uint64
    L.elp_fetch_sam_bytes.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    L.elp_fetch_sam.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
    L.elp_set_ingest_filter.argtypes = [C.c_void_p, C.c_uint32, C.c_int32]
    L.elp_n_filtered.restype = C.c_uint64
    L.elp_n_filtered.argtypes = [C.c_void_p]
    L.elp_append_bam.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    L.elp_append_sam.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
    L.elp_bqsr_gather.argtypes = [C.c_void_p]
    L.elp_bqsr_tables_get.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.elp_bqsr_tables_put.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.elp_bqsr_tables_device.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    L.elp_bqsr_finalize.argtypes = [C.c_void_p, C.c_char_p]
    L.elp_bqsr_empirical_get.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.elp_bqsr_apply.argtypes = [C.c_void_p]
    L.elp_fetch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.elp_debug_adapt.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.elp_kernel_stats.argtypes = [C.c_void_p, C.POINTER(ElpKernelStat), C.c_int]
    L.elp_synchronize.argtypes = [C.c_void_p]
    L.elp_reset_stats.argtypes = [C.c_void_p]
    L.elp_timer_start.argtypes = [C.c_void_p]
    L.elp_timer_stop.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    L.elp_debug_sort_u64.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int]
    L.elp_debug_sort_u128.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int]
    L.elp_optical_n_libraries.argtypes = [C.c_void_p]
    L.elp_optical_library_name.restype = C.c_char_p
    L.elp_optical_library_name.argtypes = [C.c_void_p, C.c_int32]
    L.elp_optical_metrics.argtypes = [C.c_void_p, C.c_int32, C.POINTER(ElpDupMetrics)]
    L.elp_optical_histogram.restype = C.c_int64
    L.elp_optical_histogram.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]
    L.elp_optical_merge.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]
    L.elp_print_duplicates_metrics.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p]
    L.elp_bgzf_inflate_bound.restype = C.c_int64
    L.elp_bgzf_inflate_bound.argtypes = [C.c_void_p, C.c_uint64]
    L.elp_bgzf_inflate.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_int]
    L.elp_bgzf_deflate_bound.restype = C.c_uint64
    L.elp_bgzf_deflate_bound.argtypes = [C.c_uint64]
    L.elp_bgzf_deflate.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int]
    L.elp_bam_header_size.restype = C.c_int64
    L.elp_bam_header_size.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_int32)]
    _lib = L
    return L
