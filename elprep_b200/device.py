"""Thin Python handle on an ``elp_ctx`` (the C ABI of include/elprep_b200.h).  Plumbing only: every
method is one C call; errors surface as ``ElprepError`` carrying the reference's panic text."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import SO_COORDINATE, SO_KEEP  # noqa: F401


class ElprepError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[{code}] {msg}")
        self.code = code


def _vp(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _cstrs(items):
    arr = (C.c_char_p * max(1, len(items)))()
    for i, s in enumerate(items):
        arr[i] = None if s is None else s.encode()
    return arr


class Context:
    """One device context = one (*sam.Sam) being filled, sorted, duplicate-marked and recalibrated."""

    NQ, NCTX = 94, 16

    def __init__(self, header, device=0, max_cycle=500, quantize_levels=0, sqq=None, prefix="GATK", optical_pixel_distance=100, profile=False):
        self.L = _lib.load()
        self.header = header
        self.max_cycle = max_cycle
        names = _cstrs(header.contig_names())
        self._clen = header.contig_lengths()
        ids = _cstrs([r["ID"] for r in header.RG])
        lbs = _cstrs([r.get("LB") for r in header.RG])
        pus = _cstrs([r.get("PU") for r in header.RG])
        sq = np.ascontiguousarray(sqq if sqq is not None else [], dtype=np.uint8)
        cfg = _lib.ElpConfig(device, len(header.SQ), names, _vp(self._clen), len(header.RG), ids, lbs, pus, max_cycle, quantize_levels,
                             _vp(sq) if sq.size else None, int(sq.size), prefix.encode(), optical_pixel_distance, int(profile))
        h = C.c_void_p()
        rc = self.L.elp_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise ElprepError(rc, (self.L.elp_last_error(None) or b"").decode())
        self.h = h
        self._keep = (names, ids, lbs, pus, sq)
        self._keep_opts = dict(quantize_levels=quantize_levels, sqq=list(sqq) if sqq is not None else None)

    def close(self):
        if getattr(self, "h", None):
            self.L.elp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise ElprepError(rc, (self.L.elp_last_error(self.h) or b"").decode())

    # ---- side inputs ----
    def set_reference(self, contig, bases):
        b = np.ascontiguousarray(bases, dtype=np.uint8)
        self._ck(self.L.elp_set_reference(self.h, contig, _vp(b), b.size))

    def set_known_sites(self, contig, start_end, already_flat=True):
        se = np.ascontiguousarray(start_end, dtype=np.int32).reshape(-1)
        self._ck(self.L.elp_set_known_sites(self.h, contig, _vp(se) if se.size else None, se.size // 2, int(already_flat)))

    # ---- phases ----
    def reserve(self, n_reads, n_bases, n_cigar, n_qname):
        self._ck(self.L.elp_reserve(self.h, n_reads, n_bases, n_cigar, n_qname))

    def reset(self):
        self._ck(self.L.elp_reset(self.h))

    def append(self, batch):
        b = _lib.ElpBatch()
        b.n = batch.n
        for k in ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg", "qname_off", "qname", "cigar_off", "cigar", "seq", "qual", "opt_flags"):
            setattr(b, k, _vp(getattr(batch, k)))
        b.l_seq = _vp(batch.lseq)
        self._ck(self.L.elp_append_batch(self.h, C.byref(b)))

    def append_async(self, batch):
        """queue the upload and return; ``batch`` (page-locked) must stay alive and unchanged until append_wait()"""
        b = _lib.ElpBatch()
        b.n = batch.n
        for k in ("refid", "pos", "flag", "mapq", "nref", "pnext", "tlen", "rg", "qname_off", "qname", "cigar_off", "cigar", "seq", "qual", "opt_flags"):
            setattr(b, k, _vp(getattr(batch, k)))
        b.l_seq = _vp(batch.lseq)
        self._ck(self.L.elp_append_batch_async(self.h, C.byref(b)))

    def append_wait(self):
        self._ck(self.L.elp_append_wait(self.h))

    def fetch_async(self, out, first=0, n=None):
        """out = (record_index u32[n], flag u16[n], qual_off u64[n+1] or None, qual u8[]) page-locked; complete after fetch_wait()"""
        n = self.n - first if n is None else n
        idx, flag, qoff, qual = out
        self._ck(self.L.elp_fetch_async(self.h, first, n, _vp(idx), _vp(flag), _vp(qoff), _vp(qual), qual.size if qual is not None else 0))

    def fetch_wait(self):
        self._ck(self.L.elp_fetch_wait(self.h))

    def set_ingest_filter(self, mask=0, min_mapq=0):
        self._ck(self.L.elp_set_ingest_filter(self.h, mask, min_mapq))

    def set_output_filter(self, mask=0, remove=(), keep=None):
        """the write-phase filters of fetch_bam / fetch_sam (elp_set_output_filter): mask of _lib.OUT_REMOVE_DUPLICATES and
        _lib.OUT_REMOVE_OPTIONAL_READS; remove: RemoveOptionalFields tags; keep: KeepOptionalFields tags ([] keeps none, None: no keep filter)"""
        remove = [t.encode() if isinstance(t, str) else bytes(t) for t in remove]
        if keep is not None:
            mask |= _lib.OUT_KEEP_FIELDS
        keep = [t.encode() if isinstance(t, str) else bytes(t) for t in (keep or ())]
        ra, ka = (C.c_char_p * max(1, len(remove)))(*remove), (C.c_char_p * max(1, len(keep)))(*keep)
        self._ck(self.L.elp_set_output_filter(self.h, mask, ra, len(remove), ka, len(keep)))

    def n_output(self):
        """output records fetch_bam / fetch_sam write (those that pass the record filters of set_output_filter); 0 before sort_markdup"""
        return int(self.L.elp_n_output(self.h))

    def _n_out(self, first):
        k = self.n_output()
        if k == 0 and self.L.elp_fetch_opt_flags(self.h, 0, 0, None) != 0:
            k = self.n                                                    # before sort_markdup: the fetch reports the refusal
        return k - first

    def set_target_regions(self, contig, start_end, already_flat=False):
        se = np.ascontiguousarray(start_end, dtype=np.int32).reshape(-1)
        self._ck(self.L.elp_set_target_regions(self.h, contig, _vp(se) if se.size else None, se.size // 2, int(already_flat)))

    def clean_sam(self):
        """filters.CleanSam over the reads appended so far; returns the number of rewritten CIGARs"""
        k = C.c_uint64()
        self._ck(self.L.elp_clean_sam(self.h, C.byref(k)))
        return int(k.value)

    def fetch_opt_flags(self, first=0, n=None):
        n = self.n - first if n is None else n
        out = np.zeros(n, np.uint8)
        self._ck(self.L.elp_fetch_opt_flags(self.h, first, n, _vp(out)))
        return out

    def debug_cigar(self):
        off = np.zeros(self.n + 1, np.uint64)
        cap = 64 * max(1, self.n)
        cg = np.zeros(cap, np.uint32)
        self._ck(self.L.elp_debug_cigar(self.h, _vp(off), _vp(cg), cap))
        return off, cg[:int(off[-1])]

    def n_filtered(self):
        return int(self.L.elp_n_filtered(self.h))

    def append_bam(self, records, record_off=None):
        """records: uint8 array of consecutive BAM alignment records (each with its block_size); record_off: uint64[n+1] or None"""
        rec = np.ascontiguousarray(records, dtype=np.uint8)
        off = np.ascontiguousarray(record_off, dtype=np.uint64) if record_off is not None else None
        self._ck(self.L.elp_append_bam(self.h, _vp(rec), rec.size, _vp(off), (off.size - 1) if off is not None else 0))

    def append_sam(self, text):
        """text: bytes or a uint8 array of SAM alignment lines (no header; the last line may lack its newline)"""
        if isinstance(text, (bytes, bytearray, memoryview)):
            buf = bytes(text)
            self._ck(self.L.elp_append_sam(self.h, buf, len(buf)))
        else:
            t = np.ascontiguousarray(text, dtype=np.uint8)
            self._ck(self.L.elp_append_sam(self.h, C.cast(_vp(t), C.c_char_p), t.size))

    @property
    def n(self):
        return int(self.L.elp_n_reads(self.h))

    def sort_markdup(self, sorting_order=SO_COORDINATE, mark_duplicates=True):
        """mark_duplicates: False/0, True/1 (MarkDuplicates(false)) or 2 (= _lib.MARKDUP_OPTICAL: also the duplication metrics)"""
        self._ck(self.L.elp_sort_markdup(self.h, sorting_order, int(mark_duplicates)))

    # ---- duplication metrics (filters.MarkOpticalDuplicates) ----
    def optical_libraries(self):
        return [self.L.elp_optical_library_name(self.h, i).decode() for i in range(int(self.L.elp_optical_n_libraries(self.h)))]

    def optical_metrics(self):
        """-> list over slots of dict(counters..., estimated_library_size, percent_duplication, roi, hist=[{key: count}] * 3)"""
        out = []
        for slot in range(int(self.L.elp_optical_n_libraries(self.h))):
            m = _lib.ElpDupMetrics()
            self._ck(self.L.elp_optical_metrics(self.h, slot, C.byref(m)))
            d = {k: int(getattr(m, k)) for k in _lib.ElpDupMetrics.COUNTERS}
            d["estimated_library_size"] = int(m.estimated_library_size)
            d["percent_duplication"] = float(m.percent_duplication)
            d["roi"] = list(m.roi) if m.has_roi else None
            d["paired_reads_examined"] = int(m.paired_reads_examined)
            hs = []
            for which in range(3):
                n = int(self.L.elp_optical_histogram(self.h, slot, which, None, None, 0))
                if n < 0:
                    raise ElprepError(-1, "elp_optical_histogram failed")
                keys, cnt = np.zeros(n, np.int64), np.zeros(n, np.int64)
                self.L.elp_optical_histogram(self.h, slot, which, _vp(keys), _vp(cnt), n)
                hs.append({int(k): int(v) for k, v in zip(keys, cnt)})
            d["hist"] = hs
            out.append(d)
        return out

    def optical_merge(self, slot, counters=None, hist=None):
        """add another worker's numbers (mergeDuplicatesCtrMaps): counters = 7 ints in DuplicatesCtr order except that
        counters[1] counts paired READS (that worker's paired_reads_examined); hist = 3 dicts"""
        c7 = np.ascontiguousarray(counters, dtype=np.int64) if counters is not None else None
        if c7 is not None:
            self._ck(self.L.elp_optical_merge(self.h, slot, _vp(c7), 0, None, None, 0))
        for which, h in enumerate(hist or []):
            keys = np.array(sorted(h), dtype=np.int64)
            cnt = np.array([h[k] for k in sorted(h)], dtype=np.int64)
            if keys.size:
                self._ck(self.L.elp_optical_merge(self.h, slot, None, which, _vp(keys), _vp(cnt), keys.size))

    def print_duplicates_metrics(self, path, command_line="", started_on=""):
        self._ck(self.L.elp_print_duplicates_metrics(self.h, path.encode(), command_line.encode(), started_on.encode()))

    def bqsr_gather(self):
        self._ck(self.L.elp_bqsr_gather(self.h))

    def table_shape(self):
        return (int(self.L.elp_bqsr_n_cov(self.h)), 94, 1 + (2 * self.max_cycle + 1) + 16, 2)

    def cov_names(self):
        return [self.L.elp_bqsr_cov_name(self.h, i).decode() for i in range(int(self.L.elp_bqsr_n_cov(self.h)))]

    def tables_get(self):
        t = np.zeros(self.table_shape(), dtype=np.int64)
        self._ck(self.L.elp_bqsr_tables_get(self.h, _vp(t), t.size))
        return t

    def tables_put(self, t):
        t = np.ascontiguousarray(t, dtype=np.int64)
        self._ck(self.L.elp_bqsr_tables_put(self.h, _vp(t), t.size))

    # ---- several GPUs: NCCL behind the C ABI (elprep_b200/csrc/comm.cu) ----
    @staticmethod
    def comm_unique_id():
        """rank 0: the 128-byte NCCL id every rank passes to comm_init (ship it with any host channel)"""
        L = _lib.load()
        buf = (C.c_uint8 * 128)()
        rc = L.elp_comm_unique_id(buf)
        if rc != 0:
            raise ElprepError(rc, "elp_comm_unique_id failed (libnccl.so.2 not loadable?)")
        return bytes(buf)

    def comm_init(self, unique_id, rank, world):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._ck(self.L.elp_comm_init(self.h, buf, rank, world))

    def comm_set_partition(self, contig_owner):
        o = np.ascontiguousarray(contig_owner, dtype=np.int32)
        self._ck(self.L.elp_comm_set_partition(self.h, _vp(o)))

    def tables_allreduce(self):
        self._ck(self.L.elp_bqsr_tables_allreduce(self.h))

    def optical_allreduce(self):
        self._ck(self.L.elp_optical_allreduce(self.h))

    def tables_clear(self):
        self._ck(self.L.elp_bqsr_tables_clear(self.h))

    def write_elrecal(self, path):
        """gob of filters.BaseRecalibratorTables, what `--bqsr-tables-only` leaves for the merge step"""
        self._ck(self.L.elp_bqsr_tables_write_elrecal(self.h, path.encode()))

    def add_elrecal(self, path):
        """LoadAndCombineBQSRTables for one file: its counters are added to the context's tables"""
        self._ck(self.L.elp_bqsr_tables_add_elrecal(self.h, path.encode()))

    def optical_write_gob(self, path):
        self._ck(self.L.elp_optical_write_gob(self.h, path.encode()))

    def optical_add_gob(self, path):
        self._ck(self.L.elp_optical_add_gob(self.h, path.encode()))

    def tables_device(self):
        p, n = C.c_void_p(), C.c_uint64()
        self._ck(self.L.elp_bqsr_tables_device(self.h, C.byref(p), C.byref(n)))
        return p.value, int(n.value)

    def bqsr_finalize(self, report_path=None):
        self._ck(self.L.elp_bqsr_finalize(self.h, report_path.encode() if report_path else None))

    def empirical_get(self):
        e = np.zeros(self.table_shape()[:3], dtype=np.uint8)
        self._ck(self.L.elp_bqsr_empirical_get(self.h, _vp(e), e.size))
        return e

    def bqsr_apply(self):
        self._ck(self.L.elp_bqsr_apply(self.h))

    def fetch(self, first=0, n=None, want_qual=True, out=None):
        """returns (record_index u64[n], flag u16[n], qual_off u64[n+1], qual u8[]) for output records [first, first+n)."""
        n = self.n - first if n is None else n
        if out is None:
            qb = int(self.L.elp_fetch_qual_bytes(self.h, first, n)) if want_qual else 0
            out = (np.empty(n, np.uint64), np.empty(n, np.uint16), np.empty(n + 1, np.uint64), np.empty(max(qb, 1), np.uint8))
        idx, flag, qoff, qual = out
        self._ck(self.L.elp_fetch(self.h, first, n, _vp(idx), _vp(flag), _vp(qoff), _vp(qual) if want_qual else None, qual.size))
        return idx, flag, qoff, qual

    def fetch_bam(self, first=0, n=None):
        """-> (uint8 record bytes, uint64 record offsets [n+1]) of output records [first, first+n) (of those that pass the output filter),
        FLAG, MAPQ and QUAL patched"""
        n = self._n_out(first) if n is None else n
        nb = int(self.L.elp_fetch_bam_bytes(self.h, first, n))
        out, off = np.empty(max(nb, 1), np.uint8), np.empty(n + 1, np.uint64)
        self._ck(self.L.elp_fetch_bam(self.h, first, n, _vp(out), out.size, _vp(off)))
        return out[:nb], off

    def fetch_sam(self, first=0, n=None):
        """-> (uint8 SAM text, uint64 line offsets [n+1]) of output records [first, first+n): FormatAlignment of each stored record with
        FLAG, MAPQ and QUAL patched, one '\\n'-terminated alignment line per record, no header (records as in fetch_bam)"""
        n = self._n_out(first) if n is None else n
        nb = int(self.L.elp_fetch_sam_bytes(self.h, first, n)) if n else 0
        out, off = np.empty(max(nb, 1), np.uint8), np.empty(n + 1, np.uint64)
        self._ck(self.L.elp_fetch_sam(self.h, first, n, _vp(out), out.size, _vp(off)))
        return out[:nb], off

    def debug_adapt(self):
        u, s = np.zeros(self.n, np.int32), np.zeros(self.n, np.int32)
        self._ck(self.L.elp_debug_adapt(self.h, _vp(u), _vp(s)))
        return u, s

    def launch_count(self):
        return int(self.L.elp_launch_count(self.h))

    def synchronize(self):
        self._ck(self.L.elp_synchronize(self.h))

    def reset_stats(self):
        self._ck(self.L.elp_reset_stats(self.h))

    def timer_start(self):
        self._ck(self.L.elp_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_double()
        self._ck(self.L.elp_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def kernel_stats(self):
        arr = (_lib.ElpKernelStat * 64)()
        k = self.L.elp_kernel_stats(self.h, arr, 64)
        return {arr[i].name.decode(): dict(launches=int(arr[i].launches), ms=float(arr[i].ms), alg_bytes=float(arr[i].alg_bytes)) for i in range(k)}

    def debug_join_hash(self):
        """per read, the (library, QNAME) hash of the mate join (0 for reads that are not true pairs)"""
        q = np.zeros(self.n, np.uint64)
        self._ck(self.L.elp_debug_join_hash(self.h, _vp(q)))
        return q

    def debug_coord_chunk_keys(self, chunk):
        """per read in arrival order, chunk `chunk` of the coordinate sort's long-tie key (layout in elp_debug_coord_chunk_keys)"""
        k = np.zeros(self.n, np.uint64)
        self._ck(self.L.elp_debug_coord_chunk_keys(self.h, chunk, _vp(k)))
        return k

    def debug_sort_u64(self, keys, vals, key_bits, lo_bit=None):
        """stable sort by bits [lo_bit, lo_bit + key_bits) (lo_bit None: the call without a range)"""
        keys = np.ascontiguousarray(keys, dtype=np.uint64).copy()
        vals = np.ascontiguousarray(vals, dtype=np.uint32).copy()
        if lo_bit is None:
            self._ck(self.L.elp_debug_sort_u64(self.h, _vp(keys), _vp(vals), keys.size, key_bits))
        else:
            self._ck(self.L.elp_debug_sort_u64_range(self.h, _vp(keys), _vp(vals), keys.size, lo_bit, key_bits))
        return keys, vals

    def debug_sort_u128(self, hi, lo, vals, key_bits, lo_bit=None):
        hi = np.ascontiguousarray(hi, dtype=np.uint64).copy()
        lo = np.ascontiguousarray(lo, dtype=np.uint64).copy()
        vals = np.ascontiguousarray(vals, dtype=np.uint32).copy()
        if lo_bit is None:
            self._ck(self.L.elp_debug_sort_u128(self.h, _vp(hi), _vp(lo), _vp(vals), hi.size, key_bits))
        else:
            self._ck(self.L.elp_debug_sort_u128_range(self.h, _vp(hi), _vp(lo), _vp(vals), hi.size, lo_bit, key_bits))
        return hi, lo, vals
