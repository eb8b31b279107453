// ctx.h -- the device context behind the C ABI (include/elprep_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include "common.cuh"
#include "radix_sort.cuh"

// Owners of device and page-locked host memory.  Every allocation has exactly one owner, which frees it when it is destroyed; owners
// move but never copy.  Kernels take the raw pointer (.p), or a trivially copyable argument struct built from raw pointers, never an
// owner.  g_live_allocations counts the allocations all owners of the process hold (elp_debug_live_allocations).
extern std::atomic<int64_t> g_live_allocations;

template <class T, bool PINNED> struct Owned {
    T* p = nullptr;
    size_t cap = 0;   // elements
    Owned() = default;
    Owned(Owned&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    Owned& operator=(Owned&& o) noexcept {
        if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
        return *this;
    }
    ~Owned() { release(); }
    // exactly n elements (the fixed buffers); reallocates, without keeping the contents, only when n exceeds the capacity
    cudaError_t fit(size_t n, unsigned host_flags = cudaHostAllocDefault) {
        if (n <= cap) return cudaSuccess;
        release();
        T* q = nullptr;
        const cudaError_t e = PINNED ? cudaHostAlloc(&q, n * sizeof(T), host_flags) : cudaMalloc(&q, n * sizeof(T));
        if (e != cudaSuccess) return e;
        p = q; cap = n; g_live_allocations++;
        return cudaSuccess;
    }
    void release() {
        if (p) { if (PINNED) cudaFreeHost(p); else cudaFree(p); g_live_allocations--; }
        p = nullptr; cap = 0;
    }
};

// growable device buffer
template <class T> struct DBuf : Owned<T, false> {
    // at least n elements, with room to grow; keeps the first `keep` elements
    cudaError_t reserve(size_t n, cudaStream_t s, size_t keep = 0) {
        if (n <= this->cap) return cudaSuccess;
        DBuf q;
        cudaError_t e = q.fit(n + n / 8 + 64);
        if (e != cudaSuccess) return e;
        if (this->p && keep) { e = cudaMemcpyAsync(q.p, this->p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s); if (e != cudaSuccess) return e; }
        if (this->p) cudaStreamSynchronize(s);
        Owned<T, false>::operator=(std::move(q));
        return cudaSuccess;
    }
};
template <class T> using HBuf = Owned<T, true>;   // page-locked host memory (cudaHostAlloc)

// duplication metrics of one library (filters.DuplicatesCtr, mark-optical-duplicates.go:95-110): the seven counters in the
// reference's field order and the three count histograms (all, non-optical, optical)
struct DupCounters { int64_t ctr[7] = {0, 0, 0, 0, 0, 0, 0}; std::map<int64_t, int64_t> hist[3]; };
#define REFHOT_PAD 512
#define ARENA_FRONT_PAD 64   // QUAL / SEQ arenas start at this offset: kernels read aligned windows that may begin before a read
#define OPT_NCTR 8
#define OPT_HBINS 1024
#define OPT_OVF_CAP (1 << 16)

// Per-contig table on the device, indexed by REFID: the interval tables (RegionTable: per contig the flattened, start-sorted (start, end)
// pairs, n counts pairs) and the reference (per contig the one-hot nibbles, d at the payload, n counts bases).  d[i] is the view of contig
// i (null: nothing).  It points into own[i], the buffer elp_set_* made for that contig, or into `block`, the one allocation the last
// elp_load_* filled for every contig; the block lives until the next load or the context's end, whatever elp_set_* replaced since.
// The kernels read the views through d_ptrs and d_n, uploaded when dirty (table_upload).
template <class T> struct ContigTable {
    std::vector<T*> d; std::vector<uint64_t> n;
    std::vector<DBuf<T>> own;
    DBuf<T> block;
    DBuf<const T*> d_ptrs; DBuf<uint64_t> d_n;
    bool dirty = true;
    void resize(int nc) { d.assign(nc, nullptr); n.assign(nc, 0); own.clear(); own.resize(nc); dirty = true; }
    // contig i loses its view and its own buffer (elp_set_* then allocates own[i] and points d[i] into it)
    void clear(int i) { own[i].release(); d[i] = nullptr; n[i] = 0; dirty = true; }
    // every contig replaced by the views into b (elp_load_*)
    void install(DBuf<T>&& b, std::vector<T*>&& views, std::vector<uint64_t>&& counts) {
        block = std::move(b); own.clear(); own.resize(views.size());
        d = std::move(views); n = std::move(counts); dirty = true;
    }
};
using RegionTable = ContigTable<int32_t>;

// "*" and every @SQ SN, sorted bytewise.  id: the refid of dictTable / AddREFID ("*" -> -1, an @SQ SN -> its index, the last of equal
// names wins).  all[all_off[e], all_off[e + 1]): every @SQ index with entry e's name, in header order ("*" has none).  The view the
// kernels take (text_parse.cuh name_entry, refid_of).
struct NameDict {
    uint8_t* names = nullptr; uint32_t* off = nullptr; int32_t* id = nullptr;
    uint32_t* all_off = nullptr; int32_t* all = nullptr;
    int n = 0;
};
// its owner: one per context, uploaded on first use (name_dict_upload, text_parse.cuh) by elp_append_sam and elp_load_known_sites
struct NameDictBufs {
    DBuf<uint8_t> names; DBuf<uint32_t> off; DBuf<int32_t> id; DBuf<uint32_t> all_off; DBuf<int32_t> all;
    int n = 0;   // entries; 0 until uploaded
    NameDict view() const { return NameDict{names.p, off.p, id.p, all_off.p, all.p, n}; }
};

// the radix sort's device workspace (sort.cu)
struct SortWorkspace {
    DBuf<uint32_t> ghist, gofs;   // [MAX_PASSES][RADIX]
    DBuf<uint32_t> counters;      // [MAX_PASSES]
    DBuf<uint32_t> status;        // [passes][tiles][RADIX]
};

// State of a module that the context owns through a StatePtr; each module defines free_state for its type, where the type is complete.
struct SamState; struct SamOutState; struct BgzfStream; struct DeflateState; struct SitesStage; struct RelabelState;
void free_state(SamState* p); void free_state(SamOutState* p); void free_state(BgzfStream* p); void free_state(DeflateState* p); void free_state(SitesStage* p);
void free_state(RelabelState* p);
struct FreeState { template <class T> void operator()(T* p) const { free_state(p); } };
template <class T> using StatePtr = std::unique_ptr<T, FreeState>;

struct KernelStat { uint64_t launches = 0; double ms = 0, alg_bytes = 0; };
struct PendingEvent { std::string name; cudaEvent_t a, b; double alg_bytes; };

// dense BQSR table geometry: [n_cov][94][1 + (2*max_cycle+1) + 16][2]
struct TableGeom {
    int n_cov = 0, max_cycle = 500;
    __host__ __device__ int ncols() const { return 1 + (2 * max_cycle + 1) + 16; }
    __host__ __device__ size_t cells() const { return (size_t)n_cov * 94 * ncols(); }
    __host__ __device__ size_t idx(int cov, int q, int col) const { return ((size_t)cov * 94 + q) * ncols() + col; }
    __host__ __device__ int col_cycle(int cyc) const { return 1 + cyc + max_cycle; }
    __host__ __device__ int col_ctx(int ctx) const { return 1 + (2 * max_cycle + 1) + ctx; }
};

struct elp_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_in = nullptr, copy_out = nullptr;   // upload / download streams of the asynchronous append / fetch
    cudaEvent_t ev_in = nullptr, ev_staged = nullptr, ev_out = nullptr;
    HBuf<uint8_t> h_stage; size_t stage_off = 0;         // page-locked staging of upload_small
    std::string err;
    std::mutex append_mu;
    bool profile = false;

    // ---- header-derived ----
    int n_contigs = 0;
    std::vector<int32_t> contig_len;
    std::vector<std::string> contig_names;
    int n_rg = 0;
    std::vector<int32_t> rg_lib, rg_cov;       // per @RG
    int n_lib = 0;
    std::vector<std::string> cov_names;
    std::vector<std::string> lib_names;       // [n_lib]
    int max_cycle = 500, quantize_levels = 0, optical_pixel_distance = 100;
    std::vector<uint8_t> sqq;
    std::string prefix = "GATK";
    DBuf<int32_t> d_rg_lib;          // [n_rg]
    DBuf<int32_t> d_rg_cov;          // [n_rg]
    DBuf<int32_t> d_contig_len;      // [n_contigs]

    // ---- reference genome + known sites (device) ----
    ContigTable<uint8_t> ref;                // elp_set_reference / elp_load_reference: one-hot nibbles (bqsr_gather.cu pack_reference), REFHOT_PAD
                                             // bytes in front of each view and 64 behind; n: the contig's bases
    uint64_t ref_chunk = 0;                  // elp_debug_set_reference_chunk: bytes per staging chunk of elp_load_reference (0: the default)
    RegionTable known_sites;                 // elp_set_known_sites / elp_load_known_sites (survives elp_reset)
    StatePtr<SitesStage> sites;              // page-locked and device staging of elp_load_known_sites (known_sites.cu)
    uint64_t sites_chunk = 0;                // elp_debug_set_sites_chunk: bytes per staging chunk (0: the default)

    // ---- reads, arrival order (SoA columns) ----
    uint64_t n = 0, n_qname = 0, n_cigar = 0, n_qual = 0, n_seq = 0;
    DBuf<int32_t> refid, pos, nref, pnext, tlen, rg;
    DBuf<uint16_t> flag;
    DBuf<uint8_t> mapq;
    DBuf<uint8_t> optf;                       // elp_batch.opt_flags (ELP_OPT_SR ...)
    DBuf<uint64_t> qname_off, cigar_off, qual_off, seq_off;   // [n+1]
    DBuf<uint8_t> qname, seq, qual;
    DBuf<uint32_t> cigar;
    DBuf<uint8_t> bam_raw; DBuf<uint64_t> bam_off;   // staging of elp_append_bam: raw records and their offsets
    DBuf<uint8_t> bam_all; DBuf<uint64_t> bam_all_off; uint64_t n_bam = 0, bam_reads = 0;   // all raw records (for elp_fetch_bam) and the start of every read's record
    DBuf<uint64_t> bam_start;                 // starts of the records that pass the ingest filters
    uint32_t filter_mask = 0; int32_t filter_min_mapq = 0; uint64_t n_filtered = 0;   // elp_set_ingest_filter (record predicates)
    bool clear_dup = false;                   // elp_set_ingest_filter ELP_FILTER_CLEAR_DUPLICATE_FLAG: 0x400 cleared in the FLAG column at ingest
    // write-phase filters of elp_fetch_bam / elp_fetch_sam (elp_set_output_filter; survive elp_reset)
    uint32_t out_mask = 0;                    // record bits (ELP_OUT_REMOVE_DUPLICATES, ELP_OUT_REMOVE_OPTIONAL_READS)
    DBuf<uint32_t> d_out_drop; bool out_fields = false;        // 65 536-bit tag table (bit set: the field is dropped); out_fields: some bit is set
    DBuf<uint32_t> out_sel; uint64_t n_out = 0; bool out_sel_valid = false;   // output positions of the records that pass, built on first use
    bool rg_replace = false;                 // --replace-read-group (elp_set_replace_read_group; survives elp_reset): every read is in @RG 0 and
                                             // the byte outputs write its RG field as RG:Z:rg_ids[0] (d_rg_names)
    // --rename-chromosomes / --replace-reference-sequences (elp_set_input_dictionary; survives elp_reset).  elp_config holds the output
    // dictionary; the input's @SQ (in_len, unrenamed) bounds the stored records' refID / next_refID.  The input name table is the input's
    // names followed by the SAM extension (REPLACE only: the RNAME texts that reach a replacement entry without being an input name);
    // d_remap[table index] is the output contig (-1: none), with one more entry, -1, for a SAM RNAME that reaches nothing under REPLACE.
    uint32_t dict_mode = 0;                  // ELP_DICT_* bits; 0: off
    std::vector<std::string> in_tab;         // the input name table as the file spells it (the extension included)
    std::vector<int32_t> in_len;             // [n_in] LN of the input's @SQ
    int n_in = 0;                            // input @SQ entries
    DBuf<int32_t> d_remap;                   // [in_tab.size() + 1]
    DBuf<int32_t> d_clean_len;               // [n_contigs] CleanSam's LN per output contig: the input LN of its name (last entry), else 0
    NameDictBufs in_dict;                    // elp_append_sam's RNAME / RNEXT lookup over in_tab while dict_mode is set (built on first use)
    // several input files (elp_add_input / elp_select_input / elp_set_tag_rename; survive elp_reset).  elp_config holds the merged header;
    // each input's @SQ maps to the merged dictionary, and the composed RG / PG maps of the merge rename the first RG / PG value of every
    // record.  While any of them is set, every appended record is rewritten at ingest (merge_inputs.cu: relabel_records).
    struct InputDict { std::vector<std::string> names; std::vector<int32_t> len, remap; };   // @SQ SN / LN, merged index of each SN
    std::vector<InputDict> inputs;
    int cur_input = -1;                      // elp_select_input
    std::vector<std::pair<std::string, std::string>> tag_ren[2];   // old -> new value: [0] RG, [1] PG
    StatePtr<RelabelState> relabel;          // device tables and staging of the rewrite (merge_inputs.cu)
    RegionTable regions;                     // --filter-non-overlapping-reads: the ingest filter ELP_FILTER_TARGET_REGIONS (elp_set_target_regions)
    RegionTable bqsr_regions;                // --target-regions: elp_filter_target_regions after marking (elp_set_bqsr_target_regions); both survive elp_reset
    uint64_t n_cleaned = 0;                  // reads whose CIGAR elp_clean_sam rewrote
    bool has_contig_names = false;           // elp_config.contig_names was given (elp_append_sam resolves RNAME / RNEXT against it)
    StatePtr<SamState> sam;                  // device staging of elp_append_sam (sam_ingest.cu)
    NameDictBufs names;                      // RNAME / RNEXT and known-sites chromosome dictionary
    uint64_t n_sam_lost_names = 0;           // reads of elp_append_sam whose RNAME / RNEXT text the stored record cannot reproduce (elp_fetch_sam refuses)
    StatePtr<SamOutState> sam_out;           // @SQ names and float staging of elp_fetch_sam (sam_format.cu)
    StatePtr<BgzfStream> bgzf;               // carried bytes and device staging of elp_append_bgzf / elp_debug_inflate (bgzf_inflate.cu)
    StatePtr<DeflateState> bgzf_out;         // device scratch of elp_fetch_bgzf / elp_debug_deflate (bgzf_deflate.cu)
    bool bgzf_open = false;                  // a BGZF file is open (elp_append_bgzf until elp_append_bgzf_end or elp_reset): the other appends
                                             // and elp_sort_markdup refuse, as the file's records are not all in yet
    DBuf<uint8_t> d_rg_names; DBuf<uint32_t> d_rg_name_off; std::vector<std::string> rg_ids;   // @RG IDs for the RG:Z match
    DBuf<int32_t> lseq_stage;       // staging for l_seq of the batch being appended
    DBuf<uint64_t> off_stage;       // staging for batch-relative offsets

    // ---- per-read temps (arrival order) ----
    DBuf<int32_t> upos, score;
    DBuf<uint64_t> qhash;
    DBuf<DeviceRanges> d_ranges;
    DeviceRanges h_ranges{};
    DBuf<uint32_t> d_err;            // device error word
    bool adapted = false;

    // ---- sort scratch ----
    DBuf<uint64_t> keys_a, keys_b;           // u64 keys, or u128 keys as pairs (2 words per key)
    DBuf<uint32_t> vals_a, vals_b;
    SortWorkspace ws;
    DBuf<uint32_t> mate;                      // [n] mate index or 0xffffffff
    DBuf<uint32_t> pair_a, pair_b, scan_tmp, scan_blk;
    DBuf<int32_t> pair_score;                 // [npairs] summed phred score of both mates of a pair (duplicate marking)
    DBuf<uint64_t> tie_bits;                  // [2][chunks] OR and AND of each chunk key over the long tie runs (coordinate sort)
    DBuf<uint8_t> bytes_tmp;
    DBuf<uint4> bq_recs, bq_segs;             // BQSR count kernel: work records of the eligible reads, segment table
    DBuf<uint32_t> d_bq_small;                // class histogram, region bases, list counters, segment counts, work-queue heads
    DBuf<uint32_t> d_qpresent;                // [4] bit q set iff QUAL value q (0..127) occurs in the arena (maintained at ingest)
    uint32_t h_qpresent[4] = {0, 0, 0, 0};    // its host copy, taken with h_ranges (phase_adapt, elp_filter_target_regions)

    // ---- output order ----
    bool sorted = false;                      // columns below valid
    uint64_t n_sorted = 0;                    // records in output order: n after the sort, the kept reads after elp_filter_target_regions
    DBuf<uint32_t> perm;                      // [n_sorted] arrival index of k-th output record
    DBuf<int32_t> s_refid, s_pos, s_nref, s_pnext, s_tlen, s_rg, s_lseq;
    DBuf<uint16_t> s_flag;
    DBuf<uint8_t> s_mapq, s_optf;
    DBuf<uint64_t> s_qual_off, s_seq_off, s_cigar_off, s_out_off;   // s_out_off[n+1]: offsets of the output qual stream
    DBuf<uint32_t> s_ncigar;
    DBuf<uint8_t> qual_out;                   // recalibrated QUAL in output order
    bool qual_out_valid = false;
    uint64_t qual_out_total = 0;              // bytes of the output QUAL stream

    // ---- BQSR ----
    TableGeom geom;
    DBuf<int64_t> d_tables;                   // dense [cells][2]
    DBuf<uint8_t> d_emp;                      // [cells] EmpiricalQuality (elp_bqsr_finalize)
    DBuf<double> d_fin;                       // [n_cov][2] reported quality of the combined read-group entry, read-group term dG
    DBuf<uint8_t> d_qmaps;                    // quantization map [0, 94), static --sqq map at [96, 350) (bqsr_finalize.cu)
    bool gathered = false, finalized = false;
    uint64_t gather_eligible = 0;             // reads the last elp_bqsr_gather recalibrated (what the roofline line charges)
    DBuf<uint8_t> d_lut;                      // [n_cov][94][2*lut_maxcyc+1][17]
    int lut_maxcyc = 0;
    DBuf<uint8_t> d_cov_exists;               // [n_cov]
    DBuf<uint8_t> d_unobs;                    // [n_cov] recalibrated byte of a QUAL value without table entries (QUAL 94..255)
    DBuf<uint8_t> d_clut; DBuf<uint16_t> d_rowtab;   // compact apply table for the shared-memory kernel: [cycle][covariate][slot][17], QUAL -> slot offset
    uint32_t clut_bytes = 0, clut_blk = 0, clut_S17 = 0; int clut_Lc = 0; uint32_t clut_present[4] = {0, 0, 0, 0};

    // ---- duplication metrics (optical.cu) ----
    DBuf<unsigned long long> d_opt_ctr, d_opt_hist, d_opt_ovf; DBuf<uint32_t> d_opt_small;
    std::vector<DupCounters> opt;             // [n_lib + 1], slot 0 = "Unknown Library"
    bool opt_valid = false;

    // ---- several GPUs (comm.cu) ----
    void* comm = nullptr;                     // ncclComm_t
    int rank = 0, world = 1;
    DBuf<int32_t> d_owner;                    // [n_contigs] rank owning each contig
    uint64_t n_ghost = 0, sp_sent_total = 0;  // visiting mates appended behind the local reads during duplicate marking; records this rank sent
    std::vector<uint32_t> sp_send, sp_recv;   // records to / from every rank
    DBuf<uint4> sp_sendbuf, sp_recvbuf; DBuf<uint32_t> sp_sent_idx;
    bool any_rank_entering = true;

    // ---- measurement ----
    uint64_t launches = 0;
    std::map<std::string, KernelStat> stats;
    std::vector<PendingEvent> pending;
    std::vector<cudaEvent_t> event_pool;
    cudaEvent_t timer_a = nullptr, timer_b = nullptr;

    ~elp_ctx();   // api.cu: the streams and events; the owners free the memory

    int fail(int code, const char* fmt, ...) {
        char buf[1024];
        va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
        err = buf;
        return code;
    }
    // bracket one kernel launch: counts it and, when profiling, records a CUDA-event pair on the launching stream
    cudaEvent_t get_event() {
        if (!event_pool.empty()) { cudaEvent_t e = event_pool.back(); event_pool.pop_back(); return e; }
        cudaEvent_t e; cudaEventCreate(&e); return e;
    }
    void begin(const char* name, double alg_bytes) {
        launches++;
        if (!profile) return;
        PendingEvent pe; pe.name = name; pe.alg_bytes = alg_bytes; pe.a = get_event(); pe.b = get_event();
        cudaEventRecord(pe.a, stream);
        pending.push_back(pe);
    }
    void end() {
        if (!profile) return;
        cudaEventRecord(pending.back().b, stream);
    }
    void set_pending_bytes(const char* name, double bytes) { for (auto& pe : pending) if (pe.name == name) pe.alg_bytes = bytes; }
    void resolve_events() {
        if (pending.empty()) return;
        cudaStreamSynchronize(stream);
        for (auto& pe : pending) {
            float ms = 0; cudaEventElapsedTime(&ms, pe.a, pe.b);
            KernelStat& s = stats[pe.name]; s.launches++; s.ms += ms; s.alg_bytes += pe.alg_bytes;
            event_pool.push_back(pe.a); event_pool.push_back(pe.b);
        }
        pending.clear();
    }
};

#define CUDA_TRY(ctx, call)                                                                                   \
    do {                                                                                                      \
        cudaError_t e__ = (call);                                                                             \
        if (e__ != cudaSuccess) return (ctx)->fail(E_CUDA, "CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, cudaGetErrorString(e__)); \
    } while (0)

#define LAUNCH_CHECK(ctx) CUDA_TRY(ctx, cudaGetLastError())
#define TRY(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)

inline unsigned nblk(uint64_t n, int t) { return (unsigned)((n + t - 1) / t); }

template <class T> int grow(elp_ctx* c, DBuf<T>& b, size_t need, size_t keep = 0) {
    cudaError_t e = b.reserve(need, c->stream, keep);
    if (e != cudaSuccess) return c->fail(e == cudaErrorMemoryAllocation ? E_NOMEM : E_CUDA, "device allocation of %zu bytes failed: %s", need * sizeof(T), cudaGetErrorString(e));
    return E_OK;
}

// the views and counts of a per-contig table -> d_ptrs / d_n.  Uploads go on the context's stream and are waited for: a pageable cudaMemcpy
// may return before its DMA has landed, and the (non-blocking) stream of the kernels that read the table does not wait for it.
template <class T> int table_upload(elp_ctx* c, ContigTable<T>& t) {
    if (!t.dirty) return E_OK;
    const size_t nc = std::max(1, c->n_contigs);
    CUDA_TRY(c, t.d_ptrs.fit(nc)); CUDA_TRY(c, t.d_n.fit(nc));
    if (c->n_contigs) {
        CUDA_TRY(c, cudaMemcpyAsync(t.d_ptrs.p, t.d.data(), c->n_contigs * sizeof(void*), cudaMemcpyHostToDevice, c->stream));
        CUDA_TRY(c, cudaMemcpyAsync(t.d_n.p, t.n.data(), c->n_contigs * 8, cudaMemcpyHostToDevice, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    t.dirty = false;
    return E_OK;
}

// ---- internal phase entry points (implemented in the .cu files) ----
// stable sort by key bits [lo_bit, lo_bit + key_bits); the bits below lo_bit do not take part in the order
int radix_sort_u32(elp_ctx* c, uint32_t* keys_a, uint32_t* keys_b, uint32_t* vals_a, uint32_t* vals_b, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit = 0);
int radix_sort_u64(elp_ctx* c, uint64_t* keys_a, uint64_t* keys_b, uint32_t* vals_a, uint32_t* vals_b, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit = 0);
int radix_sort_u128(elp_ctx* c, uint64_t* keys_a, uint64_t* keys_b, uint32_t* vals_a, uint32_t* vals_b, uint64_t n, int key_bits, bool* result_in_b, const char* tag, int lo_bit = 0);
int exclusive_scan_u32_to_u64(elp_ctx* c, const uint32_t* in, uint64_t* out, uint64_t n);   // out[n+1]
int exclusive_scan_u64(elp_ctx* c, const uint64_t* in, uint64_t* out, uint64_t n, uint64_t base);          // out[n+1], out[0]=base
int phase_adapt(elp_ctx* c);
int phase_markdup(elp_ctx* c, bool optical);
int phase_optical(elp_ctx* c, uint64_t npairs, const uint64_t* sorted_keys, const uint32_t* sorted_vals, int key_words);   // key_words: 1 (u64 keys) or 2 (u128 as lo,hi)
int phase_coordinate_sort(elp_ctx* c, int order);   // 0 keep, 1 coordinate, 2 queryname
int phase_bqsr_gather(elp_ctx* c);
int phase_bqsr_finalize(elp_ctx* c, const char* report_path);
int phase_bqsr_apply(elp_ctx* c);
int build_apply_lut(elp_ctx* c, int Lc);   // bqsr_finalize.cu
int build_compact_lut(elp_ctx* c);
int bqsr_empirical_copy(elp_ctx* c, uint8_t* emp);   // device EmpiricalQuality -> host (synchronises)
int pack_reference(elp_ctx* c, int contig, const uint8_t* bases, uint64_t n);   // bases: n host bytes
int check_device_errors(elp_ctx* c);
int upload_small(elp_ctx* c, void* dst, const void* src, size_t bytes);   // api.cu: host -> device without the copy engine
int comm_allreduce_ranges(elp_ctx* c, int local_rc);   // comm.cu: returns local_rc, or a peer's error code
int spread_exchange_begin(elp_ctx* c);
int spread_exchange_end(elp_ctx* c);
int exclusive_scan_u64_from_u32(elp_ctx* c, const uint32_t* in, uint64_t* out, uint64_t n, uint64_t base);   // out[n+1], out[0] = base
int qual_presence_update(elp_ctx* c, uint64_t first_byte, uint64_t n_bytes);   // api.cu: called by both ingest paths
int bam_ingest_core(elp_ctx* c, uint64_t n_bytes, uint64_t nrec, bool sam_records = false);   // bam_ingest.cu: records staged in bam_raw / bam_off -> reads (elp_append_bam, elp_append_sam)
// elp_set_input_dictionary: the refID bound of the stored records (BAM: the input's @SQ; elp_append_sam's records: its name table and the
// unreached-name entry), the remap table (null while off), and whether bam_keep_kernel runs (a record predicate or the REPLACE drop)
inline int ingest_ref_bound(const elp_ctx* c, bool sam_records) { return c->dict_mode ? (sam_records ? (int)c->in_tab.size() + 1 : c->n_in) : c->n_contigs; }
inline const int32_t* ingest_remap(const elp_ctx* c) { return c->dict_mode ? c->d_remap.p : nullptr; }
inline bool ingest_keep_on(const elp_ctx* c) { return c->filter_mask || c->filter_min_mapq > 0 || (c->dict_mode & 2u /* ELP_DICT_REPLACE */); }
int out_select(elp_ctx* c, const uint32_t** sel, uint64_t* n_out);
int rg_names_upload(elp_ctx* c);   // bam_ingest.cu: @RG IDs -> d_rg_names / d_rg_name_off, once per context   // bam_ingest.cu: the record filters' selection (sel null and n_out = n_sorted without record bits)
std::vector<std::string> sam_print_names(const elp_ctx* c);
// merge_inputs.cu: whether appended records are rewritten; the refID bound of the selected input's records; ELP_ESTATE when inputs exist
// and none is selected; the rewrite itself (raw / off / n_bytes in and out)
bool relabel_on(const elp_ctx* c);
int relabel_ref_bound(const elp_ctx* c);
int relabel_check_selected(elp_ctx* c, const char* who);
int relabel_records(elp_ctx* c, const uint8_t** raw, uint64_t* off, uint64_t* n_bytes, uint64_t nrec, bool sam_records);   // bam_ingest.cu: the names elp_fetch_sam prints for the stored refIDs
int region_set(elp_ctx* c, RegionTable& t, const char* who, int32_t contig, const int32_t* se, uint64_t n_intervals, int already_flat);   // bam_ingest.cu
int build_output_columns(elp_ctx* c, const uint32_t* perm, uint64_t n_out, bool refilter);   // coordsort.cu: s_* columns and s_out_off of perm[0, n_out)
int phase_target_filter(elp_ctx* c, uint64_t* n_removed);   // target_regions.cu
void bgzf_stream_reset(elp_ctx* c);   // bgzf_inflate.cu: forget the open file (elp_reset)
struct BgzfBlock;
int bgzf_inflate_run(elp_ctx* c, const char* who, const uint8_t* in, uint64_t n_in, const std::vector<BgzfBlock>& blocks, uint64_t total, uint8_t* out);   // bgzf_inflate.cu: whole blocks -> out
int bgzf_deflate_run(elp_ctx* c, const uint8_t* in, uint64_t n, int write_eof, uint8_t* out, uint64_t* out_n);   // bgzf_deflate.cu: in[0, n) on the device -> BGZF at out
