// merge_inputs.cu -- several input files in one context, as `elprep filter` / `elprep sfm` take a directory of inputs
// (sam.MergeInputs, sam/merge-inputs.go:16-219; sam/split-merge.go:230-311).
//
// The caller merges the input headers on the host (elprep_b200.sam.MergeInputs, elprep::MergeInputs) and creates the context from the
// merged header.  It then describes each file's @SQ (elp_add_input), selects the file it is about to append (elp_select_input), and
// hands over the composed RG / PG value maps of the merge's update filters (elp_set_tag_rename).
//
// Every record of an append is rewritten on the device, before the ingest filters see it, into the record the reference writes with
// the merged header: refID and next_refID through the selected input's map to the merged dictionary, and the value of the first RG and
// PG field through the rename maps (aln.SetRG / SetPG: SmallMap.Set in place, block_size rewritten).  From then on the records are
// those of a file with the merged header: the ingest filters, the RG column, CleanSam, the stored records of elp_fetch_bam / _bgzf /
// _sam and the output field filter work on them unchanged.  Two kernels:
//   relabel_measure_kernel  one thread per record: the record's structure, the spans of the values it replaces, its new length
//   relabel_emit_kernel     one warp per record: the bytes at their new offsets, block_size and refIDs patched
// A record the measure finds malformed is copied as it is, so that bam_ingest_core refuses it as it would without this pass.
#include <algorithm>
#include <map>
#include <set>
#include "ctx.h"
#include "../../include/elprep_b200.h"

namespace {

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

constexpr int BAM_FIXED = 36;

// the values of one record that the rewrite replaces, in record order: [a, e) is the old value (behind the type byte, before the NUL),
// s the rename entry that gives the new one (-1: none; then a = e = the record's length).  ok: the record is well-formed and is rewritten.
struct Sub { uint32_t a, e; int32_t s; };
struct Relabel { Sub x[2]; uint32_t ok; };

struct RelabelArgs {
    uint64_t n; const uint8_t* raw; const uint64_t* off;       // records and their offsets (off[n] = bytes)
    const int32_t* remap; int n_sq;                             // the selected input's @SQ -> merged index, or null (SAM records)
    const uint8_t* ren; const uint32_t* ren_off; int n_ren[2];  // rename entries: old / new value of entry k at 2k / 2k + 1; RG first
    Relabel* sub; uint32_t* len;                                // [n] per record
    const uint64_t* new_off; uint8_t* out;                      // emit
    uint32_t* err;
};

// index of the entry of tag t (0 RG, 1 PG) whose old value is r[a, e), or -1
__device__ int32_t ren_find(const RelabelArgs& A, int t, const uint8_t* r, uint32_t a, uint32_t e) {
    const int first = t ? A.n_ren[0] : 0, last = first + A.n_ren[t];
    for (int k = first; k < last; k++) {
        const uint32_t s = A.ren_off[2 * k], l = A.ren_off[2 * k + 1] - s;
        if (l != e - a) continue;
        bool same = true;
        for (uint32_t q = 0; q < l && same; q++) same = A.ren[s + q] == r[a + q];
        if (same) return k;
    }
    return -1;
}

__global__ void __launch_bounds__(256) relabel_measure_kernel(RelabelArgs A) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const uint64_t st = A.off[i], rec = A.off[i + 1] - st;
    const uint8_t* r = A.raw + st;
    Relabel R{};
    R.x[0] = R.x[1] = Sub{(uint32_t)rec, (uint32_t)rec, -1};
    bool ok = rec >= BAM_FIXED && rec < (1ull << 32) && (uint64_t)rd32(r) + 4 == rec;
    if (ok) {   // the structure as check_record (bam_ingest.cu) reads it
        const uint32_t l_name = r[12], n_cig = rd16(r + 16);
        const int32_t l_seq = (int32_t)rd32(r + 20);
        const uint64_t lsq = l_seq < 0 ? 0ull : (uint64_t)(uint32_t)l_seq;
        uint64_t x = BAM_FIXED + (uint64_t)l_name + 4ull * n_cig + ((lsq + 1) >> 1) + lsq;
        ok = l_name >= 1 && l_seq >= 0 && lsq <= rec && x <= rec;
        bool seen[2] = {false, false};
        int ns = 0;
        while (ok && x + 3 <= rec) {
            const uint8_t t0 = r[x], t1 = r[x + 1], ty = r[x + 2];
            const int t = (t0 == 'R' && t1 == 'G') ? 0 : ((t0 == 'P' && t1 == 'G') ? 1 : -1);
            x += 3;
            uint64_t sz = 0; bool str = false;
            switch (ty) {
                case 'A': case 'c': case 'C': sz = 1; break;
                case 's': case 'S': sz = 2; break;
                case 'i': case 'I': case 'f': sz = 4; break;
                case 'Z': case 'H': str = true; break;
                case 'B': {
                    if (x + 5 > rec) { ok = false; break; }
                    const uint8_t sub = r[x]; const uint64_t cnt = rd32(r + x + 1);
                    const uint64_t es = (sub == 'c' || sub == 'C') ? 1 : ((sub == 's' || sub == 'S') ? 2 : ((sub == 'i' || sub == 'I' || sub == 'f') ? 4 : 0));
                    if (!es || cnt * es > rec) { ok = false; break; }
                    sz = 5 + cnt * es; break;
                }
                default: ok = false;
            }
            if (!ok) break;
            uint64_t e = x + sz;
            if (str) { e = x; while (e < rec && r[e] != 0) e++; if (e >= rec) { ok = false; break; } }
            else if (e > rec) { ok = false; break; }
            // aln.TAGS.Get finds the first field of the tag; the filter's rID.(string) panics on any other type than Z
            if (t >= 0 && !seen[t] && A.n_ren[t]) {
                seen[t] = true;
                if (ty != 'Z') atomicOr(A.err, DERR_BAM_TAGTYPE);
                else {
                    const int32_t s = ren_find(A, t, r, (uint32_t)x, (uint32_t)e);
                    if (s >= 0) R.x[ns++] = Sub{(uint32_t)x, (uint32_t)e, 2 * s + 1};
                }
            }
            x = str ? e + 1 : e;
        }
        ok = ok && x == rec;
    }
    if (ok && A.remap) {
        const int32_t refid = (int32_t)rd32(r + 4), nref = (int32_t)rd32(r + 24);
        if (refid >= A.n_sq || nref >= A.n_sq) { atomicOr(A.err, DERR_BAM_INPUT_REF); ok = false; }
    }
    uint64_t m = rec;
    if (!ok) R.x[0] = R.x[1] = Sub{(uint32_t)rec, (uint32_t)rec, -1};
    for (int k = 0; k < 2; k++) if (R.x[k].s >= 0) m = m - (R.x[k].e - R.x[k].a) + (A.ren_off[R.x[k].s + 1] - A.ren_off[R.x[k].s]);
    R.ok = ok;
    A.sub[i] = R; A.len[i] = (uint32_t)m;
}

// one warp per record: output byte j comes from the record, a new value, the record behind the first replaced value, the second new value,
// or the record behind the second replaced value
__global__ void __launch_bounds__(256) relabel_emit_kernel(RelabelArgs A) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= A.n) return;
    const uint8_t* r = A.raw + A.off[i];
    const uint64_t ob = A.new_off[i], m = A.new_off[i + 1] - ob;
    uint8_t* o = A.out + ob;
    const Relabel R = A.sub[i];
    const uint8_t* v0 = A.ren + (R.x[0].s >= 0 ? A.ren_off[R.x[0].s] : 0);
    const uint8_t* v1 = A.ren + (R.x[1].s >= 0 ? A.ren_off[R.x[1].s] : 0);
    const uint32_t l0 = R.x[0].s >= 0 ? A.ren_off[R.x[0].s + 1] - A.ren_off[R.x[0].s] : 0;
    const uint32_t l1 = R.x[1].s >= 0 ? A.ren_off[R.x[1].s + 1] - A.ren_off[R.x[1].s] : 0;
    int32_t ids[2] = {0, 0};
    if (R.ok && A.remap) {
        for (int k = 0; k < 2; k++) { const int32_t id = (int32_t)rd32(r + (k ? 24 : 4)); ids[k] = id < 0 ? id : A.remap[id]; }
    }
    for (uint64_t j = lane; j < m; j += 32) {
        uint8_t v;
        if (j < R.x[0].a) v = r[j];
        else if (j < R.x[0].a + l0) v = v0[j - R.x[0].a];
        else {
            const uint64_t q = j - R.x[0].a - l0 + R.x[0].e;                 // position in the record behind the first value
            if (q < R.x[1].a) v = r[q];
            else if (q < R.x[1].a + l1) v = v1[q - R.x[1].a];
            else v = r[q - R.x[1].a - l1 + R.x[1].e];
        }
        if (R.ok) {
            if (j < 4) v = (uint8_t)((uint32_t)(m - 4) >> (8 * j));
            else if (A.remap && ((j >= 4 && j < 8) || (j >= 24 && j < 28))) v = (uint8_t)((uint32_t)ids[j >= 24] >> (8 * (j & 3)));
        }
        o[j] = v;
    }
}

}  // namespace

struct RelabelState {
    DBuf<uint8_t> ren; DBuf<uint32_t> ren_off;   // the rename entries (elp_set_tag_rename), uploaded on first use
    bool uploaded = false;
    DBuf<int32_t> remap; int remap_input = -1;   // the map of input remap_input
    DBuf<Relabel> sub; DBuf<uint32_t> len;
    DBuf<uint8_t> raw; DBuf<uint64_t> off;       // the rewritten records of the call
};
void free_state(RelabelState* S) { delete S; }

static RelabelState& relabel_state(elp_ctx* c) {
    if (!c->relabel) c->relabel.reset(new RelabelState());
    return *c->relabel;
}

bool relabel_on(const elp_ctx* c) { return !c->inputs.empty() || !c->tag_ren[0].empty() || !c->tag_ren[1].empty(); }

int relabel_ref_bound(const elp_ctx* c) { return c->inputs.empty() ? c->n_contigs : (int)c->inputs[c->cur_input].len.size(); }

int relabel_check_selected(elp_ctx* c, const char* who) {
    if (!c->inputs.empty() && c->cur_input < 0) return c->fail(E_STATE, "%s: the context has inputs (elp_add_input) but none is selected (elp_select_input)", who);
    return E_OK;
}

// nrec records at raw / off (off[nrec] = *n_bytes) -> their rewritten form in the state's raw; off is overwritten with the new offsets
int relabel_records(elp_ctx* c, const uint8_t** raw, uint64_t* off, uint64_t* n_bytes, uint64_t nrec, bool sam_records) {
    RelabelState& S = relabel_state(c);
    cudaStream_t s = c->stream;
    if (!S.uploaded) {
        std::vector<uint8_t> b; std::vector<uint32_t> o(1, 0);
        for (int t = 0; t < 2; t++)
            for (auto& kv : c->tag_ren[t]) {
                b.insert(b.end(), kv.first.begin(), kv.first.end()); o.push_back((uint32_t)b.size());
                b.insert(b.end(), kv.second.begin(), kv.second.end()); o.push_back((uint32_t)b.size());
            }
        CUDA_TRY(c, S.ren.fit(std::max<size_t>(b.size(), 1))); CUDA_TRY(c, S.ren_off.fit(o.size()));
        if (!b.empty()) CUDA_TRY(c, cudaMemcpyAsync(S.ren.p, b.data(), b.size(), cudaMemcpyHostToDevice, s));
        CUDA_TRY(c, cudaMemcpyAsync(S.ren_off.p, o.data(), o.size() * 4, cudaMemcpyHostToDevice, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));   // (b / o are pageable host memory)
        S.uploaded = true;
    }
    // SAM records resolved RNAME / RNEXT against elp_config's names, the merged dictionary: only the BAM refIDs go through the input's map
    const bool remap = !sam_records && !c->inputs.empty();
    if (remap && S.remap_input != c->cur_input) {
        const std::vector<int32_t>& m = c->inputs[c->cur_input].remap;
        CUDA_TRY(c, S.remap.fit(std::max<size_t>(m.size(), 1)));
        if (!m.empty()) CUDA_TRY(c, cudaMemcpyAsync(S.remap.p, m.data(), m.size() * 4, cudaMemcpyHostToDevice, s));
        CUDA_TRY(c, cudaStreamSynchronize(s));
        S.remap_input = c->cur_input;
    }
    TRY(grow(c, S.sub, nrec + 1, 0)); TRY(grow(c, S.len, nrec + 8, 0)); TRY(grow(c, S.off, nrec + 2, 0));
    RelabelArgs A{};
    A.n = nrec; A.raw = *raw; A.off = off; A.remap = remap ? S.remap.p : nullptr; A.n_sq = relabel_ref_bound(c);
    A.ren = S.ren.p; A.ren_off = S.ren_off.p; A.n_ren[0] = (int)c->tag_ren[0].size(); A.n_ren[1] = (int)c->tag_ren[1].size();
    A.sub = S.sub.p; A.len = S.len.p; A.err = c->d_err.p;
    c->begin("relabel_measure", (double)*n_bytes + 24.0 * (double)nrec);
    relabel_measure_kernel<<<nblk(nrec, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    TRY(exclusive_scan_u32_to_u64(c, S.len.p, S.off.p, nrec));
    uint64_t total = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&total, S.off.p + nrec, 8, cudaMemcpyDeviceToHost, s));
    TRY(check_device_errors(c));   // synchronizes
    TRY(grow(c, S.raw, total + 64, 0));
    A.new_off = S.off.p; A.out = S.raw.p;
    c->begin("relabel_emit", (double)*n_bytes + (double)total);
    relabel_emit_kernel<<<nblk(nrec * 32, 256), 256, 0, s>>>(A);
    c->end(); LAUNCH_CHECK(c);
    CUDA_TRY(c, cudaMemcpyAsync(off, S.off.p, (nrec + 1) * 8, cudaMemcpyDeviceToDevice, s));
    *raw = S.raw.p; *n_bytes = total;
    return E_OK;
}

extern "C" int elp_add_input(elp_ctx* c, const char* const* names, const int32_t* lengths, int32_t n_sq) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (n_sq < 0 || (n_sq && (!names || !lengths))) return c->fail(E_INVAL, "elp_add_input: bad input dictionary (n_sq = %d)", n_sq);
    if (c->n || c->sorted || c->bgzf_open) return c->fail(E_STATE, "elp_add_input: the context holds reads (call it after elp_create or elp_reset)");
    if (c->dict_mode) return c->fail(E_INVAL, "elp_add_input: the context has an input dictionary (elp_set_input_dictionary); the two do not combine");
    if ((int)c->inputs.size() >= ELP_MAX_INPUTS) return c->fail(E_LIMIT, "elp_add_input: more than %d inputs", ELP_MAX_INPUTS);
    if (n_sq && !c->has_contig_names) return c->fail(E_INVAL, "elp_add_input: the context was created without elp_config.contig_names");
    std::map<std::string, int32_t> first;                      // memberOfSequenceDictionary: the first entry with the name
    for (int j = c->n_contigs - 1; j >= 0; j--) first[c->contig_names[j]] = j;
    elp_ctx::InputDict d;
    for (int32_t i = 0; i < n_sq; i++) {
        if (!names[i]) return c->fail(E_INVAL, "elp_add_input: name %d is null", i);
        auto it = first.find(names[i]);
        if (it == first.end()) return c->fail(E_INVAL, "elp_add_input: @SQ %d of the input, '%s', is not in the merged dictionary (elp_config.contig_names)", i, names[i]);
        d.names.push_back(names[i]); d.len.push_back(lengths[i]); d.remap.push_back(it->second);
    }
    c->inputs.push_back(std::move(d));
    return (int)c->inputs.size() - 1;
}

extern "C" int elp_select_input(elp_ctx* c, int32_t input) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    if (input < 0 || input >= (int32_t)c->inputs.size()) return c->fail(E_INVAL, "elp_select_input: input %d is not one of the %zu added (elp_add_input)", input, c->inputs.size());
    if (c->bgzf_open) return c->fail(E_STATE, "elp_select_input while a BGZF file is open (elp_append_bgzf_end first)");
    if (c->sorted) return c->fail(E_STATE, "elp_select_input after elp_sort_markdup (call elp_reset first)");
    c->cur_input = input;
    return ELP_OK;
}

extern "C" int elp_set_tag_rename(elp_ctx* c, const char* tag, const char* const* old_ids, const char* const* new_ids, int32_t n) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::lock_guard<std::mutex> lk(c->append_mu);
    const int t = (tag && tag[0] == 'R' && tag[1] == 'G' && !tag[2]) ? 0 : ((tag && tag[0] == 'P' && tag[1] == 'G' && !tag[2]) ? 1 : -1);
    if (t < 0) return c->fail(E_INVAL, "elp_set_tag_rename: the tag must be \"RG\" or \"PG\"");
    if (n < 0 || (n && (!old_ids || !new_ids))) return c->fail(E_INVAL, "elp_set_tag_rename: bad rename list (n = %d)", n);
    if (c->n || c->sorted || c->bgzf_open) return c->fail(E_STATE, "elp_set_tag_rename: the context holds reads (call it after elp_create or elp_reset)");
    if (c->dict_mode) return c->fail(E_INVAL, "elp_set_tag_rename: the context has an input dictionary (elp_set_input_dictionary); the two do not combine");
    std::vector<std::pair<std::string, std::string>> v;
    std::set<std::string> seen;
    for (int32_t i = 0; i < n; i++) {
        if (!old_ids[i] || !new_ids[i]) return c->fail(E_INVAL, "elp_set_tag_rename: entry %d is null", i);
        if (!seen.insert(old_ids[i]).second) return c->fail(E_INVAL, "elp_set_tag_rename: the old value '%s' is given twice", old_ids[i]);
        v.emplace_back(old_ids[i], new_ids[i]);
    }
    c->tag_ren[t] = std::move(v);
    if (c->relabel) c->relabel->uploaded = false;
    return ELP_OK;
}
