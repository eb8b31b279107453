// gob.cu -- the two intermediate files an `elprep sfm` run exchanges between its filter workers, in Go's encoding/gob wire format
// (SURVEY.md 8f row 3), so that a GPU worker can sit inside a run whose other steps are the reference's own:
//   .elrecal   gob of filters.BaseRecalibratorTables{QualityScores, Cycles, Contexts map[bqsrTableKey]*bqsrEntry}
//              written by (*BaseRecalibratorTables).PrintBQSRTablesToIntermediateFile (filters/print-bqsr.go:300-308, `--bqsr-tables-only`),
//              read and summed by LoadAndCombineBQSRTables (:310-329, `--bqsr-apply`)
//   metrics    gob of map[string]*DuplicatesCtr -- only the seven exported counters travel (filters/mark-optical-duplicates.go:96-110);
//              PrintDuplicatesMetricsToIntermediateFile (:701-709), LoadAndCombineDuplicateMetrics (:711-731)
// Host code, no GPU work beyond moving the dense tables.  The writer emits the message sequence Go's encoder emits in a fresh process
// (type ids from 64); the reader is a general decoder of the type definitions in the stream, so it does not depend on those ids.
// UNVERIFIED against a Go binary (none in this image): the format follows the encoding/gob specification; tests/test_gob.py pins the
// encoder primitives on the byte example of that specification and checks writer and reader against an independent restatement.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include "../../include/elprep_b200.h"
#include "ctx.h"

namespace {

// ---------------------------------------------------------------- encoder
struct Enc {
    std::string b;
    void u(uint64_t v) {                     // unsigned: < 128 one byte, else negated byte count then big-endian bytes
        if (v < 128) { b.push_back((char)v); return; }
        unsigned char tmp[8]; int n = 0;
        while (v) { tmp[n++] = (unsigned char)(v & 255); v >>= 8; }
        b.push_back((char)(unsigned char)(256 - n));
        while (n) b.push_back((char)tmp[--n]);
    }
    void i(int64_t v) { u(v < 0 ? ((uint64_t)(~v) << 1) | 1 : (uint64_t)v << 1); }     // sign in bit 0
    void s(const std::string& x) { u(x.size()); b += x; }
};
std::string frame(const std::string& payload) { Enc e; e.u(payload.size()); return e.b + payload; }

void common_type(Enc& e, const std::string& name, int id) {      // CommonType{Name string; Id typeId}
    int prev = -1;
    if (!name.empty()) { e.u(1); e.s(name); prev = 0; }
    e.u(1 - prev); e.i(id);
    e.u(0);
}
std::string def_struct(int id, const std::string& name, const std::vector<std::pair<std::string, int>>& fields) {
    Enc e; e.i(-id);
    e.u(3);                                  // wireType.StructT (field 2)
    e.u(1); common_type(e, name, id);        // structType.CommonType
    e.u(1); e.u(fields.size());              // structType.Field []fieldType
    for (auto& f : fields) { e.u(1); e.s(f.first); e.u(1); e.i(f.second); e.u(0); }
    e.u(0); e.u(0);
    return frame(e.b);
}
std::string def_map(int id, const std::string& name, int key, int elem) {
    Enc e; e.i(-id);
    e.u(4);                                  // wireType.MapT (field 3)
    e.u(1); common_type(e, name, id);
    e.u(1); e.i(key); e.u(1); e.i(elem);
    e.u(0); e.u(0);
    return frame(e.b);
}
constexpr int T_INT = 2, T_UINT = 3, T_STRING = 6;

// struct fields: (delta, value) pairs, zero values omitted
struct SEnc { Enc& e; int prev = -1; void fu(int f, uint64_t v) { if (v) { e.u(f - prev); e.u(v); prev = f; } } void fi(int f, int64_t v) { if (v) { e.u(f - prev); e.i(v); prev = f; } }
              void fs(int f, const std::string& v) { if (!v.empty()) { e.u(f - prev); e.s(v); prev = f; } } void open(int f) { e.u(f - prev); prev = f; } void end() { e.u(0); } };

// ---------------------------------------------------------------- decoder
struct Val;
using ValP = std::shared_ptr<Val>;
struct Val { int kind = 0; /* 0 int, 1 uint, 2 string, 3 struct, 4 map, 5 slice, 6 float/other skipped */ int64_t i = 0; uint64_t u = 0; std::string s;
             std::map<std::string, ValP> fields; std::vector<std::pair<ValP, ValP>> kv; std::vector<ValP> items; };
struct TypeDef { int kind = 0; /* 3 struct, 4 map, 5 slice, 7 array */ std::vector<std::pair<std::string, int>> fields; int key = 0, elem = 0; int64_t len = 0; };
struct Dec {
    const unsigned char* p; const unsigned char* end; bool bad = false; std::map<int, TypeDef> types;
    uint64_t u() {
        if (p >= end) { bad = true; return 0; }
        unsigned c = *p++;
        if (c < 128) return c;
        int n = 256 - (int)c;
        if (n > 8 || p + n > end) { bad = true; return 0; }
        uint64_t v = 0; while (n--) v = (v << 8) | *p++;
        return v;
    }
    int64_t i() { uint64_t x = u(); return (x & 1) ? ~(int64_t)(x >> 1) : (int64_t)(x >> 1); }
    std::string s() { uint64_t n = u(); if (bad || (uint64_t)(end - p) < n) { bad = true; return ""; } std::string r((const char*)p, (size_t)n); p += n; return r; }
    // CommonType -> (name, id)
    void common(std::string& name, int& id) { int f = -1; for (;;) { uint64_t d = u(); if (bad || !d) return; f += (int)d; if (f == 0) name = s(); else if (f == 1) id = (int)i(); else { bad = true; return; } } }
    void type_def(int id) {
        TypeDef t; int f = -1;
        for (;;) {
            uint64_t d = u(); if (bad) return; if (!d) break; f += (int)d;
            std::string nm; int cid = 0; int g = -1;
            if (f == 2) {            // structType{CommonType; Field []fieldType}
                t.kind = 3;
                for (;;) { uint64_t d2 = u(); if (bad) return; if (!d2) break; g += (int)d2;
                    if (g == 0) common(nm, cid);
                    else if (g == 1) { uint64_t n = u(); for (uint64_t k = 0; k < n && !bad; k++) { std::string fn; int fid = 0; int h = -1; for (;;) { uint64_t d3 = u(); if (bad || !d3) break; h += (int)d3; if (h == 0) fn = s(); else if (h == 1) fid = (int)i(); else { bad = true; } } t.fields.push_back({fn, fid}); } }
                    else { bad = true; return; } }
            } else if (f == 3) {     // mapType{CommonType; Key, Elem typeId}
                t.kind = 4;
                for (;;) { uint64_t d2 = u(); if (bad) return; if (!d2) break; g += (int)d2; if (g == 0) common(nm, cid); else if (g == 1) t.key = (int)i(); else if (g == 2) t.elem = (int)i(); else { bad = true; return; } }
            } else if (f == 1) {     // sliceType{CommonType; Elem}
                t.kind = 5;
                for (;;) { uint64_t d2 = u(); if (bad) return; if (!d2) break; g += (int)d2; if (g == 0) common(nm, cid); else if (g == 1) t.elem = (int)i(); else { bad = true; return; } }
            } else if (f == 0) {     // arrayType{CommonType; Elem; Len}
                t.kind = 7;
                for (;;) { uint64_t d2 = u(); if (bad) return; if (!d2) break; g += (int)d2; if (g == 0) common(nm, cid); else if (g == 1) t.elem = (int)i(); else if (g == 2) t.len = i(); else { bad = true; return; } }
            } else { bad = true; return; }   // GobEncoder / marshaler types do not occur in these files
        }
        types[id] = t;
    }
    ValP value(int id, int depth = 0) {
        auto v = std::make_shared<Val>();
        if (depth > 32) bad = true;          // (a crafted self-referential type must not recurse through the whole file)
        if (bad) return v;
        switch (id) {
            case 1: v->kind = 1; v->u = u(); return v;                 // bool
            case 2: v->kind = 0; v->i = i(); return v;
            case 3: v->kind = 1; v->u = u(); return v;
            case 4: v->kind = 6; v->u = u(); return v;                 // float: byte-reversed bits, kept raw
            case 5: case 6: v->kind = 2; v->s = s(); return v;
            default: break;
        }
        auto it = types.find(id);
        if (it == types.end()) { bad = true; return v; }
        const TypeDef& t = it->second;
        if (t.kind == 3) {
            v->kind = 3; int f = -1;
            for (;;) { uint64_t d = u(); if (bad || !d) break; if (d > (1u << 20)) { bad = true; break; } f += (int)d; if (f < 0 || f >= (int)t.fields.size()) { bad = true; break; } v->fields[t.fields[f].first] = value(t.fields[f].second, depth + 1); }
        } else if (t.kind == 4) {
            v->kind = 4; uint64_t n = u();
            for (uint64_t k = 0; k < n && !bad; k++) { ValP a = value(t.key, depth + 1); ValP b = value(t.elem, depth + 1); v->kv.push_back({a, b}); }
        } else if (t.kind == 5 || t.kind == 7) {
            v->kind = 5; uint64_t n = u();
            for (uint64_t k = 0; k < n && !bad; k++) v->items.push_back(value(t.elem, depth + 1));
        } else bad = true;
        return v;
    }
    // one Encode()d value: type definitions, then the value message
    ValP top() {
        for (;;) {
            uint64_t len = u(); if (bad || (uint64_t)(end - p) < len) { bad = true; return nullptr; }
            const unsigned char* mend = p + len;
            int64_t id = i();
            if (id < 0) { Dec sub{p, mend, false, {}}; sub.types.swap(types); sub.type_def((int)-id); types.swap(sub.types); if (sub.bad) { bad = true; return nullptr; } p = mend; continue; }
            Dec sub{p, mend, false, {}}; sub.types.swap(types);
            auto it = sub.types.find((int)id);
            if (it == sub.types.end() || it->second.kind != 3) sub.u();       // singleton: a zero field delta precedes a value that is not a struct
            ValP v = sub.value((int)id);
            types.swap(sub.types);
            if (sub.bad) { bad = true; return nullptr; }
            p = mend;
            return v;
        }
    }
};

int64_t geti(const Val& s, const char* f) { auto it = s.fields.find(f); if (it == s.fields.end()) return 0; return it->second->kind == 1 ? (int64_t)it->second->u : it->second->i; }
std::string gets(const Val& s, const char* f) { auto it = s.fields.find(f); return it == s.fields.end() ? std::string() : it->second->s; }

bool read_file(const char* path, std::string& out) {
    FILE* f = fopen(path, "rb"); if (!f) return false;
    char buf[1 << 16]; size_t n;
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) out.append(buf, n);
    fclose(f); return true;
}
bool write_file(const char* path, const std::string& data) {
    FILE* f = fopen(path, "wb"); if (!f) return false;
    const bool ok = fwrite(data.data(), 1, data.size(), f) == data.size();
    return fclose(f) == 0 && ok;
}

}  // namespace

extern "C" {

int elp_bqsr_tables_clear(elp_ctx* c) {
    if (!c) return ELP_EINVAL;
    cudaSetDevice(c->device);
    CUDA_TRY(c, cudaMemsetAsync(c->d_tables.p, 0, c->geom.cells() * 2 * sizeof(int64_t), c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    c->gathered = true; c->finalized = false;
    return ELP_OK;
}

int elp_bqsr_tables_write_elrecal(elp_ctx* c, const char* path) {
    if (!c || !path) return ELP_EINVAL;
    cudaSetDevice(c->device);
    if (!c->gathered) return c->fail(E_STATE, "elp_bqsr_tables_write_elrecal before elp_bqsr_gather / elp_bqsr_tables_put");
    const TableGeom& g = c->geom;
    std::vector<int64_t> t(g.cells() * 2);
    CUDA_TRY(c, cudaMemcpyAsync(t.data(), c->d_tables.p, t.size() * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    // type ids of a fresh Go process: BaseRecalibratorTables 64, bqsrTableKey 65, bqsrEntry 66, bqsrTable 67 (a map gets its id after its key and element)
    std::string out = def_struct(64, "BaseRecalibratorTables", {{"QualityScores", 67}, {"Cycles", 67}, {"Contexts", 67}});
    out += def_map(67, "bqsrTable", 65, 66);
    out += def_struct(65, "bqsrTableKey", {{"Qual", T_UINT}, {"Covariate", T_INT}, {"ReadGroup", T_STRING}});
    out += def_struct(66, "bqsrEntry", {{"EmpiricalQuality", T_UINT}, {"Observations", T_INT}, {"Mismatches", T_INT}});
    Enc e; e.i(64);
    SEnc top{e};
    for (int table = 0; table < 3; table++) {
        const int c0 = table == 0 ? 0 : (table == 1 ? 1 : g.col_ctx(0)), c1 = table == 0 ? 1 : (table == 1 ? g.col_ctx(0) : g.ncols());
        uint64_t count = 0;
        for (int cv = 0; cv < g.n_cov; cv++) for (int q = 0; q < 94; q++) for (int col = c0; col < c1; col++) if (t[2 * g.idx(cv, q, col)] > 0) count++;
        top.open(table);                       // maps are sent even when empty (NewBaseRecalibratorTables makes them non-nil)
        e.u(count);
        for (int cv = 0; cv < g.n_cov; cv++) for (int q = 0; q < 94; q++) for (int col = c0; col < c1; col++) {
            const int64_t obs = t[2 * g.idx(cv, q, col)], mis = t[2 * g.idx(cv, q, col) + 1];
            if (obs <= 0) continue;
            const int64_t covariate = table == 0 ? 0 : (table == 1 ? (int64_t)(col - 1 - g.max_cycle) : (int64_t)(2 | ((col - g.col_ctx(0)) << 4)));   // cycle / context key (bqsr.go:64-76)
            SEnc k{e}; k.fu(0, (uint64_t)q); k.fi(1, covariate); k.fs(2, c->cov_names[cv]); k.end();
            SEnc v{e}; v.fi(1, obs); v.fi(2, mis); v.end();          // EmpiricalQuality is still 0 before FinalizeBQSRTables: omitted
        }
    }
    top.end();
    out += frame(e.b);
    if (!write_file(path, out)) return c->fail(E_INVAL, "cannot write %s", path);
    return ELP_OK;
}

int elp_bqsr_tables_add_elrecal(elp_ctx* c, const char* path) {
    if (!c || !path) return ELP_EINVAL;
    cudaSetDevice(c->device);
    std::string data;
    if (!read_file(path, data)) return c->fail(E_INVAL, "cannot read %s", path);
    Dec d{(const unsigned char*)data.data(), (const unsigned char*)data.data() + data.size(), false, {}};
    ValP v = d.top();
    if (!v || d.bad || v->kind != 3) return c->fail(E_INVAL, "%s: not a gob stream of filters.BaseRecalibratorTables", path);
    const TableGeom& g = c->geom;
    std::vector<int64_t> t(g.cells() * 2);
    CUDA_TRY(c, cudaMemcpyAsync(t.data(), c->d_tables.p, t.size() * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    const char* names[3] = {"QualityScores", "Cycles", "Contexts"};
    for (int table = 0; table < 3; table++) {
        auto it = v->fields.find(names[table]);
        if (it == v->fields.end()) continue;
        if (it->second->kind != 4) return c->fail(E_INVAL, "%s: field %s is not a map", path, names[table]);
        for (auto& kv : it->second->kv) {
            if (kv.first->kind != 3 || kv.second->kind != 3) return c->fail(E_INVAL, "%s: malformed table entry", path);
            const int64_t q = geti(*kv.first, "Qual"), cov = geti(*kv.first, "Covariate");
            const std::string rg = gets(*kv.first, "ReadGroup");
            int cv = -1;
            for (int k = 0; k < g.n_cov; k++) if (c->cov_names[k] == rg) cv = k;
            if (cv < 0) return c->fail(E_INVAL, "%s: read group covariate \"%s\" is not in this context's header", path, rg.c_str());
            if (q < 0 || q >= 94) return c->fail(E_LIMIT, "%s: QUAL %lld outside 0..93", path, (long long)q);
            int col;
            if (table == 0) col = 0;
            else if (table == 1) { if (cov < -g.max_cycle || cov > g.max_cycle) return c->fail(E_CYCLE, "cycle value exceeds maximum cycle value"); col = g.col_cycle((int)cov); }
            else { if ((cov & 15) != 2 || (cov >> 4) < 0 || (cov >> 4) > 15) return c->fail(E_INVAL, "%s: context key %lld is not a 2-mer key", path, (long long)cov); col = g.col_ctx((int)(cov >> 4)); }
            t[2 * g.idx(cv, (int)q, col)] += geti(*kv.second, "Observations");          // bqsrTable.merge (filters/bqsr.go): counters add
            t[2 * g.idx(cv, (int)q, col) + 1] += geti(*kv.second, "Mismatches");
        }
    }
    CUDA_TRY(c, cudaMemcpyAsync(c->d_tables.p, t.data(), t.size() * 8, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    c->gathered = true; c->finalized = false;
    return ELP_OK;
}

int elp_optical_write_gob(elp_ctx* c, const char* path) {
    if (!c || !path) return ELP_EINVAL;
    if (!c->opt_valid) return c->fail(E_STATE, "elp_optical_write_gob before elp_sort_markdup(.., ELP_MARKDUP_OPTICAL)");
    // map[string]*DuplicatesCtr: element struct 64, then the (unnamed) map 65
    const char* fn[7] = {"UnpairedReadsExamined", "ReadPairsExamined", "SecondaryOrSupplementaryReads", "UnmappedReads", "UnpairedReadDuplicates", "ReadPairDuplicates", "ReadPairOpticalDuplicates"};
    std::vector<std::pair<std::string, int>> fields; for (auto f : fn) fields.push_back({f, T_INT});
    std::string out = def_map(65, "", T_STRING, 64);
    out += def_struct(64, "DuplicatesCtr", fields);
    Enc e; e.i(65); e.u(0);                                     // a map is not a struct: singleton marker
    uint64_t count = 0;
    for (size_t s = 0; s < c->opt.size(); s++) { bool any = false; for (int k = 0; k < 7; k++) any |= c->opt[s].ctr[k] != 0; if (any) count++; }
    e.u(count);
    for (size_t s = 0; s < c->opt.size(); s++) {
        bool any = false; for (int k = 0; k < 7; k++) any |= c->opt[s].ctr[k] != 0;
        if (!any) continue;                                        // the reference creates a library's counter on its first read
        e.s(s == 0 ? std::string("Unknown Library") : c->lib_names[s - 1]);
        SEnc v{e};
        for (int k = 0; k < 7; k++) v.fi(k, k == 1 ? c->opt[s].ctr[1] / 2 : c->opt[s].ctr[k]);   // ctr[1] counts paired READS here; the file holds pairs (:504-506)
        v.end();
    }
    out += frame(e.b);
    if (!write_file(path, out)) return c->fail(E_INVAL, "cannot write %s", path);
    return ELP_OK;
}

int elp_optical_add_gob(elp_ctx* c, const char* path) {
    if (!c || !path) return ELP_EINVAL;
    std::string data;
    if (!read_file(path, data)) return c->fail(E_INVAL, "cannot read %s", path);
    Dec d{(const unsigned char*)data.data(), (const unsigned char*)data.data() + data.size(), false, {}};
    ValP v = d.top();
    if (!v || d.bad || v->kind != 4) return c->fail(E_INVAL, "%s: not a gob stream of map[string]*DuplicatesCtr", path);
    if (c->opt.size() != (size_t)c->n_lib + 1) c->opt.assign((size_t)c->n_lib + 1, DupCounters());
    const char* fn[7] = {"UnpairedReadsExamined", "ReadPairsExamined", "SecondaryOrSupplementaryReads", "UnmappedReads", "UnpairedReadDuplicates", "ReadPairDuplicates", "ReadPairOpticalDuplicates"};
    for (auto& kv : v->kv) {
        if (kv.first->kind != 2 || kv.second->kind != 3) return c->fail(E_INVAL, "%s: malformed entry", path);
        int slot = -1;
        if (kv.first->s == "Unknown Library") slot = 0;
        for (int l = 0; l < c->n_lib; l++) if (c->lib_names[l] == kv.first->s) slot = l + 1;
        if (slot < 0) return c->fail(E_INVAL, "%s: library \"%s\" is not in this context's header", path, kv.first->s.c_str());
        for (int k = 0; k < 7; k++) c->opt[slot].ctr[k] += (k == 1 ? 2 : 1) * geti(*kv.second, fn[k]);     // mergeDuplicatesCtrMaps (:451-466); pairs -> paired reads
    }
    c->opt_valid = true;
    return ELP_OK;
}

}  // extern "C"
