// bqsr_finalize.cu -- BQSR between gather and apply (replaces FinalizeBQSRTables, filters/bqsr.go:677-694,
// initializeCombinedBQSRTable :655-674, the quantizers :708-899, estimateHierarchicalBayesianQuality :901-919 as memoised
// by ApplyBQSR :973-1000, and PrintBQSRTables, filters/print-bqsr.go:49-298).
//
// The arithmetic is IEEE double with Go's math functions (gomath.hpp) in the reference's operation order.  It runs on the
// device, on the context's stream, with no host synchronisation between gather and apply:
//   fin_emp       EmpiricalQuality of every table cell, one thread per cell
//   fin_tail      one CTA: the combined per-read-group entries, the quantization map, the "unobserved QUAL" byte per covariate
//   fin_lut       one CTA per (covariate, QUAL) row: the apply look-up table indexed by (read-group covariate, reported qual,
//                 cycle, context) -- exactly the memo the reference fills lazily per worker
//   fin_clut      the compact table of bqsr_apply2_kernel, copied out of the full one
// This file is compiled with -fmad=false (csrc/Makefile): a fused multiply-add would round differently from the host and from Go.
// The recalibration report stays host code, fed by one copy of the tables and of EmpiricalQuality made only when a report is asked for.
// Reference non-determinism fixed here: the combined per-read-group entry accumulates in ascending-qual order
// (the reference iterates a Go map, :657-668).
#include <algorithm>
#include <cfloat>
#include <cstdio>
#include <mutex>
#include <string>
#include <vector>
#include "ctx.h"
#include "gomath.hpp"

namespace {

#define PRIOR_CACHE {   /* embedded data, filters/bqsr.go:569-591: log10(0.9*exp(-d^2/0.5)), last = -MaxFloat64 */ \
    -0.045757490560675115, -0.9143464543671788, -3.5201133457866898, -7.863058164819208, -13.943180911464733, -21.760481585723266, \
    -31.314960187594806, -42.606616717079355, -55.63545117417691, -70.40146355888747, -86.90465387121104, -105.14502211114761, \
    -125.1225682786972, -146.83729237385978, -170.2891943966354, -195.47827434702398, -222.4045322250256, -251.06796803064023, \
    -281.46858176386786, -313.60637342472336, -1.7976931348623157e308}
#ifndef __CUDA_ARCH__
const double kPriorCache[21] = PRIOR_CACHE;
#endif
__constant__ double c_prior[21] = PRIOR_CACHE;

struct BinTerms { double l[61], m[61]; };   // per-bin constants of log10BinomialProbability (:607-613): l = i/-10, m = log10(1 - 10^l)
BinTerms make_bin_terms() {
    BinTerms b;
    for (int i = 0; i < 61; i++) { b.l[i] = (double)i / -10.0; b.m[i] = (b.l[i] == 0.0) ? 0.0 : gomath::Log10(1.0 - gomath::Pow(10, b.l[i])); }
    return b;
}
const BinTerms& bin_terms() { static const BinTerms b = make_bin_terms(); return b; }
__constant__ BinTerms c_bin;   // the host's BinTerms, copied once per device (ensure_fin_state): the same bits by construction

GM_HD inline double log10_gamma(int64_t n) { return gomath::Lgamma((double)n) * 0.4342944819032518; }   // :598-601

// calculateEmpiricalQuality (:644-649) = calculateBayesianEstimateOfEmpiricalQuality (:623-642) on the smoothed counts
struct Entry {
    int64_t n, k; double coef;
    GM_HD Entry(int64_t obs, int64_t mis) {
        n = obs + 2; k = mis + 1;
        const int64_t maxObs = 2147483647 - 1;
        if (n > maxObs) { k = (int64_t)gomath::Round((double)k * ((double)maxObs / (double)n)); n = maxObs; }
        coef = log10_gamma(n + 1) - log10_gamma(k + 1) - log10_gamma(n - k + 1);   // log10BinomialCoefficient :603-605
    }
    GM_HD uint8_t empirical(double prior) const {
#ifdef __CUDA_ARCH__
        const BinTerms& B = c_bin; const double* P = c_prior;
#else
        const BinTerms& B = bin_terms(); const double* P = kPriorCache;
#endif
        double best = -DBL_MAX; int bi = 0;
        for (int i = 0; i < 61; i++) {
            int d = (int)((double)i - prior); if (d < 0) d = -d; if (d > 20) d = 20;   // log10QualEmpiricalPrior :593-596
            const double p1 = P[d];
            const double p2 = (B.l[i] == 0.0) ? -DBL_MAX : (coef + B.l[i] * (double)k) + B.m[i] * (double)(n - k);   // n is never 0 here (obs+2)
            const double post = p1 + p2;
            if (best < post) { best = post; bi = i; }
        }
        return (uint8_t)(bi < 93 ? bi : 93);
    }
};

GM_HD inline double q2err(double phred) { return gomath::Pow(10, phred / -10); }
GM_HD inline double q2prob(double phred) { return 1 - gomath::Pow(10, phred / -10); }

struct Combined { bool exists = false; double reported = 0; int64_t obs = 0, mis = 0; uint8_t emp = 0; };

struct Tables {   // the dense tables, in host memory (report) or device memory (kernels)
    TableGeom g; const int64_t* t;
    GM_HD int64_t obs(int cov, int q, int col) const { return t[2 * g.idx(cov, q, col)]; }
    GM_HD int64_t mis(int cov, int q, int col) const { return t[2 * g.idx(cov, q, col) + 1]; }
};

GM_HD Combined combine(const Tables& T, int cov) {   // :655-674
    Combined c;
    for (int q = 0; q < 94; q++) {
        const int64_t eo = T.obs(cov, q, 0), em = T.mis(cov, q, 0);
        if (eo <= 0) continue;
        if (c.exists) {
            const double sumErrors = (double)c.obs * q2err(c.reported) + (double)eo * q2err((double)q);
            c.obs += eo; c.mis += em;
            c.reported = -10 * gomath::Log10(sumErrors / (double)c.obs);
        } else { c.exists = true; c.reported = (double)q; c.obs = eo; c.mis = em; }
    }
    if (c.exists) c.emp = Entry(c.obs, c.mis).empirical(c.reported);
    return c;
}

GM_HD int err_prob_to_quality(double prob) {   // :701-706
    if (prob == 0.0) return 93;
    int q = (int)gomath::Round(-10 * gomath::Log10(prob));
    return q > 93 ? 93 : (q < 1 ? 1 : q);
}

std::vector<uint8_t> static_quantized(std::vector<uint8_t> quals) {   // initializeStaticQuantizedScores :710-743
    std::vector<uint8_t> ss(254, 0);
    for (int i = 0; i < 6; i++) ss[i] = (uint8_t)i;
    if (quals.size() == 1) { for (int i = 6; i < 254; i++) ss[i] = quals[0]; return ss; }
    std::sort(quals.begin(), quals.end());
    uint8_t prevQual = 6; double prevProb = q2prob((double)prevQual);
    for (uint8_t nextQual : quals) {
        for (uint8_t i = prevQual; i < nextQual; i++) {
            const double nextProb = q2prob((double)nextQual), iProb = q2prob((double)i);
            ss[i] = (iProb - prevProb > nextProb - iProb) ? nextQual : prevQual;
            prevProb = nextProb; prevQual = nextQual;
        }
    }
    for (int i = prevQual; i < 254; i++) ss[i] = prevQual;
    return ss;
}

struct QInterval { int next; double errorRate; int64_t nobs, leafNobs, nerrors; };
GM_HD double calc_error_rate(int64_t nobs, int64_t nerr) { return nobs == 0 ? 0.0 : (double)(nerr + 1) / (double)(nobs + 1); }
double leaf_penalty(int k, const std::vector<QInterval>& iv, double globalErrorRate) {   // :780-786
    if (k <= 6) return 0.0;
    return gomath::Fabs(gomath::Log10(iv[k].errorRate) - gomath::Log10(globalErrorRate)) * (double)iv[k].leafNobs;
}
double merge_penalty(int i, int j, const std::vector<QInterval>& iv) {   // :795-818
    const int64_t mn = iv[i].nobs + iv[j].nobs, me = iv[i].nerrors + iv[j].nerrors;
    const double mer = calc_error_rate(mn, me);
    if (mer == 0) return 0.0;
    double sumI = 0, sumJ = 0;
    for (int k = i; k < j; k++) sumI += leaf_penalty(k, iv, mer);
    const int kend = iv[j].next >= 0 ? iv[j].next : (int)iv.size();
    for (int k = j; k < kend; k++) sumJ += leaf_penalty(k, iv, mer);
    return sumI + sumJ;
}
// initializeQuantizedQualityScores :863-899
void quantized(const Tables& T, const std::vector<uint8_t>& emp, int levels, std::vector<int64_t>& qmap, std::vector<uint8_t>& scores) {
    qmap.assign(94, 0); scores.assign(94, 0);
    if (levels == 0) { for (int i = 0; i < 94; i++) scores[i] = (uint8_t)i; return; }
    for (int cov = 0; cov < T.g.n_cov; cov++) for (int q = 0; q < 94; q++) if (T.obs(cov, q, 0) > 0) qmap[emp[T.g.idx(cov, q, 0)]] += T.obs(cov, q, 0);
    std::vector<QInterval> iv(94);
    for (int i = 0; i < 94; i++) { const double er = q2err((double)i); iv[i] = {i + 1 == 94 ? -1 : i + 1, er, qmap[i], qmap[i], (int64_t)((double)qmap[i] * er)}; }
    for (int n = 94; n > levels;) {   // mergeQuantizationIntervals :852-861 / mergeMinimalPenaltyQuantizationIntervals :820-850
        int i = 0, j = iv[0].next;
        if (j < 0) break;
        int minI = 0; double mp = merge_penalty(i, j, iv);
        for (;;) { i = j; j = iv[i].next; if (j < 0) break; const double p = merge_penalty(i, j, iv); if (p < mp) { minI = i; mp = p; } }
        QInterval& a = iv[minI]; const QInterval b = iv[a.next];
        a.next = b.next; a.nobs += b.nobs; a.nerrors += b.nerrors;
        n--;
    }
    for (int i = 0; i >= 0;) {
        const bool leaf = iv[i].next < 0 ? (i == 93) : (iv[i].next == i + 1);
        const uint8_t qs = leaf ? (uint8_t)i : (uint8_t)err_prob_to_quality(calc_error_rate(iv[i].nobs, iv[i].nerrors));
        const int kend = iv[i].next >= 0 ? iv[i].next : 94;
        for (int k = i; k < kend; k++) scores[k] = qs;
        i = iv[i].next;
    }
}

// ---- report (filters/print-bqsr.go) ----
int ilen(long long v) { char b[32]; return std::snprintf(b, sizeof b, "%lld", v); }
std::string context_text(int ctx) { const char* B = "ACGT"; std::string s; s += B[ctx & 3]; s += B[(ctx >> 2) & 3]; return s; }   // keyToString, bqsr.go:166-178
struct Row { std::string rg; int q; std::string text; bool cycle; int64_t obs, mis; uint8_t emp; };

void put(std::string& out, const char* fmt, ...) {
    char buf[512]; va_list ap; va_start(ap, fmt); std::vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap); out += buf;
}

int write_report(elp_ctx* c, const Tables& T, const std::vector<uint8_t>& emp, const std::vector<Combined>& comb, const char* path) {
    const char* P = c->prefix.c_str();
    std::string o;
    put(o, "#:%sReport.v1.1:5\n#:%sTable:2:17:%%s:%%s:;\n#:%sTable:Arguments:Recalibration argument collection values used in this run\n", P, P, P);
    static const char* const kArgs[][2] = {{"Argument", "Value"}, {"binary_tag_name", "null"}, {"covariate", "ReadGroupCovariate,QualityScoreCovariate,ContextCovariate,CycleCovariate"},
        {"default_platform", "null"}, {"deletions_default_quality", "45"}, {"force_platform", "null"}, {"indels_context_size", "3"}, {"insertions_default_quality", "45"},
        {"low_quality_tail", "2"}, {"maximum_cycle_value", "500"}, {"mismatches_context_size", "2"}, {"mismatches_default_quality", "-1"}, {"no_standard_covs", "false"},
        {"quantizing_levels", "16"}, {"recalibration_report", "null"}, {"run_without_dbsnp", "false"}, {"solid_nocall_strategy", "THROW_EXCEPTION"}, {"solid_recal_mode", "SET_Q_ZERO"}};
    for (auto& a : kArgs) put(o, "%-26s  %-72s\n", a[0], a[1]);
    o += "\n";
    {   // quantization table, always 16 levels (print-bqsr.go:33,49-76)
        std::vector<int64_t> obs; std::vector<uint8_t> sc; quantized(T, emp, 16, obs, sc);
        put(o, "#:%sTable:3:%d:%%d:%%d:%%d:;\n#:%sTable:Quantized:Quality quantization map\n", P, 94, P);
        int w1 = 12, w2 = 5, w3 = 14;
        for (int i = 0; i < 94; i++) { w1 = std::max(w1, ilen(i)); w2 = std::max(w2, ilen(obs[i])); w3 = std::max(w3, ilen(sc[i])); }
        put(o, "%-*s  %-*s  %-*s\n", w1, "QualityScore", w2, "Count", w3, "QuantizedScore");
        for (int i = 0; i < 94; i++) put(o, "%*d  %*lld  %*d\n", w1, i, w2, (long long)obs[i], w3, (int)sc[i]);
        o += "\n";
    }
    {   // RecalTable0 (print-bqsr.go:78-122)
        std::vector<int> covs;
        for (int cv = 0; cv < T.g.n_cov; cv++) if (comb[cv].exists) covs.push_back(cv);
        std::sort(covs.begin(), covs.end(), [&](int a, int b) { return c->cov_names[a] < c->cov_names[b]; });
        int wrg = 9, wemp = 16, wrep = 18, wobs = 12, werr = 6; char b[64];
        for (int cv : covs) {
            wrg = std::max(wrg, (int)c->cov_names[cv].size()); wemp = std::max(wemp, ilen(comb[cv].emp) + 5);
            wrep = std::max(wrep, std::snprintf(b, sizeof b, "%.4f", comb[cv].reported)); wobs = std::max(wobs, ilen(comb[cv].obs)); werr = std::max(werr, ilen(comb[cv].mis) + 3);
        }
        put(o, "#:%sTable:6:%d:%%s:%%s:%%.4f:%%.4f:%%d:%%.2f:;\n#:%sTable:RecalTable0:\n", P, (int)covs.size(), P);
        put(o, "%-*s  %-9s  %-*s  %-*s  %-*s  %-*s\n", wrg, "ReadGroup", "EventType", wemp, "EmpiricalQuality", wrep, "EstimatedQReported", wobs, "Observations", werr, "Errors");
        for (int cv : covs)
            put(o, "%-*s  %-9s  %*d.0000  %*.4f  %*lld  %*lld.00\n", wrg, c->cov_names[cv].c_str(), "M", wemp - 5, (int)comb[cv].emp, wrep, comb[cv].reported, wobs,
                (long long)comb[cv].obs, werr - 3, (long long)comb[cv].mis);
        o += "\n";
    }
    auto row_less = [](const Row& a, const Row& b) { if (a.rg != b.rg) return a.rg < b.rg; if (a.q != b.q) return a.q < b.q; return a.text < b.text; };
    {   // RecalTable1 (print-bqsr.go:124-175)
        std::vector<Row> rows;
        for (int cv = 0; cv < T.g.n_cov; cv++) for (int q = 0; q < 94; q++) if (T.obs(cv, q, 0) > 0) rows.push_back({c->cov_names[cv], q, "", false, T.obs(cv, q, 0), T.mis(cv, q, 0), emp[T.g.idx(cv, q, 0)]});
        int wrg = 9, wq = 12, wemp = 16, wobs = 12, werr = 6;
        for (auto& r : rows) { wrg = std::max(wrg, (int)r.rg.size()); wq = std::max(wq, ilen(r.q)); wemp = std::max(wemp, ilen(r.emp) + 5); wobs = std::max(wobs, ilen(r.obs)); werr = std::max(werr, ilen(r.mis) + 3); }
        put(o, "#:%sTable:6:%d:%%s:%%d:%%s:%%.4f:%%d:%%.2f:;\n#:%sTable:RecalTable1:\n", P, (int)rows.size(), P);
        put(o, "%-*s  %-*s  %-9s  %-*s  %-*s  %-*s\n", wrg, "ReadGroup", wq, "QualityScore", "EventType", wemp, "EmpiricalQuality", wobs, "Observations", werr, "Errors");
        std::sort(rows.begin(), rows.end(), row_less);
        for (auto& r : rows) put(o, "%-*s  %*d  %-9s  %*d.0000  %*lld  %*lld.00\n", wrg, r.rg.c_str(), wq, r.q, "M", wemp - 5, (int)r.emp, wobs, (long long)r.obs, werr - 3, (long long)r.mis);
        o += "\n";
    }
    {   // RecalTable2 (print-bqsr.go:183-266): cycles and contexts, ordered by (read group, qual, TEXT of the covariate value)
        std::vector<Row> rows;
        for (int cv = 0; cv < T.g.n_cov; cv++) for (int q = 0; q < 94; q++) {
            for (int cy = -T.g.max_cycle; cy <= T.g.max_cycle; cy++) { const int col = T.g.col_cycle(cy); if (T.obs(cv, q, col) > 0) rows.push_back({c->cov_names[cv], q, std::to_string(cy), true, T.obs(cv, q, col), T.mis(cv, q, col), emp[T.g.idx(cv, q, col)]}); }
            for (int x = 0; x < 16; x++) { const int col = T.g.col_ctx(x); if (T.obs(cv, q, col) > 0) rows.push_back({c->cov_names[cv], q, context_text(x), false, T.obs(cv, q, col), T.mis(cv, q, col), emp[T.g.idx(cv, q, col)]}); }
        }
        int wrg = 9, wq = 12, wcv = 14, wemp = 16, wobs = 12, werr = 6;
        for (auto& r : rows) { wrg = std::max(wrg, (int)r.rg.size()); wq = std::max(wq, ilen(r.q)); wcv = std::max(wcv, (int)r.text.size()); wemp = std::max(wemp, ilen(r.emp) + 5); wobs = std::max(wobs, ilen(r.obs)); werr = std::max(werr, ilen(r.mis) + 3); }
        put(o, "#:%sTable:8:%d:%%s:%%d:%%s:%%s:%%s:%%.4f:%%d:%%.2f:;\n#:%sTable:RecalTable2:\n", P, (int)rows.size(), P);
        put(o, "%-*s  %-*s  %-*s  %-13s  %-9s  %-*s  %-*s  %-*s\n", wrg, "ReadGroup", wq, "QualityScore", wcv, "CovariateValue", "CovariateName", "EventType", wemp, "EmpiricalQuality", wobs, "Observations", werr, "Errors");
        std::sort(rows.begin(), rows.end(), row_less);
        for (auto& r : rows)
            put(o, "%-*s  %*d  %-*s  %-13s  %-9s  %*d.0000  %*lld  %*lld.00\n", wrg, r.rg.c_str(), wq, r.q, wcv, r.text.c_str(), r.cycle ? "Cycle" : "Context", "M", wemp - 5, (int)r.emp,
                wobs, (long long)r.obs, werr - 3, (long long)r.mis);
        o += "\n";
    }
    FILE* f = std::fopen(path, "w");
    if (!f) return c->fail(E_INVAL, "cannot create recalibration report %s", path);
    std::fwrite(o.data(), 1, o.size(), f);
    std::fclose(f);
    return E_OK;
}


// ---- device finalize ----
constexpr int FIN_T = 128;   // threads of the one-CTA tail kernel and of a LUT row; the tail's quantizer needs >= 94

// recalibrated byte of an estimate (ApplyBQSR :996-1000): quant[clamp(round(est))], then the static map when --sqq is set.
// qmaps: [0, 94) the quantization map, [QMAP_STAT, QMAP_STAT + 254) the static one
constexpr int QMAP_STAT = 96, QMAP_BYTES = QMAP_STAT + 256;
__device__ __forceinline__ uint8_t final_q(double est, const uint8_t* qmaps, int have_stat) {
    int r = (int)gomath::Round(est); r = max(1, min(r, 93));
    uint8_t nq = qmaps[r];
    if (have_stat) nq = qmaps[QMAP_STAT + nq];
    return nq;
}

// FinalizeBQSRTables: EmpiricalQuality of every existing entry with prior = its reported qual (:677-694); 0 where there is none
__global__ void fin_emp_kernel(const int64_t* __restrict__ t, TableGeom g, uint8_t* __restrict__ emp) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.cells()) return;
    const int64_t o = t[2 * i];
    emp[i] = o > 0 ? Entry(o, t[2 * i + 1]).empirical((double)(int)((i / (size_t)g.ncols()) % 94)) : 0;
}

// mergeQuantizationIntervals' penalty of merging interval i with the next one, j (:795-818), over the leaves' constants in shared memory
__device__ double fin_merge_penalty(int i, int j, const int* nxt, const long long* nobs, const long long* nerr, const long long* leafn, const double* leaflog) {
    const double mer = calc_error_rate(nobs[i] + nobs[j], nerr[i] + nerr[j]);
    if (mer == 0) return 0.0;
    const double lg = gomath::Log10(mer);
    double sumI = 0, sumJ = 0;
    for (int k = i; k < j; k++) sumI += k <= 6 ? 0.0 : gomath::Fabs(leaflog[k] - lg) * (double)leafn[k];   // leaf_penalty :780-786
    const int kend = nxt[j] >= 0 ? nxt[j] : 94;
    for (int k = j; k < kend; k++) sumJ += k <= 6 ? 0.0 : gomath::Fabs(leaflog[k] - lg) * (double)leafn[k];
    return sumI + sumJ;
}

// one CTA: the combined per-read-group entries (:655-674) -> fin[2 cov] = reported quality, fin[2 cov + 1] = its EmpiricalQuality minus
// it (the read-group term dG of :959-964); the quantization map (:863-899) -> qmaps[0, 94); the byte of a QUAL without table entries
__global__ void __launch_bounds__(FIN_T) fin_tail_kernel(const int64_t* __restrict__ t, TableGeom g, const uint8_t* __restrict__ emp, int levels, int have_stat,
                                                         double* __restrict__ fin, uint8_t* __restrict__ qmaps, uint8_t* __restrict__ cov_exists, uint8_t* __restrict__ unobs) {
    const Tables T{g, t};
    const int tid = threadIdx.x;
    for (int cv = tid; cv < g.n_cov; cv += FIN_T) {   // one covariate per thread
        const Combined cb = combine(T, cv);
        fin[2 * cv] = cb.reported;
        fin[2 * cv + 1] = cb.exists ? (double)cb.emp - cb.reported : 0.0;
        cov_exists[cv] = cb.exists ? 1 : 0;
    }
    __shared__ uint8_t quant[94];
    if (levels == 0) {
        for (int i = tid; i < 94; i += FIN_T) quant[i] = (uint8_t)i;
    } else {
        __shared__ long long qmap[94], nobs[94], nerr[94];
        __shared__ double leaflog[94];
        __shared__ int nxt[94];
        __shared__ bool head[94];
        __shared__ double wp[FIN_T / 32]; __shared__ int wi[FIN_T / 32];
        __shared__ int s_min;
        for (int i = tid; i < 94; i += FIN_T) qmap[i] = 0;
        __syncthreads();
        for (int j = tid; j < g.n_cov * 94; j += FIN_T) {
            const int cv = j / 94, q = j % 94;
            const int64_t o = T.obs(cv, q, 0);
            if (o > 0) atomicAdd(reinterpret_cast<unsigned long long*>(&qmap[emp[g.idx(cv, q, 0)]]), (unsigned long long)o);   // integer: order free
        }
        __syncthreads();
        for (int i = tid; i < 94; i += FIN_T) {
            const double er = q2err((double)i);
            nxt[i] = i + 1 == 94 ? -1 : i + 1; nobs[i] = qmap[i]; nerr[i] = (long long)((double)qmap[i] * er); leaflog[i] = gomath::Log10(er); head[i] = true;
        }
        __syncthreads();
        // mergeMinimalPenaltyQuantizationIntervals (:820-850): every pair of neighbouring intervals is priced at once; the minimum with the
        // lowest start wins, as the serial scan's strict '<' keeps the first
        for (int n = 94; n > levels; n--) {
            bool valid = tid < 94 && head[tid] && nxt[tid] >= 0;
            double p = valid ? fin_merge_penalty(tid, nxt[tid], nxt, nobs, nerr, qmap, leaflog) : 0.0;
            int idx = valid ? tid : 0x7fffffff;
            for (int o = 16; o; o >>= 1) {
                const double p2 = __shfl_down_sync(0xffffffffu, p, o); const int i2 = __shfl_down_sync(0xffffffffu, idx, o);
                const bool v2 = i2 != 0x7fffffff;
                if (v2 && (idx == 0x7fffffff || p2 < p || (p2 == p && i2 < idx))) { p = p2; idx = i2; }
            }
            if ((tid & 31) == 0) { wp[tid >> 5] = p; wi[tid >> 5] = idx; }
            __syncthreads();
            if (tid == 0) {
                double bp = wp[0]; int bi = wi[0];
                for (int w = 1; w < FIN_T / 32; w++)
                    if (wi[w] != 0x7fffffff && (bi == 0x7fffffff || wp[w] < bp || (wp[w] == bp && wi[w] < bi))) { bp = wp[w]; bi = wi[w]; }
                if (bi != 0x7fffffff) { const int b = nxt[bi]; nxt[bi] = nxt[b]; nobs[bi] += nobs[b]; nerr[bi] += nerr[b]; head[b] = false; }
                s_min = bi;
            }
            __syncthreads();
            if (s_min == 0x7fffffff) break;   // a single interval is left
        }
        if (tid == 0)
            for (int i = 0; i >= 0;) {
                const bool leaf = nxt[i] < 0 ? (i == 93) : (nxt[i] == i + 1);
                const uint8_t qs = leaf ? (uint8_t)i : (uint8_t)err_prob_to_quality(calc_error_rate(nobs[i], nerr[i]));
                const int kend = nxt[i] >= 0 ? nxt[i] : 94;
                for (int k = i; k < kend; k++) quant[k] = qs;
                i = nxt[i];
            }
    }
    __syncthreads();
    for (int i = tid; i < 94; i += FIN_T) qmaps[i] = quant[i];
    __syncthreads();
    // a QUAL value without any table entry (never observed, or above 93): only the read-group term (:901-919 with three map misses)
    for (int cv = tid; cv < g.n_cov; cv += FIN_T) unobs[cv] = cov_exists[cv] ? final_q(0.0 + fin[2 * cv + 1] + fin[2 * cv], qmaps, have_stat) : 0;
}

// the apply look-up table (ApplyBQSR :936-1006): recalibrated QUAL for (covariate, QUAL, cycle in [-Lc, Lc], context), one CTA per
// (covariate, QUAL) row of (2 Lc + 1) x 17 bytes; QUAL 0..5 and covariates without entries stay 0
__global__ void __launch_bounds__(FIN_T) fin_lut_kernel(const int64_t* __restrict__ t, TableGeom g, const double* __restrict__ fin, const uint8_t* __restrict__ qmaps, int have_stat,
                                                        const uint8_t* __restrict__ cov_exists, int Lc, uint8_t* __restrict__ lut) {
    const Tables T{g, t};
    const int cv = blockIdx.x / 94, q = blockIdx.x % 94, ncyc = 2 * Lc + 1, tid = threadIdx.x;
    uint8_t* row = lut + ((size_t)cv * 94 + q) * ncyc * 17;
    const int row_bytes = ncyc * 17;
    if (q < 6 || !cov_exists[cv]) { for (int i = tid; i < row_bytes; i += FIN_T) row[i] = 0; return; }
    // globalQualityScorePrior = -1 -> epsilon is always the read group's reportedQuality (:959-964)
    const double eps = fin[2 * cv], dG = fin[2 * cv + 1];
    const int64_t o0 = T.obs(cv, q, 0);
    double dQ = 0;
    if (o0 > 0) dQ = (double)Entry(o0, T.mis(cv, q, 0)).empirical(dG + eps) - dG - eps;
    const double cp = dQ + dG + eps;
    if (o0 <= 0) {   // QUAL never observed: no cycle/context entries either
        const uint8_t b = final_q(cp + 0.0, qmaps, have_stat);
        for (int i = tid; i < row_bytes; i += FIN_T) row[i] = b;
        return;
    }
    __shared__ double dctx[17]; __shared__ bool hctx[17];
    if (tid < 16) { const int col = g.col_ctx(tid); hctx[tid] = T.obs(cv, q, col) > 0; dctx[tid] = hctx[tid] ? (double)Entry(T.obs(cv, q, col), T.mis(cv, q, col)).empirical(cp) - cp : 0.0; }
    if (tid == 16) { hctx[16] = false; dctx[16] = 0; }
    __syncthreads();
    for (int cy = -Lc + tid; cy <= Lc; cy += FIN_T) {
        const int col = g.col_cycle(cy);
        const bool hc = T.obs(cv, q, col) > 0;
        const double dcy = hc ? (double)Entry(T.obs(cv, q, col), T.mis(cv, q, col)).empirical(cp) - cp : 0.0;
        uint8_t* dst = row + (size_t)(cy + Lc) * 17;
        for (int x = 0; x < 17; x++) {
            double dC = 0;
            if (hc) dC = dcy;
            if (hctx[x]) dC += dctx[x];
            dst[x] = final_q(cp + dC, qmaps, have_stat);
        }
    }
}

struct ClutArgs {
    const uint8_t* lut; const uint8_t* unobs; uint8_t* clut; uint16_t* rowtab;
    uint32_t bytes, blk, used; int Lc, S, n_slots;
    uint8_t slot_q[88]; uint16_t rowtab_h[256];
};
// the compact table of bqsr_apply2_kernel (see build_compact_lut), one thread per byte
__global__ void fin_clut_kernel(ClutArgs A) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 256) A.rowtab[i] = A.rowtab_h[i];
    if (i >= A.bytes) return;
    const uint32_t ncyc = 2u * (uint32_t)A.Lc + 1u, cyb = i / A.blk, off = i % A.blk, S17 = (uint32_t)A.S * 17u;
    uint8_t v = 0;
    if (cyb >= 32 && cyb < 32 + ncyc && off < A.used) {
        const uint32_t cy = cyb - 32, cv = off / S17, r = off % S17, sl = r / 17, x = r % 17;
        v = (int)sl < A.n_slots ? A.lut[(((size_t)cv * 94 + A.slot_q[sl]) * ncyc + cy) * 17 + x] : A.unobs[cv];
    }
    A.clut[i] = v;
}

// BinTerms into constant memory, once per device; the device buffers of the finalize, once per context
int ensure_fin_state(elp_ctx* c) {
    static std::mutex mu; static bool bin_set[64] = {false};
    {
        std::lock_guard<std::mutex> lk(mu);
        if (!bin_set[c->device & 63]) { CUDA_TRY(c, cudaMemcpyToSymbol(c_bin, &bin_terms(), sizeof(BinTerms))); bin_set[c->device & 63] = true; }
    }
    const int nc = std::max(1, c->geom.n_cov);
    CUDA_TRY(c, c->d_emp.fit(std::max<size_t>(1, c->geom.cells())));
    CUDA_TRY(c, c->d_fin.fit(2 * (size_t)nc));
    CUDA_TRY(c, c->d_cov_exists.fit(nc));
    CUDA_TRY(c, c->d_unobs.fit(nc));
    if (!c->d_qmaps.p) {   // the static quantization (initializeStaticQuantizedScores) depends on --sqq only
        CUDA_TRY(c, c->d_qmaps.fit(QMAP_BYTES));
        std::vector<uint8_t> m(QMAP_BYTES, 0);
        if (!c->sqq.empty()) { const std::vector<uint8_t> ss = static_quantized(c->sqq); std::copy(ss.begin(), ss.end(), m.begin() + QMAP_STAT); }
        int rc = upload_small(c, c->d_qmaps.p, m.data(), m.size()); if (rc) return rc;
    }
    return E_OK;
}

}  // namespace

int phase_bqsr_finalize(elp_ctx* c, const char* report_path) {
    if (!c->gathered) return c->fail(E_STATE, "elp_bqsr_finalize called before elp_bqsr_gather / elp_bqsr_tables_put");
    const TableGeom& g = c->geom;
    const size_t cells = g.cells();
    { int rc = ensure_fin_state(c); if (rc) return rc; }
    if (cells) {
        c->begin("bqsr_fin_emp", (double)cells * 17);
        fin_emp_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, c->stream>>>(c->d_tables.p, g, c->d_emp.p);
        c->end(); LAUNCH_CHECK(c);
    }
    c->begin("bqsr_fin_tail", (double)g.n_cov * 94 * 16);
    fin_tail_kernel<<<1, FIN_T, 0, c->stream>>>(c->d_tables.p, g, c->d_emp.p, c->quantize_levels, c->sqq.empty() ? 0 : 1, c->d_fin.p, c->d_qmaps.p, c->d_cov_exists.p, c->d_unobs.p);
    c->end(); LAUNCH_CHECK(c);
    if (report_path) {   // the report is host text: one copy of the tables and of EmpiricalQuality
        std::vector<int64_t> h_tables(cells * 2); std::vector<uint8_t> h_emp(cells);
        CUDA_TRY(c, cudaMemcpyAsync(h_tables.data(), c->d_tables.p, cells * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaMemcpyAsync(h_emp.data(), c->d_emp.p, cells, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        Tables T{g, h_tables.data()};
        std::vector<Combined> comb(g.n_cov);
        for (int cv = 0; cv < g.n_cov; cv++) comb[cv] = combine(T, cv);
        int rc = write_report(c, T, h_emp, comb, report_path); if (rc) return rc;
    }
    c->finalized = true;
    // the apply look-up table covers the cycles of the reads loaded so far; elp_bqsr_apply rebuilds it if longer reads arrive
    // later (apply-only workers: tables_put -> finalize -> append -> sort -> apply)
    if (c->n) { int rc = phase_adapt(c); if (rc) return rc; }
    return build_apply_lut(c, std::max(1, std::min(c->max_cycle, std::max(c->h_ranges.lseq_max, 1))));
}

int build_apply_lut(elp_ctx* c, int Lc) {
    if (!c->finalized) return c->fail(E_STATE, "apply look-up table requested before elp_bqsr_finalize");
    const TableGeom& g = c->geom;
    const size_t bytes = (size_t)g.n_cov * 94 * (2 * Lc + 1) * 17;
    CUDA_TRY(c, c->d_lut.fit(bytes + 16));
    if (g.n_cov) {
        c->begin("bqsr_fin_lut", (double)bytes);
        fin_lut_kernel<<<(unsigned)(g.n_cov * 94), FIN_T, 0, c->stream>>>(c->d_tables.p, g, c->d_fin.p, c->d_qmaps.p, c->sqq.empty() ? 0 : 1, c->d_cov_exists.p, Lc, c->d_lut.p);
        c->end(); LAUNCH_CHECK(c);
    }
    c->lut_maxcyc = Lc;
    c->clut_Lc = 0;                // rebuilt on the next apply
    return E_OK;
}

// The apply table compacted for bqsr_apply2_kernel: only the QUAL values >= 6 that occur in the QUAL arena get rows ("slots"); layout
// [cycle + Lc + 32][covariate][slot][17] with 32 zero cycles of margin on both sides (lanes index up to 31 bases past a read's end) and an
// odd number of bytes per cycle (bank spread).  When some QUAL above 93 occurs (presence bits 94..127; bit 127 stands for 128..255), one more
// slot holds every covariate's "unobserved QUAL" byte and QUAL 94..255 map to it.  Rebuilt whenever the full table or the set of QUAL
// values changes.  The presence bits are the host copy phase_adapt (or elp_filter_target_regions) took with the range summary.
int build_compact_lut(elp_ctx* c) {
    const uint32_t* present = c->h_qpresent;
    if (c->clut_Lc == c->lut_maxcyc && memcmp(present, c->clut_present, 16) == 0) return E_OK;
    memcpy(c->clut_present, present, 16);
    c->clut_Lc = 0; c->clut_bytes = 0;
    ClutArgs A{};
    A.n_slots = 0;
    for (int q = 6; q < 94; q++) if ((present[q >> 5] >> (q & 31)) & 1u) A.slot_q[A.n_slots++] = (uint8_t)q;
    const bool above93 = (present[2] >> 30) != 0 || present[3] != 0;   // bits 94..127
    const int S = A.n_slots + (above93 ? 1 : 0), Lc = c->lut_maxcyc, ncyc = 2 * Lc + 1, n_cov = c->geom.n_cov;
    if (S == 0 || n_cov == 0 || !c->d_lut.p) return E_OK;
    uint32_t blk = (uint32_t)(n_cov * S * 17); if (!(blk & 1)) blk++;
    const size_t bytes = ((size_t)(ncyc + 64) * blk + 15) / 16 * 16;
    if (bytes > 80 * 1024) return E_OK;                               // too large for two CTAs per SM: the global-memory kernel serves
    for (int sl = 0; sl < A.n_slots; sl++) A.rowtab_h[A.slot_q[sl]] = (uint16_t)(sl * 17);
    if (above93) for (int q = 94; q < 256; q++) A.rowtab_h[q] = (uint16_t)((S - 1) * 17);
    CUDA_TRY(c, c->d_clut.fit(bytes));
    A.lut = c->d_lut.p; A.unobs = c->d_unobs.p; A.clut = c->d_clut.p; A.rowtab = c->d_rowtab.p;
    A.bytes = (uint32_t)bytes; A.blk = blk; A.used = (uint32_t)(n_cov * S * 17); A.Lc = Lc; A.S = S;
    c->begin("bqsr_fin_clut", 2.0 * (double)bytes);
    fin_clut_kernel<<<(unsigned)((bytes + 255) / 256), 256, 0, c->stream>>>(A);
    c->end(); LAUNCH_CHECK(c);
    c->clut_bytes = (uint32_t)bytes; c->clut_blk = blk; c->clut_S17 = (uint32_t)(S * 17); c->clut_Lc = Lc;
    return E_OK;
}

int bqsr_empirical_copy(elp_ctx* c, uint8_t* emp) {
    if (c->geom.cells()) {
        CUDA_TRY(c, cudaMemcpyAsync(emp, c->d_emp.p, c->geom.cells(), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    return E_OK;
}
