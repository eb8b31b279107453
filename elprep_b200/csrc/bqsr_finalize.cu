// bqsr_finalize.cu -- host side of BQSR between gather and apply (replaces FinalizeBQSRTables, filters/bqsr.go:677-694,
// initializeCombinedBQSRTable :655-674, the quantizers :708-899, estimateHierarchicalBayesianQuality :901-919 as memoised
// by ApplyBQSR :973-1000, and PrintBQSRTables, filters/print-bqsr.go:49-298).
//
// The tables are tiny (<= a few 10^5 integer cells), the arithmetic is IEEE double with Go's math functions
// (gomath.hpp) and must be evaluated in the reference's operation order, so this runs on the host between two kernels.
// Everything the apply kernel needs is folded into ONE byte look-up table indexed by
// (read-group covariate, reported qual, cycle, context) -- exactly the memo the reference fills lazily per worker.
// Reference non-determinism fixed here: the combined per-read-group entry accumulates in ascending-qual order
// (the reference iterates a Go map, :657-668).
#include <algorithm>
#include <cfloat>
#include <cstdio>
#include <string>
#include <thread>
#include <vector>
#include "ctx.h"
#include "gomath.hpp"

namespace {

const double kPriorCache[21] = {   // embedded data, filters/bqsr.go:569-591: log10(0.9*exp(-d^2/0.5)), last = -MaxFloat64
    -0.045757490560675115, -0.9143464543671788, -3.5201133457866898, -7.863058164819208, -13.943180911464733, -21.760481585723266,
    -31.314960187594806, -42.606616717079355, -55.63545117417691, -70.40146355888747, -86.90465387121104, -105.14502211114761,
    -125.1225682786972, -146.83729237385978, -170.2891943966354, -195.47827434702398, -222.4045322250256, -251.06796803064023,
    -281.46858176386786, -313.60637342472336, -1.7976931348623157e308};

struct BinTerms {   // per-bin constants of log10BinomialProbability (:607-613): l = i/-10, m = log10(1 - 10^l)
    double l[61], m[61];
    BinTerms() { for (int i = 0; i < 61; i++) { l[i] = (double)i / -10.0; m[i] = (l[i] == 0.0) ? 0.0 : gomath::Log10(1.0 - gomath::Pow(10, l[i])); } }
};
const BinTerms& bin_terms() { static BinTerms b; return b; }

inline double log10_gamma(int64_t n) { return gomath::Lgamma((double)n) * 0.4342944819032518; }   // :598-601

// calculateEmpiricalQuality (:644-649) = calculateBayesianEstimateOfEmpiricalQuality (:623-642) on the smoothed counts
struct Entry {
    int64_t n, k; double coef;
    Entry(int64_t obs, int64_t mis) {
        n = obs + 2; k = mis + 1;
        const int64_t maxObs = 2147483647 - 1;
        if (n > maxObs) { k = (int64_t)gomath::Round((double)k * ((double)maxObs / (double)n)); n = maxObs; }
        coef = log10_gamma(n + 1) - log10_gamma(k + 1) - log10_gamma(n - k + 1);   // log10BinomialCoefficient :603-605
    }
    uint8_t empirical(double prior) const {
        const BinTerms& B = bin_terms();
        double best = -DBL_MAX; int bi = 0;
        for (int i = 0; i < 61; i++) {
            int d = (int)((double)i - prior); if (d < 0) d = -d; if (d > 20) d = 20;   // log10QualEmpiricalPrior :593-596
            const double p1 = kPriorCache[d];
            const double p2 = (B.l[i] == 0.0) ? -DBL_MAX : (coef + B.l[i] * (double)k) + B.m[i] * (double)(n - k);   // n is never 0 here (obs+2)
            const double post = p1 + p2;
            if (best < post) { best = post; bi = i; }
        }
        return (uint8_t)std::min(bi, 93);
    }
};

inline double q2err(double phred) { return gomath::Pow(10, phred / -10); }
inline double q2prob(double phred) { return 1 - gomath::Pow(10, phred / -10); }

struct Combined { bool exists = false; double reported = 0; int64_t obs = 0, mis = 0; uint8_t emp = 0; };

struct Tables {
    const TableGeom& g; const int64_t* t;
    int64_t obs(int cov, int q, int col) const { return t[2 * g.idx(cov, q, col)]; }
    int64_t mis(int cov, int q, int col) const { return t[2 * g.idx(cov, q, col) + 1]; }
};

Combined combine(const Tables& T, int cov) {   // :655-674
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

int err_prob_to_quality(double prob) {   // :701-706
    if (prob == 0.0) return 93;
    int q = (int)gomath::Round(-10 * gomath::Log10(prob));
    return std::max(std::min(q, 93), 1);
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
double calc_error_rate(int64_t nobs, int64_t nerr) { return nobs == 0 ? 0.0 : (double)(nerr + 1) / (double)(nobs + 1); }
double leaf_penalty(int k, const std::vector<QInterval>& iv, double globalErrorRate) {   // :780-786
    if (k <= 6) return 0.0;
    return std::fabs(gomath::Log10(iv[k].errorRate) - gomath::Log10(globalErrorRate)) * (double)iv[k].leafNobs;
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

// run f(i) for i in [0,n) on a few host threads (the per-entry posteriors are independent)
template <class F> void host_parallel_for(int n, F f) {
    const int nt = std::max(1, std::min<int>({8, (int)std::thread::hardware_concurrency(), n}));
    if (nt == 1) { for (int i = 0; i < n; i++) f(i); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++) th.emplace_back([=]() { for (int i = t; i < n; i += nt) f(i); });
    for (auto& x : th) x.join();
}

}  // namespace

int build_apply_lut(elp_ctx* c, int Lc);

int phase_bqsr_finalize(elp_ctx* c, const char* report_path) {
    if (!c->gathered) return c->fail(E_STATE, "elp_bqsr_finalize called before elp_bqsr_gather / elp_bqsr_tables_put");
    const TableGeom& g = c->geom;
    const size_t cells = g.cells();
    c->h_tables.resize(cells * 2);
    CUDA_TRY(c, cudaMemcpyAsync(c->h_tables.data(), c->d_tables, cells * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    Tables T{g, c->h_tables.data()};
    // FinalizeBQSRTables: EmpiricalQuality of every existing entry with prior = its reported qual (:677-694)
    c->h_emp.assign(cells, 0);
    host_parallel_for(g.n_cov * 94, [&](int row) {
        const int cv = row / 94, q = row % 94;
        for (int col = 0; col < g.ncols(); col++) {
            const int64_t o = T.obs(cv, q, col);
            if (o > 0) c->h_emp[g.idx(cv, q, col)] = Entry(o, T.mis(cv, q, col)).empirical((double)q);
        }
    });
    std::vector<Combined> comb(g.n_cov);
    for (int cv = 0; cv < g.n_cov; cv++) comb[cv] = combine(T, cv);
    if (report_path) { int rc = write_report(c, T, c->h_emp, comb, report_path); if (rc) return rc; }

    c->finalized = true;
    // the apply look-up table covers the cycles of the reads loaded so far; elp_bqsr_apply rebuilds it if longer reads arrive
    // later (apply-only workers: tables_put -> finalize -> append -> sort -> apply)
    if (c->n) { int rc = phase_adapt(c); if (rc) return rc; }
    return build_apply_lut(c, std::max(1, std::min(c->max_cycle, std::max(c->h_ranges.lseq_max, 1))));
}

// ---- the apply look-up table (ApplyBQSR :936-1006): recalibrated QUAL for (covariate, QUAL, cycle in [-Lc, Lc], context) ----
int build_apply_lut(elp_ctx* c, int Lc) {
    if (!c->finalized) return c->fail(E_STATE, "apply look-up table requested before elp_bqsr_finalize");
    const TableGeom& g = c->geom;
    Tables T{g, c->h_tables.data()};
    std::vector<Combined> comb(g.n_cov);
    for (int cv = 0; cv < g.n_cov; cv++) comb[cv] = combine(T, cv);
    std::vector<int64_t> qmap; std::vector<uint8_t> quant;
    quantized(T, c->h_emp, c->quantize_levels, qmap, quant);
    std::vector<uint8_t> stat; const bool have_stat = !c->sqq.empty();
    if (have_stat) stat = static_quantized(c->sqq);
    const int ncyc = 2 * Lc + 1;
    std::vector<uint8_t> lut((size_t)g.n_cov * 94 * ncyc * 17, 0);
    std::vector<uint8_t> cov_exists(g.n_cov, 0), unobs(g.n_cov, 0);
    std::vector<double> dGv(g.n_cov, 0.0);
    auto final_q = [&](double est) { int r = (int)gomath::Round(est); r = std::max(1, std::min(r, 93)); uint8_t nq = quant[r]; if (have_stat) nq = stat[nq]; return nq; };
    for (int cv = 0; cv < g.n_cov; cv++) {
        if (!comb[cv].exists) continue;
        cov_exists[cv] = 1;
        // globalQualityScorePrior = -1 -> epsilon is always the read group's reportedQuality (:959-964)
        dGv[cv] = (double)Entry(comb[cv].obs, comb[cv].mis).empirical(comb[cv].reported) - comb[cv].reported;
        // a QUAL value without any table entry (never observed, or above 93): only the read-group term (:901-919 with three map misses)
        unobs[cv] = final_q(0.0 + dGv[cv] + comb[cv].reported);
    }
    host_parallel_for(g.n_cov * 88, [&](int job) {
        const int cv = job / 88, q = 6 + job % 88;
        if (!comb[cv].exists) return;
        const double eps = comb[cv].reported, dG = dGv[cv];
        double dQ = 0;
        if (T.obs(cv, q, 0) > 0) dQ = (double)Entry(T.obs(cv, q, 0), T.mis(cv, q, 0)).empirical(dG + eps) - dG - eps;
        const double cp = dQ + dG + eps;
        uint8_t* row = &lut[((size_t)cv * 94 + q) * ncyc * 17];
        if (T.obs(cv, q, 0) <= 0) { std::memset(row, final_q(cp + 0.0), (size_t)ncyc * 17); return; }   // QUAL never observed: no cycle/context entries either
        double dctx[17]; bool hctx[17];
        for (int x = 0; x < 16; x++) { const int col = g.col_ctx(x); hctx[x] = T.obs(cv, q, col) > 0; dctx[x] = hctx[x] ? (double)Entry(T.obs(cv, q, col), T.mis(cv, q, col)).empirical(cp) - cp : 0.0; }
        hctx[16] = false; dctx[16] = 0;
        for (int cy = -Lc; cy <= Lc; cy++) {
            const int col = g.col_cycle(cy);
            const bool hc = T.obs(cv, q, col) > 0;
            const double dcy = hc ? (double)Entry(T.obs(cv, q, col), T.mis(cv, q, col)).empirical(cp) - cp : 0.0;
            uint8_t* dst = row + (size_t)(cy + Lc) * 17;
            for (int x = 0; x < 17; x++) {
                double dC = 0;
                if (hc) dC = dcy;
                if (hctx[x]) dC += dctx[x];
                dst[x] = final_q(cp + dC);
            }
        }
    });
    if (c->lut_cap < lut.size() + 16) {
        if (c->d_lut) { cudaFree(c->d_lut); c->d_lut = nullptr; }
        CUDA_TRY(c, cudaMalloc(&c->d_lut, lut.size() + 16));
        c->lut_cap = lut.size() + 16;
    }
    { int rcu = upload_small(c, c->d_lut, lut.data(), lut.size()); if (rcu) return rcu; }
    if (!c->d_cov_exists) CUDA_TRY(c, cudaMalloc(&c->d_cov_exists, std::max(1, g.n_cov)));
    { int rcu = upload_small(c, c->d_cov_exists, cov_exists.data(), g.n_cov); if (rcu) return rcu; }
    if (!c->d_unobs) CUDA_TRY(c, cudaMalloc(&c->d_unobs, std::max(1, g.n_cov)));
    { int rcu = upload_small(c, c->d_unobs, unobs.data(), g.n_cov); if (rcu) return rcu; }
    c->h_unobs.swap(unobs);
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    c->lut_maxcyc = Lc;
    c->h_lut.swap(lut);            // kept for the compact shared-memory table (build_compact_lut)
    c->clut_Lc = 0;                // rebuilt on the next apply
    return E_OK;
}

// The apply table compacted for bqsr_apply2_kernel: only the QUAL values >= 6 that occur in the QUAL arena get rows ("slots"); layout
// [cycle + Lc + 32][covariate][slot][17] with 32 zero cycles of margin on both sides (lanes index up to 31 bases past a read's end) and an
// odd number of bytes per cycle (bank spread).  When some QUAL above 93 occurs (presence bits 94..127; bit 127 stands for 128..255), one more
// slot holds every covariate's "unobserved QUAL" byte and QUAL 94..255 map to it.  Rebuilt whenever the full table or the set of QUAL
// values changes.
int build_compact_lut(elp_ctx* c) {
    uint32_t present[4] = {0, 0, 0, 0};
    CUDA_TRY(c, cudaMemcpyAsync(present, c->d_qpresent, 16, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (c->clut_Lc == c->lut_maxcyc && memcmp(present, c->clut_present, 16) == 0) return E_OK;
    memcpy(c->clut_present, present, 16);
    c->clut_Lc = 0; c->clut_bytes = 0;
    std::vector<int> slots;
    for (int q = 6; q < 94; q++) if ((present[q >> 5] >> (q & 31)) & 1u) slots.push_back(q);
    const bool above93 = (present[2] >> 30) != 0 || present[3] != 0;   // bits 94..127
    const int S = (int)slots.size() + (above93 ? 1 : 0), Lc = c->lut_maxcyc, ncyc = 2 * Lc + 1, n_cov = c->geom.n_cov;
    if (S == 0 || n_cov == 0 || c->h_lut.empty()) return E_OK;
    uint32_t blk = (uint32_t)(n_cov * S * 17); if (!(blk & 1)) blk++;
    const size_t bytes = ((size_t)(ncyc + 64) * blk + 15) / 16 * 16;
    if (bytes > 80 * 1024) return E_OK;                               // too large for two CTAs per SM: the global-memory kernel serves
    std::vector<uint8_t> t(bytes, 0); std::vector<uint16_t> rowtab(256, 0);
    for (int sl = 0; sl < (int)slots.size(); sl++) rowtab[slots[sl]] = (uint16_t)(sl * 17);
    if (above93) for (int q = 94; q < 256; q++) rowtab[q] = (uint16_t)((S - 1) * 17);
    for (int cy = 0; cy < ncyc; cy++) for (int cv = 0; cv < n_cov; cv++) {
        for (int sl = 0; sl < (int)slots.size(); sl++)
            memcpy(&t[(size_t)(cy + 32) * blk + (size_t)(cv * S + sl) * 17], &c->h_lut[(((size_t)cv * 94 + slots[sl]) * ncyc + cy) * 17], 17);
        if (above93) memset(&t[(size_t)(cy + 32) * blk + (size_t)(cv * S + S - 1) * 17], c->h_unobs[cv], 17);
    }
    if (c->clut_cap < bytes) { if (c->d_clut) cudaFree(c->d_clut); c->d_clut = nullptr; CUDA_TRY(c, cudaMalloc(&c->d_clut, bytes)); c->clut_cap = bytes; }
    if (!c->d_rowtab) CUDA_TRY(c, cudaMalloc(&c->d_rowtab, 512));
    { int rcu = upload_small(c, c->d_clut, t.data(), bytes); if (rcu) return rcu; }
    { int rcu = upload_small(c, c->d_rowtab, rowtab.data(), 512); if (rcu) return rcu; }
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    c->clut_bytes = (uint32_t)bytes; c->clut_blk = blk; c->clut_S17 = (uint32_t)(S * 17); c->clut_Lc = Lc;
    return E_OK;
}
