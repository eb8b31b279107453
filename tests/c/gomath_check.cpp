// gomath_check.cpp -- the finalize's Go math (elprep_b200/csrc/gomath.hpp, compiled here as plain host C++ the way g++ sees it outside
// nvcc) against the oracle's restatement (oracle/gomath.c), bit for bit over a sweep of arguments.  Both must be compiled without
// floating-point contraction.  Prints the number of comparisons and "OK", or the first mismatch.
#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
#include "gomath.hpp"
#include "gomath.h"

static uint64_t bits_of(double x) { uint64_t u; std::memcpy(&u, &x, 8); return u; }
static long n_checked = 0;
static bool same(const char* fn, double a, double b, double x, double y) {
    n_checked++;
    if (bits_of(a) == bits_of(b)) return true;
    std::printf("MISMATCH %s(%.17g, %.17g): header %.17g, oracle %.17g\n", fn, x, y, a, b);
    return false;
}

int main() {
    std::mt19937_64 rng(20261017);
    std::vector<double> xs;
    for (int i = 1; i < 4000; i++) xs.push_back((double)i);                    // integer counts (Lgamma of n + 1, k + 1, n - k + 1)
    for (int i = 0; i < 94; i++) xs.push_back(std::pow(10.0, i / -10.0));     // error rates of every QUAL
    for (double x : {2147483646.0, 2147483647.0, 6442450941.0, 1e15, 2.8823037615171174e17, 0.5, 0.70710678118654746, 1.0, 2.0, 8.0,
                     1.4616321449683622, 0.9, 0.2316321449683623, 4.9406564584124654e-324, 2.2250738585072014e-308})
        xs.push_back(x);
    std::uniform_real_distribution<double> u01(0.0, 1.0), uexp(-300.0, 300.0), uq(-10.0, 100.0);
    for (int i = 0; i < 20000; i++) { xs.push_back(u01(rng) * 10.0); xs.push_back(std::pow(10.0, uexp(rng))); xs.push_back(1.0 + u01(rng) * 1e-6); }
    bool ok = true;
    for (double x : xs) {
        int e1 = 0, e2 = 0;
        const double f1 = gomath::Frexp(x, e1), f2 = gm_frexp(x, &e2);
        ok &= same("Frexp", f1, f2, x, 0) && e1 == e2;
        ok &= same("Log", gomath::Log(x), gm_log(x), x, 0);
        ok &= same("Log2", gomath::Log2(x), gm_log2(x), x, 0);
        ok &= same("Log10", gomath::Log10(x), gm_log10(x), x, 0);
        ok &= same("Lgamma", gomath::Lgamma(x), gm_lgamma(x), x, 0);
        ok &= same("Round", gomath::Round(x * 0.37 - 20), gm_round(x * 0.37 - 20), x * 0.37 - 20, 0);
        ok &= same("Round", gomath::Round(x - 0.5), gm_round(x - 0.5), x - 0.5, 0);
        if (x < 700) ok &= same("Exp", gomath::Exp(-x), gm_exp(-x), -x, 0), ok &= same("Exp", gomath::Exp(x), gm_exp(x), x, 0);
        ok &= same("Ldexp", gomath::Ldexp(x, -1070), gm_ldexp(x, -1070), x, -1070);
        if (!ok) break;
    }
    for (int i = 0; i < 200000 && ok; i++) {   // Pow(10, phred / -10) over reported qualities, and Pow of the quantizer's inputs
        const double q = i < 1000 ? (double)(i % 100) : uq(rng);
        ok &= same("Pow", gomath::Pow(10, q / -10), gm_pow(10, q / -10), 10, q / -10);
        const double x = u01(rng) * 20.0, y = uq(rng) / 7.0;
        ok &= same("Pow", gomath::Pow(x, y), gm_pow(x, y), x, y);
    }
    for (double y : {0.0, 1.0, 0.5, -0.5, -1.0, 2.0, -9.3})
        for (double x : {0.1, 0.5, 10.0, 3.0}) ok &= same("Pow", gomath::Pow(x, y), gm_pow(x, y), x, y);
    std::printf("%ld comparisons\n%s\n", n_checked, ok ? "OK" : "FAILED");
    return ok ? 0 : 1;
}
