// gomath.hpp -- the Go standard-library math functions the BQSR finalize step depends on, restated for the
// product's finalize (filters/bqsr.go:561-706 call math.Pow, math.Lgamma, math.Log10 via filters/unpedantic.go:28-30,
// math.Round).  Bit-level behaviour matters: QUAL bytes are argmaxes and truncations of these values.  Algorithms: FreeBSD
// msun e_log.c / e_exp.c / e_lgamma_r.c as used by Go's pure-Go math package, and Go's own pow.go / log10.go.
// One source for host and device (bqsr_finalize_dev.cu): the two give the same bits only when neither contracts a*b+c into
// a fused multiply-add (amd64 Go does not fuse), so host code is compiled with -ffp-contract=off and device code with
// -fmad=false.  Only IEEE-exact primitives are used (+ - * /, sqrt, round, bit casts), never the platform's log/exp/pow.
// Only the domain the path needs is covered (finite positive arguments).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define GM_HD __host__ __device__
#else
#define GM_HD
#endif

namespace gomath {

GM_HD inline uint64_t bits(double x) {
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t u; std::memcpy(&u, &x, 8); return u;
#endif
}
GM_HD inline double from_bits(uint64_t u) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)u);
#else
    double x; std::memcpy(&x, &u, 8); return x;
#endif
}
GM_HD inline bool IsNaN(double x) { return (bits(x) & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL; }
GM_HD inline bool IsInf(double x) { return (bits(x) & 0x7fffffffffffffffULL) == 0x7ff0000000000000ULL; }
GM_HD inline double Fabs(double x) { return from_bits(bits(x) & 0x7fffffffffffffffULL); }
GM_HD inline double CopySign(double x, double s) { return from_bits((bits(x) & 0x7fffffffffffffffULL) | (bits(s) & 0x8000000000000000ULL)); }
GM_HD inline double Inf() { return from_bits(0x7ff0000000000000ULL); }
GM_HD inline double NaN() { return from_bits(0x7ff8000000000000ULL); }

GM_HD inline double Frexp(double f, int& e) {
    e = 0;
    if (f == 0 || IsInf(f) || IsNaN(f)) return f;
    if (Fabs(f) < 2.2250738585072014e-308) { f *= 4503599627370496.0; e = -52; }
    uint64_t x = bits(f);
    e += (int)((x >> 52) & 0x7ff) - 1022;
    x = (x & ~(0x7ffULL << 52)) | (1022ULL << 52);
    return from_bits(x);
}
GM_HD inline double Ldexp(double frac, int exp) {
    if (frac == 0 || IsInf(frac) || IsNaN(frac)) return frac;
    int e; frac = Frexp(frac, e);
    exp += e - 1;   // frac is in [0.5,1): unbiased exponent -1
    if (exp < -1075) return CopySign(0.0, frac);
    if (exp > 1023) return frac < 0 ? -Inf() : Inf();
    double m = 1;
    if (exp < -1022) { exp += 53; m = 1.0 / 9007199254740992.0; }
    uint64_t x = (bits(frac) & ~(0x7ffULL << 52)) | ((uint64_t)(exp + 1023) << 52);
    return m * from_bits(x);
}
GM_HD inline double Log(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10;
    const double L1 = 6.666666666666735130e-01, L2 = 3.999999999940941908e-01, L3 = 2.857142874366239149e-01, L4 = 2.222219843214978396e-01,
                 L5 = 1.818357216161805012e-01, L6 = 1.531383769920937332e-01, L7 = 1.479819860511658591e-01;
    if (IsNaN(x) || (IsInf(x) && x > 0)) return x;
    if (x < 0) return NaN();
    if (x == 0) return -Inf();
    int ki; double f1 = Frexp(x, ki);
    if (f1 < 0.70710678118654752440084436210484904) { f1 *= 2; ki--; }
    const double f = f1 - 1, k = (double)ki;
    const double s = f / (2 + f), s2 = s * s, s4 = s2 * s2;
    const double t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)));
    const double t2 = s4 * (L2 + s4 * (L4 + s4 * L6));
    const double R = t1 + t2, hfsq = 0.5 * f * f;
    return k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f);
}
GM_HD inline double Log2(double x) { int e; const double frac = Frexp(x, e); if (frac == 0.5) return (double)(e - 1); return Log(frac) * 1.4426950408889634 + (double)e; }
GM_HD inline double Log10(double x) { return Log2(x) * 0.3010299956639812; }
GM_HD inline double Exp(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10, Log2e = 1.44269504088896338700e+00;
    const double P1 = 1.66666666666666657415e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
                 P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
    if (IsNaN(x) || (IsInf(x) && x > 0)) return x;
    if (IsInf(x)) return 0;
    if (x > 7.09782712893383973096e+02) return Inf();
    if (x < -7.45133219101941108420e+02) return 0;
    if (-3.725290298461914e-09 < x && x < 3.725290298461914e-09) return 1 + x;
    int k = 0;
    if (x < 0) k = (int)(Log2e * x - 0.5); else if (x > 0) k = (int)(Log2e * x + 0.5);
    const double hi = x - (double)k * Ln2Hi, lo = (double)k * Ln2Lo;
    const double r = hi - lo, t = r * r;
    const double c = r - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
    const double y = 1 - ((lo - (r * c) / (2 - c)) - hi);
    return Ldexp(y, k);
}
// math.Pow for x > 0 finite, y finite
GM_HD inline double Pow(double x, double y) {
    if (y == 0 || x == 1) return 1;
    if (y == 1) return x;
    if (y == 0.5) return ::sqrt(x);
    if (y == -0.5) return 1 / ::sqrt(x);
    double ay = Fabs(y), yi, yf;
    if (ay < 1) { yi = 0; yf = ay; }
    else { uint64_t b = bits(ay); const unsigned e = (unsigned)((b >> 52) & 0x7ff) - 1023; if (e < 52) b &= ~((1ULL << (52 - e)) - 1); yi = from_bits(b); yf = ay - yi; }
    double a1 = 1.0; int ae = 0;
    if (yf != 0) { if (yf > 0.5) { yf--; yi++; } a1 = Exp(yf * Log(x)); }
    int xe; double x1 = Frexp(x, xe);
    for (int64_t i = (int64_t)yi; i != 0; i >>= 1) {
        if (xe < -(1 << 12) || (1 << 12) < xe) { ae += xe; break; }
        if (i & 1) { a1 *= x1; ae += xe; }
        x1 *= x1; xe <<= 1;
        if (x1 < .5) { x1 += x1; xe--; }
    }
    if (y < 0) { a1 = 1 / a1; ae = -ae; }
    return Ldexp(a1, ae);
}
// math.Lgamma for x > 0
GM_HD inline double Lgamma(double x) {
    constexpr double A[] = {7.72156649015328655494e-02, 3.22467033424113591611e-01, 6.73523010531292681824e-02, 2.05808084325167332806e-02,
        7.38555086081402883957e-03, 2.89051383673415629091e-03, 1.19270763183362067845e-03, 5.10069792153511336608e-04, 2.20862790713908385557e-04,
        1.08011567247583939954e-04, 2.52144565451257326939e-05, 4.48640949618915160150e-05};
    constexpr double Rr[] = {1.0, 1.39200533467621045958e+00, 7.21935547567138069525e-01, 1.71933865632803078993e-01, 1.86459191715652901344e-02,
        7.77942496381893596434e-04, 7.32668430744625636189e-06};
    constexpr double S[] = {-7.72156649015328655494e-02, 2.14982415960608852501e-01, 3.25778796408930981787e-01, 1.46350472652464452805e-01,
        2.66422703033638609560e-02, 1.84028451407337715652e-03, 3.19475326584100867617e-05};
    constexpr double T[] = {4.83836122723810047042e-01, -1.47587722994593911752e-01, 6.46249402391333854778e-02, -3.27885410759859649565e-02,
        1.79706750811820387126e-02, -1.03142241298341437450e-02, 6.10053870246291332635e-03, -3.68452016781138256760e-03, 2.25964780900612472250e-03,
        -1.40346469989232843813e-03, 8.81081882437654011382e-04, -5.38595305356740546715e-04, 3.15632070903625950361e-04, -3.12754168375120860518e-04,
        3.35529192635519073543e-04};
    constexpr double U[] = {-7.72156649015328655494e-02, 6.32827064025093366517e-01, 1.45492250137234768737e+00, 9.77717527963372745603e-01,
        2.28963728064692451092e-01, 1.33810918536787660377e-02};
    constexpr double V[] = {1.0, 2.45597793713041134822e+00, 2.12848976379893395361e+00, 7.69285150456672783825e-01, 1.04222645593369134254e-01,
        3.21709242282423911810e-03};
    constexpr double W[] = {4.18938533204672725052e-01, 8.33333333333329678849e-02, -2.77777777728775536470e-03, 7.93650558643019558500e-04,
        -5.95187557450339963135e-04, 8.36339918996282139126e-04, -1.63092934096575273989e-03};
    const double Ymin = 1.461632144968362245, Tc = 1.46163214496836224576e+00, Tf = -1.21486290535849611461e-01, Tt = -3.63867699703950536541e-18;
    if (IsNaN(x) || IsInf(x)) return x;
    if (x <= 0) return x == 0 ? Inf() : NaN();
    if (x < 8.470329472543003e-22) return -Log(x);
    if (x == 1 || x == 2) return 0;
    double lg;
    if (x < 2) {
        double y; int i;
        if (x <= 0.9) {
            lg = -Log(x);
            if (x >= (Ymin - 1 + 0.27)) { y = 1 - x; i = 0; } else if (x >= (Ymin - 1 - 0.23)) { y = x - (Tc - 1); i = 1; } else { y = x; i = 2; }
        } else {
            lg = 0;
            if (x >= (Ymin + 0.27)) { y = 2 - x; i = 0; } else if (x >= (Ymin - 0.23)) { y = x - Tc; i = 1; } else { y = x - 1; i = 2; }
        }
        if (i == 0) {
            const double z = y * y;
            const double p1 = A[0] + z * (A[2] + z * (A[4] + z * (A[6] + z * (A[8] + z * A[10]))));
            const double p2 = z * (A[1] + z * (+A[3] + z * (A[5] + z * (A[7] + z * (A[9] + z * A[11])))));
            const double p = y * p1 + p2;
            lg += (p - 0.5 * y);
        } else if (i == 1) {
            const double z = y * y, w = z * y;
            const double p1 = T[0] + w * (T[3] + w * (T[6] + w * (T[9] + w * T[12])));
            const double p2 = T[1] + w * (T[4] + w * (T[7] + w * (T[10] + w * T[13])));
            const double p3 = T[2] + w * (T[5] + w * (T[8] + w * (T[11] + w * T[14])));
            const double p = z * p1 - (Tt - w * (p2 + y * p3));
            lg += (Tf + p);
        } else {
            const double p1 = y * (U[0] + y * (U[1] + y * (U[2] + y * (U[3] + y * (U[4] + y * U[5])))));
            const double p2 = 1 + y * (V[1] + y * (V[2] + y * (V[3] + y * (V[4] + y * V[5]))));
            lg += (-0.5 * y + p1 / p2);
        }
        return lg;
    }
    if (x < 8) {
        const int i = (int)x; const double y = x - (double)i;
        const double p = y * (S[0] + y * (S[1] + y * (S[2] + y * (S[3] + y * (S[4] + y * (S[5] + y * S[6]))))));
        const double q = 1 + y * (Rr[1] + y * (Rr[2] + y * (Rr[3] + y * (Rr[4] + y * (Rr[5] + y * Rr[6])))));
        lg = 0.5 * y + p / q;
        double z = 1.0;
        switch (i) {
        case 7: z *= (y + 6); [[fallthrough]];
        case 6: z *= (y + 5); [[fallthrough]];
        case 5: z *= (y + 4); [[fallthrough]];
        case 4: z *= (y + 3); [[fallthrough]];
        case 3: z *= (y + 2); lg += Log(z);
        }
        return lg;
    }
    if (x < 288230376151711744.0) {
        const double t = Log(x), z = 1 / x, y = z * z;
        const double w = W[0] + z * (W[1] + y * (W[2] + y * (W[3] + y * (W[4] + y * (W[5] + y * W[6])))));
        return (x - 0.5) * (t - 1) + w;
    }
    return x * (Log(x) - 1);
}
GM_HD inline double Round(double x) { return ::round(x); }   // half away from zero

}  // namespace gomath
