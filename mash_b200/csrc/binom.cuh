// binom.cuh -- P[Binomial(n, r) >= x] in double precision on the device.
//
// This is the quantity the reference obtains from gsl_cdf_binomial_Q(x-1, r, n) / Boost.Math
// (reference CommandDistance.cpp:444-446, CommandScreen.cpp:611-613).  Direct summation of the pmf from x
// towards the tail with geometrically decreasing terms; below the mean the complementary lower tail is summed instead.
// The first term C(n,x) r^x (1-r)^(n-x) is built from exact factors in double-double arithmetic (no lgamma, no log/exp):
// r^x and (1-r)^(n-x) by binary exponentiation and C(n,x) as a running product of integers, each carried as hi + lo with
// a power-of-two exponent aside.  A plain double exponent (n-x) log2(1-r) has an absolute error of |y| 2^-53, which is the
// relative error of the result: 5e-12 at n = 1e5, r = 0.5.  With the products in double-double the error is that of the
// tail sum, which grows with its length, not with n: within 1e-12 of 60-digit truth (worst 1.3e-14 on an H100) for n
// up to 1e5 and r from 1e-9 to 0.999 (tests/test_gpu_pvalue_precision.py; SURVEY.md appendix C).
#pragma once
#include <cstdint>

namespace mashgpu {

// Double-double products on frexp-normalised operands: hi in [0.5, 1), |lo| <= ulp(hi) / 2, the value (hi + lo) * 2^e.
// The _rn intrinsics keep the error-free transformations intact: nvcc must not contract p + e into an FMA.
struct DDScaled { double hi, lo; long long e; };

__device__ __forceinline__ DDScaled dd_renorm(double p, double err, long long e)
{
    const double s = __dadd_rn(p, err);
    double lo = __dsub_rn(err, __dsub_rn(s, p));
    double hi = s;
    if (hi < 0.5) { hi *= 2.0; lo *= 2.0; e -= 1; }       // the product of two values in [0.5, 1) lies in [0.25, 1)
    return DDScaled{hi, lo, e};
}

__device__ __forceinline__ DDScaled dd_mul(const DDScaled &a, const DDScaled &b)
{
    const double p = __dmul_rn(a.hi, b.hi);
    double err = __fma_rn(a.hi, b.hi, -p);
    err = __fma_rn(a.hi, b.lo, __fma_rn(a.lo, b.hi, err));
    return dd_renorm(p, err, a.e + b.e);
}

// v as DDScaled for a double v > 0
__device__ __forceinline__ DDScaled dd_from(double v)
{
    int k;
    const double m = frexp(v, &k);
    return DDScaled{m, 0.0, k};
}

constexpr DDScaled DD_ONE{0.5, 0.0, 1};

// v^m by binary exponentiation: relative error ~ 2 log2(m) 2^-104
__device__ __forceinline__ DDScaled dd_pow(DDScaled v, uint64_t m)
{
    DDScaled acc = DD_ONE;
    while (m) {
        if (m & 1) acc = dd_mul(acc, v);
        m >>= 1;
        if (m) v = dd_mul(v, v);
    }
    return acc;
}

// 1 - r as DDScaled, exactly (Fast2Sum: 1 >= r)
__device__ __forceinline__ DDScaled dd_one_minus(double r)
{
    const double q = __dsub_rn(1.0, r);
    const double ql = __dsub_rn(__dsub_rn(1.0, q), r);
    int k;
    const double m = frexp(q, &k);
    return DDScaled{m, ldexp(ql, -k), k};
}

// Table of C(n0, x), x = 0..n0, as mant * 2^expo, built on the host in long double (dist.cu: n0 = the job's sketch size,
// which is the denominator of almost every pair).  With it the first term costs 2 log2(n)-step powers instead of
// min(x, n-x) multiply steps -- the p-value of a pair with many shared hashes used to cost more than its merge.
struct BinomTable { const double *mant; const int *expo; uint64_t n0; };

// C(n, x) r^x (1-r)^(n-x) as mant * 2^expo (mant may be far from 1; only the product is meaningful).  C(n, x) comes from the
// table when n == tab.n0, else as the exact products (n-c+1)..n over 1..c in double-double, c = min(x, n-x).
__device__ __forceinline__ void binom_pmf_scaled(uint64_t x, double r, uint64_t n, const BinomTable *tab, double &mant, int &expo)
{
    DDScaled t = dd_mul(dd_pow(dd_from(r), x), dd_pow(dd_one_minus(r), n - x));
    double m;
    long long e = t.e;
    if (tab && tab->mant && n == tab->n0) {
        m = tab->mant[x] * (t.hi + t.lo);
        e += tab->expo[x];
    } else {
        const uint64_t c = x < n - x ? x : n - x;
        DDScaled num = DD_ONE, den = DD_ONE;
        for (uint64_t i = 1; i <= c; i++) {
            num = dd_mul(num, dd_from((double)(n - c + i)));
            den = dd_mul(den, dd_from((double)i));
        }
        num = dd_mul(num, t);
        m = (num.hi + num.lo) / (den.hi + den.lo);
        e = num.e - den.e;
    }
    // the result can be far below the double range (it underflows to 0): clamp so the int conversion is safe
    mant = m;
    expo = (int)(e < -1000000 ? -1000000 : (e > 1000000 ? 1000000 : e));
}

__device__ __forceinline__ double binomial_upper_tail(uint64_t x, double r, uint64_t n, const BinomTable *tab = nullptr)
{
    if (x == 0) return 1.0;
    if (x > n) return 0.0;
    if (!(r > 0.0)) return 0.0;
    if (r >= 1.0) return 1.0;
    const double odds = r / (1.0 - r);
    if ((double)x >= ((double)n + 1.0) * r) {
        double m; int e;
        binom_pmf_scaled(x, r, n, tab, m, e);
        double sum = 1.0, t = 1.0;
        for (uint64_t i = x; i < n; i++) {
            t *= ((double)(n - i) / (double)(i + 1)) * odds;
            sum += t;
            if (t < sum * 1e-18) break;
        }
        return ldexp(m * sum, e < -100000 ? -100000 : e);
    } else {
        const uint64_t xm = x - 1;
        double m; int e;
        binom_pmf_scaled(xm, r, n, tab, m, e);
        double sum = 1.0, t = 1.0;
        for (uint64_t i = xm; i > 0; i--) {
            t *= ((double)i / (double)(n - i + 1)) / odds;
            sum += t;
            if (t < sum * 1e-18) break;
        }
        return 1.0 - ldexp(m * sum, e < -100000 ? -100000 : e);
    }
}

// pValue, reference CommandDistance.cpp:427-448
__device__ __forceinline__ double mash_pvalue(uint64_t x, uint64_t len_ref, uint64_t len_qry, double kmer_space, uint64_t sketch_size,
                                              const BinomTable *tab = nullptr)
{
    if (x == 0) return 1.0;
    const double pX = 1. / (1. + kmer_space / (double)len_ref);
    const double pY = 1. / (1. + kmer_space / (double)len_qry);
    const double r = pX * pY / (pX + pY - pX * pY);
    return binomial_upper_tail(x, r, sketch_size, tab);
}

}  // namespace mashgpu
