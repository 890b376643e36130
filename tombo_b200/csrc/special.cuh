// special.cuh -- fp64 special functions of the level tests (group_stats.cu) and of the Fisher
// windows (fisher.cuh), host and device.
//
//   tb2_kolmogorov_sf(y)      scipy.special.kolmogorov == stats.kstwobign.sf
//   tb2_t_two_sided_p(df, t)  2 * scipy.special.stdtr(df, t) for t <= 0
//   tb2_chi2_sf_even(y, k)    scipy.stats.chi2.sf(2 y, 2 k)
//   tb2_div12(P)              Python's int / 12 (correctly rounded) for a 128-bit P
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define TB2_HD __host__ __device__ __forceinline__
#else
#define TB2_HD inline
#endif

// Kolmogorov's limiting distribution, survival function.  Same two regimes as scipy
// (cutover 0.82): for small y the Jacobi-theta form of the CDF,
//   cdf = sqrt(2 pi) / y * sum_{k>=1} exp(-(2k-1)^2 pi^2 / (8 y^2)),   sf = 1 - cdf
// (sf >= 0.5 there, so the subtraction loses nothing); for large y the alternating series
//   sf = 2 * sum_{k>=1} (-1)^(k-1) exp(-2 k^2 y^2),
// whose terms fall so fast that the sum has full relative precision down to underflow.
TB2_HD double tb2_kolmogorov_sf(double y)
{
    if (y != y) return y;
    if (y <= 0.0) return 1.0;
    if (y <= 0.82) {
        const double f = -(M_PI * M_PI) / (8.0 * y * y);
        double s = 0.0;
        for (int k = 1; k < 32; ++k) {
            const double m = (double)(2 * k - 1);
            const double t = exp(m * m * f);
            s += t;
            if (t <= 1e-18 * s) break;
        }
        return 1.0 - 2.5066282746310002 / y * s;      // sqrt(2 pi)
    }
    const double f = -2.0 * y * y;
    double s = 0.0, sign = 1.0;
    for (int k = 1; k < 64; ++k) {
        const double t = exp((double)k * (double)k * f);
        s += sign * t;
        if (t <= 1e-18 * s) break;
        sign = -sign;
    }
    return 2.0 * s;
}

// continued fraction of the regularised incomplete beta (modified Lentz)
TB2_HD double tb2_betacf(double a, double b, double x)
{
    const double tiny = 1e-300, eps = 1e-16;
    const double qab = a + b, qap = a + 1.0, qam = a - 1.0;
    double c = 1.0, d = 1.0 - qab * x / qap;
    if (fabs(d) < tiny) d = tiny;
    d = 1.0 / d;
    double h = d;
    for (int m = 1; m <= 5000; ++m) {
        const double m2 = 2.0 * m;
        double aa = m * (b - m) * x / ((qam + m2) * (a + m2));
        d = 1.0 + aa * d; if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c; if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        h *= d * c;
        aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2));
        d = 1.0 + aa * d; if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c; if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (fabs(del - 1.0) < eps) break;
    }
    return h;
}

// lgamma(a + 0.5) - lgamma(a).  For large a the two lgamma values cancel (at a = 1e4 they are
// ~8e4, so their rounding alone costs ~1e-11 relative in the p-value); there the difference
// comes from Stirling's series directly:
//   (a - 1/2) log1p(b/a) + b log(a + b) - b + S(a + b) - S(a),
//   S(x) = 1/(12x) - 1/(360x^3) + 1/(1260x^5) - 1/(1680x^7)
// (the next term is below 1e-16 for a >= 20).
TB2_HD double tb2_stirling_tail(double x)
{
    const double r = 1.0 / x, r2 = r * r;
    return r * (1.0 / 12.0 - r2 * (1.0 / 360.0 - r2 * (1.0 / 1260.0 - r2 * (1.0 / 1680.0))));
}

TB2_HD double tb2_lgamma_half_ratio(double a)
{
    const double b = 0.5;
    if (a < 20.0) return lgamma(a + b) - lgamma(a);
    return (a - 0.5) * log1p(b / a) + b * log(a + b) - b +
           (tb2_stirling_tail(a + b) - tb2_stirling_tail(a));
}

// 2 * stdtr(df, t) for t <= 0, i.e. I_x(df/2, 1/2) with x = df / (df + t^2).  x and 1 - x
// are formed separately (log x = -log1p(t^2/df)) so neither loses digits to cancellation.
TB2_HD double tb2_t_two_sided_p(double df, double t)
{
    if (t != t || !(df > 0.0)) return NAN;
    const double t2 = t * t;
    if (t2 == 0.0) return 1.0;
    if (isinf(t2)) return 0.0;
    const double a = 0.5 * df, b = 0.5;
    const double x = df / (df + t2), y = t2 / (df + t2);
    const double lx = -log1p(t2 / df), ly = log(y);
    // log B(a, 1/2) = lgamma(a) + lgamma(1/2) - lgamma(a + 1/2); lgamma(1/2) = log(sqrt(pi))
    const double front = exp(tb2_lgamma_half_ratio(a) - 0.57236494292470008707 + a * lx + b * ly);
    if (x < (a + 1.0) / (a + b + 2.0)) return front * tb2_betacf(a, b, x) / a;
    return 1.0 - front * tb2_betacf(b, a, y) / b;
}

// ---------------------------------------------------------------------------
// scipy.stats.chi2.sf(2 y, 2 k) = Q(k, y) = exp(-y) * sum_{i<k} y^i / i!, the Poisson
// probability P(N <= k - 1), N ~ Poisson(y).  Fisher's method over a window of k p-values
// asks for it with y = -sum log p.
//
// y < 700: the closed form, operation for operation.  exp(-y) is a normal double and the sum
// stays below e^700, so nothing under- or overflows; every term is a product of at most
// 2 i roundings, so the relative error stays within about 2 (y + 10 sqrt(y)) u.  The loop
// stops once the terms decrease (i > y) and adding one no longer changes the sum: every
// later term is smaller still, so the result is the same as summing all k terms.
//
// y >= 700: exp(-y) would underflow before the sum makes up for it (and for y beyond ~12 000
// the sum overflows, 0 * inf = NaN).  Instead the largest term of the sum, j = min(k - 1,
// floor(y)), is evaluated in logarithms with Loader's saddle-point form
//   log p(j; y) = -stirlerr(j) - bd0(j, y) - log(2 pi j) / 2,
// which has no lgamma cancellation at large j, and the other terms are summed outward from it
// as ratios p(j-1)/p(j) = j / y and p(j+1)/p(j) = y / (j+1) until they are negligible:
// the terms fall off like a Gaussian of width sqrt(y) around the mode (or geometrically below
// it), so at most min(k, ~40 sqrt(y)) ratios are taken.  Rounding log p(j; y), whose size is
// up to ~y, costs ~y u relative after exp; the ratio sum adds a few u per term.
// ---------------------------------------------------------------------------

// stirlerr(n) = log(n!) - log(sqrt(2 pi n) (n/e)^n) for an integer n >= 1
TB2_HD double tb2_stirlerr(double n)
{
    if (n <= 15.0)
        return lgamma(n + 1.0) - (n + 0.5) * log(n) + n - 0.91893853320467274178;  // log sqrt(2 pi)
    const double r = 1.0 / n, r2 = r * r;
    return r * (1.0 / 12.0 - r2 * (1.0 / 360.0 - r2 * (1.0 / 1260.0 - r2 * (1.0 / 1680.0 -
                r2 * (1.0 / 1188.0)))));
}

// bd0(x, m) = x log(x / m) + m - x >= 0, with the series in v = (x - m) / (x + m) where the
// direct form cancels
TB2_HD double tb2_bd0(double x, double m)
{
    if (fabs(x - m) < 0.1 * (x + m)) {
        double v = (x - m) / (x + m);
        double s = (x - m) * v, ej = 2.0 * x * v;
        v = v * v;
        for (int j = 1; j < 1000; ++j) {
            ej *= v;
            const double s1 = s + ej / (double)(2 * j + 1);
            if (s1 == s) break;
            s = s1;
        }
        return s;
    }
    return x * log(x / m) + m - x;
}

TB2_HD double tb2_chi2_sf_even(double y, int k)
{
    if (y != y) return y;
    if (y < 700.0) {
        double term = 1.0, sum = 1.0;
        for (int i = 1; i < k; ++i) {
            term *= y / (double)i;
            const double prev = sum;
            sum += term;
            if (sum == prev && (double)i > y) break;
        }
        return exp(-y) * sum;
    }
    if (isinf(y)) return 0.0;
    const double jt = fmin((double)(k - 1), floor(y));       // the largest term
    const double lp = jt == 0.0 ? -y
                                : -tb2_stirlerr(jt) - tb2_bd0(jt, y) - 0.5 * log(6.283185307179586477 * jt);
    if (lp < -760.0) return 0.0;                              // Q < e^-740
    const double eps = 1e-17;
    double s = 1.0, t = 1.0;
    for (double j = jt; j >= 1.0; j -= 1.0) {                // p(j - 1) / p(j) = j / y
        t *= j / y;
        s += t;
        if (t < eps * s) break;
    }
    t = 1.0;
    for (double j = jt + 1.0; j <= (double)(k - 1); j += 1.0) {   // p(j) / p(j - 1) = y / j
        t *= y / j;
        s += t;
        if (t < eps * s) break;
    }
    return exp(lp) * s;
}

// p / 12 correctly rounded to double, as Python's int / int evaluates tot * (tot + 1) / 12
// for the U test's rhou.  Requires p < 2^124 (tot < 2^62).
TB2_HD double tb2_div12(unsigned __int128 p)
{
    const unsigned __int128 two53 = (unsigned __int128)1 << 53;
    if (p < two53) return (double)(unsigned long long)p / 12.0;    // one IEEE division of exact operands
    // scale by 2^k so that the quotient has at least 53 integer bits, round the quotient to
    // 53 significant bits (nearest, ties to even) from its integer remainder, scale back
    int k = 0;
    while ((p << k) / 12 < two53) ++k;                              // k <= 4
    const unsigned __int128 pk = p << k, q = pk / 12;
    const unsigned r = (unsigned)(pk % 12);
    int sh = 0;
    while ((q >> sh) >= two53) ++sh;
    unsigned long long m = (unsigned long long)(q >> sh);
    // fraction below the kept bits, times 12: rem * 12 + r against half = 6 * 2^sh
    const unsigned __int128 rem = q & ((((unsigned __int128)1) << sh) - 1);
    const unsigned __int128 f12 = rem * 12 + r, half12 = (unsigned __int128)6 << sh;
    if (f12 > half12 || (f12 == half12 && (m & 1))) ++m;
    return ldexp((double)m, sh - k);
}
