// k2c_core.cuh -- the body of K2c site_continuous (include/strelka_b200.h, "K2c site_continuous"): the germline caller's
// continuous-frequency site model.  Everything that decides a byte of the output is here, compiled __device__ by nvcc and as plain C++ by
// g++ (tests/cpp/k2c_core_host.cpp and oracle/continuous_oracle.cpp), with the mirrored libm of sx_libm_mirror_d.h and unfused arithmetic
// (-fmad=false / -ffp-contract=off): the host and the device give the same bits.  k2c_continuous.cu adds only the kernels' index arithmetic.
//
// The two functions the reference takes from Boost.Math (applications/starling/starling_continuous_variant_caller.cpp):
//
//   getAlleleSequencingErrorQscore(a, n, q, maxq) = a == 0 ? 0 : min(maxq, floor(-10 log10(gamma_p(a, n * 10^(-q/10))) + 0.5)),
//       maxq where gamma_p is 0.  For integer a, gamma_p(a, L) = P(Poisson(L) >= a) = e^-L sum_{k >= a} L^k / k!.  Below, a > L sums that
//       tail from its first term up; a <= L takes 1 - e^-L sum_{k < a} L^k / k!, summed from its last term down (P >= about 0.4 there, so
//       the subtraction loses nothing that matters).  Each first term is exp(-L + k ln L - ln k!), ln k! exact through 18! and Stirling's
//       series with four correction terms above (truncation below 1e-15).
//       Error bound of x = -10 log10(P): the first term's exponent is a sum of magnitude M = L + k |ln L| + ln k!, each operation within
//       half an ulp and log / exp within one, so its absolute error is below 8 eps M; the series adds below (terms + 2) eps relative.  In
//       phred units (10 / ln 10 = 4.343) that is below 4.343 * (8 M + terms + 2) * 1.2e-16.  The bound used, K2C_QBOUND_ABS +
//       K2C_QBOUND_REL * (M + terms), is more than 25 times that.  A value of x + 0.5 within it of an integer in 1..maxq sets
//       SX_CONT_ST_QSCORE_TIE; none occurs for n <= 16384 (tests/golden/continuous_ref.npz holds the reference's qscores over that grid).
//
//   strandBias(fa, ra, fo, ro) = max(fwdLnp, revLnp) - lnp over log(pdf(binomial(trials, p), k)) terms.  pdf is evaluated as
//       C(n, k) p^k (1-p)^(n-k) in the log domain, with Boost's cases p == 0, p == 1 and k == n, and rounded through exp to a double before its
//       log, as the reference narrows Boost's long double pdf to double: a pdf below the least subnormal is 0 and its log -inf.
#pragma once

#include <math.h>
#include <stdint.h>

#include "strelka_b200.h"
#include "sx_libm_mirror_d.h"

#if defined(__CUDACC__)
#define K2C_HD __device__ __forceinline__
#else
#include <cstring>
#define K2C_HD static inline
#endif

constexpr double K2C_QBOUND_ABS = 1e-9;
constexpr double K2C_QBOUND_REL = 1e-13;
constexpr double K2C_PHRED_PER_LN = 4.3429448190325182765; // 10 / ln 10

// one sample's tier1 column: cleaned calls by strand (0 reverse, 1 forward) and base (4: ANY), and the raw call count
struct k2c_counts
{
    uint32_t n[2][5];
    uint32_t raw;
};

K2C_HD uint32_t k2c_base_of(const uint32_t call) { return ((call >> 6) & 15u) < 4u ? ((call >> 6) & 15u) : 4u; }
K2C_HD bool k2c_is_filtered(const uint32_t call) { return ((call >> 12) & 1u) != 0; }
K2C_HD uint32_t k2c_is_fwd(const uint32_t call) { return (call >> 10) & 1u; }

// base_to_id of the reference base: A C G T -> 0..3, anything else ('N') -> 4 (ANY)
K2C_HD uint32_t k2c_ref_id(const char c)
{
    return c == 'A' ? 0u : c == 'C' ? 1u : c == 'G' ? 2u : c == 'T' ? 3u : 4u;
}

K2C_HD double k2c_from_bits(const uint64_t bits)
{
#if defined(__CUDACC__)
    return __longlong_as_double(static_cast<long long>(bits));
#else
    double d;
    std::memcpy(&d, &bits, sizeof d);
    return d;
#endif
}
K2C_HD double k2c_nan() { return k2c_from_bits(0xfff8000000000000ull); } // the x86-64 default NaN the reference's arithmetic produces
K2C_HD double k2c_neg_inf() { return k2c_from_bits(0xfff0000000000000ull); }

// ln k!
K2C_HD double k2c_ln_fact(const uint32_t k)
{
    if (k <= 18)
    {
        double f = 1.0;
        for (uint32_t i = 2; i <= k; ++i) f = f * static_cast<double>(i); // exact through 18!
        return sx_log(f);
    }
    const double x = static_cast<double>(k), r = 1.0 / x, r2 = r * r;
    const double series = r * (1.0 / 12.0 - r2 * (1.0 / 360.0 - r2 * (1.0 / 1260.0 - r2 * (1.0 / 1680.0))));
    return x * sx_log(x) - x + 0.5 * sx_log(6.283185307179586477 * x) + series;
}

struct k2c_q
{
    int32_t gq;
    uint32_t status;
};

// getAlleleSequencingErrorQscore; err_rate = qphred_to_error_prob(expected_qscore) (the host's std::pow(10., -q / 10.))
K2C_HD k2c_q k2c_qscore(const uint32_t a, const uint32_t n, const double err_rate, const int32_t max_q)
{
    k2c_q r{0, 0};
    if (a == 0)
    {
        r.gq = 0; // gamma_p = 1 -> qphred 0 (max_q >= 0)
        return r;
    }
    const double L = static_cast<double>(n) * err_rate;
    if (!(L > 0.0))
    {
        r.gq = max_q; // gamma_p(a, 0) = 0
        return r;
    }
    const double lnL = sx_log(L);
    double x, mag;
    uint32_t terms = 0;
    if (static_cast<double>(a) > L)
    {
        const double lf = k2c_ln_fact(a);
        const double e = static_cast<double>(a) * lnL - L - lf;
        mag = L + static_cast<double>(a) * (lnL < 0 ? -lnL : lnL) + lf;
        // the tail's sum relative to its first term: 1 + L/(a+1) + L^2/((a+1)(a+2)) + ...
        double s = 1.0, t = 1.0;
        for (uint32_t k = a + 1;; ++k)
        {
            t = t * (L / static_cast<double>(k));
            s = s + t;
            ++terms;
            if (t < s * 1e-17) break;
        }
        x = -(e + sx_log(s)) * K2C_PHRED_PER_LN;
    }
    else
    {
        // 1 - e^-L sum_{k < a} L^k / k!, from k = a - 1 down (the terms shrink going down because k <= L)
        const uint32_t k0 = a - 1;
        const double lf = k2c_ln_fact(k0);
        const double e = static_cast<double>(k0) * lnL - L - lf;
        mag = L + static_cast<double>(k0) * (lnL < 0 ? -lnL : lnL) + lf;
        double t = sx_exp(e), q = t;
        for (uint32_t k = k0; k > 0; --k)
        {
            t = t * (static_cast<double>(k) / L);
            q = q + t;
            ++terms;
            if (t < q * 1e-17) break;
        }
        const double p = 1.0 - q;
        if (!(p > 0.0))
        {
            r.gq = max_q;
            return r;
        }
        x = -10.0 * sx_log10(p);
    }
    const double bound = K2C_QBOUND_ABS + K2C_QBOUND_REL * (mag + static_cast<double>(terms));
    const double y = x + 0.5;
    if (!(y < static_cast<double>(max_q) + 1.0)) // max_q on both sides of max_q + 1; also x >= 3070 (the reference's log10 floor) and x = +inf
    {
        r.gq = max_q;
        return r;
    }
    const double fl = floor(y);
    r.gq = static_cast<int32_t>(fl);
    if (r.gq > max_q) r.gq = max_q;
    // the boundaries 1..max_q nearest y
    const double up = fl + 1.0;
    if ((y - fl < bound && fl >= 1.0) || (up - y < bound && up >= 1.0 && up <= static_cast<double>(max_q))) r.status = SX_CONT_ST_QSCORE_TIE;
    return r;
}

// binomialLogDensity(trials, successes, p) of the reference, narrowed as there
K2C_HD double k2c_binom_ln(const uint32_t n, const uint32_t k, const double p)
{
    if (n == 0) return 0.0;
    const double NEG_INF = k2c_neg_inf();
    if (p == 0.0) return k == 0 ? 0.0 : NEG_INF;
    if (p == 1.0) return k == n ? 0.0 : NEG_INF;
    double lp;
    if (k == n)
        lp = static_cast<double>(n) * sx_log(p);
    else
    {
        const double lc = k2c_ln_fact(n) - k2c_ln_fact(k) - k2c_ln_fact(n - k);
        lp = lc + static_cast<double>(k) * sx_log(p) + static_cast<double>(n - k) * sx_log1p(-p);
    }
    if (lp > 0.0) lp = 0.0; // a pdf is at most 1
    return sx_log(sx_exp(lp));
}

K2C_HD double k2c_safe_frac(const uint32_t a, const uint32_t b) { return b == 0 ? 0.0 : static_cast<double>(a) / static_cast<double>(b); }

// starling_continuous_variant_caller::strandBias
K2C_HD double k2c_strand_bias(const uint32_t fa, const uint32_t ra, const uint32_t fo, const uint32_t ro)
{
    const uint32_t ft = fa + fo, rt = ra + ro, tot = ft + rt;
    if (tot == 0) return 0.0;
    const double ff = k2c_safe_frac(fa, ft), rf = k2c_safe_frac(ra, rt), af = k2c_safe_frac(fa + ra, tot);
    const double err = 0.005;
    const double fwd = k2c_binom_ln(ft, fa, ff) + k2c_binom_ln(rt, ra, err);
    const double rev = k2c_binom_ln(ft, fa, err) + k2c_binom_ln(rt, ra, rf);
    const double lnp = k2c_binom_ln(ft, fa, af) + k2c_binom_ln(rt, ra, af);
    const double mx = (fwd < rev) ? rev : fwd; // std::max
    const double sb = mx - lnp;
    return sb != sb ? k2c_nan() : sb;
}

// updateSiteSampleInfo's clamp: std::min(M, std::max(-M, sb))
K2C_HD double k2c_clamp_sb(const double sb, const double M)
{
    const double lo = (-M < sb) ? sb : -M;
    return (lo < M) ? lo : M;
}

// the alt locus `alt` of a site whose samples have counts c[0..S): does some sample's AF exceed min_het_vf?
K2C_HD bool k2c_alt_reportable(const k2c_counts* c, const uint32_t S, const uint32_t alt, const double min_het_vf)
{
    for (uint32_t s = 0; s < S; ++s)
    {
        const uint32_t tot = c[s].n[0][0] + c[s].n[0][1] + c[s].n[0][2] + c[s].n[0][3] + c[s].n[1][0] + c[s].n[1][1] + c[s].n[1][2] + c[s].n[1][3];
        if (k2c_safe_frac(c[s].n[0][alt] + c[s].n[1][alt], tot) > min_het_vf) return true;
    }
    return false;
}

// the loci a site reports, in record order, into loci[]; returns how many (0 for a skipped site)
K2C_HD uint32_t k2c_site_loci(const k2c_counts* c, const uint32_t S, const uint32_t ref, const bool forced, const double min_het_vf, uint8_t* loci)
{
    if (!forced)
    {
        bool empty = true;
        for (uint32_t s = 0; s < S; ++s) empty = empty && c[s].raw == 0;
        if (empty) return 0;
    }
    uint32_t m = 0;
    for (uint32_t b = 0; b < 4; ++b)
        if (b != ref && (forced || k2c_alt_reportable(c, S, b, min_het_vf))) loci[m++] = static_cast<uint8_t>(b);
    if (m == 0) loci[m++] = SX_CONT_REF_LOCUS;
    return m;
}

// the (locus, sample) entry; `alt` is the locus's alt base or SX_CONT_REF_LOCUS
K2C_HD sx_cont_sample k2c_entry(const k2c_counts& c, const uint32_t ref, const uint32_t alt, const sx_cont_opts& o, const double err_rate)
{
    sx_cont_sample e;
    const bool is_ref = alt == SX_CONT_REF_LOCUS;
    e.ref_fwd = ref < 4 ? c.n[1][ref] : 0u;
    e.ref_rev = ref < 4 ? c.n[0][ref] : 0u;
    e.alt_fwd = is_ref ? 0u : c.n[1][alt];
    e.alt_rev = is_ref ? 0u : c.n[0][alt];
    const uint32_t fwd = c.n[1][0] + c.n[1][1] + c.n[1][2] + c.n[1][3], rev = c.n[0][0] + c.n[0][1] + c.n[0][2] + c.n[0][3];
    e.non_confident_fwd = fwd - e.ref_fwd - e.alt_fwd;
    e.non_confident_rev = rev - e.ref_rev - e.alt_rev;
    e.total_depth = fwd + rev;
    e.allele_depth = is_ref ? e.ref_fwd + e.ref_rev : e.alt_fwd + e.alt_rev;
    e.used = fwd + rev + c.n[0][4] + c.n[1][4];
    e.unused = c.raw - e.used;
    e.af = k2c_safe_frac(e.allele_depth, e.total_depth);
    e.gt = is_ref ? SX_CONT_GT_HOMREF : (e.af >= 1.0 - o.min_het_vf) ? SX_CONT_GT_HOM : (e.af < o.min_het_vf) ? SX_CONT_GT_HOMREF : SX_CONT_GT_HET;
    const k2c_q q = k2c_qscore(e.allele_depth, e.total_depth, err_rate, o.max_qscore);
    e.gq = q.gq;
    e.status = q.status;
    if (is_ref)
        e.strand_bias = 0.0;
    else
    {
        const uint32_t all_fwd = fwd + c.n[1][4], all_rev = rev + c.n[0][4];
        e.strand_bias = k2c_clamp_sb(k2c_strand_bias(e.alt_fwd, e.alt_rev, all_fwd - e.alt_fwd, all_rev - e.alt_rev), o.max_abs_sample_strand_bias);
    }
    for (int i = 0; i < 7; ++i) e.pad[i] = 0;
    return e;
}

// the locus record; qual = the largest gq of the locus's sample entries
K2C_HD sx_cont_locus k2c_locus(const k2c_counts* c, const uint32_t S, const int32_t pos, const uint32_t ref, const uint32_t alt, const bool forced,
                               const int32_t qual)
{
    sx_cont_locus l;
    l.pos = pos;
    l.alt = static_cast<uint8_t>(alt);
    l.ref = static_cast<uint8_t>(ref);
    l.forced = forced ? 1 : 0;
    for (int i = 0; i < 5; ++i) l.pad[i] = 0;
    l.sb_fwd_alt = l.sb_rev_alt = l.sb_fwd_other = l.sb_rev_other = 0;
    l.qual = 0;
    l.strand_bias = 0.0;
    if (alt == SX_CONT_REF_LOCUS) return l;
    for (uint32_t s = 0; s < S; ++s)
    {
        const uint32_t fwd = c[s].n[1][0] + c[s].n[1][1] + c[s].n[1][2] + c[s].n[1][3] + c[s].n[1][4];
        const uint32_t rev = c[s].n[0][0] + c[s].n[0][1] + c[s].n[0][2] + c[s].n[0][3] + c[s].n[0][4];
        l.sb_fwd_alt += c[s].n[1][alt];
        l.sb_rev_alt += c[s].n[0][alt];
        l.sb_fwd_other += fwd - c[s].n[1][alt];
        l.sb_rev_other += rev - c[s].n[0][alt];
    }
    l.qual = qual > 0 ? qual : 0;
    l.strand_bias = k2c_strand_bias(l.sb_fwd_alt, l.sb_rev_alt, l.sb_fwd_other, l.sb_rev_other);
    return l;
}
