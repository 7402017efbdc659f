/* b200_crf_math.h -- the numerics contract of the CRF decoder.
 *
 * The reference decoder (dorado/basecall/decode/beam_search.cpp:42-45, :94-98, :503 and
 * CPUDecoder.cpp:29-34, :130) evaluates exp/log/log1p/pow/log10 through libm and libtorch, whose
 * last-bit behaviour is platform specific and cannot be reproduced on a GPU.  Because the beam
 * search is full of hard thresholds, "bit-identical" output needs bit-identical transcendentals, so
 * this header pins them: every function below is built only from IEEE-754 binary32 add / mul / fma /
 * div (all correctly rounded on x86-64 and on sm_90a) in a fixed order.  The CUDA kernels
 * (dorado_b200/csrc/decode.cu) and the CPU oracle (oracle/crf_oracle.c) both include this file, so
 * the two produce the same bits by construction.  Accuracy versus libm: <= 2 ulp over the ranges
 * the decoder uses (tests/test_host_cpu.py::test_numerics_contract_accuracy).
 *
 * Compile rules: C side with -ffp-contract=off (oracle/Makefile); CUDA side uses the explicit
 * __f*_rn intrinsics, which nvcc never contracts.
 */
#ifndef B200_CRF_MATH_H
#define B200_CRF_MATH_H

#include <stdint.h>

#if defined(__CUDA_ARCH__)
#define B200_MATH_FN static __device__ __forceinline__
#define B200_FMA(a, b, c) __fmaf_rn((a), (b), (c))
#define B200_MUL(a, b) __fmul_rn((a), (b))
#define B200_ADD(a, b) __fadd_rn((a), (b))
#define B200_SUB(a, b) __fsub_rn((a), (b))
#define B200_DIV(a, b) __fdiv_rn((a), (b))
#define B200_F2U(x) __float_as_uint(x)
#define B200_U2F(x) __uint_as_float(x)
#else
#include <math.h>
#include <string.h>
#define B200_MATH_FN static inline
#define B200_FMA(a, b, c) fmaf((a), (b), (c))
#define B200_MUL(a, b) ((a) * (b))
#define B200_ADD(a, b) ((a) + (b))
#define B200_SUB(a, b) ((a) - (b))
#define B200_DIV(a, b) ((a) / (b))
static inline uint32_t b200_f2u_(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    return u;
}
static inline float b200_u2f_(uint32_t u) {
    float x;
    memcpy(&x, &u, 4);
    return x;
}
#define B200_F2U(x) b200_f2u_(x)
#define B200_U2F(x) b200_u2f_(x)
#endif

#define B200_FLT_LOWEST (-3.402823466e+38f)

B200_MATH_FN float b200_fmaxf(float a, float b) { return a > b ? a : b; }

/* exp(x) for any finite x <= ~88; returns 0 below -86 (results there would be subnormal).
 * Written without control flow (clamp, evaluate, select): the scans evaluate five of these per state and block, and with an
 * early return the GPU compiler kept five branch regions that ran one after the other instead of interleaving. */
B200_MATH_FN float b200_expf(float x) {
    const float xc = x < -86.0f ? -86.0f : (x > 88.0f ? 88.0f : x);
    /* n = round-to-nearest-even(x / ln2) via the 1.5*2^23 trick: the integer sits in the low mantissa bits of t + big */
    const float t = B200_MUL(xc, 1.44269504088896341f);
    const float big = 12582912.0f;
    const float tb = B200_ADD(t, big);
    const float n = B200_SUB(tb, big);
    float r = B200_FMA(n, -0.693359375f, xc);
    r = B200_FMA(n, 2.12194440e-4f, r);
    float p = 1.9875691500e-4f;
    p = B200_FMA(p, r, 1.3981999507e-3f);
    p = B200_FMA(p, r, 8.3334519073e-3f);
    p = B200_FMA(p, r, 4.1665795894e-2f);
    p = B200_FMA(p, r, 1.6666665459e-1f);
    p = B200_FMA(p, r, 5.0000001201e-1f);
    const float r2 = B200_MUL(r, r);
    p = B200_FMA(p, r2, r);
    p = B200_ADD(p, 1.0f);
    /* 2^n: bits(t + big) = 0x4B400000 + n for |n| < 2^22, and 0x4B400000 << 23 == 0 (mod 2^32), so the exponent field is
     * (bits << 23) + bias -- one integer instruction, no float -> int conversion */
    const float scale = B200_U2F((B200_F2U(tb) << 23) + 0x3f800000u);
    const float y = B200_MUL(p, scale);
    return x < -86.0f ? 0.0f : y;
}

/* exp(x) for x <= 0 (the arguments of a max-shifted sum): b200_expf without the upper clamp, bit-identical there. */
B200_MATH_FN float b200_expf_nonpos(float x) {
    const float xc = x < -86.0f ? -86.0f : x;
    const float t = B200_MUL(xc, 1.44269504088896341f);
    const float big = 12582912.0f;
    const float tb = B200_ADD(t, big);
    const float n = B200_SUB(tb, big);
    float r = B200_FMA(n, -0.693359375f, xc);
    r = B200_FMA(n, 2.12194440e-4f, r);
    float p = 1.9875691500e-4f;
    p = B200_FMA(p, r, 1.3981999507e-3f);
    p = B200_FMA(p, r, 8.3334519073e-3f);
    p = B200_FMA(p, r, 4.1665795894e-2f);
    p = B200_FMA(p, r, 1.6666665459e-1f);
    p = B200_FMA(p, r, 5.0000001201e-1f);
    const float r2 = B200_MUL(r, r);
    p = B200_FMA(p, r2, r);
    p = B200_ADD(p, 1.0f);
    const float scale = B200_U2F((B200_F2U(tb) << 23) + 0x3f800000u);
    const float y = B200_MUL(p, scale);
    return x < -86.0f ? 0.0f : y;
}

/* log(x) for normal x > 0. */
B200_MATH_FN float b200_logf(float x) {
    const uint32_t ix = B200_F2U(x);
    int32_t e = (int32_t)((ix >> 23) & 0xffu) - 126;
    float m = B200_U2F((ix & 0x007fffffu) | 0x3f000000u); /* [0.5, 1) */
    if (m < 0.707106781186547524f) {
        e -= 1;
        m = B200_SUB(B200_ADD(m, m), 1.0f);
    } else {
        m = B200_SUB(m, 1.0f);
    }
    const float z = B200_MUL(m, m);
    float y = 7.0376836292e-2f;
    y = B200_FMA(y, m, -1.1514610310e-1f);
    y = B200_FMA(y, m, 1.1676998740e-1f);
    y = B200_FMA(y, m, -1.2420140846e-1f);
    y = B200_FMA(y, m, 1.4249322787e-1f);
    y = B200_FMA(y, m, -1.6668057665e-1f);
    y = B200_FMA(y, m, 2.0000714765e-1f);
    y = B200_FMA(y, m, -2.4999993993e-1f);
    y = B200_FMA(y, m, 3.3333331174e-1f);
    y = B200_MUL(B200_MUL(y, m), z);
    const float fe = (float)e;
    y = B200_FMA(fe, -2.12194440e-4f, y);
    y = B200_FMA(z, -0.5f, y);
    float r = B200_ADD(m, y);
    r = B200_FMA(fe, 0.693359375f, r);
    return r;
}

/* log1p(x) for x in [0, 1]: log(u) corrected for the rounding of u = 1 + x. */
B200_MATH_FN float b200_log1pf(float x) {
    const float u = B200_ADD(1.0f, x);
    const float c = B200_SUB(x, B200_SUB(u, 1.0f)); /* exact rounding error of 1 + x */
    return B200_ADD(b200_logf(u), B200_DIV(c, u));
}

/* beam_search.cpp:42-45 */
B200_MATH_FN float b200_log_sum_exp(float x, float y) {
    const float d = B200_SUB(x, y);
    const float ad = d < 0.0f ? -d : d;
    const float mx = b200_fmaxf(x, y);
    if (ad < 17.0f) {
        return B200_ADD(mx, b200_log1pf(b200_expf(-ad)));
    }
    return mx;
}

/* CPUDecoder.cpp:29-34: logsumexp over {stay, step0..3}: max-shifted, summed in this order. */
B200_MATH_FN float b200_lse5(float v_stay, float v0, float v1, float v2, float v3) {
    float m = b200_fmaxf(v_stay, v0);
    m = b200_fmaxf(m, v1);
    m = b200_fmaxf(m, v2);
    m = b200_fmaxf(m, v3);
    /* every argument is <= 0 (m is the maximum) */
    float s = b200_expf_nonpos(B200_SUB(v_stay, m));
    s = B200_ADD(s, b200_expf_nonpos(B200_SUB(v0, m)));
    s = B200_ADD(s, b200_expf_nonpos(B200_SUB(v1, m)));
    s = B200_ADD(s, b200_expf_nonpos(B200_SUB(v2, m)));
    s = B200_ADD(s, b200_expf_nonpos(B200_SUB(v3, m)));
    return B200_ADD(m, b200_logf(s));
}

/* ---- double-precision helpers (same rule: only correctly rounded IEEE-754 binary64 operations, fixed order) ---- */
#if defined(__CUDA_ARCH__)
#define B200_DFMA(a, b, c) __fma_rn((a), (b), (c))
#define B200_DMUL(a, b) __dmul_rn((a), (b))
#define B200_DADD(a, b) __dadd_rn((a), (b))
#define B200_DSUB(a, b) __dsub_rn((a), (b))
#define B200_DDIV(a, b) __ddiv_rn((a), (b))
#define B200_D2U(x) ((uint64_t)__double_as_longlong(x))
#define B200_U2D(x) __longlong_as_double((long long)(x))
#define B200_D2F(x) __double2float_rn(x)
#else
#define B200_DFMA(a, b, c) fma((a), (b), (c))
#define B200_DMUL(a, b) ((a) * (b))
#define B200_DADD(a, b) ((a) + (b))
#define B200_DSUB(a, b) ((a) - (b))
#define B200_DDIV(a, b) ((a) / (b))
static inline uint64_t b200_d2u_(double x) {
    uint64_t u;
    memcpy(&u, &x, 8);
    return u;
}
static inline double b200_u2d_(uint64_t u) {
    double x;
    memcpy(&x, &u, 8);
    return x;
}
#define B200_D2U(x) b200_d2u_(x)
#define B200_U2D(x) b200_u2d_(x)
#define B200_D2F(x) ((float)(x))
#endif

/* beam_search.cpp:503: std::pow(p, 0.4f) for p in [0, 1] (float arguments, i.e. powf with the exponent
 * 0.4f = 0.4000000059604644775390625).  The reference's value comes from the host libm; glibc 2.39's powf is within
 * 1 ulp and differs from the correctly rounded result for 0.06 % of the arguments (measured,
 * tests/test_host_cpu.py::test_pow0p4_against_libm).  The per-base quality is 1 - sum(p^0.4)/sum(...), which
 * cancels, so a 1-ulp difference here moves quality characters; the contract therefore evaluates
 * exp(0.4f * log(p)) in binary64 (relative error < 1e-15) and rounds once to binary32: the correctly rounded powf except
 * when the exact value lies within ~1e-8 ulp of a rounding boundary.  Subnormal arguments are handled exactly (binary64
 * holds them as normal numbers). */
B200_MATH_FN float b200_pow0p4f(float p) {
    if (p <= 0.0f) {
        return 0.0f;
    }
    if (p >= 1.0f) {
        return 1.0f;
    }
    /* log(x), x = m * 2^e with m in [sqrt(1/2), sqrt(2)):  log m = 2 atanh(s), s = (m - 1) / (m + 1) */
    const double x = (double)p;
    const uint64_t ix = B200_D2U(x);
    int64_t e = (int64_t)((ix >> 52) & 0x7ffu) - 1023;
    double m = B200_U2D((ix & 0x000fffffffffffffull) | 0x3ff0000000000000ull); /* [1, 2) */
    if (m > 1.4142135623730951) {
        m = B200_DMUL(m, 0.5);
        e += 1;
    }
    const double s = B200_DDIV(B200_DSUB(m, 1.0), B200_DADD(m, 1.0));
    const double s2 = B200_DMUL(s, s);
    double q = 1.0 / 23.0;
    q = B200_DFMA(q, s2, 1.0 / 21.0);
    q = B200_DFMA(q, s2, 1.0 / 19.0);
    q = B200_DFMA(q, s2, 1.0 / 17.0);
    q = B200_DFMA(q, s2, 1.0 / 15.0);
    q = B200_DFMA(q, s2, 1.0 / 13.0);
    q = B200_DFMA(q, s2, 1.0 / 11.0);
    q = B200_DFMA(q, s2, 1.0 / 9.0);
    q = B200_DFMA(q, s2, 1.0 / 7.0);
    q = B200_DFMA(q, s2, 1.0 / 5.0);
    q = B200_DFMA(q, s2, 1.0 / 3.0);
    double lm = B200_DFMA(B200_DMUL(s, s2), q, s); /* atanh(s) */
    lm = B200_DADD(lm, lm);
    const double fe = (double)e;
    /* ln2 split so that fe * hi is exact (fdlibm's constants) */
    double lx = B200_DFMA(fe, 1.90821492927058770002e-10, lm);
    lx = B200_DFMA(fe, 6.93147180369123816490e-01, lx);
    /* y = 0.4f * log(x) in [-41.4, 0);  exp(y) = 2^n * exp(r) */
    const double y = B200_DMUL(lx, 0.4000000059604644775390625);
    const double t = B200_DMUL(y, 1.44269504088896338700e+00);
    const double big = 6755399441055744.0; /* 1.5 * 2^52: round to nearest even */
    const double n = B200_DSUB(B200_DADD(t, big), big);
    double r = B200_DFMA(n, -6.93147180369123816490e-01, y);
    r = B200_DFMA(n, -1.90821492927058770002e-10, r);
    double ex = 1.0 / 6227020800.0; /* 1/13! */
    ex = B200_DFMA(ex, r, 1.0 / 479001600.0);
    ex = B200_DFMA(ex, r, 1.0 / 39916800.0);
    ex = B200_DFMA(ex, r, 1.0 / 3628800.0);
    ex = B200_DFMA(ex, r, 1.0 / 362880.0);
    ex = B200_DFMA(ex, r, 1.0 / 40320.0);
    ex = B200_DFMA(ex, r, 1.0 / 5040.0);
    ex = B200_DFMA(ex, r, 1.0 / 720.0);
    ex = B200_DFMA(ex, r, 1.0 / 120.0);
    ex = B200_DFMA(ex, r, 1.0 / 24.0);
    ex = B200_DFMA(ex, r, 1.0 / 6.0);
    ex = B200_DFMA(ex, r, 0.5);
    ex = B200_DFMA(ex, r, 1.0);
    ex = B200_DFMA(ex, r, 1.0);
    const int64_t ni = (int64_t)n;
    const double scale = B200_U2D((uint64_t)(ni + 1023) << 52);
    return B200_D2F(B200_DMUL(ex, scale));
}

/* beam_search.cpp:94-98: per-base quality character
 *     err = 1 - base_prob / total_prob;  q = -10 * log10(err) * scale + shift;  clamp(q, 1, 50);  char(33.5 + q)
 * As a function of err this is a quantiser with at most 50 output characters, so instead of approximating the host
 * libm's log10f (glibc's differs from the correctly rounded value for 4 % of the arguments) the engine places the bin
 * edges exactly: b200_qtable_build() (host) bisects the reference expression, evaluated with the host's own log10f, over
 * the bit patterns of err in (0, 1] and records every value at which the character changes; b200_qtable_lookup()
 * (host and device) is a search over those edges.  The result is the reference's character for every err, on the libm
 * of the machine the engine runs on -- the same libm the reference would use there. */
#define B200_QTABLE_CAP 96
typedef struct b200_qtable {
    uint32_t n;                      /* number of edges */
    uint32_t edge[B200_QTABLE_CAP];  /* ascending bit patterns of positive floats: the character changes AT edge[i] */
    uint8_t ch[B200_QTABLE_CAP + 1]; /* ch[i] for edge[i-1] <= bits(err) < edge[i] */
    uint8_t ch_nonpositive;          /* err <= 0 (log10 -> -inf -> q = +inf -> 50) */
    uint8_t pad[2];
} b200_qtable;

B200_MATH_FN char b200_qtable_lookup(const b200_qtable* tb, float base_prob, float total_prob) {
    const float e = B200_SUB(1.0f, B200_DIV(base_prob, total_prob));
    if (!(e > 0.0f)) {
        return (char)tb->ch_nonpositive;
    }
    const uint32_t u = B200_F2U(e);
    /* number of edges <= u */
    uint32_t lo = 0, hi = tb->n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (tb->edge[mid] <= u) {
            lo = mid + 1;
        } else {
            hi = mid;
        }
    }
    return (char)tb->ch[lo];
}

/* Host side (also parsed, as host code, in nvcc's device pass: no device intrinsics below). */
#include <math.h>
#include <string.h>
static inline float b200_host_u2f_(uint32_t u) {
    float x;
    memcpy(&x, &u, 4);
    return x;
}
/* The reference expression, operation by operation (beam_search.cpp:94-98), on the host libm. */
static inline char b200_qchar_libm(float err, float scale, float shift) {
    float bp = -10.0f * log10f(err);
    float q = bp * scale + shift;
    q = (q < 1.0f) ? 1.0f : ((50.0f < q) ? 50.0f : q); /* std::clamp */
    return (char)(33.5f + q);
}

static inline void b200_qtable_scan_(b200_qtable* tb, uint32_t lo, uint32_t hi, float scale, float shift, int* overflow) {
    /* invariant: the character at lo is already the last recorded one; find every change in (lo, hi] */
    const char clo = b200_qchar_libm(b200_host_u2f_(lo), scale, shift);
    const char chi = b200_qchar_libm(b200_host_u2f_(hi), scale, shift);
    if (clo == chi) {
        return; /* monotone quantiser: equal ends => constant in between (checked densely by the tests) */
    }
    if (hi - lo == 1) {
        if (tb->n >= B200_QTABLE_CAP) {
            *overflow = 1;
            return;
        }
        tb->edge[tb->n] = hi;
        tb->ch[tb->n + 1] = (uint8_t)chi;
        tb->n += 1;
        return;
    }
    const uint32_t mid = lo + (hi - lo) / 2;
    b200_qtable_scan_(tb, lo, mid, scale, shift, overflow);
    b200_qtable_scan_(tb, mid, hi, scale, shift, overflow);
}

/* Returns 0 on success, -1 if the expression is not a quantiser this table can hold (non-finite scale / shift). */
static inline int b200_qtable_build(float scale, float shift, b200_qtable* tb) {
    memset(tb, 0, sizeof(*tb));
    if (!(scale == scale) || !(shift == shift) || scale - scale != 0.0f || shift - shift != 0.0f) {
        return -1;
    }
    int overflow = 0;
    const uint32_t first = 1u, last = 0x3f800000u; /* smallest subnormal .. 1.0f */
    tb->ch_nonpositive = (uint8_t)b200_qchar_libm(0.0f, scale, shift);
    tb->ch[0] = (uint8_t)b200_qchar_libm(b200_host_u2f_(first), scale, shift);
    b200_qtable_scan_(tb, first, last, scale, shift, &overflow);
    return overflow ? -1 : 0;
}

#endif /* B200_CRF_MATH_H */
