/* llm_b200/csrc/libm_f32.h -- glibc's expf and logf (x86-64, the FMA build its ifunc picks on AVX2 hosts), restated so that the GPU computes the
 * same bits as the host's libm.
 *
 * Why: the reference's perplexity loop (crates/llm-base/src/inference_session.rs:514-589, util::softmax) calls Rust's f32::exp / f32::ln, which on
 * x86_64-linux-gnu are glibc's expf / logf.  CUDA's expf / logf, and rounding a double exp / log, differ from them on about 1e-4 of all inputs.
 *
 * The algorithms and their constants are those of glibc's sysdeps/ieee754/flt-32/e_expf.c, e_exp2f_data.c, e_logf.c and e_logf_data.c, which
 * come from ARM's optimized-routines (MIT licence).  Every double operation is written with an explicit rounding intrinsic (the device's
 * __dmul_rn / __dadd_rn / __fma_rn; on the host plain operators with -ffp-contract=off and fma()), in the order and with the fused multiply-adds
 * the FMA build of glibc executes, so that no compiler contraction can change a result.
 *
 * The same source is compiled by nvcc for the kernels (ppl.cu) and by gcc for the exhaustive check against the host libm
 * (tests/test_perplexity_oracle.py).  Plain C, no CUDA headers needed on the host side. */
#ifndef LLM_B200_LIBM_F32_H
#define LLM_B200_LIBM_F32_H
#include <stdint.h>

#if defined(__CUDACC__)
#define LM_HD __host__ __device__ __forceinline__
#else
#include <math.h>
#include <string.h>
#define LM_HD static inline
#endif

#if defined(__CUDA_ARCH__)
LM_HD double lm_mul(double a, double b) { return __dmul_rn(a, b); }
LM_HD double lm_add(double a, double b) { return __dadd_rn(a, b); }
LM_HD double lm_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
LM_HD float lm_fmul(float a, float b) { return __fmul_rn(a, b); }
LM_HD float lm_f(double a) { return __double2float_rn(a); }
LM_HD double lm_i2d(int32_t k) { return __int2double_rn(k); }
LM_HD uint32_t lm_fbits(float x) { return __float_as_uint(x); }
LM_HD float lm_bitsf(uint32_t u) { return __uint_as_float(u); }
LM_HD uint64_t lm_dbits(double x) { return (uint64_t)__double_as_longlong(x); }
LM_HD double lm_bitsd(uint64_t u) { return __longlong_as_double((long long)u); }
#else
LM_HD double lm_mul(double a, double b) { return a * b; }
LM_HD double lm_add(double a, double b) { return a + b; }
LM_HD double lm_fma(double a, double b, double c) { return fma(a, b, c); }
LM_HD float lm_fmul(float a, float b) { return a * b; }
LM_HD float lm_f(double a) { return (float)a; }
LM_HD double lm_i2d(int32_t k) { return (double)k; }
LM_HD uint32_t lm_fbits(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
LM_HD float lm_bitsf(uint32_t u) { float x; memcpy(&x, &u, 4); return x; }
LM_HD uint64_t lm_dbits(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }
LM_HD double lm_bitsd(uint64_t u) { double x; memcpy(&x, &u, 8); return x; }
#endif

/* __exp2f_data.tab: bits of 2^(i/32), minus i << 47 so that adding ki << 47 puts the exponent of 2^(ki/32) in place */
#define LM_EXP2F_TAB { \
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, 0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, \
    0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, 0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull, \
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, 0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, \
    0x3feea11473eb0187ull, 0x3feea589994cce13ull, 0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull, \
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, 0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, \
    0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull }

/* __logf_data.tab: {invc, logc} of the 16 subintervals of [0x3f330000, 2 * 0x3f330000) */
#define LM_LOGF_TAB { \
    {0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2}, {0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2}, {0x1.49539f0f010b0p+0, -0x1.01eae7f513a67p-2}, \
    {0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3}, {0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3}, {0x1.25e227b0b8ea0p+0, -0x1.1aa2bc79c8100p-3}, \
    {0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4}, {0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4}, {0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5}, \
    {0x1.0p+0, 0x0.0p+0}, {0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5}, {0x1.ca4b31f026aa0p-1, 0x1.c5e53aa362eb4p-4}, \
    {0x1.b2036576afce6p-1, 0x1.526e57720db08p-3}, {0x1.9c2d163a1aa2dp-1, 0x1.bc2860d224770p-3}, {0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2}, \
    {0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2} }

#if defined(__CUDACC__)
static __device__ const uint64_t lm_exp2f_tab_d[32] = LM_EXP2F_TAB;
static __device__ const double lm_logf_tab_d[16][2] = LM_LOGF_TAB;
#endif
static const uint64_t lm_exp2f_tab_h[32] = LM_EXP2F_TAB;
static const double lm_logf_tab_h[16][2] = LM_LOGF_TAB;

LM_HD uint64_t lm_exp2f_tab(uint32_t i) {
#if defined(__CUDA_ARCH__)
    return lm_exp2f_tab_d[i];
#else
    return lm_exp2f_tab_h[i];
#endif
}
LM_HD double lm_logf_tab(uint32_t i, int which) {
#if defined(__CUDA_ARCH__)
    return lm_logf_tab_d[i][which];
#else
    return lm_logf_tab_h[i][which];
#endif
}

/* expf: exp(x) = 2^(k/32) * 2^(r/32), k = round(x * 32/ln2), r = x * 32/ln2 - k in [-1/2, 1/2], 2^(r/32) by a degree-3 polynomial */
LM_HD float lm_expf(float x) {
    const double InvLn2N = 0x1.71547652b82fep+5, Shift = 0x1.8p+52;
    const double C0 = 0x1.c6af84b912394p-20, C1 = 0x1.ebfce50fac4f3p-13, C2 = 0x1.62e42ff0c52d6p-6;
    const uint32_t abstop = (lm_fbits(x) >> 20) & 0x7ff;
    if (abstop >= 0x42b) {                                      /* |x| >= 88 or x is nan */
        if (lm_fbits(x) == 0xff800000u) return 0.0f;             /* -inf */
        if (abstop >= 0x7f8) return x + x;                      /* +inf, nan */
        if (x > 0x1.62e42ep6f) return lm_bitsf(0x7f800000u);    /* overflow: +inf */
        if (x < -0x1.9fe368p6f) return 0.0f;                    /* exp(x) < 2^-150: underflow to +0 */
        if (x < -0x1.9d1d9ep6f) return lm_fmul(0x1.4p-75f, 0x1.4p-75f);   /* exp(x) in (2^-150, 2^-149): the least subnormal */
    }
    const double xd = (double)x;
    double kd = lm_fma(InvLn2N, xd, Shift);                     /* z + Shift, fused: the FMA build contracts z = InvLn2N * xd into both uses */
    const uint64_t ki = lm_dbits(kd);
    kd = lm_add(kd, -Shift);
    const double r = lm_fma(InvLn2N, xd, -kd);
    const uint64_t t = lm_exp2f_tab((uint32_t)(ki % 32)) + (ki << 47);
    const double s = lm_bitsd(t);
    const double z = lm_fma(C0, r, C1);
    const double r2 = lm_mul(r, r);
    double y = lm_fma(C2, r, 1.0);
    y = lm_fma(z, r2, y);
    y = lm_mul(y, s);
    return lm_f(y);
}

/* logf: x = 2^k z with z in [0x3f330000, 2 * 0x3f330000); log(x) = log1p(z/c - 1) + log(c) + k ln2, c near the centre of z's subinterval */
LM_HD float lm_logf(float x) {
    const double Ln2 = 0x1.62e42fefa39efp-1;
    const double A0 = -0x1.00ea348b88334p-2, A1 = 0x1.5575b0be00b6ap-2, A2 = -0x1.ffffef20a4123p-2;
    const uint32_t OFF = 0x3f330000u;
    uint32_t ix = lm_fbits(x);
    if (ix == 0x3f800000u) return 0.0f;                         /* log(1) = +0 */
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {        /* x < 0x1p-126, inf or nan */
        if (ix * 2 == 0) return lm_bitsf(0xff800000u);          /* log(+-0) = -inf */
        if (ix == 0x7f800000u) return x;                        /* log(inf) = inf */
        if ((ix & 0x80000000u) || ix * 2 >= 0xff000000u) return lm_bitsf(0x7fc00000u);   /* negative or nan: nan */
        ix = lm_fbits(lm_fmul(x, 0x1p23f));                     /* subnormal: normalize */
        ix -= 23u << 23;
    }
    const uint32_t tmp = ix - OFF;
    const uint32_t i = (tmp >> 19) % 16;
    const int32_t k = (int32_t)tmp >> 23;
    const uint32_t iz = ix - (tmp & 0xff800000u);
    const double invc = lm_logf_tab(i, 0), logc = lm_logf_tab(i, 1);
    const double z = (double)lm_bitsf(iz);
    const double r = lm_fma(z, invc, -1.0);
    const double y0 = lm_fma(lm_i2d(k), Ln2, logc);
    const double r2 = lm_mul(r, r);
    double y = lm_fma(A1, r, A2);
    y = lm_fma(A0, r2, y);
    y = lm_fma(y, r2, lm_add(y0, r));
    return lm_f(y);
}

#endif /* LLM_B200_LIBM_F32_H */
