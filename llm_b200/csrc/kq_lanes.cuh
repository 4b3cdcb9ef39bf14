// llm_b200/csrc/kq_lanes.cuh -- the lane arithmetic of ggml_vec_dot_q{2,3,4,5,6}_K_q8_K (AVX2 build) for one super-block, in the order kquants.cu's
// header documents.  A warp holds one weight row: lane = 8 * part + L owns byte column L of two of the eight 32-byte groups.  kq_load reads what the
// lane needs of a weight super-block once; kq_step folds one Q8_K super-block of one activation row into that row's chains (integer partials met by
// shuffles, then the 8-lane f32 FMA chain and the type's mins chain); kq_finish reduces them to the dot product (valid in every lane).
// Each output is therefore one complete dot product in the reference's order, however many activation rows a warp walks with one kq_load.
#pragma once
#include "kernels.cuh"

namespace b200 {
namespace kq {

constexpr int QKK = 256;
struct __align__(4) BlockQ8K { float d; int8_t qs[QKK]; int16_t bsums[QKK / 16]; };   // LC/k_quants.h:112-117
static_assert(sizeof(BlockQ8K) == 292, "block_q8_K");

__device__ __forceinline__ uint32_t ld_u32_a2(const uint8_t *p) {        // 4 bytes from a 2-byte aligned address (block_q6_K is 210 bytes)
    return (uint32_t)*(const uint16_t *)p | ((uint32_t)*(const uint16_t *)(p + 2) << 16);
}
__device__ __forceinline__ float h2f(const uint8_t *p) { return __half2float(*(const __half *)p); }

// 6-bit scale / min j of block_q4_K / block_q5_K (the utmp shuffles of LC/k_quants.c:2604-2609 = get_scale_min_k4, :316-324)
__device__ __forceinline__ int k4_scale(const uint8_t *q, int j) { return j < 4 ? (q[j] & 63) : ((q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4)); }
__device__ __forceinline__ int k4_min(const uint8_t *q, int j) { return j < 4 ? (q[j + 4] & 63) : ((q[j + 4] >> 4) | ((q[j] >> 6) << 4)); }
// 6-bit signed scale si of block_q3_K (the aux[] shuffles of LC/k_quants.c:1907-1913)
__device__ __forceinline__ int k3_scale(const uint8_t *s, int si) {
    const int wd = si >> 2, c = si & 3;
    return (int)(((s[(wd & 1) * 4 + c] >> (4 * (wd >> 1))) & 0xF) | (((s[8 + c] >> (2 * wd)) & 3) << 4)) - 32;
}

template <int TYPE> struct Bytes;
template <> struct Bytes<T_Q2_K> { static constexpr int N = 84, QS = 16; };      // scales[16] qs[64] d dmin   (LC/k_quants.h:34-39)
template <> struct Bytes<T_Q3_K> { static constexpr int N = 110, QS = 32; };     // hmask[32] qs[64] scales[12] d (:52-57)
template <> struct Bytes<T_Q4_K> { static constexpr int N = 144, QS = 16; };     // d dmin scales[12] qs[128]
template <> struct Bytes<T_Q5_K> { static constexpr int N = 176, QS = 48; };     // d dmin scales[12] qh[32] qs[128]
template <> struct Bytes<T_Q6_K> { static constexpr int N = 210, QS = 0; };      // ql[128] qh[64] scales[16] d

// one lane's share of a weight super-block
struct Lane {
    float d, dmin;          // fp16 d / dmin of the block
    uint32_t w, h;          // quant words (Q3_K: hmask; Q5_K: high bits; Q6_K: high 2-bit word)
    int s0, s1, m0, m1;     // the two sub-block scales this lane's groups use; the mins of its bsums pair
};

template <int TYPE>
__device__ __forceinline__ Lane kq_load(const uint8_t *wb, int lane) {
    const int L = lane & 7, part = lane >> 3;
    Lane r;
    r.dmin = 0.f; r.h = 0; r.m0 = r.m1 = 0;
    if (TYPE == T_Q2_K || TYPE == T_Q3_K) {
        // 2-bit planes: group (j, k) = bits 2k of qs[32j ..] against q8[128j + 32k ..]; sub-block scale index 8j + 2k + (L >= 4) (get_scale_shuffle_q3k)
        const int j = part >> 1, k0 = 2 * (part & 1);
        const int si0 = 8 * j + 2 * k0 + (L >= 4), si1 = si0 + 2;
        if (TYPE == T_Q2_K) {
            r.d = h2f(wb + 80); r.dmin = h2f(wb + 82);
            r.m0 = wb[2 * L] >> 4; r.m1 = wb[2 * L + 1] >> 4;
            r.w = *(const uint32_t *)(wb + 16 + 32 * j + 4 * L);
            r.s0 = wb[si0] & 0xF; r.s1 = wb[si1] & 0xF;
        } else {
            r.d = h2f(wb + 108);
            r.h = ld_u32_a2(wb + 4 * L);
            r.w = ld_u32_a2(wb + 32 + 32 * j + 4 * L);
            r.s0 = k3_scale(wb + 96, si0); r.s1 = k3_scale(wb + 96, si1);
        }
    } else if (TYPE == T_Q6_K) {
        const int j = part >> 1, hs = part & 1;
        r.d = h2f(wb + 208);
        r.w = ld_u32_a2(wb + 64 * j + 32 * hs + 4 * L);
        r.h = ld_u32_a2(wb + 128 + 32 * j + 4 * L);
        const int8_t *sc = (const int8_t *)(wb + 192);
        r.s0 = sc[2 * (4 * j + hs) + (L >= 4)]; r.s1 = sc[2 * (4 * j + hs + 2) + (L >= 4)];
    } else {
        r.d = h2f(wb); r.dmin = h2f(wb + 2);
        const uint8_t *scq = wb + 4;
        r.w = *(const uint32_t *)(wb + Bytes<TYPE>::QS + 32 * part + 4 * L);
        if (TYPE == T_Q5_K) r.h = *(const uint32_t *)(wb + 16 + 4 * L);
        r.s0 = k4_scale(scq, 2 * part); r.s1 = k4_scale(scq, 2 * part + 1);
        const int t = lane & 3;                                        // prod[t] of :2614-2617 (every lane carries the copy of its t)
        r.m0 = k4_min(scq, 2 * t); r.m1 = k4_min(scq, 2 * t + 1);
    }
    return r;
}

// acc: lane L's entry of the 8-lane f32 accumulator; accm: Q4_K's 4-lane / Q5_K's scalar mins accumulator
template <int TYPE>
__device__ __forceinline__ void kq_step(const Lane &r, const BlockQ8K *__restrict__ xb, int lane, float &acc, float &accm) {
    const int L = lane & 7, part = lane >> 3;
    const float yd = xb->d;
    int p;
    if (TYPE == T_Q2_K || TYPE == T_Q3_K) {
        const int j = part >> 1;
        float d;
        if (TYPE == T_Q2_K) {
            d = __fmul_rn(yd, r.d);
            const float dmin = __fmul_rn(-yd, r.dmin);
            const int prod = r.m0 * (int)xb->bsums[2 * L] + r.m1 * (int)xb->bsums[2 * L + 1];
            acc = __fmaf_rn(dmin, (float)prod, acc);                  // the mins go into the SAME accumulator, before the quants (:1350)
        } else {
            d = __fmul_rn(yd, r.d);
        }
        p = 0;
#pragma unroll
        for (int kk = 0; kk < 2; kk++) {
            const int k = 2 * (part & 1) + kk;
            const uint32_t lo = (r.w >> (2 * k)) & 0x03030303u;
            const int xw = *(const int *)(xb->qs + 128 * j + 32 * k + 4 * L);
            const int sc = kk ? r.s1 : r.s0;
            if (TYPE == T_Q2_K) p += sc * __dp4a((int)lo, xw, 0);
            else {
                const uint32_t q3h = ((~(r.h >> (4 * j + k))) & 0x01010101u) << 2;       // 4 where the high bit is NOT set (:1936-1948)
                p += sc * (__dp4a((int)lo, xw, 0) - __dp4a((int)q3h, xw, 0));
            }
        }
        p += __shfl_xor_sync(0xffffffffu, p, 8);
        p += __shfl_xor_sync(0xffffffffu, p, 16);
        acc = __fmaf_rn(d, (float)p, acc);
    } else if (TYPE == T_Q6_K) {
        const float d = __fmul_rn(yd, r.d);
        const int j = part >> 1, hs = part & 1;
        p = 0;
#pragma unroll
        for (int kk = 0; kk < 2; kk++) {                              // groups k = hs and hs + 2 of this 128-element half share the ql bytes
            const int k = hs + 2 * kk;
            const uint32_t nib = (kk ? (r.w >> 4) : r.w) & 0x0F0F0F0Fu;
            const uint32_t q = nib | (((r.h >> (2 * k)) & 0x03030303u) << 4);
            const int xw = *(const int *)(xb->qs + 128 * j + 32 * k + 4 * L);
            const int dot = __dp4a((int)q, xw, 0) - 32 * __dp4a(0x01010101, xw, 0);
            p += (kk ? r.s1 : r.s0) * dot;
        }
        p += __shfl_xor_sync(0xffffffffu, p, 8);
        p += __shfl_xor_sync(0xffffffffu, p, 16);
        acc = __fmaf_rn(d, (float)p, acc);
    } else {
        const float d = __fmul_rn(yd, r.d), dmin = __fmul_rn(-yd, r.dmin);
        uint32_t lo = r.w & 0x0F0F0F0Fu, hi = (r.w >> 4) & 0x0F0F0F0Fu;
        if (TYPE == T_Q5_K) {
            lo |= ((r.h >> (2 * part)) & 0x01010101u) << 4;
            hi |= ((r.h >> (2 * part + 1)) & 0x01010101u) << 4;
        }
        const int x0 = *(const int *)(xb->qs + 64 * part + 4 * L), x1 = *(const int *)(xb->qs + 64 * part + 32 + 4 * L);
        p = r.s0 * __dp4a((int)lo, x0, 0) + r.s1 * __dp4a((int)hi, x1, 0);
        p += __shfl_xor_sync(0xffffffffu, p, 8);
        p += __shfl_xor_sync(0xffffffffu, p, 16);
        acc = __fmaf_rn(d, (float)p, acc);
        const int t = lane & 3;
        const int q8a = (int)(int16_t)(xb->bsums[4 * t] + xb->bsums[4 * t + 1]), q8b = (int)(int16_t)(xb->bsums[4 * t + 2] + xb->bsums[4 * t + 3]);
        int prod = r.m0 * q8a + r.m1 * q8b;
        if (TYPE == T_Q5_K) {
            prod += __shfl_xor_sync(0xffffffffu, prod, 1);
            prod += __shfl_xor_sync(0xffffffffu, prod, 2);
        }
        accm = __fmaf_rn(dmin, (float)prod, accm);
    }
}

template <int TYPE>
__device__ __forceinline__ float kq_finish(float acc, float accm) {
    float v = acc;                                                        // hsum_float_8: ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7))
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 2));
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 1));
    if (TYPE == T_Q4_K) {                                                 // (m0+m2) + (m1+m3)
        accm = __fadd_rn(accm, __shfl_xor_sync(0xffffffffu, accm, 2));
        accm = __fadd_rn(accm, __shfl_xor_sync(0xffffffffu, accm, 1));
    }
    if (TYPE == T_Q4_K || TYPE == T_Q5_K) v = __fadd_rn(v, accm);
    return v;
}

}  // namespace kq
}  // namespace b200
