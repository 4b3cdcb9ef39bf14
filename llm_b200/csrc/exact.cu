// llm_b200/csrc/exact.cu -- BIT-EXACT counterparts of the mat-mul kernels: same bits as the reference's AVX2 CPU path.
//
// Why they exist (DESIGN.md "chaos"): the reference graph re-quantizes activations to Q8 before every weight mat-mul and
// rounds Q / softmax rows to fp16 before the attention mat-muls.  Those roundings are discontinuous, and on a multi-layer
// model a 1e-7 perturbation of ONE mat-mul (e.g. merely re-associating the final horizontal sum of ggml_vec_dot_q4_0_q8_0)
// already moves the logits by ~1e-2 (tests/test_chaos.py reproduces this on the CPU with the oracle alone).  The north-star
// bar of 1e-3 against the reference CPU path is therefore reachable only by reproducing its f32 operation ORDER, not just
// its integer arithmetic.  These kernels do exactly that:
//
//   ggml_vec_dot_q*_q8_* (AVX2, LC/ggml.c:2434-2457, 2702-2735, 2916-2938, 3166-3191, 3315-3336):
//       one __m256 accumulator = 8 f32 lanes; lane L accumulates, block after block IN ORDER,
//       acc_L = fma(d_w*d_x, (float)sum_{t<4} w[4L+t]*x[4L+t], acc_L);  result = hsum_float_8(acc) (+ summs),
//       hsum_float_8 (LC/ggml.c:608-616) = ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)).
//   Here: 4 threads per weight row; thread w owns lanes w and w+4 -- which is exactly word w of a packed GGML block
//   (low nibbles = elements 4w..4w+3 = lane w, high nibbles = elements 16+4w.. = lane w+4) -- walks the blocks in order with
//   two dp4a + two fma, and the 4 threads finish with the hsum tree through two xor-shuffles.
//
//   ggml_vec_dot_f16 (AVX, LC/ggml.c:2325-2359, macros :1876-1975): 4 accumulators x 8 lanes, element k goes to lane k % 32,
//       fma in order; GGML_F32x8_REDUCE: (s0+s2)+(s1+s3), then lanes (q + q+4), then hadd, hadd; leftovers (n % 32) are added
//       in DOUBLE on top.  Here: one warp per dot product, lane l = element k % 32, shuffle tree with offsets 16, 8, 4, 1, 2.
#include <type_traits>

#include "f32dot.cuh"
#include "kernels.cuh"

namespace b200 {

// ---- weight block word access: word w (bytes 4w..4w+3 of qs) of block i, unpacked to the two int8x4 the AVX code multiplies ----
template <int TYPE>
__device__ __forceinline__ void load_word(const QWeight &w, int64_t i, int wd, int &lo, int &hi, float &d, float &m) {
    m = 0.f;
    if (TYPE == T_Q8_0) {
        lo = (int)__ldg((const uint32_t *)(w.qs + i * 32) + wd);          // elements 4w..4w+3      -> lane w
        hi = (int)__ldg((const uint32_t *)(w.qs + i * 32) + 4 + wd);      // elements 16+4w..       -> lane w+4
        d = f16_bits_to_f32(__ldg((const uint16_t *)w.dm + i));
        return;
    }
    const uint32_t q = __ldg((const uint32_t *)(w.qs + i * 16) + wd);
    uint32_t l = q & 0x0F0F0F0Fu, h = (q >> 4) & 0x0F0F0F0Fu;
    if (TYPE == T_Q5_0 || TYPE == T_Q5_1) {
        const uint32_t qh = __ldg(w.qh + i);
        l |= spread4_to_bit4(qh >> (4 * wd));
        h |= spread4_to_bit4(qh >> (16 + 4 * wd));
    }
    if (TYPE == T_Q4_0) {   // bx - 8 (LC/ggml.c:2445-2447): per byte, no carries
        uint32_t u = l ^ 0x08080808u; l = u | ((u & 0x08080808u) * 30u);
        u = h ^ 0x08080808u; h = u | ((u & 0x08080808u) * 30u);
    }
    if (TYPE == T_Q5_0) {   // (nibble | ~bit<<4) == q5 - 16 (LC/ggml.c:2924-2927)
        uint32_t u = l ^ 0x10101010u; l = u | ((u & 0x10101010u) * 14u);
        u = h ^ 0x10101010u; h = u | ((u & 0x10101010u) * 14u);
    }
    lo = (int)l; hi = (int)h;
    if (TYPE == T_Q4_1 || TYPE == T_Q5_1) {
        const uint32_t dm = __ldg((const uint32_t *)w.dm + i);
        d = f16_bits_to_f32((uint16_t)(dm & 0xffffu)); m = f16_bits_to_f32((uint16_t)(dm >> 16));
    } else {
        d = f16_bits_to_f32(__ldg((const uint16_t *)w.dm + i));
    }
}

constexpr int EX_THREADS = 128;   // 32 rows per CTA, 4 threads per row

// dst[t*ldd + row] for TOK activation rows starting at token t0 (TOK = 1: the decode mat-vec)
template <int TYPE, int TOK>
__global__ void __launch_bounds__(EX_THREADS) mm_exact_kernel(const QWeight w, const int8_t *__restrict__ xq, const float2 *__restrict__ xds,
                                                              float *__restrict__ dst, int64_t ldd, int64_t B,
                                                              const float *__restrict__ addend, int64_t lda) {
    constexpr bool Q81 = (TYPE == T_Q4_1 || TYPE == T_Q5_1);
    const int wd = threadIdx.x & 3;
    const int64_t row_raw = (int64_t)blockIdx.x * (EX_THREADS / 4) + (threadIdx.x >> 2);
    const int64_t row = row_raw < w.N ? row_raw : w.N - 1;          // clamp: whole quads stay converged for the shuffles
    const int64_t t0 = (int64_t)blockIdx.y * TOK;
    const int nb = (int)w.nb;
    float a_lo[TOK], a_hi[TOK], summs[TOK];
#pragma unroll
    for (int t = 0; t < TOK; t++) { a_lo[t] = 0.f; a_hi[t] = 0.f; summs[t] = 0.f; }

#pragma unroll 4
    for (int b = 0; b < nb; b++) {
        int lo, hi; float dw, mw;
        load_word<TYPE>(w, row * nb + b, wd, lo, hi, dw, mw);
#pragma unroll
        for (int t = 0; t < TOK; t++) {
            const int64_t tok = t0 + t < B ? t0 + t : B - 1;
            const int32_t *xb = (const int32_t *)(xq + (tok * nb + b) * QK);
            const int xl = __ldg(xb + wd), xh = __ldg(xb + 4 + wd);
            const float2 xs = __ldg(xds + tok * nb + b);
            const float d = __fmul_rn(dw, xs.x);                           // _mm256_set1_ps(d_w * d_x) / _mm256_mul_ps(d0v, d1v)
            a_lo[t] = __fmaf_rn(d, (float)__dp4a(lo, xl, 0), a_lo[t]);     // _mm256_fmadd_ps(d, q, acc), lane w
            a_hi[t] = __fmaf_rn(d, (float)__dp4a(hi, xh, 0), a_hi[t]);     //                             lane w + 4
            if (Q81) summs[t] = __fmaf_rn(mw, xs.y, summs[t]);             // summs += m * s  (fused in the reference build); same on all 4 threads
        }
    }
#pragma unroll
    for (int t = 0; t < TOK; t++) {
        float r = __fadd_rn(a_hi[t], a_lo[t]);                             // hsum_float_8: hi128 + lo128       -> r_w = a_{w+4} + a_w
        r = __fadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 2));              //   + movehl                         -> s_{w&1} = r_w + r_{w^2}
        r = __fadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 1));              //   + movehdup                       -> s_0 + s_1
        if (Q81) r = __fadd_rn(r, summs[t]);                               // hsum_float_8(acc) + summs
        if (wd == 0 && row_raw < w.N && t0 + t < B) {
            const int64_t o = (t0 + t) * ldd + row;
            dst[o] = addend ? __fadd_rn(r, addend[(t0 + t) * lda + row]) : r;
        }
    }
}

template <int TYPE>
static void launch_exact(const QWeight &w, const int8_t *xq, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    const unsigned gx = (unsigned)((w.N + EX_THREADS / 4 - 1) / (EX_THREADS / 4));
    if (B == 1)      mm_exact_kernel<TYPE, 1><<<dim3(gx, 1), EX_THREADS, 0, st>>>(w, xq, xds, dst, ldd, B, addend, lda);
    else if (B <= 4) mm_exact_kernel<TYPE, 4><<<dim3(gx, 1), EX_THREADS, 0, st>>>(w, xq, xds, dst, ldd, B, addend, lda);
    else             mm_exact_kernel<TYPE, 8><<<dim3(gx, (unsigned)((B + 7) / 8)), EX_THREADS, 0, st>>>(w, xq, xds, dst, ldd, B, addend, lda);
    B200_CHECK(cudaGetLastError());
}

void mul_mat_q_exact(const QWeight &w, const int8_t *xq, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    if (w.N == 0 || B == 0) return;
    switch (w.type) {
        case T_Q4_0: launch_exact<T_Q4_0>(w, xq, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q4_1: launch_exact<T_Q4_1>(w, xq, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q5_0: launch_exact<T_Q5_0>(w, xq, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q5_1: launch_exact<T_Q5_1>(w, xq, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q8_0: launch_exact<T_Q8_0>(w, xq, xds, dst, ldd, B, addend, lda, st); break;
        default: B200_ASSERT(!"mul_mat_q_exact: unsupported weight type");
    }
}

// ---- the attention mat-muls on the KV cache: one warp per output element ------------------------------------------------------------
// dst[i2][i1][i0] = dot(src0[i2/(ne12/ne02)][i0][0..ne00), src1[i2][i1][0..ne00)).  `causal_past` >= 0 skips outputs with
// i0 > causal_past + i1 (they are overwritten with -inf by diag_mask_inf before anyone reads them; llama lib.rs:274-276).
// F32 = false: an f16 cache, ggml_vec_dot_f16 on src1 rounded to fp16 (leftovers in double); F32 = true: an f32 cache, ggml_vec_dot_f32 on src1
// as it is (leftovers in float, f32dot.cuh).  Both share the 32 chains and the reduction tree.
template <bool F32> struct AttnSrc0 { using T = __half; };
template <> struct AttnSrc0<true> { using T = float; };
template <bool F32> __device__ __forceinline__ float attn_a(const typename AttnSrc0<F32>::T *a, int64_t k) {
    if constexpr (F32) return a[k]; else return __half2float(a[k]);
}
template <bool F32> __device__ __forceinline__ float attn_b(const float *b, int64_t k) {   // from_float of the vec_dot_type (F32: none)
    if constexpr (F32) return b[k]; else return __half2float(__float2half_rn(b[k]));
}

constexpr int F16X_WARPS = 8;
template <bool F32>
__device__ __forceinline__ void mul_mat_attn_warp(const char *__restrict__ src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                                                  const char *__restrict__ src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                                                  char *__restrict__ dst, int64_t nbd1, int64_t nbd2, int causal_past,
                                                  unsigned bx, unsigned by, unsigned bz) {   // the output block (the grid's, or a batched row's)
    using T0 = typename AttnSrc0<F32>::T;
    const int lane = threadIdx.x & 31;
    const int64_t i0 = (int64_t)bx * F16X_WARPS + (threadIdx.x >> 5);
    const int64_t i1 = by, i2 = bz;
    if (i0 >= ne01) return;
    if (causal_past >= 0 && i0 > causal_past + i1) return;
    const int64_t i02 = i2 / (ne12 / ne02);
    const T0 *a = (const T0 *)(src0 + i02 * nb02 + i0 * nb01);
    const float *b = (const float *)(src1 + i2 * nb12 + i1 * nb11);
    const int64_t np = ne00 & ~(int64_t)31;
    float s = 0.f;
    for (int64_t k = lane; k < np; k += 32)                       // sum[j][q] with l = j*8 + q: GGML_F16_VEC_FMA / GGML_F32_VEC_FMA in order of i
        s = __fmaf_rn(attn_a<F32>(a, k), attn_b<F32>(b, k), s);
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 16));        // x[0] += x[2]; x[1] += x[3]
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 8));         // x[0] += x[1]
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 4));         // t0 = lo128 + hi128
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 1));         // hadd
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 2));         // hadd
    if (lane == 0) {
        float r;
        if constexpr (F32) {
            r = f32_leftovers(s, (int)(ne00 - np), [&](int i) { return a[np + i]; }, [&](int i) { return b[np + i]; });
        } else {
            double sumf = (double)s;
            for (int64_t k = np; k < ne00; ++k)                    // leftovers: double += (double)(f32 product)
                sumf += (double)__fmul_rn(__half2float(a[k]), __half2float(__float2half_rn(b[k])));
            r = (float)sumf;
        }
        *(float *)(dst + i2 * nbd2 + i1 * nbd1 + i0 * 4) = r;
    }
}
__global__ void __launch_bounds__(F16X_WARPS * 32) mul_mat_f16_exact_kernel(const char *__restrict__ src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                                                                            const char *__restrict__ src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                                                                            char *__restrict__ dst, int64_t nbd1, int64_t nbd2, int causal_past) {
    mul_mat_attn_warp<false>(src0, ne00, ne01, ne02, nb01, nb02, src1, ne11, ne12, nb11, nb12, dst, nbd1, nbd2, causal_past,
                              blockIdx.x, blockIdx.y, blockIdx.z);
}
__global__ void __launch_bounds__(F16X_WARPS * 32) mul_mat_f32_exact_kernel(const char *__restrict__ src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                                                                            const char *__restrict__ src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                                                                            char *__restrict__ dst, int64_t nbd1, int64_t nbd2, int causal_past) {
    mul_mat_attn_warp<true>(src0, ne00, ne01, ne02, nb01, nb02, src1, ne11, ne12, nb11, nb12, dst, nbd1, nbd2, causal_past,
                              blockIdx.x, blockIdx.y, blockIdx.z);
}

// ---- batched version: shared-memory tiles, 4 threads per dot, 8 dots per thread --------------------------------------------------------
// CTA = 16 src0 rows x 32 src1 rows (512 dots), 64 elements of the reduction per stage, operands staged as f32 (src0: f16 -> f32 or f32,
// src1: f32 -> f16 -> f32, the rounding ggml_compute_forward_mul_mat applies before the f16 dot, or f32 as it is).  The 32 chains of
// ggml_vec_dot_f16 / ggml_vec_dot_f32 (chain l over elements k = l mod 32, sequential in k) are split over the 4 threads of a quad as
// l in {4u..4u+3} u {16+4u..16+4u+3}: two 16-byte shared loads per operand row and step, and the reduction tree (offsets 16, 8, 4, then the two
// hadds) is: in-thread, quad shuffle 2, quad shuffle 1, in-thread -- the reference's association exactly.  Inner loop per thread and 32-element
// step: 12 LDS.128 + 64 FFMA.
constexpr int FT_A = 16, FT_B = 32, FT_K = 64, FT_STRIDE = FT_K + 4, FT_THREADS = 256;      // stride 68 floats: quads of a quarter-warp hit disjoint banks
static_assert(FT_B == ATTN_TILE_ROWS, "a ragged step's tile table counts query tiles of FT_B rows");

template <bool F32>
__device__ __forceinline__ void mul_mat_attn_tiled(const char *__restrict__ src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                                                   const char *__restrict__ src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                                                   char *__restrict__ dst, int64_t nbd1, int64_t nbd2, int causal_past,
                                                   unsigned bx, unsigned by, unsigned bz) {   // the output tile (the grid's, or a ragged step's)
    using T0 = typename AttnSrc0<F32>::T;
    using RA = typename std::conditional<F32, float4, uint2>::type;                   // one thread's 4 src0 elements
    __shared__ __align__(16) float sa[2][FT_A][FT_STRIDE];
    __shared__ __align__(16) float sb[2][FT_B][FT_STRIDE];
    const int tid = threadIdx.x, u = tid & 3, bq = (tid >> 2) & 7, ap = tid >> 5;        // quad (ap, bq): src0 rows 2ap, 2ap+1 x src1 rows 4bq..4bq+3
    const int64_t a0 = (int64_t)bx * FT_A, b0 = (int64_t)by * FT_B, i2 = bz;
    if (causal_past >= 0 && a0 > causal_past + (b0 + FT_B - 1 < ne11 - 1 ? b0 + FT_B - 1 : ne11 - 1)) return;      // whole tile above the diagonal
    const int64_t i02 = i2 / (ne12 / ne02);
    const char *A = src0 + i02 * nb02, *Bm = src1 + i2 * nb12;
    const int64_t np = ne00 & ~(int64_t)31;

    // fill plan: src0 tile = 16 rows x 64 elements = 256 x 4 elements (one per thread); src1 tile = 32 rows x 64 floats = 512 x 16 B (two per thread)
    const int far = tid >> 4, fac = (tid & 15) * 4;                  // src0: row, first of 4 elements
    const int fbr = tid >> 3, fbc = (tid & 7) * 4;                   // src1: rows fbr and fbr (+0) with columns fbc, fbc + 32
    const int64_t arow = a0 + far < ne01 ? a0 + far : ne01 - 1, brow = b0 + fbr < ne11 ? b0 + fbr : ne11 - 1;
    const T0 *ga = (const T0 *)(A + arow * nb01);
    const float *gb = (const float *)(Bm + brow * nb11);
    RA ra; float4 rb0, rb1;
    auto fetch = [&](int64_t k0) {                                   // elements past np are never used by the main loop: read them as zero
        if constexpr (F32) ra = k0 + fac < np ? *(const float4 *)(ga + k0 + fac) : make_float4(0.f, 0.f, 0.f, 0.f);
        else ra = k0 + fac < np ? *(const uint2 *)(ga + k0 + fac) : make_uint2(0u, 0u);
        rb0 = k0 + fbc < np ? *(const float4 *)(gb + k0 + fbc) : make_float4(0.f, 0.f, 0.f, 0.f);
        rb1 = k0 + 32 + fbc < np ? *(const float4 *)(gb + k0 + 32 + fbc) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto r16 = [](float v) { if constexpr (F32) return v; else return __half2float(__float2half_rn(v)); };
    auto stash = [&](int buf) {
        if constexpr (F32) {
            *(float4 *)&sa[buf][far][fac] = ra;
        } else {
            const __half2 h0 = *(const __half2 *)&ra.x, h1 = *(const __half2 *)&ra.y;
            const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
            *(float4 *)&sa[buf][far][fac] = make_float4(f0.x, f0.y, f1.x, f1.y);
        }
        *(float4 *)&sb[buf][fbr][fbc] = make_float4(r16(rb0.x), r16(rb0.y), r16(rb0.z), r16(rb0.w));
        *(float4 *)&sb[buf][fbr][32 + fbc] = make_float4(r16(rb1.x), r16(rb1.y), r16(rb1.z), r16(rb1.w));
    };

    float acc[2][4][8];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int e = 0; e < 8; e++) acc[i][j][e] = 0.f;

    const int nchunks = (int)((np + FT_K - 1) / FT_K);
    if (nchunks > 0) { fetch(0); stash(0); }
    __syncthreads();
    for (int c = 0; c < nchunks; c++) {
        const int buf = c & 1;
        if (c + 1 < nchunks) fetch((int64_t)(c + 1) * FT_K);
        const int steps = np - (int64_t)c * FT_K >= FT_K ? 2 : 1;    // np is a multiple of 32
#pragma unroll
        for (int st = 0; st < 2; st++) {
            if (st >= steps) break;
            float4 av[2][2], bv[4][2];
#pragma unroll
            for (int i = 0; i < 2; i++) { av[i][0] = *(const float4 *)&sa[buf][2 * ap + i][st * 32 + 4 * u]; av[i][1] = *(const float4 *)&sa[buf][2 * ap + i][st * 32 + 16 + 4 * u]; }
#pragma unroll
            for (int j = 0; j < 4; j++) { bv[j][0] = *(const float4 *)&sb[buf][4 * bq + j][st * 32 + 4 * u]; bv[j][1] = *(const float4 *)&sb[buf][4 * bq + j][st * 32 + 16 + 4 * u]; }
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    float *a = acc[i][j];
                    a[0] = __fmaf_rn(av[i][0].x, bv[j][0].x, a[0]); a[1] = __fmaf_rn(av[i][0].y, bv[j][0].y, a[1]);
                    a[2] = __fmaf_rn(av[i][0].z, bv[j][0].z, a[2]); a[3] = __fmaf_rn(av[i][0].w, bv[j][0].w, a[3]);
                    a[4] = __fmaf_rn(av[i][1].x, bv[j][1].x, a[4]); a[5] = __fmaf_rn(av[i][1].y, bv[j][1].y, a[5]);
                    a[6] = __fmaf_rn(av[i][1].z, bv[j][1].z, a[6]); a[7] = __fmaf_rn(av[i][1].w, bv[j][1].w, a[7]);
                }
        }
        if (c + 1 < nchunks) stash(buf ^ 1);
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            float *a = acc[i][j];
            float r[4];
#pragma unroll
            for (int e = 0; e < 4; e++) r[e] = __fadd_rn(a[e], a[e + 4]);                                        // chain l += chain l + 16
#pragma unroll
            for (int e = 0; e < 4; e++) r[e] = __fadd_rn(r[e], __shfl_xor_sync(0xffffffffu, r[e], 2));             // l += l + 8   (valid in u = 0, 1)
#pragma unroll
            for (int e = 0; e < 4; e++) r[e] = __fadd_rn(r[e], __shfl_xor_sync(0xffffffffu, r[e], 1));             // l += l + 4   (valid in u = 0)
            const float s = __fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3]));                               // the two hadds
            const int64_t i0 = a0 + 2 * ap + i, i1 = b0 + 4 * bq + j;
            if (u == 0 && i0 < ne01 && i1 < ne11 && !(causal_past >= 0 && i0 > causal_past + i1)) {
                float out;
                if constexpr (F32) {
                    const float *al = (const float *)(A + i0 * nb01), *bl = (const float *)(Bm + i1 * nb11);
                    out = f32_leftovers(s, (int)(ne00 - np), [&](int k) { return al[np + k]; }, [&](int k) { return bl[np + k]; });
                } else {
                    double sumf = (double)s;
                    if (np < ne00) {                                                                               // leftovers: double += (double)(f32 product)
                        const __half *al = (const __half *)(A + i0 * nb01);
                        const float *bl = (const float *)(Bm + i1 * nb11);
                        for (int64_t k = np; k < ne00; ++k) sumf += (double)__fmul_rn(__half2float(al[k]), r16(bl[k]));
                    }
                    out = (float)sumf;
                }
                *(float *)(dst + i2 * nbd2 + i1 * nbd1 + i0 * 4) = out;
            }
        }
}
__global__ void __launch_bounds__(FT_THREADS) mul_mat_f16_tiled_kernel(const char *__restrict__ src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                                                                       const char *__restrict__ src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                                                                       char *__restrict__ dst, int64_t nbd1, int64_t nbd2, int causal_past) {
    mul_mat_attn_tiled<false>(src0, ne00, ne01, ne02, nb01, nb02, src1, ne11, ne12, nb11, nb12, dst, nbd1, nbd2, causal_past,
                              blockIdx.x, blockIdx.y, blockIdx.z);
}
// (FT_THREADS, 1): without the one-CTA hint ptxas caps the f32 form at 128 registers and spills 24 bytes inside the main loop; it needs 145
__global__ void __launch_bounds__(FT_THREADS, 1) mul_mat_f32_tiled_kernel(const char *__restrict__ src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                                                                       const char *__restrict__ src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                                                                       char *__restrict__ dst, int64_t nbd1, int64_t nbd2, int causal_past) {
    mul_mat_attn_tiled<true>(src0, ne00, ne01, ne02, nb01, nb02, src1, ne11, ne12, nb11, nb12, dst, nbd1, nbd2, causal_past,
                              blockIdx.x, blockIdx.y, blockIdx.z);
}

// the tiled kernel wants src0 rows aligned to its 4-element loads (8 bytes f16, 16 bytes f32) and 16-byte aligned src1 rows; a handful of src1
// rows is cheaper one warp per dot
template <bool F32>
static void mul_mat_attn(const void *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                         const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                         float *dst, int64_t nbd1, int64_t nbd2, int causal_past, cudaStream_t st) {
    if (ne01 == 0 || ne11 == 0 || ne12 == 0) return;
    B200_ASSERT(ne12 % ne02 == 0 && ne11 <= 65535 && ne12 <= 65535);
    const int64_t al = F32 ? 16 : 8;
    const bool aligned = ((uintptr_t)src0 % al == 0) && nb01 % al == 0 && nb02 % al == 0 && ((uintptr_t)src1 % 16 == 0) && nb11 % 16 == 0 && nb12 % 16 == 0;
    if (ne11 >= 8 && aligned) {
        dim3 grid((unsigned)((ne01 + FT_A - 1) / FT_A), (unsigned)((ne11 + FT_B - 1) / FT_B), (unsigned)ne12);
        (F32 ? mul_mat_f32_tiled_kernel : mul_mat_f16_tiled_kernel)<<<grid, FT_THREADS, 0, st>>>((const char *)src0, ne00, ne01, ne02, nb01, nb02, (const char *)src1, ne11,
                                                                                                ne12, nb11, nb12, (char *)dst, nbd1, nbd2, causal_past);
    } else {
        dim3 grid((unsigned)((ne01 + F16X_WARPS - 1) / F16X_WARPS), (unsigned)ne11, (unsigned)ne12);
        (F32 ? mul_mat_f32_exact_kernel : mul_mat_f16_exact_kernel)<<<grid, F16X_WARPS * 32, 0, st>>>((const char *)src0, ne00, ne01, ne02, nb01, nb02, (const char *)src1,
                                                                                                      ne11, ne12, nb11, nb12, (char *)dst, nbd1, nbd2, causal_past);
    }
    B200_CHECK(cudaGetLastError());
}

void mul_mat_f16_exact(const __half *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                       const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                       float *dst, int64_t nbd1, int64_t nbd2, int causal_past, cudaStream_t st) {
    mul_mat_attn<false>(src0, ne00, ne01, ne02, nb01, nb02, src1, ne11, ne12, nb11, nb12, dst, nbd1, nbd2, causal_past, st);
}

void mul_mat_f32_exact(const float *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                       const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                       float *dst, int64_t nbd1, int64_t nbd2, int causal_past, cudaStream_t st) {
    mul_mat_attn<true>(src0, ne00, ne01, ne02, nb01, nb02, src1, ne11, ne12, nb11, nb12, dst, nbd1, nbd2, causal_past, st);
}

// ---- the same two mat-muls for a batched step: each chunk on its own cache and positions (kernels.cuh: BatchStep) ----------------------------
// Warp form: row warp[blockIdx.z] of the step, one output per warp, as mul_mat_f16_exact_kernel / mul_mat_f32_exact_kernel with one src1 row:
// the same dot, chains, tree and leftovers.  KQ: grid (max_n_kv / 8, n_head, n_warp); outputs past the row's pos exit at once.
template <bool F32>
__global__ void __launch_bounds__(F16X_WARPS * 32) attn_kq_rows_kernel(const BatchRow *__restrict__ rows, const int32_t *__restrict__ warp, size_t layer_off,
                                                                       const float *__restrict__ q, int64_t q_ld, int64_t q_hs, int hd, int n_head, int n_head_kv,
                                                                       int n_ctx, float *__restrict__ kq) {
    constexpr int64_t es = F32 ? 4 : 2;
    const int64_t gqa = (int64_t)n_head_kv * hd;
    const int z = warp[blockIdx.z];
    const BatchRow &r = rows[z];
    const char *K = (const char *)r.K + layer_off * es;
    mul_mat_attn_warp<F32>(K, hd, r.n_kv, n_head_kv, gqa * es, hd * es, (const char *)(q + z * q_ld), 1, n_head, 0, q_hs * 4,
                           (char *)(kq + (int64_t)z * n_head * n_ctx), 0, (int64_t)n_ctx * 4, r.pos,
                           blockIdx.x, 0, blockIdx.y);
}
// KQV: grid (hd / 8, n_head, n_warp); out row z holds the merged heads [n_head][hd]
template <bool F32>
__global__ void __launch_bounds__(F16X_WARPS * 32) attn_kqv_rows_kernel(const BatchRow *__restrict__ rows, const int32_t *__restrict__ warp, size_t layer_off,
                                                                        const float *__restrict__ kq, int hd, int n_head, int n_head_kv, int n_ctx,
                                                                        float *__restrict__ out, int64_t ld_out) {
    constexpr int64_t es = F32 ? 4 : 2;
    const int z = warp[blockIdx.z];
    const BatchRow &r = rows[z];
    const char *V = (const char *)r.V + layer_off * es;
    mul_mat_attn_warp<F32>(V, r.n_kv, hd, n_head_kv, (int64_t)n_ctx * es, (int64_t)n_ctx * hd * es, (const char *)(kq + (int64_t)z * n_head * n_ctx),
                           1, n_head, 0, (int64_t)n_ctx * 4, (char *)(out + z * ld_out), 0, (int64_t)hd * 4, -1,
                           blockIdx.x, 0, blockIdx.y);
}

// Tiled form: tile {chunk, query tile} = tiles[blockIdx.y], each chunk addressed as its single evaluate addresses its own buffers -- its cache at
// layer_off, its q rows inside the step's qkv rows, its kq rows n_head * n_ctx apart, causal_past = n_past -- with the step's kq layout
// [rows][n_head][n_ctx] and merged output rows.  KQ: grid (max_n_kv / 16, n_tiles, n_head); tiles past the chunk's n_kv exit at once, as do
// whole tiles above the diagonal.
template <bool F32>
__device__ __forceinline__ void attn_kq_tile(const BatchChunk *__restrict__ chunks, const int2 *__restrict__ tiles, size_t layer_off, const float *__restrict__ q,
                                             int64_t q_ld, int64_t q_hs, int hd, int n_head, int n_head_kv, int n_ctx, float *__restrict__ kq) {
    constexpr int64_t es = F32 ? 4 : 2;
    const int2 t = tiles[blockIdx.y];
    const BatchChunk c = chunks[t.x];
    const int64_t n_kv = (int64_t)c.n_past + c.n, gqa = (int64_t)n_head_kv * hd;
    if ((int64_t)blockIdx.x * FT_A >= n_kv) return;                      // the whole CTA: before the tile's first barrier
    mul_mat_attn_tiled<F32>((const char *)c.K + layer_off * es, hd, n_kv, n_head_kv, gqa * es, hd * es,
                            (const char *)(q + (int64_t)c.row0 * q_ld), c.n, n_head, q_ld * 4, q_hs * 4,
                            (char *)(kq + (int64_t)c.row0 * n_head * n_ctx), (int64_t)n_head * n_ctx * 4, (int64_t)n_ctx * 4, c.n_past,
                            blockIdx.x, (unsigned)t.y, blockIdx.z);
}
// KQV: grid (hd / 16, n_tiles, n_head); the dot runs over the chunk's n_kv columns
template <bool F32>
__device__ __forceinline__ void attn_kqv_tile(const BatchChunk *__restrict__ chunks, const int2 *__restrict__ tiles, size_t layer_off, const float *__restrict__ kq,
                                              int hd, int n_head, int n_head_kv, int n_ctx, float *__restrict__ out, int64_t ld_out) {
    constexpr int64_t es = F32 ? 4 : 2;
    const int2 t = tiles[blockIdx.y];
    const BatchChunk c = chunks[t.x];
    mul_mat_attn_tiled<F32>((const char *)c.V + layer_off * es, (int64_t)c.n_past + c.n, hd, n_head_kv, (int64_t)n_ctx * es, (int64_t)n_ctx * hd * es,
                            (const char *)(kq + (int64_t)c.row0 * n_head * n_ctx), c.n, n_head, (int64_t)n_head * n_ctx * 4, (int64_t)n_ctx * 4,
                            (char *)(out + (int64_t)c.row0 * ld_out), ld_out * 4, (int64_t)hd * 4, -1,
                            blockIdx.x, (unsigned)t.y, blockIdx.z);
}
// the launch bounds of mul_mat_f16_tiled_kernel / mul_mat_f32_tiled_kernel (the f32 form needs the one-CTA hint not to spill)
__global__ void __launch_bounds__(FT_THREADS) attn_kq_tiles_f16_kernel(const BatchChunk *__restrict__ chunks, const int2 *__restrict__ tiles, size_t layer_off,
                                                                       const float *__restrict__ q, int64_t q_ld, int64_t q_hs, int hd, int n_head, int n_head_kv,
                                                                       int n_ctx, float *__restrict__ kq) {
    attn_kq_tile<false>(chunks, tiles, layer_off, q, q_ld, q_hs, hd, n_head, n_head_kv, n_ctx, kq);
}
__global__ void __launch_bounds__(FT_THREADS, 1) attn_kq_tiles_f32_kernel(const BatchChunk *__restrict__ chunks, const int2 *__restrict__ tiles, size_t layer_off,
                                                                          const float *__restrict__ q, int64_t q_ld, int64_t q_hs, int hd, int n_head, int n_head_kv,
                                                                          int n_ctx, float *__restrict__ kq) {
    attn_kq_tile<true>(chunks, tiles, layer_off, q, q_ld, q_hs, hd, n_head, n_head_kv, n_ctx, kq);
}
__global__ void __launch_bounds__(FT_THREADS) attn_kqv_tiles_f16_kernel(const BatchChunk *__restrict__ chunks, const int2 *__restrict__ tiles, size_t layer_off,
                                                                        const float *__restrict__ kq, int hd, int n_head, int n_head_kv, int n_ctx,
                                                                        float *__restrict__ out, int64_t ld_out) {
    attn_kqv_tile<false>(chunks, tiles, layer_off, kq, hd, n_head, n_head_kv, n_ctx, out, ld_out);
}
__global__ void __launch_bounds__(FT_THREADS, 1) attn_kqv_tiles_f32_kernel(const BatchChunk *__restrict__ chunks, const int2 *__restrict__ tiles, size_t layer_off,
                                                                           const float *__restrict__ kq, int hd, int n_head, int n_head_kv, int n_ctx,
                                                                           float *__restrict__ out, int64_t ld_out) {
    attn_kqv_tile<true>(chunks, tiles, layer_off, kq, hd, n_head, n_head_kv, n_ctx, out, ld_out);
}

// mul_mat_attn's alignment test on a chunk's KQ (K rows gqa apart, q rows q_ld apart, heads hd / q_hs apart) and KQV (V rows n_ctx apart, kq rows
// n_head * n_ctx apart, heads n_ctx apart), for both cache types and every chunk's first row: the buffers themselves are cudaMalloc'd
bool attn_tiles_aligned(int hd, int64_t q_ld, int64_t q_hs, int n_ctx) {
    return hd % 4 == 0 && q_ld % 4 == 0 && q_hs % 4 == 0 && n_ctx % 4 == 0;
}

int attn_kq_step(const BatchStep &p, size_t layer_off, const float *q, int64_t q_ld, int64_t q_hs, int hd, int n_head, int n_head_kv, int n_ctx,
                 float *kq, cudaStream_t st) {
    B200_ASSERT(p.n_warp <= 65535 && p.n_tiles <= 65535 && n_head <= 65535 && n_head % n_head_kv == 0);
    const bool f32 = p.kv_type == T_F32;
    int L = 0;
    if (p.n_warp) {
        const dim3 grid((unsigned)((p.max_n_kv_warp + F16X_WARPS - 1) / F16X_WARPS), (unsigned)n_head, (unsigned)p.n_warp);
        (f32 ? attn_kq_rows_kernel<true> : attn_kq_rows_kernel<false>)<<<grid, F16X_WARPS * 32, 0, st>>>(p.rows, p.warp, layer_off, q, q_ld, q_hs, hd, n_head,
                                                                                                         n_head_kv, n_ctx, kq);
        B200_CHECK(cudaGetLastError()); L++;
    }
    if (p.n_tiles) {
        const dim3 grid((unsigned)((p.max_n_kv_tiles + FT_A - 1) / FT_A), (unsigned)p.n_tiles, (unsigned)n_head);
        (f32 ? attn_kq_tiles_f32_kernel : attn_kq_tiles_f16_kernel)<<<grid, FT_THREADS, 0, st>>>(p.chunks, p.tiles, layer_off, q, q_ld, q_hs, hd, n_head, n_head_kv,
                                                                                                n_ctx, kq);
        B200_CHECK(cudaGetLastError()); L++;
    }
    return L;
}

int attn_kqv_step(const BatchStep &p, size_t layer_off, const float *kq, int hd, int n_head, int n_head_kv, int n_ctx, float *out, int64_t ld_out,
                  cudaStream_t st) {
    B200_ASSERT(p.n_warp <= 65535 && p.n_tiles <= 65535 && n_head <= 65535 && n_head % n_head_kv == 0);
    const bool f32 = p.kv_type == T_F32;
    int L = 0;
    if (p.n_warp) {
        const dim3 grid((unsigned)((hd + F16X_WARPS - 1) / F16X_WARPS), (unsigned)n_head, (unsigned)p.n_warp);
        (f32 ? attn_kqv_rows_kernel<true> : attn_kqv_rows_kernel<false>)<<<grid, F16X_WARPS * 32, 0, st>>>(p.rows, p.warp, layer_off, kq, hd, n_head, n_head_kv,
                                                                                                           n_ctx, out, ld_out);
        B200_CHECK(cudaGetLastError()); L++;
    }
    if (p.n_tiles) {
        const dim3 grid((unsigned)((hd + FT_A - 1) / FT_A), (unsigned)p.n_tiles, (unsigned)n_head);
        (f32 ? attn_kqv_tiles_f32_kernel : attn_kqv_tiles_f16_kernel)<<<grid, FT_THREADS, 0, st>>>(p.chunks, p.tiles, layer_off, kq, hd, n_head, n_head_kv, n_ctx,
                                                                                                  out, ld_out);
        B200_CHECK(cudaGetLastError()); L++;
    }
    return L;
}

}  // namespace b200
