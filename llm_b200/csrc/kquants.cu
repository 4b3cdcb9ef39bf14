// llm_b200/csrc/kquants.cu -- K-quant weights Q2_K .. Q6_K (256-element super-blocks, LC/k_quants.h:28-120): bit-exact mat-mul against Q8_K activations.
//
// Serves ggml_compute_forward_mul_mat (LC/ggml.c:10397-10586) when src0 is Q2_K / Q3_K / Q4_K / Q5_K / Q6_K: type_traits[] pairs them with
// vec_dot_type = Q8_K (LC/ggml.c:1700-1737), i.e. the INIT phase runs quantize_row_q8_K on every src1 row and the COMPUTE phase calls
// ggml_vec_dot_q{2,3,4,5,6}_K_q8_K (LC/k_quants.c:1240, :1763, :2492, :3023, :3592) once per (weight row, src1 row).
//
// What "the reference's result" is (the x86 build of crates/ggml/sys/build.rs: -mavx2 -mfma -mf16c, QK_K = 256):
//   * quantize_row_q8_K_reference (LC/k_quants.c:1133-1168): the FIRST element of largest magnitude gives iscale = -128/max, q = min(127, nearest_int(iscale*x)),
//     d = 1/iscale, bsums = sums of 16.  gcc contracts nearest_int's `iscale*x + 12582912.f` into ONE fused multiply-add (default -ffp-contract=fast; verified in the
//     disassembly of oracle/_ref: vfmadd132ps) -- so does this file (__fmaf_rn); a separately rounded product differs in the last bit for ~1e-3 of the inputs.
//   * the AVX2 dot products keep 8 int32 lanes per super-block (lane L = bytes 4L..4L+3 of every 32-byte group, each group weighted by its 6-bit / 8-bit sub-block
//     scale: all integer, exact) and ONE 8-lane f32 accumulator: acc_L = fma(d, (float)sumi_L, acc_L) per super-block in order, d = y.d * fp16(x.d); the result is
//     hsum_float_8(acc) (LC/k_quants.c:1193-1199) plus the "mins" term: Q4_K keeps 4 f32 lanes acc_m[t] = fma(dmin, (float)prod[t], acc_m[t]) reduced as
//     (m0+m2)+(m1+m3) (:2618-2620, :2652-2655); Q5_K a scalar summs = fma(dmin, (float)(prod0+..+prod3), summs) (:3157-3160; contracted, vfmadd231ss);
//     Q2_K folds its mins into the SAME 8 lanes first: acc_L = fma(dmin, (float)(m[2L] bsums[2L] + m[2L+1] bsums[2L+1]), acc_L) (:1346-1350).
// lane = 8*part + L owns byte column L of two of the eight 32-byte groups; the integer partials meet by shuffles, every lane then carries the f32
// chain of its L (kq_lanes.cuh).  Two kernels, chosen by the batch size: below 32 tokens (decode included) one warp per (weight row, token); from
// 32 tokens on a tiled GEMM that stages 8 weight rows' super-blocks and 32 tokens' Q8_K blocks in shared memory once per super-block index.
#include "kq_lanes.cuh"

namespace b200 {

namespace {

using kq::QKK;
using kq::BlockQ8K;

__device__ __forceinline__ int nearest_int_fma(float a, float b) {        // nearest_int(a*b) of LC/k_quants.c:36-42 as compiled (see the header)
    const float val = __fmaf_rn(a, b, 12582912.f);
    return (__float_as_int(val) & 0x007fffff) - 0x00400000;
}

// one warp per super-block; lane holds elements 8*lane .. 8*lane+7
__global__ void __launch_bounds__(128) quantize_q8k_kernel(const float *__restrict__ x, int64_t ldx, BlockQ8K *__restrict__ y, int64_t nsb, int64_t total) {
    const int lane = threadIdx.x & 31;
    const int64_t gw = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (gw >= total) return;
    const int64_t row = gw / nsb, sb = gw % nsb;
    const float *src = x + row * ldx + sb * QKK + lane * 8;
    float v[8];
    *(float4 *)&v[0] = *(const float4 *)src; *(float4 *)&v[4] = *(const float4 *)(src + 4);
    float amax = 0.f, mx = 0.f;
    int idx = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { const float ax = fabsf(v[j]); if (ax > amax) { amax = ax; mx = v[j]; idx = lane * 8 + j; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {                                   // largest magnitude, ties to the lower index (the scalar loop's strict `>`)
        const float oa = __shfl_xor_sync(0xffffffffu, amax, o), om = __shfl_xor_sync(0xffffffffu, mx, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (oa > amax || (oa == amax && oi < idx)) { amax = oa; mx = om; idx = oi; }
    }
    BlockQ8K *yb = y + gw;
    int q[8];
    float d = 0.f;
    if (amax == 0.f) {
#pragma unroll
        for (int j = 0; j < 8; j++) q[j] = 0;
    } else {
        const float iscale = __fdiv_rn(-128.f, mx);
#pragma unroll
        for (int j = 0; j < 8; j++) { const int t = nearest_int_fma(iscale, v[j]); q[j] = t < 127 ? t : 127; }
        d = __fdiv_rn(1.f, iscale);
    }
    int s8 = 0;
    uint32_t w0 = 0, w1 = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) { s8 += q[j] + q[j + 4]; w0 |= (uint32_t)(q[j] & 0xff) << (8 * j); w1 |= (uint32_t)(q[j + 4] & 0xff) << (8 * j); }
    *(uint32_t *)(yb->qs + lane * 8) = w0; *(uint32_t *)(yb->qs + lane * 8 + 4) = w1;
    const int s16 = s8 + __shfl_xor_sync(0xffffffffu, s8, 1);
    if ((lane & 1) == 0) yb->bsums[lane >> 1] = (int16_t)s16;
    if (lane == 0) yb->d = d;
}

// ---- short batches (B < KQ_GEMM_MIN, decode included): one warp per (weight row, token) --------------------------------------------------------
// The warp walks its row's super-blocks in order through kq_load / kq_step (kq_lanes.cuh).  With N / 4 x B CTAs in flight it keeps more loads
// outstanding than a tile that reuses weights can at these batch sizes, and it is the faster kernel there (DESIGN.md §4 has the measurements).
// n_past_inc (nullable): incremented once, for a decode graph whose last node this is.
template <int TYPE>
__global__ void __launch_bounds__(128) mul_mat_kq_warp_kernel(const uint8_t *__restrict__ W, const kq::BlockQ8K *__restrict__ X, float *__restrict__ dst,
                                                              int64_t ldd, int64_t N, int nsb, const float *__restrict__ addend, int64_t lda, int *n_past_inc) {
    const int lane = threadIdx.x & 31;
    if (n_past_inc && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *n_past_inc = *n_past_inc + 1;
    const int64_t n = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5), b = blockIdx.y;
    if (n >= N) return;
    constexpr int BB = kq::Bytes<TYPE>::N;
    const uint8_t *wrow = W + n * nsb * BB;
    const kq::BlockQ8K *xrow = X + b * nsb;
    float acc = 0.f, accm = 0.f;
    for (int i = 0; i < nsb; i++) kq::kq_step<TYPE>(kq::kq_load<TYPE>(wrow + (int64_t)i * BB, lane), xrow + i, lane, acc, accm);
    const float v = kq::kq_finish<TYPE>(acc, accm);
    if (lane == 0) dst[b * ldd + n] = addend ? __fadd_rn(v, addend[b * lda + n]) : v;
}

// ---- batches of KQ_GEMM_MIN tokens and more (prefill): the tiled GEMM ------------------------------------------------------------------------------------------------------
// A CTA owns GROWS weight rows (one per warp) x GTOK token rows.  Per super-block index it stages the GROWS weight super-blocks and the GTOK Q8_K
// super-blocks in shared memory once; each warp reads its weight super-block once (kq_load) and folds it into the chains of all GTOK tokens
// (kq_step), so each weight byte serves GTOK tokens and each activation byte GROWS rows.  Every output is still one complete
// ggml_vec_dot_q*_K_q8_K in the reference's order.  The CTAs of consecutive indices take the token tiles of the same rows, so a matrix larger
// than L2 comes from HBM about once per call.
constexpr int GROWS = 8, GTOK = 32;
template <int TYPE> struct KqTile { static constexpr int PITCH = (kq::Bytes<TYPE>::N + 4 + 15) / 16 * 16; };

template <int TYPE>
__global__ void __launch_bounds__(32 * GROWS) mul_mat_kq_gemm_kernel(const uint8_t *__restrict__ W, const kq::BlockQ8K *__restrict__ X, float *__restrict__ dst,
                                                                      int64_t ldd, int64_t N, int nsb, int64_t B, int64_t ntt,
                                                                      const float *__restrict__ addend, int64_t lda) {
    constexpr int BB = kq::Bytes<TYPE>::N, PITCH = KqTile<TYPE>::PITCH;
    __shared__ __align__(16) uint8_t ws[GROWS * PITCH];
    __shared__ kq::BlockQ8K xs[GTOK];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t tt = blockIdx.x % ntt, rt = blockIdx.x / ntt;
    const int64_t n0 = rt * GROWS, b0 = tt * GTOK;
    const int nr = N - n0 < GROWS ? (int)(N - n0) : GROWS, nt = B - b0 < GTOK ? (int)(B - b0) : GTOK;
    const int64_t row_bytes = (int64_t)nsb * BB;
    float acc[GTOK], accm[GTOK];
#pragma unroll
    for (int t = 0; t < GTOK; t++) { acc[t] = 0.f; accm[t] = 0.f; }
    for (int i = 0; i < nsb; i++) {
        __syncthreads();                                                  // the previous super-block's readers are done
        // weights: row r's super-block at ws + r * PITCH + (address & 3), copied as 2-byte words (blocks are 2-byte aligned), so kq_load's 4-byte
        // reads see the alignment they have in global memory
        for (int k = threadIdx.x; k < nr * (BB / 2); k += 32 * GROWS) {
            const int r = k / (BB / 2), h = k - r * (BB / 2);
            const uint8_t *src = W + (n0 + r) * row_bytes + (int64_t)i * BB;
            ((uint16_t *)(ws + r * PITCH + ((uintptr_t)src & 3)))[h] = ((const uint16_t *)src)[h];
        }
        for (int k = threadIdx.x; k < nt * 73; k += 32 * GROWS) {             // 73 words per block_q8_K
            const int t = k / 73, h = k - t * 73;
            ((uint32_t *)&xs[t])[h] = ((const uint32_t *)(X + (b0 + t) * nsb + i))[h];
        }
        __syncthreads();
        if (warp < nr) {
            const uint8_t *src = W + (n0 + warp) * row_bytes + (int64_t)i * BB;
            const kq::Lane w = kq::kq_load<TYPE>(ws + warp * PITCH + ((uintptr_t)src & 3), lane);
#pragma unroll
            for (int t = 0; t < GTOK; t++)
                if (t < nt) kq::kq_step<TYPE>(w, &xs[t], lane, acc[t], accm[t]);
        }
    }
    if (warp >= nr) return;
    const int64_t n = n0 + warp;
#pragma unroll
    for (int t = 0; t < GTOK; t++) {
        if (t >= nt) break;
        const float v = kq::kq_finish<TYPE>(acc[t], accm[t]);
        const int64_t b = b0 + t;
        if (lane == 0) dst[b * ldd + n] = addend ? __fadd_rn(v, addend[b * lda + n]) : v;
    }
}

constexpr int KQ_GEMM_MIN = 32;               // the tiled GEMM from this batch size on (one whole token tile), the warp kernel below it

template <int TYPE>
void launch_kq(const void *w_raw, const void *xq8k, float *dst, int64_t ldd, int64_t N, int64_t nsb, int64_t B, const float *addend, int64_t lda,
               int *n_past_inc, cudaStream_t st) {
    const uint8_t *w = (const uint8_t *)w_raw;
    const kq::BlockQ8K *x = (const kq::BlockQ8K *)xq8k;
    if (B < KQ_GEMM_MIN) {
        B200_ASSERT((N + 3) / 4 <= 0x7fffffffLL);
        mul_mat_kq_warp_kernel<TYPE><<<dim3((unsigned)((N + 3) / 4), (unsigned)B), 128, 0, st>>>(w, x, dst, ldd, N, (int)nsb, addend, lda, n_past_inc);
        return;
    }
    B200_ASSERT(!n_past_inc);
    const int64_t ntt = (B + GTOK - 1) / GTOK, nrt = (N + GROWS - 1) / GROWS;
    B200_ASSERT(ntt * nrt <= 0x7fffffffLL);
    mul_mat_kq_gemm_kernel<TYPE><<<(unsigned)(ntt * nrt), 32 * GROWS, 0, st>>>(w, x, dst, ldd, N, (int)nsb, B, ntt, addend, lda);
}

// ---- get_rows: dequantize_row_q{2,3,4,5,6}_K (LC/k_quants.c:352, :531, :733, :926, :1065), one thread per element --------------------------------
// As the reference's x86 build computes them: the block scale times the sub-block scale rounded first, then Q2_K / Q4_K / Q5_K contract
// `dl * q - ml` into one fused multiply-add (vfnmadd / vfmsub in the disassembly of oracle/_ref), Q3_K has no min, Q6_K rounds (d * sc) * q twice.
template <int TYPE>
__global__ void get_rows_kq_kernel(const uint8_t *__restrict__ W, int64_t nsb, const int32_t *__restrict__ ids, float *__restrict__ dst, int64_t total) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int64_t K = nsb * QKK, i = t / K, c = t - i * K;
    const int e = (int)(c % QKK);
    const uint8_t *b = W + ((int64_t)ids[i] * nsb + c / QKK) * kq::Bytes<TYPE>::N;
    float y;
    if (TYPE == T_Q2_K || TYPE == T_Q3_K) {
        const int n = e >> 7, r = e & 127, j = r >> 5, l = r & 31, is = 8 * n + 2 * j + (l >> 4);
        const int q = (b[(TYPE == T_Q2_K ? 16 : 32) + 32 * n + l] >> (2 * j)) & 3;
        if (TYPE == T_Q2_K) {
            const float dl = __fmul_rn(kq::h2f(b + 80), (float)(b[is] & 0xF)), ml = __fmul_rn(kq::h2f(b + 82), (float)(b[is] >> 4));
            y = __fmaf_rn(dl, (float)q, -ml);
        } else {
            const float dl = __fmul_rn(kq::h2f(b + 108), (float)kq::k3_scale(b + 96, is));
            y = __fmul_rn(dl, (float)(q - ((b[l] >> (4 * n + j)) & 1 ? 0 : 4)));
        }
    } else if (TYPE == T_Q6_K) {
        const int n = e >> 7, r = e & 127, g = r >> 5, l = r & 31;
        const int lo = (b[64 * n + l + 32 * (g & 1)] >> (4 * (g >> 1))) & 0xF;
        const int q = (lo | (((b[128 + 32 * n + l] >> (2 * g)) & 3) << 4)) - 32;
        const int sc = ((const int8_t *)(b + 192))[8 * n + (l >> 4) + 2 * g];
        y = __fmul_rn(__fmul_rn(kq::h2f(b + 208), (float)sc), (float)q);
    } else {
        const int j = e >> 6, hi = (e >> 5) & 1, l = e & 31, is = 2 * j + hi;
        int q = (b[kq::Bytes<TYPE>::QS + 32 * j + l] >> (4 * hi)) & 0xF;
        if (TYPE == T_Q5_K) q += (b[16 + l] >> is) & 1 ? 16 : 0;
        const float d1 = __fmul_rn(kq::h2f(b), (float)kq::k4_scale(b + 4, is)), m1 = __fmul_rn(kq::h2f(b + 2), (float)kq::k4_min(b + 4, is));
        y = __fmaf_rn(d1, (float)q, -m1);
    }
    dst[t] = y;
}

}  // namespace

size_t q8k_bytes(int64_t K, int64_t B) { return (size_t)B * (size_t)(K / QKK) * sizeof(BlockQ8K); }

void quantize_act_q8k(const float *x, int64_t ldx, void *y, int64_t K, int64_t B, cudaStream_t st) {
    B200_ASSERT(K % QKK == 0 && ldx % 4 == 0 && ((uintptr_t)x & 15) == 0);
    const int64_t nsb = K / QKK, total = nsb * B;
    if (!total) return;
    quantize_q8k_kernel<<<(unsigned)((total + 3) / 4), 128, 0, st>>>(x, ldx, (BlockQ8K *)y, nsb, total);
    B200_CHECK(cudaGetLastError());
}

void mul_mat_kq_exact(int type, const void *w_raw, const void *xq8k, float *dst, int64_t ldd, int64_t K, int64_t N, int64_t B, const float *addend, int64_t lda,
                      cudaStream_t st, int *n_past_inc) {
    B200_ASSERT(is_kquant(type) && K % QKK == 0);
    if (!N || !B) return;
    const int64_t nsb = K / QKK;
    switch (type) {
        case T_Q2_K: launch_kq<T_Q2_K>(w_raw, xq8k, dst, ldd, N, nsb, B, addend, lda, n_past_inc, st); break;
        case T_Q3_K: launch_kq<T_Q3_K>(w_raw, xq8k, dst, ldd, N, nsb, B, addend, lda, n_past_inc, st); break;
        case T_Q4_K: launch_kq<T_Q4_K>(w_raw, xq8k, dst, ldd, N, nsb, B, addend, lda, n_past_inc, st); break;
        case T_Q5_K: launch_kq<T_Q5_K>(w_raw, xq8k, dst, ldd, N, nsb, B, addend, lda, n_past_inc, st); break;
        case T_Q6_K: launch_kq<T_Q6_K>(w_raw, xq8k, dst, ldd, N, nsb, B, addend, lda, n_past_inc, st); break;
        default: B200_ASSERT(!"mul_mat_kq_exact: type");
    }
    B200_CHECK(cudaGetLastError());
}

void get_rows_kq(int type, const void *w_raw, int64_t K, const int32_t *ids, float *dst, int64_t n, cudaStream_t st) {
    B200_ASSERT(is_kquant(type) && K % QKK == 0);
    const int64_t total = n * K, nsb = K / QKK;
    if (!total) return;
    const unsigned grid = (unsigned)((total + 255) / 256);
    const uint8_t *w = (const uint8_t *)w_raw;
    switch (type) {
        case T_Q2_K: get_rows_kq_kernel<T_Q2_K><<<grid, 256, 0, st>>>(w, nsb, ids, dst, total); break;
        case T_Q3_K: get_rows_kq_kernel<T_Q3_K><<<grid, 256, 0, st>>>(w, nsb, ids, dst, total); break;
        case T_Q4_K: get_rows_kq_kernel<T_Q4_K><<<grid, 256, 0, st>>>(w, nsb, ids, dst, total); break;
        case T_Q5_K: get_rows_kq_kernel<T_Q5_K><<<grid, 256, 0, st>>>(w, nsb, ids, dst, total); break;
        case T_Q6_K: get_rows_kq_kernel<T_Q6_K><<<grid, 256, 0, st>>>(w, nsb, ids, dst, total); break;
        default: B200_ASSERT(!"get_rows_kq: type");
    }
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
