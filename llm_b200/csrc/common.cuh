// llm_b200/csrc/common.cuh -- shared device/host helpers for the H100 (sm_90a) ggml backend.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

// Error behaviour mirrors the reference backend: print and exit(1) (LC/ggml-cuda.cu:24-32). No fallback.
#define B200_CHECK(expr)                                                                                   \
    do {                                                                                                   \
        cudaError_t err_ = (expr);                                                                         \
        if (err_ != cudaSuccess) {                                                                         \
            fprintf(stderr, "llm_b200: CUDA error %d (%s) at %s:%d: %s\n", (int)err_, cudaGetErrorName(err_), \
                    __FILE__, __LINE__, cudaGetErrorString(err_));                                         \
            exit(1);                                                                                       \
        }                                                                                                  \
    } while (0)

#define B200_ASSERT(cond)                                                                         \
    do {                                                                                          \
        if (!(cond)) {                                                                            \
            fprintf(stderr, "llm_b200: assertion failed at %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            abort();                                                                              \
        }                                                                                         \
    } while (0)

namespace b200 {

// enum ggml_type values (LC/ggml.h:262-285)
enum : int { T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q8_1 = 9, T_Q2_K = 10, T_Q3_K = 11, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14,
              T_Q8_K = 15, T_I8 = 16, T_I16 = 17, T_I32 = 18 };

constexpr int QK = 32;  // elements per quant block for all five formats (LC/ggml.c:895-940)

__host__ __device__ inline bool is_quant(int t) { return t == T_Q4_0 || t == T_Q4_1 || t == T_Q5_0 || t == T_Q5_1 || t == T_Q8_0; }
// K-quants with kernels here (kquants.cu): 256-element super-blocks kept in HBM exactly as GGML lays them out (LC/k_quants.h:60-110)
__host__ __device__ inline bool is_kquant(int t) { return t >= T_Q2_K && t <= T_Q6_K; }
__host__ __device__ inline int kquant_block_bytes(int t) { return t == T_Q2_K ? 84 : t == T_Q3_K ? 110 : t == T_Q4_K ? 144 : t == T_Q5_K ? 176 : t == T_Q6_K ? 210 : 0; }
// bytes per GGML block as laid out in files / host memory
__host__ __device__ inline int ggml_block_bytes(int t) {
    switch (t) { case T_Q4_0: return 18; case T_Q4_1: return 20; case T_Q5_0: return 22; case T_Q5_1: return 24; case T_Q8_0: return 34; case T_Q8_1: return 40;
                 case T_Q2_K: return 84; case T_Q3_K: return 110; case T_Q4_K: return 144; case T_Q5_K: return 176; case T_Q6_K: return 210; case T_Q8_K: return 292; }
    return 0;
}
__host__ __device__ inline size_t ggml_type_size(int t) {  // bytes per block (block = 1 element for scalar types)
    switch (t) { case T_F32: case T_I32: return 4; case T_F16: case T_I16: return 2; case T_I8: return 1; }
    return (size_t)ggml_block_bytes(t);
}
__host__ __device__ inline int ggml_blck_size(int t) { return (t >= T_Q2_K && t <= T_Q8_K) ? 256 : (is_quant(t) || t == T_Q8_1) ? QK : 1; }
// activation quantization format paired with each weight format (type_traits[].vec_dot_type, LC/ggml.c:1645-1737)
__host__ __device__ inline int vec_dot_type(int t) { return (t == T_Q4_1 || t == T_Q5_1) ? T_Q8_1 : T_Q8_0; }
__host__ __device__ inline bool has_min(int t) { return t == T_Q4_1 || t == T_Q5_1; }
__host__ __device__ inline bool has_qh(int t) { return t == T_Q5_0 || t == T_Q5_1; }
__host__ __device__ inline int qs_bytes(int t) { return t == T_Q8_0 ? 32 : 16; }
// types a QWeight holds: the five block formats and F16 (one plane of N rows x K halves, GGML's bytes)
inline bool is_qweight_type(int t) { return is_quant(t) || t == T_F16; }
// GGML bytes per 32 elements of a QWeight row: an F16 row counts as blocks of 32 halves
inline int qweight_block_bytes(int t) { return t == T_F16 ? 64 : ggml_block_bytes(t); }

// A quantized weight matrix resident in HBM, repacked at upload from GGML's array-of-blocks (2-byte aligned, 18..34 B
// blocks) into 16-byte aligned planes so that every access is a full 128-bit transaction and TMA boxes are legal:
//   qs : [N][nb][16] packed nibbles (Q4_x, Q5_x) or [N][nb][32] int8 (Q8_0)   -- bit-identical to GGML's qs bytes
//   qh : [N][nb] uint32 fifth bits (Q5_x)
//   dm : [N][nb] fp16 d  (Q4_0, Q5_0, Q8_0)  or  [N][nb] half2 {d, m} (Q4_1, Q5_1)
// Bytes per weight are exactly GGML's (18/20/22/24/34 per 32).  An F16 weight keeps GGML's bytes in `qs` alone ([N][K] halves, row pitch 2K,
// 16-byte aligned since K % 64 == 0); nb = K/32 then counts 64-byte groups of 32 halves, so row views and chunked loads work unchanged.
struct QWeight {
    int type = 0;
    int64_t K = 0, N = 0, nb = 0;
    const uint8_t *qs = nullptr;
    const uint32_t *qh = nullptr;
    const void *dm = nullptr;
    void *base = nullptr;  // owning allocation (planes are carved from it)
    size_t bytes = 0;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// ---- the norms' row sums, bit for bit --------------------------------------------------------------------------------------------
// ggml_compute_forward_norm_f32 / _rms_norm_f32 (LC/ggml.c:10063-10175) add a row's n terms in index order in a double (ggml_float) and keep
// only the float (float)(sum / n).  The kernels add the same terms in a tree, T.  When every sum within a bound d of T gives the float T gives,
// so does the reference's in-order sum Q: x -> (float)(x / n) is monotone.  row_sum_within checks that with both ends rounded outwards; it
// fails for inf / NaN.  Otherwise the caller adds the row again in order (row_sum_in_order).
__device__ __forceinline__ bool row_sum_within(double T, double d, int64_t n) {
    const double nd = (double)n;
    if (!(fabs(T) <= 0x1.fffffffffffffp+1023) || !(d <= 0x1.fffffffffffffp+1023)) return false;
    return (float)(__dsub_rd(T, d) / nd) == (float)(__dadd_ru(T, d) / nd);
}
// Any order of adding the terms lies within gamma_{n-1} A of the exact sum (A = sum |term|, gamma_k = k u / (1 - k u), u = 2^-53), so
// |Q - T| <= 2 gamma_{n-1} A.  Enough for sums of squares, where A = T.
__device__ __forceinline__ bool row_sum_settled(double T, double A, int64_t n) {
    return row_sum_within(T, __dmul_ru(__dmul_ru((double)n, 0x1.0001p-52), A), n);    // >= 2 gamma_{n-1} A, with room for A's own tree rounding
}
// A tighter bound for sums that cancel (norm's sum x over a row of mean ~0, where the one above fails for a few rows in a thousand): the in-order
// sum's error is at most u / (1 - u) sum_k |Q_k| over its partial sums, |Q_k| <= |P_k| + 2 gamma_n A for prefix sums P_k computed in any
// order (S = sum_k |P_k|, prefix_abs_sum), and T's own error is at most gamma_depth A, depth = the most additions on one path of its tree.
__device__ __forceinline__ double row_sum_prefix_bound(double S, double A, int64_t n, int depth) {
    const double nd = (double)n;
    const double k = __dadd_ru((double)depth, __dmul_ru(__dmul_ru(4.0 * nd, nd), 0x1p-53));
    return __dmul_ru(0x1.00001p-53, __dadd_ru(S, __dmul_ru(k, A)));
}
// sum_k |x_0 + ... + x_k| over the row, from a block scan of blockDim.x-element chunks (blockDim.x a multiple of 32, at most 1024).  Call from
// all threads, on a block-uniform branch.  Out of line: it runs only where row_sum_settled fails.
static __device__ __noinline__ double prefix_abs_sum(const float *x, int64_t n) {
    __shared__ double wsum[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    double carry = 0.0, acc = 0.0;
    for (int64_t base = 0; base < n; base += blockDim.x) {
        const int64_t i = base + threadIdx.x;
        double v = i < n ? (double)__ldcg(x + i) : 0.0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const double t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
        __syncthreads();                                        // every thread has read wsum of the previous chunk
        if (lane == 31) wsum[wid] = v;
        __syncthreads();
        double off = carry, tot = carry;
        for (int w = 0; w < nw; w++) { if (w < wid) off += wsum[w]; tot += wsum[w]; }
        if (i < n) acc += fabs(off + v);
        carry = tot;
    }
    acc = warp_sum(acc);
    __syncthreads();
    if (lane == 0) wsum[wid] = acc;
    __syncthreads();
    double S = 0.0;
    for (int w = 0; w < nw; w++) S += wsum[w];
    __syncthreads();                                            // wsum is free again
    return S;
}
// The reference's sum: term(0) + term(1) + ... + term(n-1), one after another in a double.  Out of line, so that the kernels' register
// allocation is not sized by this rarely taken loop.
template <typename Term>
__device__ __noinline__ double add_in_order(int64_t n, Term term) {
    double s = 0.0;
#pragma unroll 8
    for (int64_t i = 0; i < n; i++) s += term(i);
    return s;
}
// add_in_order on thread 0, the result to every thread of the block.  Call from all threads, on a block-uniform branch.
template <typename Term>
__device__ __forceinline__ double row_sum_in_order(int64_t n, Term term) {
    __shared__ double r;
    if (threadIdx.x == 0) r = add_in_order(n, term);
    __syncthreads();
    const double v = r;
    __syncthreads();                                            // r is free again for the next row sum
    return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// streaming 128-bit load that does not pollute L1 (weights are read exactly once per mat-vec)
__device__ __forceinline__ int4 ld_stream_int4(const void *p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ld_stream_u32(const void *p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint16_t ld_stream_u16(const void *p) {
    uint16_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return r;
}

// fp16 helpers with the reference's semantics: RNE conversion (== _cvtss_sh(x, 0), LC/ggml.c:309-317)
__device__ __forceinline__ uint16_t f32_to_f16_bits(float x) { return __half_as_ushort(__float2half_rn(x)); }
__device__ __forceinline__ float f16_bits_to_f32(uint16_t h) { return __half2float(__ushort_as_half(h)); }

// spread 4 bits b0..b3 of t to bit 4 of bytes 0..3 (Q5 fifth bits -> nibble extension)
__device__ __forceinline__ uint32_t spread4_to_bit4(uint32_t t) { return (((t & 0xFu) * 0x00204081u) & 0x01010101u) << 4; }

}  // namespace b200
