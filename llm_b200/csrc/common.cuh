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
