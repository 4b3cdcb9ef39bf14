// llm_b200/csrc/f32dot.cuh -- ggml_vec_dot_f32 (LC/ggml.c:2288-2323) as the reference's AVX2 build computes it, for every kernel that restates it
// (lora.cu's LoRA patch, exact.cu's f32 attention mat-mul, decode_ops.cu's f32 cache attention):
//   * 32 f32 FMA chains, chain l over the elements k = l (mod 32) below n & ~31, in order;
//   * GGML_F32x8_REDUCE (LC/ggml.c:1897-1915) on them: chains l and l + 16, then l and l + 8, then the two 128-bit halves (l and l + 4), then
//     two hadds;
//   * the leftovers (n % 32) into the FLOAT sum: the build multiplies them in vectors of 8 and then 4 and adds each rounded product in order,
//     and the last n % 4 are scalar fused multiply-adds.
#pragma once
#include "common.cuh"

namespace b200 {

// GGML_F32x8_REDUCE on the 32 chains held by one thread
__device__ __forceinline__ float f32x8_reduce(float (&c)[32]) {
#pragma unroll
    for (int l = 0; l < 16; l++) c[l] = __fadd_rn(c[l], c[l + 16]);
#pragma unroll
    for (int l = 0; l < 8; l++) c[l] = __fadd_rn(c[l], c[l + 8]);
#pragma unroll
    for (int l = 0; l < 4; l++) c[l] = __fadd_rn(c[l], c[l + 4]);
    return __fadd_rn(__fadd_rn(c[0], c[1]), __fadd_rn(c[2], c[3]));
}

// the leftovers of one dot: s (the reduced chains) plus x(i) * y(i) for i in [0, left), left < 32, in the order and rounding of the build
template <class X, class Y>
__device__ __forceinline__ float f32_leftovers(float s, int left, X &&x, Y &&y) {
    const int nv = left & ~3;
    for (int i = 0; i < nv; i++) s = __fadd_rn(s, __fmul_rn(x(i), y(i)));
    for (int i = nv; i < left; i++) s = __fmaf_rn(x(i), y(i), s);
    return s;
}

}  // namespace b200
