// llm_b200/csrc/synth.cu -- seeded synthetic weights generated directly in HBM (there are no model files here).
// Every 2-D weight ~ N(0, 1/K) is quantized with the rule of the reference's weight quantizers
// (quantize_row_q{4_0,4_1,5_0,5_1,8_0}_reference, LC/ggml.c:943-1145) straight into the planes layout; 1-D norm gains are
// 1 + 0.1 N(0,1).  The generator is a counter-based hash, so a tensor's content depends only on (seed, tensor id, element).
#include "kernels.cuh"
#include "quant_rules.cuh"

namespace b200 {

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__device__ __forceinline__ float gauss(uint64_t seed, uint64_t idx) {
    const uint64_t u = splitmix64(seed ^ (idx * 0xD1342543DE82EF95ull));
    const float u1 = ((float)(u >> 40) + 0.5f) * (1.0f / 16777216.0f);
    const float u2 = (float)((u >> 16) & 0xFFFFFFull) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

// one warp per quant block, lane j <-> element j: seeded gaussians quantized by the reference's rule (quantize_row_*_reference,
// LC/ggml.c:943-1145) straight into the planes
__global__ void __launch_bounds__(256) synth_q_kernel(QWeight w, uint64_t seed, float sigma) {
    const int64_t blk = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (blk >= w.N * w.nb) return;
    const int lane = threadIdx.x & 31;
    const float v = gauss(seed, (uint64_t)blk * 32 + lane) * sigma;
    float d, mn;
    const int q = quantize_block_ref(w.type, v, d, mn);
    if (w.type == T_Q8_0) {
        ((int8_t *)w.qs)[blk * 32 + lane] = (int8_t)q;
    } else {
        const int hi = __shfl_down_sync(0xffffffffu, q, 16);
        if (lane < 16) ((uint8_t *)w.qs)[blk * 16 + lane] = (uint8_t)((q & 0xF) | ((hi & 0xF) << 4));
        if (has_qh(w.type)) {
            const unsigned qh = __ballot_sync(0xffffffffu, (q & 0x10) != 0);
            if (lane == 0) ((uint32_t *)w.qh)[blk] = qh;
        }
    }
    if (lane == 0) {
        if (has_min(w.type)) ((__half2 *)w.dm)[blk] = __halves2half2(__float2half_rn(d), __float2half_rn(mn));
        else ((__half *)w.dm)[blk] = __float2half_rn(d);
    }
}

// F16 weights: N(0, 1/K) rounded to fp16 (RNE), element i of the matrix drawn as element i of a quantized one
__global__ void synth_f16_kernel(__half *w, int64_t n, uint64_t seed, float sigma) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] = __float2half_rn(gauss(seed, (uint64_t)i) * sigma);
}

__global__ void synth_gain_kernel(float *g, int64_t n, uint64_t seed) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) g[i] = 1.0f + 0.1f * gauss(seed, (uint64_t)i);
}

void synth_qweight(const QWeight &w, uint64_t seed, cudaStream_t st) {
    const int64_t nblk = w.N * w.nb;
    if (nblk == 0) return;
    if (w.type == T_F16) {
        const int64_t n = w.N * w.K;
        synth_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((__half *)w.qs, n, seed, 1.0f / sqrtf((float)w.K));
        B200_CHECK(cudaGetLastError());
        return;
    }
    synth_q_kernel<<<(unsigned)((nblk + 7) / 8), 256, 0, st>>>(w, seed, 1.0f / sqrtf((float)w.K));
    B200_CHECK(cudaGetLastError());
}
__global__ void scale_shift_kernel(float *p, int64_t n, float a, float b) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = p[i] * a + b;
}
void scale_shift_f32(float *p, int64_t n, float a, float b, cudaStream_t st) {
    scale_shift_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, n, a, b);
    B200_CHECK(cudaGetLastError());
}
void synth_gain(float *g, int64_t n, uint64_t seed, cudaStream_t st) {
    synth_gain_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, n, seed);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
