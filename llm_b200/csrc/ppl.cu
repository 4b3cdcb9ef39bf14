// llm_b200/csrc/ppl.cu -- the per-row arithmetic of InferenceSession::perplexity (crates/llm-base/src/inference_session.rs:514-589) on logits in HBM.
//
// For a scored row l of n_vocab logits and its target t the reference computes (util::softmax, crates/llm-base/src/util.rs:143-151)
//   max = fold(-inf, f32::max), sum = sum of (v - max).exp() over the row, LEFT TO RIGHT in f32 from 0, p = (l[t] - max).exp() / sum,
// and adds -p.ln() to an f32 nll that runs over every chunk.  exp and ln are glibc's expf / logf (libm_f32.h restates them bit for bit).
//
// nll_rows_kernel: one CTA of 8 warps per row, every row of the batch at once.  The max is order-free (fmaxf is exact); the sum is a chain of
// n_vocab dependent adds and must stay one: the threads compute tiles of expf values into shared memory and thread 0 adds them in index order,
// one tile behind the others so that the expf work of the next tile hides under its adds.
// nll_fold_kernel: one thread folds a chunk's terms into the running nll / count in position order and writes expf(nll / count).
#include "kernels.cuh"
#include "libm_f32.h"

namespace b200 {

namespace {

constexpr int NLL_THREADS = 256;      // one CTA (8 warps) per row
constexpr int NLL_TILE = 2048;        // expf values staged per step, double-buffered; thread 0's in-order adds are the row's critical path

__device__ __forceinline__ float neg(float x) { return __uint_as_float(__float_as_uint(x) ^ 0x80000000u); }   // -x, also for +-0

// expf(l[j0 + j] - mx) for j in [0, n) into e, by the threads [t0, NLL_THREADS)
__device__ __forceinline__ void exp_tile(const float *__restrict__ l, int64_t j0, int n, float mx, float *e, int t0) {
    for (int j = threadIdx.x - t0; j < n; j += NLL_THREADS - t0) e[j] = lm_expf(__fsub_rn(l[j0 + j], mx));
}

__global__ void __launch_bounds__(NLL_THREADS) nll_rows_kernel(const float *__restrict__ logits, int64_t n_vocab, const int32_t *__restrict__ targets,
                                                               float *__restrict__ terms) {
    __shared__ __align__(16) float e[2][NLL_TILE];
    __shared__ float wmax[NLL_THREADS / 32];
    const int tid = threadIdx.x;
    const float *l = logits + (int64_t)blockIdx.x * n_vocab;
    float mx = -INFINITY;
    for (int64_t j = tid; j < n_vocab; j += NLL_THREADS) mx = fmaxf(mx, l[j]);
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) wmax[tid >> 5] = mx;
    __syncthreads();
    for (int w = 0; w < NLL_THREADS / 32; w++) mx = fmaxf(mx, wmax[w]);       // fmaxf is exact: any order gives the row's max
    // tile 0 by every thread; then, while thread 0 adds tile t in index order, warps 1.. compute tile t + 1 into the other buffer
    const int64_t n_tiles = (n_vocab + NLL_TILE - 1) / NLL_TILE;
    exp_tile(l, 0, (int)min((int64_t)NLL_TILE, n_vocab), mx, e[0], 0);
    __syncthreads();
    float sum = 0.0f;
    for (int64_t t = 0; t < n_tiles; t++) {
        if (t + 1 < n_tiles && tid >= 32) {
            const int64_t j1 = (t + 1) * NLL_TILE;
            exp_tile(l, j1, (int)min((int64_t)NLL_TILE, n_vocab - j1), mx, e[(t + 1) & 1], 32);
        }
        if (tid == 0) {
            const int n = (int)min((int64_t)NLL_TILE, n_vocab - t * NLL_TILE);
            const float *b = e[t & 1];
            const float4 *b4 = (const float4 *)b;
            int j = 0;
            for (; j + 4 <= n; j += 4) {
                const float4 v = b4[j >> 2];
                sum = __fadd_rn(sum, v.x); sum = __fadd_rn(sum, v.y); sum = __fadd_rn(sum, v.z); sum = __fadd_rn(sum, v.w);
            }
            for (; j < n; j++) sum = __fadd_rn(sum, b[j]);
        }
        __syncthreads();
    }
    if (tid == 0) {
        const float p = __fdiv_rn(lm_expf(__fsub_rn(l[targets[blockIdx.x]], mx)), sum);
        terms[blockIdx.x] = neg(lm_logf(p));
    }
}

// state: {f32 nll, pad, i64 count} carried across chunks
__global__ void nll_fold_kernel(const float *__restrict__ terms, int64_t n, PplState *state, float *ppl) {
    float nll = state->nll;
    int64_t count = state->count;
#pragma unroll 16
    for (int64_t i = 0; i < n; i++) { nll = __fadd_rn(nll, terms[i]); count++; }
    state->nll = nll;
    state->count = count;
    *ppl = lm_expf(__fdiv_rn(nll, __ll2float_rn(count)));        // (nll / count as f32).exp()
}

}  // namespace

void nll_rows(const float *logits, int64_t rows, int64_t n_vocab, const int32_t *targets, float *terms, cudaStream_t st) {
    if (rows <= 0) return;
    nll_rows_kernel<<<(unsigned)rows, NLL_THREADS, 0, st>>>(logits, n_vocab, targets, terms);
    B200_CHECK(cudaGetLastError());
}

void nll_fold(const float *terms, int64_t n, PplState *state, float *ppl, cudaStream_t st) {
    nll_fold_kernel<<<1, 1, 0, st>>>(terms, n, state, ppl);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
