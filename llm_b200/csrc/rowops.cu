// llm_b200/csrc/rowops.cu -- the warp/block-reduce kernels around the mat-muls: ggml_rms_norm / ggml_norm /
// ggml_soft_max (+scale, +diag_mask_inf) / ggml_rope / silu / gelu / add / mul / scale / cpy.
//
// All of them feed an activation quantizer further down the graph, and that quantizer is discontinuous, so every
// kernel reproduces the reference's arithmetic operation for operation (SURVEY.md §7 "hard parts"):
//   * row sums in double (ggml_float, LC/ggml.c:270) -- the only freedom taken is the order of the double additions;
//   * SiLU / GELU / exp through the 64 Ki-entry fp16 tables, built here on the HOST with the same libm formulas as
//     ggml_init (LC/ggml.c:4313-4326) and uploaded once (3 x 128 KB, L2 resident);
//   * RoPE angles from a host-built table that follows the reference's sequential f32 `theta *= theta_scale`
//     recurrence and libm cosf/sinf (LC/ggml.c:11832-11897);
//   * explicit __fmul_rn/__fmaf_rn so nvcc contracts exactly where gcc -ffp-contract=fast -mfma does.
#include <math.h>

#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "kernels.cuh"

namespace b200 {

// ---- fp16 look-up tables ------------------------------------------------------------------------------------------
static uint16_t h_f32_to_f16(float f) {   // round-to-nearest-even, == _cvtss_sh(f, 0)
    uint32_t x; memcpy(&x, &f, 4);
    const uint32_t sign = (x >> 16) & 0x8000u, ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u) return (uint16_t)(sign | 0x7c00u | (ax > 0x7f800000u ? (0x0200u | ((ax >> 13) & 0x3ffu)) : 0u));
    if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);
    if (ax < 0x33000001u) return (uint16_t)sign;
    const int e = (int)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7fffffu) | 0x800000u, base = 0; int shift = 13;
    if (e < -14) shift = 13 + (-14 - e); else { base = (uint32_t)(e + 15) << 10; m &= 0x7fffffu; }
    uint32_t q = m >> shift; const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (q & 1u))) q++;
    return (uint16_t)(sign | (base + q));
}
static float h_f16_to_f32(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu; uint32_t x;
    if (e == 0) { if (m == 0) x = sign; else { int s = 0; uint32_t mm = m; while (!(mm & 0x400u)) { mm <<= 1; s++; } x = sign | ((uint32_t)(113 - s) << 23) | ((mm & 0x3ffu) << 13); } }
    else if (e == 31) x = sign | 0x7f800000u | (m << 13);
    else x = sign | ((e + 112) << 23) | (m << 13);
    float f; memcpy(&f, &x, 4); return f;
}

const Luts &luts() {
    static Luts L = {nullptr, nullptr, nullptr};
    static std::once_flag once;
    std::call_once(once, [] {
        std::vector<uint16_t> silu(1 << 16), gelu(1 << 16), ex(1 << 16);
        for (int i = 0; i < (1 << 16); ++i) {
            const float f = h_f16_to_f32((uint16_t)i);
            // ggml_gelu_f32 (LC/ggml.c:3484-3490): the inner `1.0f + A*x*x` is one fma in the reference build
            gelu[i] = h_f32_to_f16(0.5f * f * (1.0f + tanhf(0.79788456080286535587989211986876f * f * fmaf(0.044715f * f, f, 1.0f))));
            silu[i] = h_f32_to_f16(f / (1.0f + expf(-f)));     // ggml_silu_f32, LC/ggml.c:3545-3547
            ex[i]   = h_f32_to_f16(expf(f));
        }
        uint16_t *d;
        B200_CHECK(cudaMalloc(&d, 3 * (1 << 16) * sizeof(uint16_t)));
        B200_CHECK(cudaMemcpy(d, silu.data(), (1 << 17), cudaMemcpyHostToDevice));
        B200_CHECK(cudaMemcpy(d + (1 << 16), gelu.data(), (1 << 17), cudaMemcpyHostToDevice));
        B200_CHECK(cudaMemcpy(d + (2 << 16), ex.data(), (1 << 17), cudaMemcpyHostToDevice));
        B200_CHECK(cudaDeviceSynchronize());   // legacy-stream copy/memset: not ordered with our non-blocking stream, and a pageable H2D cudaMemcpy may return before its DMA lands
        L.silu = d; L.gelu = d + (1 << 16); L.exp = d + (2 << 16);
    });
    return L;
}

__device__ __forceinline__ float lut(const uint16_t *__restrict__ t, float x) { return f16_bits_to_f32(__ldg(t + f32_to_f16_bits(x))); }

// ---- block reductions (blockDim.x <= 1024) -------------------------------------------------------------------------
__device__ __forceinline__ double block_sum(double v, double *sh) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) sh[wid] = v;
    __syncthreads();
    double t = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.0;
    if (wid == 0) { t = warp_sum(t); if (lane == 0) sh[0] = t; }
    __syncthreads();
    return sh[0];
}
__device__ __forceinline__ float block_max(float v, float *sh) {
    v = warp_max(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) sh[wid] = v;
    __syncthreads();
    float t = (threadIdx.x < nw) ? sh[threadIdx.x] : -INFINITY;
    if (wid == 0) { t = warp_max(t); if (lane == 0) sh[0] = t; }
    __syncthreads();
    return sh[0];
}

// ---- rms_norm (LC/ggml.c:10129-10175) [+ mul by gain, the next graph node] -------------------------------------------
__global__ void rms_norm_kernel(const float *__restrict__ x, float *__restrict__ y, const float *__restrict__ gain, int64_t n, float eps) {
    __shared__ double shd[32];
    const float *xr = x + (int64_t)blockIdx.x * n;
    float *yr = y + (int64_t)blockIdx.x * n;
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) { const float v = xr[i]; s += (double)__fmul_rn(v, v); }
    const double sum = block_sum(s, shd);
    const float mean = (float)(sum / (double)n);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, eps)));
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        float v = __fmul_rn(xr[i], scale);
        if (gain) v = __fmul_rn(v, gain[i]);
        yr[i] = v;
    }
}
// ---- top-k of one row: k selection passes over a strict total order (value descending, index ascending); nothing is modified, an element is
//      eligible in pass p iff it comes after the element selected in pass p-1 ----------------------------------------------------------------
__global__ void __launch_bounds__(1024) top_k_kernel(const float *__restrict__ x, int64_t n, int k, int32_t *__restrict__ ids, float *__restrict__ vals) {
    __shared__ float sv[32];
    __shared__ int si[32];
    __shared__ float last_v;
    __shared__ int last_i;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { last_v = INFINITY; last_i = -1; }
    __syncthreads();
    for (int p = 0; p < k; p++) {
        const float lv = last_v; const int li = last_i;
        float bv = -INFINITY; int bi = 0x7fffffff;
        for (int64_t i = tid; i < n; i += 1024) {
            const float v = x[i];
            const bool eligible = v < lv || (v == lv && (int)i > li);
            if (eligible && (v > bv || (v == bv && (int)i < bi))) { bv = v; bi = (int)i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            bv = sv[lane]; bi = si[lane];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) { last_v = bv; last_i = bi; ids[p] = bi; vals[p] = bv; }
        }
        __syncthreads();
    }
}

void top_k_rows(const float *x, int64_t n, int k, int32_t *ids, float *vals, cudaStream_t st) {
    B200_ASSERT(k >= 1 && k <= 1024 && n >= k && n < 0x7fffffff);
    top_k_kernel<<<1, 1024, 0, st>>>(x, n, k, ids, vals);
    B200_CHECK(cudaGetLastError());
}

void rms_norm(const float *x, float *y, const float *gain, int64_t n, int64_t rows, float eps, cudaStream_t st) {
    if (rows == 0) return;
    const int threads = n >= 4096 ? 512 : 256;
    rms_norm_kernel<<<(unsigned)rows, threads, 0, st>>>(x, y, gain, n, eps);
    B200_CHECK(cudaGetLastError());
}

// ---- norm (LC/ggml.c:10063-10111) [+ mul gain] [+ add bias] -----------------------------------------------------------
__global__ void layer_norm_kernel(const float *__restrict__ x, float *__restrict__ y, const float *__restrict__ gain, const float *__restrict__ bias, int64_t n) {
    __shared__ double shd[32];
    const float *xr = x + (int64_t)blockIdx.x * n;
    float *yr = y + (int64_t)blockIdx.x * n;
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += (double)xr[i];
    const float mean = (float)(block_sum(s, shd) / (double)n);
    double s2 = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) { const float v = __fsub_rn(xr[i], mean); s2 += (double)__fmul_rn(v, v); }
    const float variance = (float)(block_sum(s2, shd) / (double)n);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(variance, 1e-5f)));
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        float v = __fmul_rn(__fsub_rn(xr[i], mean), scale);
        if (gain) v = __fmul_rn(v, gain[i]);
        if (bias) v = __fadd_rn(v, bias[i]);
        yr[i] = v;
    }
}
void layer_norm(const float *x, float *y, const float *gain, const float *bias, int64_t n, int64_t rows, cudaStream_t st) {
    if (rows == 0) return;
    layer_norm_kernel<<<(unsigned)rows, n >= 4096 ? 512 : 256, 0, st>>>(x, y, gain, bias, n);
    B200_CHECK(cudaGetLastError());
}

// ---- scale -> diag_mask_inf -> soft_max (LC/ggml.c:10733, 11268-11316, 11352-11421), any subset, one pass over the row ---
// Row values live in shared memory between the passes (rows are <= n_ctx floats).
// ALIBI: between scale and mask, column i of a row of head r / nr gets fma(i, alibi[head], v) (ggml_alibi, LC/ggml.c:11534-11597, one fused
// multiply-add as the reference's x86 build compiles it)
template <bool ALIBI>
__device__ __forceinline__ void soft_max_body(const float *__restrict__ x, float *__restrict__ y, int64_t nc, int64_t nr, float scale, int do_scale,
                                              int n_past, int do_mask, int do_softmax, const uint16_t *__restrict__ t_exp, const float *__restrict__ alibi) {
    extern __shared__ float row[];
    __shared__ double shd[32];
    __shared__ float shf[32];
    const int64_t r = blockIdx.x;
    const int64_t j = r % nr;                       // row index inside its [nc, nr] matrix: mask col > n_past + j
    const float *xr = x + r * nc;
    float *yr = y + r * nc;
    float mx = -INFINITY;
    const float slope = ALIBI ? alibi[r / nr] : 0.f;
    for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) {
        float v = xr[i];
        if (do_scale) v = __fmul_rn(v, scale);
        if (ALIBI) v = __fmaf_rn((float)i, slope, v);
        if (do_mask && i > n_past + j) v = -INFINITY;
        row[i] = v;
        mx = fmaxf(mx, v);
    }
    if (!do_softmax) {
        __syncthreads();
        for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) yr[i] = row[i];
        return;
    }
    mx = block_max(mx, shf);
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) {
        const float v = row[i];
        float e = 0.0f;
        if (v != -INFINITY) { e = lut(t_exp, __fsub_rn(v, mx)); s += (double)e; }
        row[i] = e;
    }
    const double sum = block_sum(s, shd);
    const float inv = (float)(1.0 / sum);
    for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) yr[i] = __fmul_rn(row[i], inv);
}
__global__ void soft_max_kernel(const float *__restrict__ x, float *__restrict__ y, int64_t nc, int64_t nr, float scale, int do_scale,
                                int n_past, int do_mask, int do_softmax, const uint16_t *__restrict__ t_exp) {
    soft_max_body<false>(x, y, nc, nr, scale, do_scale, n_past, do_mask, do_softmax, t_exp, nullptr);
}
__global__ void soft_max_alibi_kernel(const float *__restrict__ x, float *__restrict__ y, int64_t nc, int64_t nr, float scale, int n_past,
                                      const uint16_t *__restrict__ t_exp, const float *__restrict__ alibi) {
    soft_max_body<true>(x, y, nc, nr, scale, 1, n_past, 1, 1, t_exp, alibi);
}
void soft_max_alibi(const float *x, float *y, int64_t nc, int64_t rows, int64_t nr, float scale, int n_past, const float *alibi, cudaStream_t st) {
    if (rows == 0 || nc == 0) return;
    const size_t smem = (size_t)nc * sizeof(float);
    static size_t smem_set = 48 * 1024;
    if (smem > smem_set) {
        B200_ASSERT(smem <= 200 * 1024);
        B200_CHECK(cudaFuncSetAttribute(soft_max_alibi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        smem_set = smem;
    }
    soft_max_alibi_kernel<<<(unsigned)rows, nc >= 1024 ? 256 : 128, smem, st>>>(x, y, nc, nr, scale, n_past, luts().exp, alibi);
    B200_CHECK(cudaGetLastError());
}
void soft_max(const float *x, float *y, int64_t nc, int64_t rows, int64_t nr, float scale, bool do_scale, int n_past, bool do_mask, bool do_softmax, cudaStream_t st) {
    if (rows == 0 || nc == 0) return;
    const size_t smem = (size_t)nc * sizeof(float);
    static size_t smem_set = 48 * 1024;
    if (smem > smem_set) {
        B200_ASSERT(smem <= 200 * 1024);
        B200_CHECK(cudaFuncSetAttribute(soft_max_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        smem_set = smem;
    }
    const int threads = nc >= 1024 ? 256 : 128;
    soft_max_kernel<<<(unsigned)rows, threads, smem, st>>>(x, y, nc, nr, scale, do_scale, n_past, do_mask, do_softmax, luts().exp);
    B200_CHECK(cudaGetLastError());
}

// ---- elementwise ---------------------------------------------------------------------------------------------------------
__global__ void unary_lut_kernel(const uint16_t *__restrict__ t, const float *__restrict__ x, float *__restrict__ y, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = lut(t, x[i]);
}
void unary_lut(int which, const float *x, float *y, int64_t n, cudaStream_t st) {
    if (n == 0) return;
    unary_lut_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(which == UNARY_GELU ? luts().gelu : luts().silu, x, y, n);
    B200_CHECK(cudaGetLastError());
}
__global__ void silu_mul_kernel(const uint16_t *__restrict__ t, const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ y, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = __fmul_rn(lut(t, a[i]), b[i]);
}
void silu_mul(const float *a, const float *b, float *y, int64_t n, cudaStream_t st) {
    if (n == 0) return;
    silu_mul_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(luts().silu, a, b, y, n);
    B200_CHECK(cudaGetLastError());
}
template <int OP>
__global__ void binary_kernel(const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ dst, int64_t n, int64_t nbe) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float bv = b[nbe == n ? i : i % nbe];
    dst[i] = OP == 0 ? __fadd_rn(a[i], bv) : __fmul_rn(a[i], bv);
}
void add_f32(const float *a, const float *b, float *dst, int64_t n, int64_t nbe, cudaStream_t st) {
    if (n == 0) return;
    binary_kernel<0><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, b, dst, n, nbe);
    B200_CHECK(cudaGetLastError());
}
void mul_f32(const float *a, const float *b, float *dst, int64_t n, int64_t nbe, cudaStream_t st) {
    if (n == 0) return;
    binary_kernel<1><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, b, dst, n, nbe);
    B200_CHECK(cudaGetLastError());
}
__global__ void scale_kernel(const float *__restrict__ a, float s, float *__restrict__ dst, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __fmul_rn(a[i], s);
}
void scale_f32(const float *a, float scale, float *dst, int64_t n, cudaStream_t st) {
    if (n == 0) return;
    scale_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, scale, dst, n);
    B200_CHECK(cudaGetLastError());
}

// ---- RoPE ---------------------------------------------------------------------------------------------------------------
// Table entry (p, i) = {cos, sin} of the i-th angle the reference's inner loop reaches for position p:
//   theta_0 = freq_scale * p ; theta_{i+1} = theta_i * theta_scale, theta_scale = powf(freq_base, -2/n_dims)
// mode 0 walks ne0/2 adjacent pairs (LC/ggml.c:11859-11874); mode 2 (NeoX) walks ne0/n_dims chunks of n_dims/2 pairs with
// theta carried across chunks (:11875-11897) -- also ne0/2 angles per row.
const RopeTable &rope_table(int n_dims, int mode, float freq_base, float freq_scale, int ne0, int n_pos_needed) {
    using Key = std::tuple<int, int, uint32_t, uint32_t, int>;
    static std::map<Key, RopeTable> cache;
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    uint32_t fb, fs; memcpy(&fb, &freq_base, 4); memcpy(&fs, &freq_scale, 4);
    const Key key{n_dims, mode & 2, fb, fs, ne0};
    auto it = cache.find(key);
    if (it != cache.end() && it->second.n_pos >= n_pos_needed) return it->second;
    int n_pos = 2048;
    while (n_pos < n_pos_needed) n_pos *= 2;
    const int half = ne0 / 2;
    std::vector<float2> h((size_t)n_pos * half);
    const float theta_scale = powf(freq_base, -2.0f / n_dims);
    for (int p = 0; p < n_pos; p++) {
        float theta = freq_scale * (float)p;
        for (int i = 0; i < half; i++) { h[(size_t)p * half + i] = make_float2(cosf(theta), sinf(theta)); theta *= theta_scale; }
    }
    float2 *d;
    B200_CHECK(cudaMalloc(&d, h.size() * sizeof(float2)));
    B200_CHECK(cudaMemcpy(d, h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice));
    B200_CHECK(cudaDeviceSynchronize());   // legacy-stream copy/memset: not ordered with our non-blocking stream, and a pageable H2D cudaMemcpy may return before its DMA lands
    // (this was a real race: the first rope launch after a table upload read a half-written table when the GPU was shared, tests/test_seam_gpt2_neox.py)
    // an outgrown table is leaked on purpose: kernels already enqueued may still read it
    RopeTable t{d, n_pos, half, n_dims, mode & 2, freq_base, freq_scale, ne0};
    cache[key] = t;
    return cache[key];
}

// one thread per rotated pair
__global__ void rope_kernel(const float *x, float *y, int64_t ne0, int64_t ne1, int64_t ne2, int64_t s1, int64_t s2,
                            int64_t ds1, int64_t ds2, int n_past, const float2 *__restrict__ cs, int half, int n_dims, int neox) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = ne2 * ne1 * half;
    if (t >= total) return;
    const int i = (int)(t % half);
    const int64_t i1 = (t / half) % ne1, i2 = t / ((int64_t)half * ne1);
    const float2 c = __ldg(cs + (int64_t)(n_past + i2) * half + i);
    int64_t e0, e1;
    if (!neox) { e0 = 2 * (int64_t)i; e1 = e0 + 1; }
    else { const int hb = n_dims / 2; const int ib = i / hb, ic = i % hb; e0 = (int64_t)ib * n_dims + ic; e1 = e0 + hb; }
    const float *src = x + i2 * s2 + i1 * s1;
    float *dst = y + i2 * ds2 + i1 * ds1;
    const float x0 = src[e0], x1 = src[e1];
    // gcc contracts `x0*c - x1*s` to fma(x0, c, -(x1*s)) and `x0*s + x1*c` to fma(x0, s, x1*c) in the reference build
    dst[e0] = __fmaf_rn(x0, c.x, -__fmul_rn(x1, c.y));
    dst[e1] = __fmaf_rn(x0, c.y, __fmul_rn(x1, c.x));
}
void rope_f32(const float *x, float *y, int64_t ne0, int64_t ne1, int64_t ne2, int64_t s1, int64_t s2, int64_t ds1, int64_t ds2,
              int n_past, const RopeTable &tab, cudaStream_t st) {
    const int64_t total = ne2 * ne1 * tab.half;
    if (total == 0) return;
    B200_ASSERT(n_past + ne2 <= tab.n_pos && tab.ne0 == ne0);
    rope_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, y, ne0, ne1, ne2, s1, s2, ds1, ds2, n_past, tab.cs, tab.half, tab.n_dims, tab.mode);
    B200_CHECK(cudaGetLastError());
}

// ---- generic strided copy (ggml_compute_forward_dup, LC/ggml.c:7815...): element order preserved, shapes may differ ----------
__global__ void cpy_kernel(const char *__restrict__ src, int st, StridedDesc s, char *__restrict__ dst, int dt, StridedDesc d, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t r = i;
    const int64_t s0 = r % s.ne[0]; r /= s.ne[0]; const int64_t s1 = r % s.ne[1]; r /= s.ne[1]; const int64_t s2 = r % s.ne[2]; const int64_t s3 = r / s.ne[2];
    r = i;
    const int64_t d0 = r % d.ne[0]; r /= d.ne[0]; const int64_t d1 = r % d.ne[1]; r /= d.ne[1]; const int64_t d2 = r % d.ne[2]; const int64_t d3 = r / d.ne[2];
    const char *sp = src + s0 * s.nb[0] + s1 * s.nb[1] + s2 * s.nb[2] + s3 * s.nb[3];
    char *dp = dst + d0 * d.nb[0] + d1 * d.nb[1] + d2 * d.nb[2] + d3 * d.nb[3];
    if (st == T_F32 && dt == T_F32) *(float *)dp = *(const float *)sp;
    else if (st == T_F32 && dt == T_F16) *(__half *)dp = __float2half_rn(*(const float *)sp);
    else if (st == T_F16 && dt == T_F16) *(__half *)dp = *(const __half *)sp;
    else *(float *)dp = __half2float(*(const __half *)sp);
}
void cpy_strided(const void *src, int src_type, const StridedDesc &s, void *dst, int dst_type, const StridedDesc &d, cudaStream_t st) {
    const int64_t n = s.ne[0] * s.ne[1] * s.ne[2] * s.ne[3];
    B200_ASSERT(n == d.ne[0] * d.ne[1] * d.ne[2] * d.ne[3]);
    B200_ASSERT((src_type == T_F32 || src_type == T_F16) && (dst_type == T_F32 || dst_type == T_F16));
    if (n == 0) return;
    cpy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const char *)src, src_type, s, (char *)dst, dst_type, d, n);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
