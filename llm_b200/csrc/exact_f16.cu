// llm_b200/csrc/exact_f16.cu -- weight mat-muls on F16 model files, bit-exact with the reference's generic F16 path.
//
// ggml_compute_forward_mul_mat with an F16 weight (LC/ggml.c:10397-10586, type traits :1650-1656) first rounds every activation row to
// fp16 (ggml_fp32_to_fp16_row, RNE), then computes each output as one ggml_vec_dot_f16 (:2325-2359): 32 f32 FMA chains -- chain l takes
// the elements k = l mod 32, in order of k -- reduced by GGML_F32x8_REDUCE.  The weight matrices here have K % 64 == 0, so there are no
// leftovers.  The reduction is (exact.cu): c[l] + c[l+16], then + 8, + 4, then the two hadds (offsets 1 and 2); as shuffle-downs on a warp
// whose lane l holds chain l that is offsets 16, 8, 4, 1, 2.
//
// The activation is rounded once per mat-mul (cvt_act_f16, the same RNE), so both kernels read fp16 operands.
//
//   * mat-vec (B == 1): HBM-bound.  Persistent CTAs; a producer warp streams 16-row x 256-element stages of the weight rows through an
//     8-stage shared-memory ring (stream_core.cuh: cp.async + mbarriers), each weight byte read once.  4 compute warps own 4 rows each,
//     lane l = chain l: per 32-element step one LDS of x and, per row, one LDS + one FMA.
//   * GEMM (B >= 2): fp32-pipe-bound by construction (one separately rounded FMA per weight x token).  A CTA computes 32 weight rows x 32
//     tokens; each warp a 16 x 8 tile with lane l holding chain l of all 128 outputs.  Operands are staged as f32 in a [step][lane][row]
//     layout, so a 32-element step costs a warp 6 conflict-free LDS.128 for 128 FMAs.  The cross-lane tree runs once per output at the end.
#include "stream_core.cuh"

namespace b200 {

using namespace stream;

namespace {

// ggml_vec_dot_f16's GGML_F32x8_REDUCE over the 32 chains held one per lane; the result is in lane 0
__device__ __forceinline__ float f16_reduce(float s) {
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 16));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 8));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 4));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 1));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 2));
    return s;
}

// ---- mat-vec -------------------------------------------------------------------------------------------------------------------
constexpr int VR = 16;                   // rows per tile
constexpr int VCH = 256;                 // elements of a row per ring stage (512 B)
constexpr int VST = 8;                   // ring stages
constexpr int V_STAGE = VR * VCH * 2;    // 8 KB
constexpr int V_RING = VST * V_STAGE;
constexpr int V_RPW = VR / (SCOMPUTE / 32);   // rows per compute warp
static_assert(VST <= SST_MAX, "ring depth");

__global__ void __launch_bounds__(STHREADS) mmv_f16_kernel(const __half *__restrict__ w, int64_t K, int64_t N, const __half *__restrict__ xh,
                                                           float *__restrict__ dst, const float *__restrict__ addend) {
    extern __shared__ __align__(128) uint8_t smem[];
    Ring R{(uint64_t *)smem, (uint64_t *)smem + SST_MAX, smem + 256, 0u, VST};
    const __half *sx = (const __half *)(R.base + V_RING);
    const int tid = threadIdx.x, lane = tid & 31;
    const int nch = (int)((K + VCH - 1) / VCH), ntiles = (int)((N + VR - 1) / VR);
    if (tid == 0) ring_init(R.full, R.empty, VST);
    __syncthreads();
    if (tid >= SCOMPUTE) {                                             // producer warp
        const uint32_t ring_u32 = smem_u32(R.base);
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t row0 = (int64_t)tile * VR;
            const int rows_valid = (int)(N - row0 < VR ? N - row0 : VR);
            for (int c = 0; c < nch; c++, R.advance()) {
                const int s = R.slot;
                const int64_t k0 = (int64_t)c * VCH;
                const int cb = (int)(K - k0 < VCH ? K - k0 : VCH);
                mbar_wait(&R.empty[s], R.phase ^ 1u);
                stream_plane<VCH * 2 / 16, VR>(ring_u32 + s * V_STAGE, VCH * 2, (const uint8_t *)(w + row0 * K + k0), K * 2, cb * 2 / 16, rows_valid, lane);
                cp_async_arrive(&R.full[s]);
            }
        }
        return;
    }
    for (int64_t i = tid; i < K / 8; i += SCOMPUTE) cp16(smem_u32(sx + 8 * i), xh + 8 * i);
    asm volatile("cp.async.wait_all;" ::: "memory");
    compute_sync();
    const int r0 = (tid >> 5) * V_RPW;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        float acc[V_RPW];
#pragma unroll
        for (int r = 0; r < V_RPW; r++) acc[r] = 0.f;
        for (int c = 0; c < nch; c++, R.advance()) {
            const int s = R.slot;
            const int64_t k0 = (int64_t)c * VCH;
            const int steps = (int)(K - k0 < VCH ? K - k0 : VCH) / 32;
            mbar_wait(&R.full[s], R.phase);
            const __half *sw = (const __half *)(R.base + s * V_STAGE) + r0 * VCH + lane;
            const __half *xs = sx + k0 + lane;
#pragma unroll 8
            for (int j = 0; j < steps; j++) {
                const float xv = __half2float(xs[32 * j]);
#pragma unroll
                for (int r = 0; r < V_RPW; r++) acc[r] = __fmaf_rn(__half2float(sw[r * VCH + 32 * j]), xv, acc[r]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&R.empty[s]);
        }
#pragma unroll
        for (int r = 0; r < V_RPW; r++) {
            const float v = f16_reduce(acc[r]);
            const int64_t row = (int64_t)tile * VR + r0 + r;
            if (lane == 0 && row < N) dst[row] = addend ? __fadd_rn(v, addend[row]) : v;
        }
    }
}

constexpr int v_smem(int64_t K) { return 256 + V_RING + (int)K * 2; }

// ---- GEMM ----------------------------------------------------------------------------------------------------------------------
constexpr int GM = 32, GN = 32;          // weight rows x tokens per CTA
constexpr int GK = 128;                  // elements per chunk (4 steps of 32)
constexpr int GP = 36;                   // floats per (step, lane) record of 32 rows: lanes of a quarter-warp land 4 banks apart
constexpr int G_THREADS = 256;
constexpr int G_OP = (GK / 32) * 32 * GP;          // floats of one operand tile
constexpr int G_SMEM = 2 * 2 * G_OP * 4;           // double-buffered weight and activation tiles (72 KB)

// Thread (q = tid % 32, g = tid / 32) of the fill owns elements [16g, 16g + 16) of operand row q: two 16-byte loads, and 16 stores to
// [step g/2][lane 16(g&1) + e][q] -- a warp stores 32 consecutive floats per instruction.
struct F16Rows {
    const __half *p; int64_t ld, rows;
    __device__ __forceinline__ void fetch(int64_t row0, int q, int g, int64_t k0, int64_t K, uint4 (&v)[2]) const {
        const int64_t r = row0 + q < rows ? row0 + q : rows - 1;
        const __half *src = p + r * ld + k0 + 16 * g;
#pragma unroll
        for (int h = 0; h < 2; h++) v[h] = k0 + 16 * g + 8 * h < K ? __ldg((const uint4 *)src + h) : make_uint4(0u, 0u, 0u, 0u);
    }
};
__device__ __forceinline__ void stash(float *tile, int q, int g, const uint4 (&v)[2]) {
    float *dst = tile + ((g >> 1) * 32 + 16 * (g & 1)) * GP + q;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const __half2 *hp = (const __half2 *)&v[h];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const float2 f = __half22float2(hp[e]);
            dst[(8 * h + 2 * e) * GP] = f.x;
            dst[(8 * h + 2 * e + 1) * GP] = f.y;
        }
    }
}

__global__ void __launch_bounds__(G_THREADS, 1) mm_f16_gemm_kernel(const __half *__restrict__ w, int64_t K, int64_t N, const __half *__restrict__ xh, int64_t B,
                                                                   float *__restrict__ dst, int64_t ldd, const float *__restrict__ addend, int64_t lda) {
    extern __shared__ __align__(16) float gsm[];
    float *sw = gsm, *sx = gsm + 2 * G_OP;                    // [buf][step][lane][GP]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rg = warp & 1, cg = warp >> 1;                  // this warp: rows 16 rg .. +15, tokens 8 cg .. +7 of the tile
    const int64_t t0 = (int64_t)blockIdx.x * GN, m0 = (int64_t)blockIdx.y * GM;
    const F16Rows W{w, K, N}, X{xh, K, B};
    const int q = lane, g = warp;
    uint4 wv[2], xv[2];

    float acc[16][8];
#pragma unroll
    for (int i = 0; i < 16; i++)
#pragma unroll
        for (int t = 0; t < 8; t++) acc[i][t] = 0.f;

    const int nch = (int)((K + GK - 1) / GK);
    W.fetch(m0, q, g, 0, K, wv); X.fetch(t0, q, g, 0, K, xv);
    stash(sw, q, g, wv); stash(sx, q, g, xv);
    __syncthreads();
    for (int c = 0; c < nch; c++) {
        const int buf = c & 1;
        const int64_t k0 = (int64_t)c * GK;
        if (c + 1 < nch) { W.fetch(m0, q, g, k0 + GK, K, wv); X.fetch(t0, q, g, k0 + GK, K, xv); }
        const int steps = K - k0 < GK ? (int)(K - k0) / 32 : GK / 32;
        const float *aw = sw + buf * G_OP + lane * GP + 16 * rg, *ax = sx + buf * G_OP + lane * GP + 8 * cg;
#pragma unroll
        for (int j = 0; j < GK / 32; j++) {
            if (j >= steps) break;
            float a[16], b[8];
#pragma unroll
            for (int u = 0; u < 4; u++) *(float4 *)&a[4 * u] = *(const float4 *)(aw + j * 32 * GP + 4 * u);
#pragma unroll
            for (int u = 0; u < 2; u++) *(float4 *)&b[4 * u] = *(const float4 *)(ax + j * 32 * GP + 4 * u);
#pragma unroll
            for (int i = 0; i < 16; i++)
#pragma unroll
                for (int t = 0; t < 8; t++) acc[i][t] = __fmaf_rn(a[i], b[t], acc[i][t]);
        }
        if (c + 1 < nch) { stash(sw + (buf ^ 1) * G_OP, q, g, wv); stash(sx + (buf ^ 1) * G_OP, q, g, xv); }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 16; i++)
#pragma unroll
        for (int t = 0; t < 8; t++) {
            const float v = f16_reduce(acc[i][t]);
            const int64_t row = m0 + 16 * rg + i, tok = t0 + 8 * cg + t;
            if (lane == 0 && row < N && tok < B) dst[tok * ldd + row] = addend ? __fadd_rn(v, addend[tok * lda + row]) : v;
        }
}

// ---- gathers and patches on F16 weights ----------------------------------------------------------------------------------------
__global__ void get_rows_f16_kernel(const __half *__restrict__ w, int64_t K, const int32_t *__restrict__ ids, float *__restrict__ dst, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int64_t r = i / K, k = i - r * K;
    dst[i] = __half2float(w[(int64_t)ids[r] * K + k]);
}

__global__ void f16_to_f32_kernel(const __half *__restrict__ src, float *__restrict__ dst, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __half2float(src[i]);
}

}  // namespace

bool mmv_f16_supported(const QWeight &w) { return w.type == T_F16 && w.K % 64 == 0 && v_smem(w.K) <= 227 * 1024; }

void mul_mat_vec_f16(const QWeight &w, const __half *xh, float *dst, const float *addend, cudaStream_t st) {
    if (w.N == 0) return;
    B200_ASSERT(mmv_f16_supported(w));
    const int smem = v_smem(w.K);
    static int smem_set = 0;
    if (smem > smem_set) {
        B200_CHECK(cudaFuncSetAttribute(mmv_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        smem_set = smem;
    }
    static int ctas_per_sm = 0, sms = 0, occ_smem = -1;
    if (!sms) { int dev; B200_CHECK(cudaGetDevice(&dev)); B200_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)); }
    if (occ_smem != smem) { B200_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, mmv_f16_kernel, STHREADS, smem)); occ_smem = smem; }
    const int64_t tiles = (w.N + VR - 1) / VR;
    const int64_t slots = (int64_t)sms * (ctas_per_sm > 0 ? ctas_per_sm : 1);
    const unsigned grid = (unsigned)(tiles < slots ? tiles : slots);
    mmv_f16_kernel<<<grid, STHREADS, smem, st>>>((const __half *)w.qs, w.K, w.N, xh, dst, addend);
    B200_CHECK(cudaGetLastError());
}

void mul_mat_f16_gemm(const QWeight &w, const __half *xh, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    if (w.N == 0 || B == 0) return;
    B200_ASSERT(w.type == T_F16 && w.K % 64 == 0 && (w.N + GM - 1) / GM <= 65535);
    static bool set = false;
    if (!set) { B200_CHECK(cudaFuncSetAttribute(mm_f16_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM)); set = true; }
    const dim3 grid((unsigned)((B + GN - 1) / GN), (unsigned)((w.N + GM - 1) / GM));    // token tiles of one weight tile run side by side (L2 reuse)
    mm_f16_gemm_kernel<<<grid, G_THREADS, G_SMEM, st>>>((const __half *)w.qs, w.K, w.N, xh, B, dst, ldd, addend, lda);
    B200_CHECK(cudaGetLastError());
}

void get_rows_f16(const QWeight &w, const int32_t *ids, float *dst, int64_t n, cudaStream_t st) {
    const int64_t total = n * w.K;
    if (total == 0) return;
    get_rows_f16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const __half *)w.qs, w.K, ids, dst, total);
    B200_CHECK(cudaGetLastError());
}

void f16_to_f32(const void *src, float *dst, int64_t n, cudaStream_t st) {
    if (n == 0) return;
    f16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const __half *)src, dst, n);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
