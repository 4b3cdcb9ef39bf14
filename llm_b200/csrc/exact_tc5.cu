// llm_b200/csrc/exact_tc5.cu -- bit-exact ggml_mul_mat for a batch of activation rows (prefill) on Hopper's warpgroup tensor cores:
// TMA-staged activations, wgmma.mma_async from shared-memory descriptors into registers, warp-specialised, one CTA per SM.
//
// Per output (token t, row n) the reference keeps eight f32 lane accumulators; for every 32-element block b IN ORDER
//     acc_L = fma(d_w[n,b] * d_x[t,b], (float)S_L, acc_L),   S_L = sum_{e<4} w[4L+e] * x[4L+e]   (integers)
// then ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)) (+ the fma chain of m_w * s_x for Q4_1 / Q5_1).  The S_L come from wgmma with a BLOCK-DIAGONAL
// B operand (DESIGN.md section 4): per half-block and warpgroup, A = 64 tokens x 16 Q8 quants, B = (16 rows x 4 lanes) x 16 weights, column
// (n, l) non-zero only at elements 4l..4l+3, scale-d = 0, so D[t][(n, l)] = S_{4h+l} exactly.  Column c = 8i + 2q + e of the fragment
// (q = lane % 4) is row 4(i/2) + q, lane 2(i%2) + e: a thread holds all eight lanes of its rows.
//
// Warps: 0 TMA producer (f16 activations [128 tokens x 64], 128B swizzle, + scales); 2-3 expanders (packed weights -> block-diagonal f16
// B operands + f32 scales); 4-11 two consumer warpgroups (tokens 0-63 / 64-127) sharing each stage's B: wgmma, the ordered fp32 chains, store.
#include <string.h>

#include "kernels.cuh"
#include "tc5.cuh"

namespace b200 {

namespace {

using namespace tc5;

constexpr int TM = 128, TN = 32, NST = 4;                         // tokens / rows per CTA, pipeline stages (2 blocks each)
constexpr int A_STAGE = TM * 64 * 2;                              // 16 KB: [128 tokens][64 elements] f16, 128-byte rows, swizzled
constexpr int B_LBO = 128, B_SBO = 272;                           // K-adjacent core matrices contiguous; 8-column groups 272 B apart (the expanders' 8-byte
                                                                  // stores then spread over the banks: 2-way instead of 8-way conflicts with 256)
constexpr int B_HALF = 16 * B_SBO;                                // one block-diagonal operand (N = 128 columns = 32 rows x 4 lanes, K = 16), no swizzle
constexpr int B_STAGE = 4 * B_HALF;                               // [block j][half h]
constexpr int W_STAGE = 2 * 2 * TN * 4;                           // weight scales of the stage: [block j][d | m][32 rows] f32
constexpr int X_STAGE = TM * 16;                                  // activation scales of the stage: [token] float4 {d, aux} x 2 blocks
constexpr int NTHREADS = 384;
// setmaxnreg re-splits the CTA's own register pool (what the launch allocated: 384 threads x 168, the __launch_bounds__(384, 1) cap)
constexpr int PROD_REGS = 56, CONS_REGS = 224;
static_assert(128 * PROD_REGS + 256 * CONS_REGS <= NTHREADS * 168, "register split exceeds the CTA's pool");
constexpr int SMEM_BYTES = 1024 + NST * (A_STAGE + B_STAGE + W_STAGE + X_STAGE) + 128;

template <int TYPE> struct Tc {
    static constexpr bool MIN = (TYPE == T_Q4_1 || TYPE == T_Q5_1), QH = (TYPE == T_Q5_0 || TYPE == T_Q5_1), Q8 = (TYPE == T_Q8_0);
    static constexpr int QS = Q8 ? 32 : 16, DM = MIN ? 4 : 2;
    static constexpr uint32_t OFF = TYPE == T_Q4_0 ? 0x64086408u : TYPE == T_Q5_0 ? 0x64106410u : TYPE == T_Q8_0 ? 0x64806480u : 0x64006400u;
};

// bytes (sel picks two of the four bytes of v) -> half2(1024 + lo, 1024 + hi) - off   (exact: the fp16 magic-number trick)
__device__ __forceinline__ uint32_t bytes_to_half2(uint32_t v, uint32_t sel, uint32_t off_h2) {
    const uint32_t p = __byte_perm(v, 0x64646464u, sel);
    __half2 a, o;
    memcpy(&a, &p, 4); memcpy(&o, &off_h2, 4);
    const __half2 h = __hsub2(a, o);
    uint32_t r; memcpy(&r, &h, 4);
    return r;
}

struct WRaw { uint4 q; uint32_t dm; uint32_t qh; };               // one (row, block) as fetched by an expander thread

template <int TYPE>
__global__ void __launch_bounds__(NTHREADS, 1) mm_exact_tc5_kernel(const __grid_constant__ CUtensorMap tmap_x, const QWeight w, const float4 *__restrict__ xdt,
                                                                     float *__restrict__ dst, int64_t ldd, int64_t B, const float *__restrict__ addend, int64_t lda) {
    using T = Tc<TYPE>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;                     // 128B-swizzled tiles need 1024-byte alignment
    uint8_t *const sptr = smem_raw + (sbase - smem_u32(smem_raw));
    const uint32_t sA = sbase, sB = sbase + NST * A_STAGE, sX = sB + NST * (B_STAGE + W_STAGE), sBar = sX + NST * X_STAGE;
    uint8_t *const pB = sptr + NST * A_STAGE;
    float *const pW = (float *)(sptr + NST * (A_STAGE + B_STAGE));
    const float4 *const pX = (const float4 *)(sptr + NST * (A_STAGE + B_STAGE + W_STAGE));
    auto bar_a_full = [&](int s) { return sBar + 8 * s; };
    auto bar_b_full = [&](int s) { return sBar + 8 * (NST + s); };
    auto bar_empty = [&](int s) { return sBar + 8 * (2 * NST + s); };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t n_base = (int64_t)blockIdx.x * TN, m_base = (int64_t)blockIdx.y * TM;
    const int nb = (int)w.nb, nstage = nb / 2;

    // ---- set-up: zero the operand buffers (the off-diagonal zeros are written once), barriers ----
    for (int i = tid; i < NST * B_STAGE / 16; i += NTHREADS) ((uint4 *)pB)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async_smem();
    if (tid == 0) {
        tma_prefetch_desc(&tmap_x);
        for (int s = 0; s < NST; s++) { mbar_init(bar_a_full(s), 1); mbar_init(bar_b_full(s), 64); mbar_init(bar_empty(s), 8); }
        fence_barrier_init();
    }
    __syncthreads();
    bool dead = false;

    if (warp < 4) {
        reg_dealloc<PROD_REGS>();
        if (warp == 0) {
            // ================= TMA producer =================
            if (lane == 0) {
                const uint32_t x_bytes = (uint32_t)(B - m_base < TM ? B - m_base : TM) * 16u;
                for (int st = 0; st < nstage; st++) {
                    const int slot = st % NST; const uint32_t par = (st / NST) & 1;
                    mbar_wait(bar_empty(slot), par ^ 1, dead);
                    mbar_expect_tx(bar_a_full(slot), A_STAGE + x_bytes);
                    tma_load_2d(sA + slot * A_STAGE, &tmap_x, st * 64, (int)m_base, bar_a_full(slot));
                    // {d, aux} of this stage's two blocks for the tile's tokens: one contiguous piece of the block-pair-major scale array
                    bulk_load(sX + slot * X_STAGE, xdt + ((size_t)st * B + m_base), x_bytes, bar_a_full(slot));
                }
            }
        } else if (warp >= 2) {
            // ================= expanders: thread (row r, half h) =================
            const int et = tid - 64, r = et >> 1, h = et & 1;
            const int64_t n = n_base + r < w.N ? n_base + r : w.N - 1;
            const uint8_t *q_ptr = w.qs + (size_t)n * nb * T::QS + (T::Q8 ? 16 * h : 0);
            const uint8_t *d_ptr = (const uint8_t *)w.dm + (size_t)n * nb * T::DM;
            const uint32_t *h_ptr = T::QH ? w.qh + (size_t)n * nb : nullptr;
            auto fetch = [&](int blk) {
                WRaw x;
                x.q = *(const uint4 *)(q_ptr + (size_t)blk * T::QS);
                x.dm = T::MIN ? *(const uint32_t *)(d_ptr + (size_t)blk * 4) : (uint32_t)*(const uint16_t *)(d_ptr + (size_t)blk * 2);
                x.qh = T::QH ? h_ptr[blk] : 0u;
                return x;
            };
            // column (r, l) of half h: non-zero K slots 4l..4l+3  ->  8 bytes at this offset inside the operand.  Column index inside the
            // 64-column operand of row slice r / 16: 16 (r % 16 / 4) + 8 (l / 2) + 2 (r % 4) + l % 2 (the fragment order of the header comment)
            uint32_t col_off[4];
#pragma unroll
            for (int l = 0; l < 4; l++) {
                const uint32_t c = (uint32_t)(64 * (r >> 4) + 16 * ((r & 15) >> 2) + 8 * (l >> 1) + 2 * (r & 3) + (l & 1));
                col_off[l] = (c >> 3) * B_SBO + (l >> 1) * B_LBO + (c & 7) * 16 + (l & 1) * 8;
            }
            auto expand = [&](const WRaw &x, int slot, int j) {
                uint8_t *out = pB + slot * B_STAGE + (j * 2 + h) * B_HALF;
                const uint32_t qw[4] = {x.q.x, x.q.y, x.q.z, x.q.w};
#pragma unroll
                for (int l = 0; l < 4; l++) {
                    uint32_t v;
                    if (T::Q8) v = qw[l] ^ 0x80808080u;                                           // int8 -> biased 0..255
                    else {
                        v = (qw[l] >> (4 * h)) & 0x0F0F0F0Fu;                                      // elements 16h + 4l .. +3
                        if (T::QH) v |= spread4_to_bit4((x.qh >> (16 * h + 4 * l)) & 0xFu);
                    }
                    uint2 f;
                    f.x = bytes_to_half2(v, 0x4140u, T::OFF);
                    f.y = bytes_to_half2(v, 0x4342u, T::OFF);
                    *(uint2 *)(out + col_off[l]) = f;
                }
                if (h == 0) {                                                                          // f32 scales: [slot][j][d | m][32 rows]
                    float *pd = pW + (slot * 2 + j) * 2 * TN;
                    if (T::MIN) { __half2 hh; memcpy(&hh, &x.dm, 4); pd[r] = __low2float(hh); pd[TN + r] = __high2float(hh); }
                    else pd[r] = __half2float(__ushort_as_half((unsigned short)x.dm));
                }
            };
            WRaw cur[2];                                                                           // the next stage's blocks are in flight while
            if (nstage > 0) { cur[0] = fetch(0); cur[1] = fetch(1); }                              // this one waits for its ring slot
            for (int st = 0; st < nstage; st++) {
                const int slot = st % NST; const uint32_t par = (st / NST) & 1;
                mbar_wait(bar_empty(slot), par ^ 1, dead);
                expand(cur[0], slot, 0);
                expand(cur[1], slot, 1);
                if (st + 1 < nstage) { cur[0] = fetch(2 * (st + 1)); cur[1] = fetch(2 * (st + 1) + 1); }
                fence_proxy_async_smem();
                mbar_arrive(bar_b_full(slot));
            }
        }
    } else {
        // ================= consumers: warpgroup g = tokens 64g .. 64g+63 of the tile, all 32 rows =================
        // thread: tokens tok0, tok0 + 8; rows 16 s + 4 jj + q (row slice s, jj < 4), all eight lanes of each
        reg_alloc<CONS_REGS>();
        const int g = (warp >> 2) - 1, q = lane & 3;
        const int tok0 = g * 64 + (warp & 3) * 16 + (lane >> 2);
        float acc[2][4][2][8];
        float summs[2][4][2];
        float d[2][32];
#pragma unroll
        for (int s = 0; s < 2; s++)
#pragma unroll
            for (int jj = 0; jj < 4; jj++)
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    summs[s][jj][u] = 0.f;
#pragma unroll
                    for (int L = 0; L < 8; L++) acc[s][jj][u][L] = 0.f;
                }
#pragma unroll
        for (int i = 0; i < 32; i++) { d[0][i] = 0.f; d[1][i] = 0.f; }

        for (int st = 0; st < nstage; st++) {
            const int slot = st % NST; const uint32_t par = (st / NST) & 1;
            mbar_wait(bar_a_full(slot), par, dead);
            mbar_wait(bar_b_full(slot), par, dead);
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const float2 x0 = ((const float2 *)(pX + slot * TM + tok0))[j], x1 = ((const float2 *)(pX + slot * TM + tok0 + 8))[j];
                const float dx[2] = {x0.x, x1.x}, sx[2] = {x0.y, x1.y};
                const float *pd = pW + (slot * 2 + j) * 2 * TN, *pm = pd + TN;
#pragma unroll
                for (int s = 0; s < 2; s++) {
                    wgmma_fence();
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const uint64_t ad = make_smem_desc(sA + slot * A_STAGE + g * 64 * 128 + j * 64 + h * 32, 16, 1024, LAYOUT_SW128);
                        const uint64_t bd = make_smem_desc(sB + slot * B_STAGE + (j * 2 + h) * B_HALF + s * 8 * B_SBO, B_LBO, B_SBO, LAYOUT_NONE);
                        wgmma_m64n64k16(d[h], ad, bd, 0u);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_regs(d[0]); fence_regs(d[1]);
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        const int row = 16 * s + 4 * jj + q;
                        const float dw = pd[row];
                        const float mw = T::MIN ? pm[row] : 0.f;
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            const float sc = __fmul_rn(dw, dx[u]);
                            if (T::MIN) summs[s][jj][u] = __fmaf_rn(mw, sx[u], summs[s][jj][u]);
#pragma unroll
                            for (int h = 0; h < 2; h++)
#pragma unroll
                                for (int il = 0; il < 2; il++)
#pragma unroll
                                    for (int e = 0; e < 2; e++)
                                        acc[s][jj][u][4 * h + 2 * il + e] = __fmaf_rn(sc, d[h][4 * (2 * jj + il) + 2 * u + e], acc[s][jj][u][4 * h + 2 * il + e]);
                        }
                    }
                }
            }
            __syncwarp();                                                                          // the stage's operands and scales are consumed
            if (lane == 0) mbar_arrive(bar_empty(slot));
        }
        // hsum_float_8 (LC/ggml.c:608-616): ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)), then + summs
#pragma unroll
        for (int s = 0; s < 2; s++)
#pragma unroll
            for (int jj = 0; jj < 4; jj++)
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int64_t m = m_base + tok0 + 8 * u, n = n_base + 16 * s + 4 * jj + q;
                    if (m < B && n < w.N) {
                        const float *a = acc[s][jj][u];
                        float v = __fadd_rn(__fadd_rn(__fadd_rn(a[0], a[4]), __fadd_rn(a[2], a[6])), __fadd_rn(__fadd_rn(a[1], a[5]), __fadd_rn(a[3], a[7])));
                        if (T::MIN) v = __fadd_rn(v, summs[s][jj][u]);
                        dst[(size_t)m * ldd + n] = addend ? __fadd_rn(v, addend[(size_t)m * lda + n]) : v;
                    }
                }
    }
}

// quantize_act with the quants written as fp16 in plain row-major [B][K] (the TMA source), same arithmetic as quantize_act_kernel (quant.cu)
template <bool Q81>
__global__ void __launch_bounds__(256) quantize_act_f16_rm_kernel(const float *__restrict__ x, int64_t ldx, __half *__restrict__ xh, float2 *__restrict__ ds,
                                                                  int64_t nbk, int64_t total_blocks, int64_t rows) {
    const int64_t blk = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (blk >= total_blocks) return;
    const int lane = threadIdx.x & 31;
    const int64_t row = blk / nbk, b = blk - row * nbk;
    const float v = x[row * ldx + b * QK + lane];
    const float amax = warp_max(fabsf(v));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
    const int q = __float2int_rn(__fmul_rn(v, id));
    const int isum = warp_sum(q);
    xh[(row * nbk + b) * QK + lane] = __int2half_rn(q);
    // scales in block-pair-major order [K/64][B] x float4 {d, aux of block 2p | d, aux of block 2p+1}: the kernel's per-stage piece is contiguous
    if (lane == 0) ds[((b >> 1) * rows + row) * 2 + (b & 1)] = Q81 ? make_float2(d, __fmul_rn(d, (float)isum)) : make_float2(__half2float(__float2half_rn(d)), (float)isum);
}

template <int TYPE>
void launch_tc5(const QWeight &w, const __half *xh, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    static bool set = false;                                        // per-process attribute (one device per process: include/llm_b200.h)
    if (!set) { B200_CHECK(cudaFuncSetAttribute(mm_exact_tc5_kernel<TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); set = true; }
    const CUtensorMap tm = make_tmap_2d_f16_sw128(xh, (uint64_t)w.K, (uint64_t)B, (uint64_t)w.K * 2, TM);
    dim3 grid((unsigned)((w.N + TN - 1) / TN), (unsigned)((B + TM - 1) / TM));
    mm_exact_tc5_kernel<TYPE><<<grid, NTHREADS, SMEM_BYTES, st>>>(tm, w, (const float4 *)xds, dst, ldd, B, addend, lda);
    B200_CHECK(cudaGetLastError());
}

}  // namespace

void quantize_act_f16_rm(int vdt, const float *x, int64_t ldx, __half *xh, float2 *ds, int64_t K, int64_t B, cudaStream_t st) {
    const int64_t nbk = K / QK, total = nbk * B;
    if (total == 0) return;
    if (vdt == T_Q8_1) quantize_act_f16_rm_kernel<true><<<(unsigned)((total + 7) / 8), 256, 0, st>>>(x, ldx, xh, ds, nbk, total, B);
    else               quantize_act_f16_rm_kernel<false><<<(unsigned)((total + 7) / 8), 256, 0, st>>>(x, ldx, xh, ds, nbk, total, B);
    B200_CHECK(cudaGetLastError());
}

int exact_tc5_check_timeout() { return tc5::check_timeout("mm_exact_tc5_kernel"); }

// xh = quantized activations as fp16, row-major [B][K]; xds = {d, aux} per (block, token) in the block-pair-major order of quantize_act_f16_rm
void mul_mat_q_exact_tc5(const QWeight &w, const __half *xh, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    if (w.N == 0 || B == 0) return;
    B200_ASSERT(w.nb % 2 == 0 && ((uintptr_t)xh & 15) == 0 && ((uintptr_t)xds & 15) == 0);
    switch (w.type) {
        case T_Q4_0: launch_tc5<T_Q4_0>(w, xh, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q4_1: launch_tc5<T_Q4_1>(w, xh, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q5_0: launch_tc5<T_Q5_0>(w, xh, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q5_1: launch_tc5<T_Q5_1>(w, xh, xds, dst, ldd, B, addend, lda, st); break;
        case T_Q8_0: launch_tc5<T_Q8_0>(w, xh, xds, dst, ldd, B, addend, lda, st); break;
        default: B200_ASSERT(!"mul_mat_q_exact_tc5: unsupported weight type");
    }
}

}  // namespace b200
