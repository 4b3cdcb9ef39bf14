// llm_b200/csrc/mmq_tc5.cu -- the north star's named kernel in its order-free ("fast", NON-conformant) form: fused per-32-element-block
// dequant -> wgmma tensor-core GEMM with TMA staging, f32 accumulation over the whole K in registers.
//
//   dst[t][n] = sum_k f16(x[t][k]) * f16(d_w[n][k/32] * (q[n][k] - off) (+ m_w))          (the reference's CUDA prefill does dequantize -> cublasSgemm in
//                                                                                          TF32: LC/ggml-cuda.cu:3121-3160, dequant :1308-1327)
// Why it is only the fast mode: the reference's CPU result depends on the AVX2 operation order (DESIGN.md section 2); this kernel rounds activations and
// dequantized weights to fp16 and lets the tensor core sum 4096+ terms in its own order -- ~1e-3 per mat-mul, ~1e-2 on logits.  The conformant wgmma
// kernel is exact_tc5.cu; this one shows what the tensor pipe does when the fp32 chain is not the bound.
//
// CTA = 128 tokens (M) x 128 weight rows (N), K stepped 64 elements per pipeline stage:
//   warp 0       TMA producer: activations f16 [128 tokens x 64] (128B swizzle), one cp.async.bulk.tensor per stage
//   warps 4-11   two consumer warpgroups (tokens 0-63 / 64-127): 4 x wgmma.m64n128k16 per stage, accumulators in registers, f32 stores (+ addend)
//   warps 12-19  dequant: thread = (weight row, block of the stage); packed nibbles (+ fifth bits) -> f16 via the 0x6400 magic, one HFMA2 per pair applies d
//                (and m), written as the 128B-swizzled K-major B operand
#include <string.h>

#include "kernels.cuh"
#include "tc5.cuh"

namespace b200 {

namespace {

using namespace tc5;

constexpr int FM = 128, FN = 128, FST = 4;
constexpr int FA = FM * 128, FB = FN * 128;                       // bytes per stage: [rows][64 f16] = 128-byte rows, swizzled
constexpr int FTHREADS = 640;                                    // TMA warpgroup + 2 consumer warpgroups + 2 dequant warpgroups
constexpr int FSMEM = 1024 + FST * (FA + FB) + 128;

template <int TYPE> struct Fq {
    static constexpr bool MIN = (TYPE == T_Q4_1 || TYPE == T_Q5_1), QH = (TYPE == T_Q5_0 || TYPE == T_Q5_1), Q8 = (TYPE == T_Q8_0);
    static constexpr int QS = Q8 ? 32 : 16, DM = MIN ? 4 : 2;
    static constexpr uint32_t OFF = TYPE == T_Q4_0 ? 0x64086408u : TYPE == T_Q5_0 ? 0x64106410u : TYPE == T_Q8_0 ? 0x64806480u : 0x64006400u;
};

struct Raw { uint4 q0, q1; uint32_t dm, qh; };                    // one (row, block): q1 only for Q8_0 (32 bytes of quants)

// two bytes of v (selected by sel) -> half2(d * (b - off) + m)
__device__ __forceinline__ uint32_t deq2(uint32_t v, uint32_t sel, uint32_t off_h2, __half2 d2, __half2 m2) {
    const uint32_t p = __byte_perm(v, 0x64646464u, sel);
    __half2 a, o;
    memcpy(&a, &p, 4); memcpy(&o, &off_h2, 4);
    const __half2 h = __hfma2(__hsub2(a, o), d2, m2);
    uint32_t r; memcpy(&r, &h, 4);
    return r;
}

template <int TYPE>
__global__ void __launch_bounds__(FTHREADS, 1) mm_fast_tc5_kernel(const __grid_constant__ CUtensorMap tmap_x, const QWeight w, float *__restrict__ dst, int64_t ldd, int64_t B,
                                                                    const float *__restrict__ addend, int64_t lda) {
    using T = Fq<TYPE>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *const sptr = smem_raw + (sbase - smem_u32(smem_raw));
    const uint32_t sA = sbase, sB = sbase + FST * FA, sBar = sB + FST * FB;
    uint8_t *const pB = sptr + FST * FA;
    auto bar_a = [&](int s) { return sBar + 8 * s; };
    auto bar_b = [&](int s) { return sBar + 8 * (FST + s); };
    auto bar_e = [&](int s) { return sBar + 8 * (2 * FST + s); };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t n_base = (int64_t)blockIdx.x * FN, m_base = (int64_t)blockIdx.y * FM;
    const int nb = (int)w.nb, nstage = nb / 2;

    if (tid == 0) {
        tma_prefetch_desc(&tmap_x);
        for (int s = 0; s < FST; s++) { mbar_init(bar_a(s), 1); mbar_init(bar_b(s), 2 * FN); mbar_init(bar_e(s), 8); }
        fence_barrier_init();
    }
    __syncthreads();
    bool dead = false;

    if (warp == 0) {
        if (lane == 0) {
            for (int st = 0; st < nstage; st++) {
                const int slot = st % FST; const uint32_t par = (st / FST) & 1;
                mbar_wait(bar_e(slot), par ^ 1, dead);
                mbar_expect_tx(bar_a(slot), FA);
                tma_load_2d(sA + slot * FA, &tmap_x, st * 64, (int)m_base, bar_a(slot));
            }
        }
    } else if (warp >= 12) {
        // ================= dequant: thread = (weight row of the tile, block j of the stage) =================
        const int r = (tid - 384) & (FN - 1), j = (tid - 384) / FN;
        const int64_t n = n_base + r < w.N ? n_base + r : w.N - 1;
        const uint8_t *q_ptr = w.qs + (size_t)n * nb * T::QS;
        const uint8_t *d_ptr = (const uint8_t *)w.dm + (size_t)n * nb * T::DM;
        const uint32_t *h_ptr = T::QH ? w.qh + (size_t)n * nb : nullptr;
        auto fetch = [&](int blk) {
            Raw x;
            x.q0 = *(const uint4 *)(q_ptr + (size_t)blk * T::QS);
            x.q1 = T::Q8 ? *(const uint4 *)(q_ptr + (size_t)blk * T::QS + 16) : make_uint4(0u, 0u, 0u, 0u);
            x.dm = T::MIN ? *(const uint32_t *)(d_ptr + (size_t)blk * 4) : (uint32_t)*(const uint16_t *)(d_ptr + (size_t)blk * 2);
            x.qh = T::QH ? h_ptr[blk] : 0u;
            return x;
        };
        const uint32_t row_off = (uint32_t)r * 128u, sw = (uint32_t)(r & 7);
        auto expand = [&](const Raw &x, int slot) {
            uint8_t *row = pB + slot * FB + row_off;
            const __half dh = __ushort_as_half((unsigned short)(x.dm & 0xffffu));
            const __half2 d2 = __half2half2(dh);
            const __half2 m2 = T::MIN ? __half2half2(__ushort_as_half((unsigned short)(x.dm >> 16))) : __float2half2_rn(0.f);
            // chunk c of the block = elements 8c .. 8c+7 (K order): two source words a, b with 4 byte-values each
#pragma unroll
            for (int c = 0; c < 4; c++) {
                uint32_t a, b;
                if (T::Q8) {
                    const uint32_t qw[8] = {x.q0.x, x.q0.y, x.q0.z, x.q0.w, x.q1.x, x.q1.y, x.q1.z, x.q1.w};
                    a = qw[2 * c] ^ 0x80808080u; b = qw[2 * c + 1] ^ 0x80808080u;
                } else {
                    const uint32_t qw[4] = {x.q0.x, x.q0.y, x.q0.z, x.q0.w};
                    const int wsel = (c & 1) * 2, sh = (c >> 1) * 4;              // c = 0,1: low nibbles of words 0,1 / 2,3; c = 2,3: high nibbles
                    a = (qw[wsel] >> sh) & 0x0F0F0F0Fu; b = (qw[wsel + 1] >> sh) & 0x0F0F0F0Fu;
                    if (T::QH) { a |= spread4_to_bit4((x.qh >> (8 * c)) & 0xFu); b |= spread4_to_bit4((x.qh >> (8 * c + 4)) & 0xFu); }
                }
                uint4 f;
                f.x = deq2(a, 0x4140u, T::OFF, d2, m2); f.y = deq2(a, 0x4342u, T::OFF, d2, m2);
                f.z = deq2(b, 0x4140u, T::OFF, d2, m2); f.w = deq2(b, 0x4342u, T::OFF, d2, m2);
                *(uint4 *)(row + (((uint32_t)(4 * j + c) ^ sw) << 4)) = f;
            }
        };
        Raw c0, c1;                                                                                // two stages in flight
        if (nstage > 0) c0 = fetch(j);
        if (nstage > 1) c1 = fetch(2 + j);
        for (int st = 0; st < nstage; st += 2) {
#pragma unroll
            for (int u = 0; u < 2; u++) {
                const int s2 = st + u;
                if (s2 >= nstage) break;
                const int slot = s2 % FST; const uint32_t par = (s2 / FST) & 1;
                mbar_wait(bar_e(slot), par ^ 1, dead);
                Raw &cur = u == 0 ? c0 : c1;
                expand(cur, slot);
                if (s2 + 2 < nstage) cur = fetch(2 * (s2 + 2) + j);
                fence_proxy_async_smem();
                mbar_arrive(bar_b(slot));
            }
        }
    } else if (warp >= 4) {
        // ================= consumers: warpgroup g = tokens 64g .. 64g+63 of the tile, all 128 rows =================
        const int g = (warp >> 2) - 1;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; i++) acc[i] = 0.f;
        for (int st = 0; st < nstage; st++) {
            const int slot = st % FST; const uint32_t par = (st / FST) & 1;
            mbar_wait(bar_a(slot), par, dead);
            mbar_wait(bar_b(slot), par, dead);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint64_t ad = make_smem_desc(sA + slot * FA + g * 64 * 128 + k * 32, 16, 1024, LAYOUT_SW128);
                const uint64_t bd = make_smem_desc(sB + slot * FB + k * 32, 16, 1024, LAYOUT_SW128);
                wgmma_m64n128k16(acc, ad, bd, (st > 0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            // the previous stage's MMAs are complete once at most this stage's group is pending: release its slot
            wgmma_wait<1>();
            if (st > 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_e((st - 1) % FST)); }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        // fragment: rows (tokens) 16 (warp % 4) + lane / 4 (+ 8), columns 8i + 2 (lane % 4) + {0, 1}
        const int64_t m0 = m_base + g * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const int64_t m = m0 + 8 * u;
            if (m >= B) continue;
            float *out = dst + (size_t)m * ldd + n_base;
            const float *add = addend ? addend + (size_t)m * lda + n_base : nullptr;
#pragma unroll
            for (int i = 0; i < 16; i++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int c = 8 * i + 2 * (lane & 3) + e;
                    if (n_base + c < w.N) out[c] = add ? acc[4 * i + 2 * u + e] + add[c] : acc[4 * i + 2 * u + e];
                }
        }
    }
}

__global__ void __launch_bounds__(256) cvt_act_f16_kernel(const float *__restrict__ x, int64_t ldx, __half *__restrict__ xh, int64_t K, int64_t total) {
    const int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 2;
    if (i >= total) return;
    const int64_t row = i / K, c = i - row * K;
    const float2 v = *(const float2 *)(x + row * ldx + c);
    *(__half2 *)(xh + i) = __floats2half2_rn(v.x, v.y);
}

template <int TYPE>
void launch_fast(const QWeight &w, const __half *xh, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    static bool set = false;
    if (!set) { B200_CHECK(cudaFuncSetAttribute(mm_fast_tc5_kernel<TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, FSMEM)); set = true; }
    const CUtensorMap tm = make_tmap_2d_f16_sw128(xh, (uint64_t)w.K, (uint64_t)B, (uint64_t)w.K * 2, FM);
    dim3 grid((unsigned)((w.N + FN - 1) / FN), (unsigned)((B + FM - 1) / FM));
    mm_fast_tc5_kernel<TYPE><<<grid, FTHREADS, FSMEM, st>>>(tm, w, dst, ldd, B, addend, lda);
    B200_CHECK(cudaGetLastError());
}

}  // namespace

void cvt_act_f16(const float *x, int64_t ldx, __half *xh, int64_t K, int64_t B, cudaStream_t st) {
    const int64_t total = K * B;
    if (total == 0) return;
    cvt_act_f16_kernel<<<(unsigned)((total / 2 + 255) / 256), 256, 0, st>>>(x, ldx, xh, K, total);
    B200_CHECK(cudaGetLastError());
}

int fast_tc5_check_timeout() { return tc5::check_timeout("mm_fast_tc5_kernel"); }

// xh = activations as fp16, row-major [B][K] (cvt_act_f16)
void mul_mat_q_fast_tc5(const QWeight &w, const __half *xh, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st) {
    if (w.N == 0 || B == 0) return;
    B200_ASSERT(w.nb % 2 == 0 && ((uintptr_t)xh & 15) == 0);
    switch (w.type) {
        case T_Q4_0: launch_fast<T_Q4_0>(w, xh, dst, ldd, B, addend, lda, st); break;
        case T_Q4_1: launch_fast<T_Q4_1>(w, xh, dst, ldd, B, addend, lda, st); break;
        case T_Q5_0: launch_fast<T_Q5_0>(w, xh, dst, ldd, B, addend, lda, st); break;
        case T_Q5_1: launch_fast<T_Q5_1>(w, xh, dst, ldd, B, addend, lda, st); break;
        case T_Q8_0: launch_fast<T_Q8_0>(w, xh, dst, ldd, B, addend, lda, st); break;
        default: B200_ASSERT(!"mul_mat_q_fast_tc5: unsupported weight type");
    }
}

}  // namespace b200
