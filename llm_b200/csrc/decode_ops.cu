// llm_b200/csrc/decode_ops.cu -- the default decode schedule: 7 fused kernels per layer, replayed from ONE CUDA graph per token.
//
//   1 norm_pack        rms_norm(x) * attn_norm -> Q8 activation records                       (llama lib.rs:183-186 + mul_mat INIT)
//   2 mmv<QKV>         [wq|wk|wv] x, epilogue: RoPE on Q/K rows, K/V rows -> cache at n_past (:190-244)
//   3 attn_fused       KQ = K . f16(Q), scale + soft_max, V^T . f16(P), epilogue: quantize the merged row -- one cluster of hd/32 CTAs per
//                      head, scores exchanged through distributed shared memory                (:246-307)
//                      (buckets past 3264 positions, 1664 on an f32 cache: the two-kernel variant attn_kq + attn_sv)
// Each attention kernel is one template over the cache's element type KT: __half, or float for an f32 cache (Q and P then stay f32).
//   4 mmv<RES>         wo x + inpSA                                                           (:310-314)
//   5 norm_pack        rms_norm(inpFF) * ffn_norm                                             (:318-321)
//   6 mmv<SILU>        [w1|w3] x (rows interleaved in 32-row pieces), epilogue: silu(w1 x) * (w3 x) quantized (:323-330)
//   7 mmv<RES>         w2 h + inpFF                                                           (:332-334)
// Everything that depends on the position reads n_past from DEVICE memory, so the captured graph is valid for every token; the
// last node increments it.  All arithmetic is the bit-exact arithmetic of exact.cu / rowops.cu.
// Variants that were tried on top of this and not kept: norm fusion, tiled weights + TMA, L2 prefetch.
#include <cooperative_groups.h>

#include <algorithm>
#include <array>
#include <map>
#include <vector>

#include "decode.h"
#include "f32dot.cuh"
#include "stream_core.cuh"
#include "tp.cuh"

namespace b200 {

using namespace stream;

// the tensor-parallel context of this process's session (tp.cuh): one copy in constant memory instead of ~120 bytes in every kernel's argument block
// (the single-GPU decode graph must not pay for it: 227 launches per token).  world == 0 / 1: single GPU.
__constant__ TpCtx c_tp;

namespace {

// Programmatic dependent launch.  Every kernel of the chain touches nothing a predecessor writes (and writes nothing at all) before
// `pdl_wait`; what runs ahead of the wait only reads the constant weights (the producer warp of the next mat-vec fills its ring).
// WHERE the dependents are released matters: triggered at kernel entry, the successors sit on SM resources the running kernel's tail needs;
// a mat-vec triggers from its producer warp as soon as every byte of the CTA is requested.
// tuning aid: per-launch timeline (DecodeParams::prof), see b200_session_decode_timeline
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void prof_begin(unsigned long long *p) { if (p && threadIdx.x == 0) { const unsigned long long t = gtime(); atomicMin(p, t); atomicMax(p + 3 * B200_PROF_SLOTS, t); } }
__device__ __forceinline__ void prof_ready(unsigned long long *p) { if (p && threadIdx.x == 0) { const unsigned long long t = gtime(); atomicMin(p + 2 * B200_PROF_SLOTS, t); atomicMax(p + 4 * B200_PROF_SLOTS, t); } }
__device__ __forceinline__ void prof_end(unsigned long long *p) { if (p && threadIdx.x == 0) atomicMax(p + B200_PROF_SLOTS, gtime()); }

__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// a launch as a programmatic dependent of its predecessor on `st`
template <typename... KArgs, typename... Args>
void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args &&...args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    B200_CHECK(cudaLaunchKernelEx(&cfg, kern, KArgs(args)...));
}

__device__ __forceinline__ float lutf(const uint16_t *t, float x) { return f16_bits_to_f32(__ldg(t + f32_to_f16_bits(x))); }
__device__ __forceinline__ float f16dot_tree(float s) {          // ggml_vec_dot_f16 reduction order, see exact.cu
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 16));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 8));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 4));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 1));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 2));
    return s;
}
// the KV cache's element type KT (__half or float): a float converted to it (f16: rounded to nearest), and one read back as a float
template <typename KT>
__device__ __forceinline__ KT kv_cast(float v) { if constexpr (sizeof(KT) == 2) return __float2half_rn(v); else return v; }
__device__ __forceinline__ float kv_load(__half v) { return __half2float(v); }
__device__ __forceinline__ float kv_load(float v) { return v; }

// ---- 1 / 6: rms_norm * gain -> records.  grid = e/128 CTAs of 256 threads; every CTA reduces the whole row (16 KB from L2) and
//      quantizes its own 4 blocks per warp pass.  STORE (the token's final norm only): each CTA also stores its own float4s of the f32 row to
//      `normed` -- rms_norm, then the separately rounded * gain: the embeddings of OutputRequest (llama lib.rs:343-348). ----------------------
template <bool TP, bool STORE = false>
__device__ __forceinline__ void norm_pack_body(const float *__restrict__ x, const float *__restrict__ gain, int4 *__restrict__ pack,
                                               int e, float eps, int q81, int off, int scale16, unsigned long long *prof, const TpSync &S,
                                               float *__restrict__ normed = nullptr) {
    const TpCtx &T = c_tp;
    __shared__ double shd[8];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_trigger();                                              // 4 CTAs: the next mat-vec fits beside this kernel and streams its first stages meanwhile
    // Tensor-parallel: the row arrives as tagged units and the records this kernel overwrites were last read by a mat-vec whose outputs the producers of
    // those units needed (tp.cuh): nothing here depends on the predecessor grid having COMPLETED, only on its units -- do not wait for its peer stores to be acknowledged.
    if (!(TP && (T.relax & 1))) pdl_wait();
    constexpr bool tp = TP;                                    // tensor-parallel: the row is an array of {value, tag} units filled by every rank (tp.cuh)
    const unsigned tag = tp ? tp_tag(T, S.in_v) : 0u;

    prof_begin(prof);
    // this CTA's 32 blocks are float4s [blockIdx.x * 256, +256) of the row: thread tid packs float4 blockIdx.x * 256 + tid, which is also
    // one of the values it sums -- the row is read once, all loads (row and gains) are in flight before the first use (one L2 round trip)
    const int mine = blockIdx.x * 256 + tid, nv = e / 4;
    const bool active = mine < nv;
    const float4 gv = active ? __ldg((const float4 *)gain + mine) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
    double s = 0.0;
    constexpr int U = 4;
    if (tp && (T.relax & 1)) {                                  // launched ahead of the data: warp 0 watches a sample of the row, the others sleep on the barrier
        if (warp == 0) tp_wait_sample(T, S.in_buf, (int64_t)e, tag, lane);
        __syncthreads();
    }
    for (int i0 = tid; i0 < nv; i0 += 256 * U) {
        float4 v[U];
        if (!tp) {
#pragma unroll
            for (int k = 0; k < U; k++) { const int i = i0 + 256 * k; v[k] = i < nv ? __ldcg((const float4 *)x + i) : make_float4(0.f, 0.f, 0.f, 0.f); }   // written by a predecessor: L2-coherent load
        } else {                                                // float4 i = units 4i .. 4i+3 = pairs 2i, 2i+1: all loads first, then the tag checks
            uint4 ra[U], rb[U];
#pragma unroll
            for (int k = 0; k < U; k++) { const int i = i0 + 256 * k; if (i < nv) { ra[k] = tp_ld2(T, S.in_buf, 2 * (int64_t)i); rb[k] = tp_ld2(T, S.in_buf, 2 * (int64_t)i + 1); } }
#pragma unroll
            for (int k = 0; k < U; k++) {
                const int i = i0 + 256 * k;
                if (i < nv) {
                    tp_fix2(T, S.in_buf, 2 * (int64_t)i, tag, ra[k]); tp_fix2(T, S.in_buf, 2 * (int64_t)i + 1, tag, rb[k]);
                    v[k] = make_float4(__uint_as_float(ra[k].x), __uint_as_float(ra[k].z), __uint_as_float(rb[k].x), __uint_as_float(rb[k].z));
                } else v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int k = 0; k < U; k++) {
            if (i0 + 256 * k == mine) xv = v[k];
            s += (double)__fmul_rn(v[k].x, v[k].x); s += (double)__fmul_rn(v[k].y, v[k].y); s += (double)__fmul_rn(v[k].z, v[k].z); s += (double)__fmul_rn(v[k].w, v[k].w);
        }
    }
    s = warp_sum(s);
    if (lane == 0) shd[warp] = s;
    __syncthreads();
    double tot = ((shd[0] + shd[1]) + (shd[2] + shd[3])) + ((shd[4] + shd[5]) + (shd[6] + shd[7]));
    if (!row_sum_settled(tot, tot, e)) {                        // every CTA has the same tot, so every CTA takes this branch
        tot = row_sum_in_order(e, [=](int64_t i) {
            float v;
            if constexpr (!TP) v = __ldcg(x + i);
            else {                                              // units this CTA's first pass has seen tagged (before the barrier)
                const uint4 u = tp_ld2(T, S.in_buf, i >> 1);
                v = __uint_as_float(i & 1 ? u.z : u.x);
            }
            return (double)__fmul_rn(v, v);
        });
    }
    const float mean = (float)(tot / (double)e);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, eps)));
    float4 v;
    v.x = __fmul_rn(__fmul_rn(xv.x, scale), gv.x); v.y = __fmul_rn(__fmul_rn(xv.y, scale), gv.y);
    v.z = __fmul_rn(__fmul_rn(xv.z, scale), gv.z); v.w = __fmul_rn(__fmul_rn(xv.w, scale), gv.w);
    if constexpr (STORE) if (active) ((float4 *)normed)[mine] = v;
    pack_quad(v, pack + (active ? mine >> 3 : 0) * 4, lane, active, q81, off, scale16);
    prof_end(prof);
}
// Two entry points: the single-GPU kernel does not carry the 24 bytes of TpSync, so its argument block stays inside ONE 64-byte line of the constant bank
// (56 B; with them, 80 B, every one of the 64 launches per token reads one more line).
__global__ void __launch_bounds__(256) norm_pack_kernel(const float *__restrict__ x, const float *__restrict__ gain, int4 *__restrict__ pack,
                                                        int e, float eps, int q81, int off, int scale16, unsigned long long *prof) {
    norm_pack_body<false>(x, gain, pack, e, eps, q81, off, scale16, prof, TpSync{});
}
__global__ void __launch_bounds__(256) norm_pack_tp_kernel(const float *__restrict__ x, const float *__restrict__ gain, int4 *__restrict__ pack,
                                                           int e, float eps, int q81, int off, int scale16, unsigned long long *prof, const TpSync S) {
    norm_pack_body<true>(x, gain, pack, e, eps, q81, off, scale16, prof, S);
}
// the final norm of a single-GPU token: norm_pack_kernel's records, and the f32 row in `normed` (8 more bytes: the block is still one 64-byte line)
__global__ void __launch_bounds__(256) norm_pack_store_kernel(const float *__restrict__ x, const float *__restrict__ gain, int4 *__restrict__ pack,
                                                              int e, float eps, int q81, int off, int scale16, unsigned long long *prof,
                                                              float *__restrict__ normed) {
    norm_pack_body<false, true>(x, gain, pack, e, eps, q81, off, scale16, prof, TpSync{}, normed);
}

// ---- mat-vec with fused epilogues --------------------------------------------------------------------------------------------------
// BIAS / GELU: GPT-NeoX (bias adds, gelu table); GELU_NB: gelu without a bias node (MPT); QKV_F32: EPI_QKV storing K / V into an f32 cache
enum { EPI_RES = 0, EPI_QKV = 1, EPI_SILU = 2, EPI_LOGITS = 3, EPI_BIAS = 4, EPI_GELU = 5, EPI_GELU_NB = 6, EPI_QKV_F32 = 7 };

struct MmvArgs {
    const int4 *xpack;            // input records
    float *dst; const float *addend;                       // EPI_RES / EPI_LOGITS
    // Two pointer groups that no launch uses together share their 32 bytes: the argument block (QWeight 72 B + this struct) then stays within four 64-byte
    // lines of the constant bank (248 B; 280 B with both groups, one more line read on every launch of the decode graph).
    union {
        struct { float *q; void *K, *V; const float2 *rope_cs; };                              // EPI_QKV / EPI_QKV_F32 (LLaMA: RoPE + KV store)
        // EPI_BIAS: dst = ((W x + bias) [+ add1]) [+ add2] in that order (ggml_add nodes of gptneox lib.rs:200,302,308-325); EPI_GELU: gelu(W x + bias) quantized
        struct { const float *bias, *add1, *add2; const uint16_t *lut_gelu; };
    };
    int rope_half, hd, e, gqa, n_ctx; const int *n_past;                                      // EPI_QKV / EPI_QKV_F32
    // EPI_SILU
    int4 *xpack_out; const uint16_t *lut_silu;
    int q81, off, scale16;
    int *n_past_inc;              // EPI_LOGITS: the last node of the token increments InferenceSession::n_past on the device
    int nst;                      // ring depth chosen by mmv_plan
    unsigned long long *prof;
    // tensor-parallel decode (tp.cuh): this rank owns rows [row0, row0 + w.N) of the full matrix; results go to buffer dst_buf of every rank
    TpSync ts; int64_t row0;
};
static_assert(sizeof(QWeight) + sizeof(MmvArgs) <= 256, "mat-vec argument block: at most four 64-byte lines of the constant bank (see the union above)");

template <int TYPE, int EPI, bool TP>
__global__ void __launch_bounds__(STHREADS) mmv_fused_kernel(const QWeight w, const MmvArgs A) {
    using T = St<TYPE>;
    extern __shared__ __align__(128) uint8_t smem[];
    Ring R{(uint64_t *)smem, (uint64_t *)smem + SST_MAX, smem + 256, 0u, (uint32_t)A.nst};
    int4 *sx = (int4 *)(R.base + T::ring_bytes(A.nst));
    const int tid = threadIdx.x;
    constexpr int G = EPI == EPI_SILU ? 2 : 1;
    prof_begin(A.prof);
    if (tid == 0) ring_init(R.full, R.empty, A.nst);
    __syncthreads();
    if (tid >= SCOMPUTE) {                                      // weights only: runs ahead of the predecessors
        produce_matvec<TYPE>(w, R, blockIdx.x, gridDim.x, tid & 31, G);
        pdl_trigger();                                          // every byte of this CTA is requested: let the successor's CTAs take the free slots
        return;
    }
    if (!(TP && (c_tp.relax & 2) && A.ts.in_buf >= 0)) pdl_wait();    // records and addend arrive as tagged units: no dependence on the predecessor's completion (tp.cuh)
    if (TP && A.ts.in_buf >= 0) {                 // tensor-parallel: the input records arrive from every rank as {word, tag} units (tp.cuh)
        const unsigned tag = tp_tag(c_tp, A.ts.in_v);
        if (c_tp.relax & 2) {                                   // launched ahead of the data: warp 0 watches a sample, the others sleep on the barrier
            if (tid < 32) tp_wait_sample(c_tp, A.ts.in_buf, (int64_t)w.nb * 16, tag, tid);
            compute_sync();
        }
        const int npair = (int)w.nb * 8;                        // a 16-byte record = 4 units = 2 pairs
        constexpr int U = 8;                                    // 16-byte loads in flight per thread
        for (int i0 = tid; i0 < npair; i0 += SCOMPUTE * U) {
            uint4 v[U];
#pragma unroll
            for (int k = 0; k < U; k++) { const int i = i0 + k * SCOMPUTE; if (i < npair) v[k] = tp_ld2(c_tp, A.ts.in_buf, i); }
#pragma unroll
            for (int k = 0; k < U; k++) {
                const int i = i0 + k * SCOMPUTE;
                if (i < npair) { tp_fix2(c_tp, A.ts.in_buf, i, tag, v[k]); ((uint2 *)sx)[i] = make_uint2(v[k].x, v[k].z); }
            }
        }
    } else {
        for (int i = tid; i < (int)w.nb * 4; i += SCOMPUTE) cp16(smem_u32(sx + i), A.xpack + i);   // all 16-byte copies in flight at once
        asm volatile("cp.async.wait_all;" ::: "memory");
    }
    float *stash = (float *)(sx + (size_t)w.nb * 4);      // 64 floats behind the records (EPI_SILU)
    compute_sync();
    prof_ready(A.prof);
    const int lane = tid & 31, warp = tid >> 5;
    if (EPI == EPI_RES || EPI == EPI_LOGITS) {
        consume_matvec<TYPE>(w, sx, R, blockIdx.x, gridDim.x, tid, [&](int64_t row, float v) {
            if ((tid & 3) != 0 || row >= w.N) return;
            const int64_t g = A.row0 + row;                      // row of the full matrix (row0 = 0 on a single GPU)
            if (TP) {                                            // addend: this rank's own slice of the gathered vector; result: to every rank
                const float out = A.ts.add_buf >= 0 ? __fadd_rn(v, tp_get_f32(c_tp, A.ts.add_buf, g, tp_tag(c_tp, A.ts.add_v))) : v;
                tp_put_f32(c_tp, A.ts.out_buf, g, out, tp_tag(c_tp, A.ts.out_v));
            } else A.dst[g] = A.addend ? __fadd_rn(v, __ldcg(A.addend + g)) : v;
        }, 1, A.prof);
        if (EPI == EPI_LOGITS && blockIdx.x == 0 && tid == 0) *A.n_past_inc = *A.n_past_inc + 1;
    } else if (EPI == EPI_QKV || EPI == EPI_QKV_F32) {
        const int p = __ldcg(A.n_past);
        consume_matvec<TYPE>(w, sx, R, blockIdx.x, gridDim.x, tid, [&](int64_t row, float v) {
            const float other = __shfl_xor_sync(0xffffffffu, v, 4);              // rotation partner: rows 2i, 2i+1 sit in adjacent quads
            if ((tid & 3) != 0 || row >= w.N) return;
            if (row < A.e + A.gqa) {                                               // ggml_rope mode 0 (LC/ggml.c:11859-11874)
                const int within = (int)(row < A.e ? row : row - A.e);
                const float2 cs = __ldg(A.rope_cs + (int64_t)p * A.rope_half + (within % A.hd) / 2);
                const bool even = (row & 1) == 0;
                const float x0 = even ? v : other, x1 = even ? other : v;
                const float out = even ? __fmaf_rn(x0, cs.x, -__fmul_rn(x1, cs.y)) : __fmaf_rn(x0, cs.y, __fmul_rn(x1, cs.x));
                if (row < A.e) A.q[row] = out;
                else if (EPI == EPI_QKV) ((__half *)A.K)[(int64_t)p * A.gqa + within] = __float2half_rn(out);
                else ((float *)A.K)[(int64_t)p * A.gqa + within] = out;
            } else {
                if (EPI == EPI_QKV) ((__half *)A.V)[(int64_t)(row - A.e - A.gqa) * A.n_ctx + p] = __float2half_rn(v);
                else ((float *)A.V)[(int64_t)(row - A.e - A.gqa) * A.n_ctx + p] = v;
            }
        });
    } else if (EPI == EPI_BIAS) {
        consume_matvec<TYPE>(w, sx, R, blockIdx.x, gridDim.x, tid, [&](int64_t row, float v) {
            if ((tid & 3) != 0 || row >= w.N) return;
            float out = A.bias ? __fadd_rn(v, __ldg(A.bias + row)) : v;
            if (A.add1) out = __fadd_rn(out, __ldcg(A.add1 + row));
            if (A.add2) out = __fadd_rn(out, __ldcg(A.add2 + row));
            A.dst[row] = out;
        }, 1, A.prof);
        if (A.n_past_inc && blockIdx.x == 0 && tid == 0) *A.n_past_inc = *A.n_past_inc + 1;
    } else if (EPI == EPI_GELU || EPI == EPI_GELU_NB) {   // one 32-row tile = one quant block of the next mat-vec's input (rows past N: zero activations)
        consume_matvec<TYPE>(w, sx, R, blockIdx.x, gridDim.x, tid, [&](int64_t row, float v) {
            if ((tid & 3) == 0) stash[row & 31] = row < w.N ? (EPI == EPI_GELU ? __fadd_rn(v, __ldg(A.bias + row)) : v) : 0.f;
            compute_sync();
            if (warp == 0) {
                const float4 a = ((const float4 *)stash)[lane & 7];
                float4 hm;
                hm.x = lutf(A.lut_gelu, a.x); hm.y = lutf(A.lut_gelu, a.y); hm.z = lutf(A.lut_gelu, a.z); hm.w = lutf(A.lut_gelu, a.w);
                pack_quad(hm, A.xpack_out + (row >> 5) * 4, lane, lane < 8, A.q81, A.off, A.scale16);
            }
            compute_sync();
        }, 1, A.prof);
    } else {   // EPI_SILU
        consume_matvec<TYPE>(w, sx, R, blockIdx.x, gridDim.x, tid, [&](int64_t row, float v) {
            if ((tid & 3) == 0) stash[row & 63] = v;
            if (((row >> 5) & 1) == 0) return;
            compute_sync();
            if (warp == 0) {
                const int w8 = lane & 7;
                const float4 a = ((const float4 *)stash)[w8], b = ((const float4 *)stash)[8 + w8];
                float4 hm;
                hm.x = __fmul_rn(lutf(A.lut_silu, a.x), b.x); hm.y = __fmul_rn(lutf(A.lut_silu, a.y), b.y);
                hm.z = __fmul_rn(lutf(A.lut_silu, a.z), b.z); hm.w = __fmul_rn(lutf(A.lut_silu, a.w), b.w);
                const int64_t blk = (A.row0 >> 6) + (row >> 6);     // block of w2's input (row0 counts this rank's interleaved w1|w3 rows)
                int4 rec;
                if (pack_quad_rec(hm, lane, lane < 8, A.q81, A.off, A.scale16, rec)) {
                    if (TP) tp_put_rec(c_tp, TPB_XF, blk * 4 + (lane & 7), rec, tp_tag(c_tp, A.ts.out_v)); else A.xpack_out[blk * 4 + (lane & 7)] = rec;
                }
            }
            compute_sync();
        }, G, A.prof);
    }
    pdl_trigger();                                              // late: this CTA has consumed its last tile
    prof_end(A.prof);
}

// ---- 3: KQ.  CTA = (64 cached positions, head); CTAs past n_kv exit at once (the grid is sized for the context bucket).  All
//      16-byte loads of the K tile are issued before the first one is consumed.
//      KT, the cache's element type: f16 rounds q to f16 (ggml_vec_dot_f16); f32 takes q as it is (ggml_vec_dot_f32: the chains and tree of
//      the f16 dot; hd % 32 == 0 leaves no leftovers). ------------------------------------------------------------------------------------
template <int HD, typename KT>
__global__ void __launch_bounds__(128) attn_kq_kernel(const float *__restrict__ q, const KT *__restrict__ Kl, float *__restrict__ kq,
                                                      const int *__restrict__ n_past, int gqa, int n_head, int n_head_kv, int n_ctx, unsigned long long *prof) {
    __shared__ __align__(16) KT qs[HD];
    __shared__ __align__(16) KT kt[64 * HD];
    pdl_trigger();
    pdl_wait();
    prof_begin(prof);
    const int n_kv = __ldcg(n_past) + 1;
    const int j0 = blockIdx.x * 64, h = blockIdx.y;
    if (j0 >= n_kv) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int hk = h / (n_head / n_head_kv);
    const int rows = n_kv - j0 < 64 ? n_kv - j0 : 64;
    constexpr int VPR = HD * (int)sizeof(KT) / 16;    // 16-byte vectors per K row
    constexpr int NV = 64 * VPR / 128;                // vectors per thread
    int4 v[NV];
#pragma unroll
    for (int u = 0; u < NV; u++) {
        const int i = tid + u * 128, rr = i / VPR, cc = i % VPR;
        v[u] = rr < rows ? __ldcg((const int4 *)(Kl + (int64_t)(j0 + rr) * gqa + hk * HD) + cc) : make_int4(0, 0, 0, 0);
    }
    for (int i = tid; i < HD; i += 128) qs[i] = kv_cast<KT>(__ldcg(q + h * HD + i));
#pragma unroll
    for (int u = 0; u < NV; u++) ((int4 *)kt)[tid + u * 128] = v[u];
    __syncthreads();
    for (int jj = warp; jj < rows; jj += 4) {
        const KT *krow = kt + jj * HD;
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < HD; k += 32) s = __fmaf_rn(kv_load(krow[k + lane]), kv_load(qs[k + lane]), s);
        s = f16dot_tree(s);                           // GGML_F32x8_REDUCE is the same tree
        if (lane == 0) kq[(int64_t)h * n_ctx + j0 + jj] = s;
    }
    prof_end(prof);
}

// ---- 4: scale + soft_max + KQV for 32 channels of one head, then quantize those 32 outputs (one block of wo's input) ---------------
//      KT, the cache's element type, is also that of the probabilities (f16: rounded, ggml_vec_dot_f16).  V tiles are 32 rows of 256 bytes
//      (KC = 128 f16 or 64 f32 positions: 4 vectors per thread); the positions past the last whole 32 are added in double (f16) or by the
//      f32 leftover rule (f32dot.cuh).  Dynamic shared memory: scores and probabilities for the whole context, a V tile, 32 leftover columns.
constexpr int KC = 128;
constexpr size_t attn_sv_smem(int n_ctx, int kv_type) {
    const size_t es = kv_type == T_F32 ? 4 : 2;
    return (size_t)n_ctx * (4 + es) + 32 * KC * 2 + 32 * 32 * es;
}
template <typename KT>
__global__ void __launch_bounds__(128) attn_sv_kernel(const float *__restrict__ kq, const KT *__restrict__ Vl, int4 *__restrict__ xpack_out,
                                                      const int *__restrict__ n_past, const uint16_t *__restrict__ lut_exp, float kq_scale,
                                                      int hd, int n_head, int n_head_kv, int n_ctx, int q81, int off, int scale16, unsigned long long *prof) {
    constexpr bool F32 = sizeof(KT) == 4;
    constexpr int TC = KC * 2 / (int)sizeof(KT);      // positions per V tile
    constexpr int TV = TC * (int)sizeof(KT) / 16;     // 16-byte vectors per row of a tile
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ double shd[8];
    __shared__ float shf[4], stash[32];
    pdl_trigger();
    pdl_wait();
    prof_begin(prof);
    const int n_kv = __ldcg(n_past) + 1;
    const int per_head = hd / 32, h = blockIdx.x / per_head, c0 = (blockIdx.x - h * per_head) * 32;
    const int hk = h / (n_head / n_head_kv);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float *sc = (float *)sm;
    KT *p = (KT *)(sm + (size_t)n_ctx * 4);
    KT *vt = (KT *)(sm + (size_t)n_ctx * (4 + sizeof(KT)));
    KT *vleft = vt + 32 * TC;
    // leftover V columns and the first V tile are requested before anything else so that their latency hides behind the soft_max
    const int np = n_kv & ~31;
    if (np < n_kv) {
        if constexpr (F32) {
            constexpr int VL = 8;                     // 16-byte vectors of 32 positions
#pragma unroll
            for (int i = tid; i < 32 * VL; i += 128) ((int4 *)vleft)[i] = __ldcg((const int4 *)(Vl + (int64_t)(hk * hd + c0 + i / VL) * n_ctx + np) + i % VL);
        } else {
            const int rr = tid >> 2, part = tid & 3;
            ((int4 *)vleft)[tid] = __ldcg((const int4 *)(Vl + (int64_t)(hk * hd + c0 + rr) * n_ctx + np) + part);
        }
    }
    int4 pre[32 * TV / 128];
    auto fetch = [&](int k0) {
#pragma unroll
        for (int u = 0; u < 32 * TV / 128; u++) {
            const int i = tid + u * 128, rr = i / TV, cc = i - rr * TV;
            pre[u] = __ldcg((const int4 *)(Vl + (int64_t)(hk * hd + c0 + rr) * n_ctx + k0) + cc);
        }
    };
    if (np > 0) fetch(0);
    float mx = -INFINITY;
    constexpr int SB = 8;                              // scores per thread per pass: 8 loads in flight
    for (int jb = 0; jb < n_kv; jb += SB * 128) {
        float sv[SB];
#pragma unroll
        for (int u = 0; u < SB; u++) { const int j = jb + tid + u * 128; sv[u] = j < n_kv ? __ldcg(kq + (int64_t)h * n_ctx + j) : 0.f; }
#pragma unroll
        for (int u = 0; u < SB; u++) { const int j = jb + tid + u * 128; if (j < n_kv) { const float v = __fmul_rn(sv[u], kq_scale); sc[j] = v; mx = fmaxf(mx, v); } }
    }
    mx = warp_max(mx);
    if (lane == 0) shf[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(shf[0], shf[1]), fmaxf(shf[2], shf[3]));
    double s = 0.0;
    for (int jb = 0; jb < n_kv; jb += SB * 128) {
        uint16_t ev16[SB];
#pragma unroll
        for (int u = 0; u < SB; u++) { const int j = jb + tid + u * 128; ev16[u] = j < n_kv ? __ldg(lut_exp + f32_to_f16_bits(__fsub_rn(sc[j], mx))) : (uint16_t)0; }
#pragma unroll
        for (int u = 0; u < SB; u++) { const int j = jb + tid + u * 128; if (j < n_kv) { const float ev = f16_bits_to_f32(ev16[u]); sc[j] = ev; s += (double)ev; } }
    }
    s = warp_sum(s);
    if (lane == 0) shd[warp] = s;
    __syncthreads();
    const float inv = (float)(1.0 / ((shd[0] + shd[1]) + (shd[2] + shd[3])));
    for (int j = tid; j < n_kv; j += 128) p[j] = kv_cast<KT>(__fmul_rn(sc[j], inv));
    float acc[8];
#pragma unroll
    for (int cc = 0; cc < 8; cc++) acc[cc] = 0.f;
    for (int k0 = 0; k0 < np; k0 += TC) {
        __syncthreads();
#pragma unroll
        for (int u = 0; u < 32 * TV / 128; u++) ((int4 *)vt)[tid + u * 128] = pre[u];
        __syncthreads();
        if (k0 + TC < np) fetch(k0 + TC);
        const int kend = np - k0 < TC ? np - k0 : TC;
#pragma unroll
        for (int cc = 0; cc < 8; cc++) {
            const KT *vrow = vt + (warp * 8 + cc) * TC;
            for (int k = lane; k < kend; k += 32) acc[cc] = __fmaf_rn(kv_load(vrow[k]), kv_load(p[k0 + k]), acc[cc]);
        }
    }
    __syncthreads();
#pragma unroll
    for (int cc = 0; cc < 8; cc++) {
        const float a = f16dot_tree(acc[cc]);
        if (lane == 0) {
            const KT *vrow = vleft + (warp * 8 + cc) * 32;
            if constexpr (F32) {
                stash[warp * 8 + cc] = f32_leftovers(a, n_kv - np, [&](int i) { return vrow[i]; }, [&](int i) { return p[np + i]; });
            } else {
                double sumf = (double)a;
                for (int k = np; k < n_kv; k++) sumf += (double)__fmul_rn(__half2float(vrow[k - np]), __half2float(p[k]));
                stash[warp * 8 + cc] = (float)sumf;
            }
        }
    }
    __syncthreads();
    if (warp == 0) pack_quad(((const float4 *)stash)[lane & 7], xpack_out + (int64_t)((h * hd + c0) / QK) * 4, lane, lane < 8, q81, off, scale16);
    prof_end(prof);
}

// ---- 3+4 fused: KQ, scale, soft_max, KQV and the quantize epilogue for one head, as ONE cluster of hd/32 CTAs ----------------------------
// CTA `part` of the cluster owns 32 channels of the head (its V rows are staged by cp.async at kernel entry, long before they are needed)
// and 1/(hd/32) of the cached positions for KQ; the scaled scores are written straight into every CTA's shared memory (DSMEM) and one
// cluster barrier later each CTA runs the soft_max on the full row and its own 32 KQV dots.  No global round trip between the phases.
//
// ggml_vec_dot_f16 (LC/ggml.c:1573-1610) keeps 32 f32 chains, chain l over elements k = l (mod 32); here thread u (0..3) of a quad owns
// chains 8u..8u+7 of one dot, so every load is a 16-byte vector, and the reduction tree (offsets 16, 8, 4, 1, 2) is two quad shuffles plus
// in-thread adds in exactly that association.
__device__ __forceinline__ float quad_tree(float (&acc)[8]) {
#pragma unroll
    for (int e = 0; e < 8; e++) acc[e] = __fadd_rn(acc[e], __shfl_xor_sync(0xffffffffu, acc[e], 2));     // chain l += chain l + 16
#pragma unroll
    for (int e = 0; e < 8; e++) acc[e] = __fadd_rn(acc[e], __shfl_xor_sync(0xffffffffu, acc[e], 1));     // l += l + 8   (valid in u == 0)
    const float r0 = __fadd_rn(acc[0], acc[4]), r1 = __fadd_rn(acc[1], acc[5]), r2 = __fadd_rn(acc[2], acc[6]), r3 = __fadd_rn(acc[3], acc[7]);   // l += l + 4
    return __fadd_rn(__fadd_rn(r0, r1), __fadd_rn(r2, r3));                                                // down 1, down 2
}
__device__ __forceinline__ void fma8(float (&acc)[8], const int4 &a, const int4 &b) {
    const __half2 *ah = (const __half2 *)&a, *bh = (const __half2 *)&b;
#pragma unroll
    for (int e = 0; e < 4; e++) {
        const float2 af = __half22float2(ah[e]), bf = __half22float2(bh[e]);
        acc[2 * e] = __fmaf_rn(af.x, bf.x, acc[2 * e]); acc[2 * e + 1] = __fmaf_rn(af.y, bf.y, acc[2 * e + 1]);
    }
}
// the f32 cache's form: chains 8u..8u+7 of a 32-element step are two 16-byte vectors of each operand
__device__ __forceinline__ void fma8(float (&acc)[8], const int4 &a0, const int4 &a1, const float4 &b0, const float4 &b1) {
    const float4 x0 = *(const float4 *)&a0, x1 = *(const float4 *)&a1;
    acc[0] = __fmaf_rn(x0.x, b0.x, acc[0]); acc[1] = __fmaf_rn(x0.y, b0.y, acc[1]); acc[2] = __fmaf_rn(x0.z, b0.z, acc[2]); acc[3] = __fmaf_rn(x0.w, b0.w, acc[3]);
    acc[4] = __fmaf_rn(x1.x, b1.x, acc[4]); acc[5] = __fmaf_rn(x1.y, b1.y, acc[5]); acc[6] = __fmaf_rn(x1.z, b1.z, acc[6]); acc[7] = __fmaf_rn(x1.w, b1.w, acc[7]);
}

//
// ALIBI (MPT, BLOOM): the score of key position j in head h is fma(j, slope[h], kq * kq_scale) -- ggml_alibi (LC/ggml.c:11534-11597) on the
// scaled scores, one fused multiply-add as the reference's x86 build compiles it; the slopes come from alibi_slopes() on the host.
//
// NV: the most 32-element steps per position and quad thread (hd / 32).  4 serves hd <= 128 (clusters of up to 4 CTAs); 8 serves hd <= 256 (GPT-J's
// 256-wide heads, clusters of up to 8 CTAs, the portable limit) and halves the positions per pass, so kv[PU][NV * CW] stays 16 int4 per thread.
//
// KT = float (an f32 cache, ggml_vec_dot_f32): a step of a quad thread is two 16-byte K vectors (CW = 2, so half the positions per pass); q and
// the probabilities stay f32 in shared memory, the V rows take twice the bytes, and the KQV leftovers are added in float (f32dot.cuh).
//
// TP: the merged row goes to every rank's exchange buffer (tp.cuh); head0 is this rank's first head.  alibi: the per-head slopes [n_head], read
// only by the ALIBI instances.  The instances that launch are listed in attn_fused_instances.
constexpr int ATH = 256;
template <bool TP, bool ALIBI, int NV, typename KT>
__global__ void __launch_bounds__(ATH) attn_fused_kernel(const float *__restrict__ q, const KT *__restrict__ Kl, const KT *__restrict__ Vl,
                                                         int4 *__restrict__ xpack_out, const int *__restrict__ n_past, const uint16_t *__restrict__ lut_exp,
                                                         float kq_scale, int hd, int n_head, int n_head_kv, int gqa, int n_ctx, int nlay, int q81, int off, int scale16,
                                                         unsigned long long *prof, const TpSync S, int head0, const float *__restrict__ alibi) {
    const TpCtx &T = c_tp;
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ double shd[ATH / 32];
    __shared__ float shf[ATH / 32], stash[32];
    prof_begin(prof);
    const int per_head = hd / 32, h = blockIdx.x / per_head, part = blockIdx.x - h * per_head, c0 = part * 32;
    const int hk = h / (n_head / n_head_kv);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, u = tid & 3;
    constexpr bool F32 = sizeof(KT) == 4;
    constexpr int CW = F32 ? 2 : 1;                              // 16-byte K vectors per 32-element step and quad thread
    constexpr int PER16 = 16 / (int)sizeof(KT);                 // cache elements per 16-byte chunk
    // shared-memory layout for nlay >= n_kv positions (the context bucket the graph was captured for, a multiple of 64: small enough that the
    // next mat-vec's CTAs fit beside this kernel's and stream their weights while it runs)
    // f16: (nlay + 32) * 2 B = 64 B mod 128 B; f32: (nlay + 4) * 4 B = 16 B mod 128 B -- either way the two columns of a quarter-warp hit different banks
    const int vstride = F32 ? nlay + 4 : nlay + 32;             // elements
    float *sc = (float *)sm;
    KT *p16 = (KT *)(sm + (size_t)nlay * 4);
    KT *q16 = p16 + nlay;
    KT *vs = (KT *)(sm + (((size_t)nlay * (4 + sizeof(KT)) + (size_t)hd * sizeof(KT) + 127) & ~(size_t)127));
    pdl_trigger();                                              // the successor (wo) only needs shared memory beside us: let it prefetch its tiles now
    // Ahead of the wait: n_past and the KV cache below it.  Of these, this token's kernels write only cache position n_past of each layer (the
    // qkv node).  The older positions were written by earlier tokens or the prefill, n_past by the previous token's last kernel or by a
    // stream-ordered copy after a rewind -- all of it complete before this token's first kernel (the embedding row, a plain stream-ordered launch
    // without the programmatic attribute, decode_ops_t / neox_ops_t) starts, and so before any kernel chained behind it by PDL, this one included.
    // So the old cache -- the whole HBM traffic of this kernel -- streams while the qkv node still runs; q, the K row at n_past and the V chunk
    // holding it are read after the wait.
    const int p = __ldcg(n_past), n_kv = p + 1;
    const int np = n_kv & ~31;
    const int64_t vrow0 = (int64_t)(hk * hd + c0) * n_ctx;
    const int cold = p / PER16;                                  // 16-byte V chunks per row wholly before position p
    for (int i = tid; i < 32 * cold; i += ATH) {                 // V rows of this CTA's 32 channels: consumed after the soft_max
        const int rr = i / cold, cc = i - rr * cold;
        cp16(smem_u32(vs + rr * vstride + cc * PER16), Vl + vrow0 + (int64_t)rr * n_ctx + cc * PER16);
    }
    const int per = (n_kv + per_head - 1) / per_head, j0 = part * per, j1 = n_kv < j0 + per ? n_kv : j0 + per;   // this CTA's KQ positions
    const int nvec = hd / 32;                                    // 32-element steps per position (i = 0..nvec-1), CW 16-byte loads each
    constexpr int PU = 16 / (NV * CW);                           // positions per quad per pass: up to PU * nvec * CW 16-byte loads in flight per thread
    int4 kv[PU][NV * CW];
    auto krow_of = [&](int j) { return Kl + (int64_t)(j < j1 ? j : j0) * gqa + hk * hd + 8 * u; };
#pragma unroll
    for (int pu = 0; pu < PU; pu++) {                            // the first pass's K rows below p
        const int j = j0 + pu * (ATH / 4) + (tid >> 2);
        const KT *krow = krow_of(j);
#pragma unroll
        for (int i = 0; i < NV; i++)
#pragma unroll
            for (int c = 0; c < CW; c++)
                if (i < nvec) kv[pu][i * CW + c] = j < j1 && j < p ? __ldcg((const int4 *)(krow + 32 * i) + c) : make_int4(0, 0, 0, 0);
    }
    pdl_wait();
    float qv = 0.f;
    if (tid < hd) qv = __ldcg(q + h * hd + tid);               // hd <= 256 = ATH
    if (tid < 32) cp16(smem_u32(vs + tid * vstride + cold * PER16), Vl + vrow0 + (int64_t)tid * n_ctx + cold * PER16);
#pragma unroll
    for (int pu = 0; pu < PU; pu++) {
        const int j = j0 + pu * (ATH / 4) + (tid >> 2);
        if (j == p && j < j1) {
            const KT *krow = krow_of(j);
#pragma unroll
            for (int i = 0; i < NV; i++)
#pragma unroll
                for (int c = 0; c < CW; c++)
                    if (i < nvec) kv[pu][i * CW + c] = __ldcg((const int4 *)(krow + 32 * i) + c);
        }
    }
    if constexpr (F32) { if (tid < hd) q16[tid] = qv; }         // ggml_vec_dot_f32: q as it is
    else { if (tid < hd) q16[tid] = __float2half_rn(qv); }
    // q16 visible inside the CTA; every CTA of the cluster is running before its shared memory is written remotely (no data is exchanged
    // yet, so the cluster barrier can be the relaxed one: no fence)
    __syncthreads();
    asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");

    // ---- KQ for this CTA's share of the positions ----
    {
        const float slope = ALIBI ? __ldg(alibi + h) : 0.f;
        for (int jb = j0; jb < j1; jb += PU * (ATH / 4)) {
            if (jb != j0) {                                      // later passes (contexts beyond PU * ATH / 4 positions per CTA)
#pragma unroll
                for (int pu = 0; pu < PU; pu++) {
                    const int j = jb + pu * (ATH / 4) + (tid >> 2);
                    const KT *krow = krow_of(j);
#pragma unroll
                    for (int i = 0; i < NV; i++)
#pragma unroll
                        for (int c = 0; c < CW; c++)
                            if (i < nvec) kv[pu][i * CW + c] = j < j1 ? __ldcg((const int4 *)(krow + 32 * i) + c) : make_int4(0, 0, 0, 0);
                }
            }
#pragma unroll
            for (int pu = 0; pu < PU; pu++) {
                const int j = jb + pu * (ATH / 4) + (tid >> 2);
                float acc[8];
#pragma unroll
                for (int e = 0; e < 8; e++) acc[e] = 0.f;
#pragma unroll
                for (int i = 0; i < NV; i++) {
                    if constexpr (F32) { if (i < nvec) fma8(acc, kv[pu][2 * i], kv[pu][2 * i + 1], *(const float4 *)(q16 + 32 * i + 8 * u), *(const float4 *)(q16 + 32 * i + 8 * u + 4)); }
                    else { if (i < nvec) fma8(acc, kv[pu][i], *(const int4 *)(q16 + 32 * i + 8 * u)); }
                }
                const float s = quad_tree(acc);
                if (j < j1 && u < per_head)                      // thread u of the quad feeds CTA u (and CTA u + 4 of a cluster of more than 4)
                    cluster.map_shared_rank(sc, u)[j] = ALIBI ? __fmaf_rn((float)j, slope, __fmul_rn(s, kq_scale)) : __fmul_rn(s, kq_scale);
                if (NV > 4 && j < j1 && u + 4 < per_head)
                    cluster.map_shared_rank(sc, u + 4)[j] = ALIBI ? __fmaf_rn((float)j, slope, __fmul_rn(s, kq_scale)) : __fmul_rn(s, kq_scale);
            }
        }
    }
    cluster.sync();

    // ---- soft_max over sc[0, n_kv) (ggml_compute_forward_soft_max_f32, LC/ggml.c:11700-11770: fp16 exp table, double row sum) ----
    float mx = -INFINITY;
    for (int j = tid; j < n_kv; j += ATH) mx = fmaxf(mx, sc[j]);
    mx = warp_max(mx);
    if (lane == 0) shf[warp] = mx;
    __syncthreads();
    mx = shf[0];
#pragma unroll
    for (int i = 1; i < ATH / 32; i++) mx = fmaxf(mx, shf[i]);
    double s = 0.0;
    constexpr int SB = 4;                                        // table look-ups in flight per thread
    for (int jb = 0; jb < n_kv; jb += SB * ATH) {
        uint16_t ev16[SB];
#pragma unroll
        for (int k = 0; k < SB; k++) { const int j = jb + tid + k * ATH; ev16[k] = j < n_kv ? __ldg(lut_exp + f32_to_f16_bits(__fsub_rn(sc[j], mx))) : (uint16_t)0; }
#pragma unroll
        for (int k = 0; k < SB; k++) { const int j = jb + tid + k * ATH; if (j < n_kv) { const float ev = f16_bits_to_f32(ev16[k]); sc[j] = ev; s += (double)ev; } }
    }
    s = warp_sum(s);
    if (lane == 0) shd[warp] = s;
    __syncthreads();
    const float inv = (float)(1.0 / (((shd[0] + shd[1]) + (shd[2] + shd[3])) + ((shd[4] + shd[5]) + (shd[6] + shd[7]))));
    if constexpr (F32) { for (int j = tid; j < n_kv; j += ATH) p16[j] = __fmul_rn(sc[j], inv); }
    else { for (int j = tid; j < n_kv; j += ATH) p16[j] = __float2half_rn(__fmul_rn(sc[j], inv)); }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();

    // ---- KQV: 32 channels x 4 threads ----
    if (tid < 128) {
        const int col = tid >> 2;
        const KT *vrow = vs + col * vstride;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; e++) acc[e] = 0.f;
        if constexpr (F32) {
#pragma unroll 4
            for (int k = 0; k < np; k += 32)
                fma8(acc, *(const int4 *)(vrow + k + 8 * u), *(const int4 *)(vrow + k + 8 * u + 4), *(const float4 *)(p16 + k + 8 * u), *(const float4 *)(p16 + k + 8 * u + 4));
        } else {
#pragma unroll 4
            for (int k = 0; k < np; k += 32) fma8(acc, *(const int4 *)(vrow + k + 8 * u), *(const int4 *)(p16 + k + 8 * u));
        }
        const float a = quad_tree(acc);
        if (u == 0) {
            if constexpr (F32) {
                stash[col] = f32_leftovers(a, n_kv - np, [&](int i) { return vrow[np + i]; }, [&](int i) { return p16[np + i]; });
            } else {
                double sumf = (double)a;
                for (int k = np; k < n_kv; k++) sumf += (double)__fmul_rn(__half2float(vrow[k]), __half2float(p16[k]));
                stash[col] = (float)sumf;
            }
        }
    }
    __syncthreads();
    if (warp == 0) {
        int4 rec;
        const int64_t blk = (int64_t)(((head0 + h) * hd + c0) / QK);       // block of wo's input: heads are global (head0 = first head of this rank)
        if (pack_quad_rec(((const float4 *)stash)[lane & 7], lane, lane < 8, q81, off, scale16, rec)) {
            if (TP) tp_put_rec(T, TPB_XD, blk * 4 + (lane & 7), rec, tp_tag(T, S.out_v)); else xpack_out[blk * 4 + (lane & 7)] = rec;
        }
    }
    prof_end(prof);
}

// ---- ring and grid plan of the decode mat-vecs ------------------------------------------------------------------------------------------------
// What one CTA takes from an SM while it is resident: shared memory (static + dynamic + the per-CTA reservation), registers as the SM allocates
// them (per warp, in units of 256), threads.  Footprints add up: a + b = both resident on one SM.
struct CtaFootprint {
    int smem = 0, regs = 0, threads = 0, ctas = 0;
    CtaFootprint operator+(const CtaFootprint &o) const { return {smem + o.smem, regs + o.regs, threads + o.threads, ctas + o.ctas}; }
};
struct SmLimits { int sms, smem, reserved, regs, threads, ctas; double hbm_bytes_per_ns; };   // per SM; hbm: the SM's share of the device's peak
const SmLimits &sm_limits() {
    static SmLimits L{};
    if (!L.sms) {
        int dev; B200_CHECK(cudaGetDevice(&dev));
        auto at = [&](cudaDeviceAttr a) { int v; B200_CHECK(cudaDeviceGetAttribute(&v, a, dev)); return v; };
        L.sms = at(cudaDevAttrMultiProcessorCount); L.smem = at(cudaDevAttrMaxSharedMemoryPerMultiprocessor);
        L.reserved = at(cudaDevAttrReservedSharedMemoryPerBlock); L.regs = at(cudaDevAttrMaxRegistersPerMultiprocessor);
        L.threads = at(cudaDevAttrMaxThreadsPerMultiProcessor); L.ctas = at(cudaDevAttrMaxBlocksPerMultiprocessor);
        // memory clock (kHz) x bus width (bits) x 2 (double data rate): 3.35 TB/s on an H100 SXM, 25 GB/s per SM
        L.hbm_bytes_per_ns = (double)at(cudaDevAttrMemoryClockRate) * 1e3 * at(cudaDevAttrGlobalMemoryBusWidth) / 8.0 * 2.0 / 1e9 / L.sms;
    }
    return L;
}
template <typename K>
CtaFootprint footprint_of(K *kern, int threads, size_t dyn_smem) {
    cudaFuncAttributes fa;
    B200_CHECK(cudaFuncGetAttributes(&fa, (const void *)kern));
    const int warps = (threads + 31) / 32;
    return {(int)(fa.sharedSizeBytes + dyn_smem) + sm_limits().reserved, warps * ((fa.numRegs * 32 + 255) / 256 * 256), warps * 32, 1};
}

// Loaded HBM latency one CTA's weight ring has to cover.  Not a device attribute: a figure fitted on one H100 80GB HBM3 at a 400 W power limit,
// where capping every ring of the 7B decode graph at 6 Q4_0 stages (61 KB) streams as fast as 8 or 12, 4 stages is slower, and w13 at 3 stages
// x 2 CTAs per SM takes 1.7x as long: ~2.4 us at that SM's 25 GB/s share (the share itself is derived from the device, sm_limits).
constexpr double kLoadedLatencyNs = 2400.0;

struct MmvPlan { int nst = 0, grid = 0, smem = 0; CtaFootprint cta; };

// the most row groups one SM streams when CTA b runs on SM b mod sms and takes groups b, b + grid, ...  A model, not a guarantee: on an idle
// GPU the block scheduler fills the SMs in CTA order, but CTAs launched under a predecessor's tail land wherever SMs free up first, so with
// CTAs of unequal share (qkv: 264 CTAs, the first 120 with 2 groups) an SM can end up with more than its fair share.  Placement never
// changes results, only how evenly the bytes are spread.
int64_t max_groups_per_sm(int64_t groups, int64_t grid, int sms) {
    int64_t worst = 0;
    for (int s = 0; s < sms && s < grid; s++) {
        int64_t t = 0;
        for (int64_t b = s; b < grid; b += sms) t += (groups - b + grid - 1) / grid;
        worst = t > worst ? t : worst;
    }
    return worst;
}

// Ring depth and grid of one mat-vec, computed once per (matrix shape, successor).  `succ` is what the node launched after this one needs
// on an SM: with room left for it, its CTAs become resident while this kernel's tail runs and start their own loads under it (the mat-vec
// producer warp streams weights ahead of griddepcontrol.wait; the attention kernel the older KV cache).  The plan:
//   * one wave, balanced: no SM streams more row groups than ceil(groups / SMs);
//   * k CTAs per SM plus one successor CTA fit the SM's shared memory, registers, threads and CTA slots;
//   * every CTA's ring, as deep as that room allows, holds at least HBM-share x latency bytes (or the CTA's whole share of the matrix):
//     the depth beyond that lets a node bank weights while its predecessor still runs;
//   * the most CTAs per SM that meet this, and at least 2 where the row groups allow: the four consumer warps of one CTA retire about
//     30 GB/s of Q4_0 weights (wo, w2), barely the SM's HBM share;
//   * if no such plan leaves room for the successor, the plan ignores it.
template <int TYPE, int EPI, bool TP>
const MmvPlan &mmv_plan(const QWeight &w, const CtaFootprint &succ) {
    using T = St<TYPE>;
    auto kern = mmv_fused_kernel<TYPE, EPI, TP>;
    static std::map<std::array<int64_t, 5>, MmvPlan> plans;
    static int smem_set = 0;
    const std::array<int64_t, 5> key{w.N, w.nb, succ.smem, succ.regs, succ.threads};
    auto it = plans.find(key);
    if (it != plans.end()) return it->second;
    const SmLimits &L = sm_limits();
    auto smem_of = [&](int nst) { return 256 + T::ring_bytes(nst) + (int)w.nb * 64 + 256; };
    if (smem_of(SST_MAX) > smem_set) {
        const int want = smem_of(SST_MAX) < 227 * 1024 ? smem_of(SST_MAX) : 227 * 1024;
        B200_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, want));
        smem_set = smem_of(SST_MAX);
    }
    const CtaFootprint base = footprint_of(kern, STHREADS, 0);
    constexpr int G = EPI == EPI_SILU ? 2 : 1;
    const int64_t groups = ((w.N + SR - 1) / SR + G - 1) / G;
    const int chunks = (int)((w.nb + SCB - 1) / SCB) * G;              // ring stages per row group
    const int64_t fair = (groups + L.sms - 1) / L.sms;
    const int min_stages = (int)(L.hbm_bytes_per_ns * kLoadedLatencyNs / T::STAGE_BYTES + 0.999);
    const int min_k = fair < 2 ? (int)fair : 2;
    MmvPlan best;
    for (int pass = 0; pass < 3 && !best.nst; pass++) {              // 2: last resort, any ring that runs
        const CtaFootprint room = pass == 0 ? succ : CtaFootprint{};
        for (int k = (int)(fair < L.ctas ? fair : L.ctas); k >= (pass < 2 ? min_k : 1) && !best.nst; k--) {
            const int64_t grid = groups < (int64_t)L.sms * k ? groups : (int64_t)L.sms * k;
            if (max_groups_per_sm(groups, grid, L.sms) > fair) continue;
            const int per_cta = (int)((groups + grid - 1) / grid) * chunks;
            int nst = 0;
            for (int c = 2; c <= SST_MAX && c <= (per_cta > 2 ? per_cta : 2); c++) {
                if (smem_of(c) > 227 * 1024) break;
                int occ = 0;
                B200_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, STHREADS, smem_of(c)));
                CtaFootprint one = base;
                one.smem += smem_of(c);
                const CtaFootprint all = CtaFootprint{k * one.smem, k * one.regs, k * one.threads, k} + room;
                if (occ < k || all.smem > L.smem || all.regs > L.regs || all.threads > L.threads || all.ctas > L.ctas) break;
                nst = c;
            }
            const int need = pass == 2 ? 2 : std::min({min_stages, per_cta, SST_MAX});
            if (nst < need || nst < 2) continue;
            best.nst = nst; best.grid = (int)grid; best.smem = smem_of(nst);
            best.cta = base; best.cta.smem += best.smem;
        }
    }
    B200_ASSERT(best.nst > 0);
    return plans.emplace(key, best).first->second;
}

template <int TYPE, int EPI, bool TP = false>
void launch_mmv(const QWeight &w, MmvArgs A, const MmvPlan &plan, cudaStream_t st) {
    A.nst = plan.nst;
    launch_k(mmv_fused_kernel<TYPE, EPI, TP>, dim3((unsigned)plan.grid), dim3(STHREADS), (size_t)plan.smem, st, w, A);
}

// The instances of attn_fused_kernel that launch, in one list: attn_fused_pick chooses from it and attn_fused_reserve opts every entry in, so no
// instance launches without its shared-memory reservation.  All of them take one parameter list; Kl and Vl point to the cache's element type.
struct AttnFusedInstance { bool tp, alibi; int nv, kv_type; const void *kern; };
template <bool TP, bool ALIBI, int NV, typename KT>
AttnFusedInstance attn_fused_entry() { return {TP, ALIBI, NV, sizeof(KT) == 4 ? T_F32 : T_F16, (const void *)attn_fused_kernel<TP, ALIBI, NV, KT>}; }
const AttnFusedInstance attn_fused_instances[] = {
    attn_fused_entry<false, false, 4, __half>(), attn_fused_entry<true, false, 4, __half>(), attn_fused_entry<false, true, 4, __half>(),
    attn_fused_entry<false, false, 8, __half>(),
    attn_fused_entry<false, false, 4, float>(), attn_fused_entry<false, true, 4, float>(), attn_fused_entry<false, false, 8, float>(),
};
// the instance for a geometry: heads of up to 256 in 32-wide slices (NV 8 past 128), ALiBi only up to 128, tensor-parallel only on an f16
// cache with heads of up to 128 and no ALiBi
const void *attn_fused_pick(bool tp, int hd, bool alibi, int kv_type) {
    B200_ASSERT(hd <= 256 && hd % 32 == 0);
    B200_ASSERT(!alibi || hd <= 128);
    B200_ASSERT(!tp || (kv_type == T_F16 && hd <= 128 && !alibi));
    const int nv = hd > 128 ? 8 : 4;
    for (const AttnFusedInstance &I : attn_fused_instances)
        if (I.tp == tp && I.alibi == alibi && I.nv == nv && I.kv_type == kv_type) return I.kern;
    B200_ASSERT(!"attn_fused_pick: no instance for this geometry");
    return nullptr;
}
// dynamic shared memory opt-in of the cluster attention kernels: one high-water mark for all of them (the attribute is per function, not per caller)
static void attn_fused_reserve(size_t bytes) {
    static size_t set = 48 * 1024;
    if (bytes <= set) return;
    for (const AttnFusedInstance &I : attn_fused_instances) B200_CHECK(cudaFuncSetAttribute(I.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    set = bytes;
}
// the same for attn_sv_kernel (both instances): one record per process.  Every decode_ops_t<TYPE, TP> launches this one kernel, so a record per
// instantiation would let a session of another weight type with a shorter context LOWER the attribute under a session that already relies on more.
static void attn_sv_reserve(size_t bytes) {
    static size_t set = 48 * 1024;
    if (bytes <= set) return;
    B200_CHECK(cudaFuncSetAttribute(attn_sv_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    B200_CHECK(cudaFuncSetAttribute(attn_sv_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    set = bytes;
}
// the positions attn_fused_kernel holds for a context bucket: the bucket rounded up to whole 64-position tiles
int attn_fused_rows(int n_kv_bucket) { return (n_kv_bucket + 63) / 64 * 64; }
// dynamic shared memory of attn_fused_kernel for a context bucket and head size hd: scores (f32), probabilities and q (f16), then 32 V rows;
// an f32 cache (kv_type T_F32): probabilities, q and the V rows in f32 (136 bytes per position)
size_t attn_fused_smem(int n_kv_bucket, int hd, int kv_type = T_F16) {
    const int nlay = attn_fused_rows(n_kv_bucket);
    if (kv_type == T_F32) return (((size_t)nlay * 8 + (size_t)hd * 4 + 127) & ~(size_t)127) + (size_t)32 * (nlay + 4) * 4;
    return (((size_t)nlay * 6 + (size_t)hd * 2 + 127) & ~(size_t)127) + (size_t)32 * (nlay + 32) * 2;
}
}  // namespace
bool attn_fused_fits(int n_kv_bucket, int hd, int kv_type) { return attn_fused_smem(n_kv_bucket, hd, kv_type) <= 227 * 1024; }
int attn_sv_f32_max_ctx() { return (int)((227 * 1024 - attn_sv_smem(0, T_F32)) / 8); }
namespace {
// one cluster of hd/32 CTAs per head, a programmatic dependent of its predecessor.  alibi: per-head slopes (the ALiBi form, single GPU only)
// or nullptr.  kv_type T_F32: Kl / Vl are an f32 cache (single GPU only)
void launch_attn_fused(cudaStream_t st, bool tp, const float *q, const void *Kl, const void *Vl, int4 *xpack_out, const int *n_past, const uint16_t *lut_exp,
                       float kq_scale, int hd, int n_head, int n_head_kv, int gqa, int n_ctx, int n_kv_bucket, int q81, int off, int scale16,
                       unsigned long long *prof, TpSync S, int head0, const float *alibi, int kv_type) {
    const void *kern = attn_fused_pick(tp, hd, alibi != nullptr, kv_type);
    int nlay = attn_fused_rows(n_kv_bucket);
    const size_t smem = attn_fused_smem(n_kv_bucket, hd, kv_type);
    attn_fused_reserve(smem);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_head * (hd / 32)); cfg.blockDim = dim3(ATH); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = hd / 32; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 2;
    // attn_fused_kernel's parameters in order (Kl and Vl as the untyped pointers they are here)
    void *args[] = {&q, &Kl, &Vl, &xpack_out, &n_past, &lut_exp, &kq_scale, &hd, &n_head, &n_head_kv, &gqa, &n_ctx, &nlay, &q81, &off, &scale16, &prof, &S, &head0, &alibi};
    B200_CHECK(cudaLaunchKernelExC(&cfg, kern, args));
}
// the footprint of the cluster attention launch_attn_fused picks for the geometry (the successor the qkv node's ring is planned against)
CtaFootprint attn_fused_footprint(bool tp, int hd, bool alibi, int kv_type, size_t smem) { return footprint_of(attn_fused_pick(tp, hd, alibi, kv_type), ATH, smem); }

// f(KT()) for the KV cache's element type KT: the choice between the f16 and f32 instances of a kernel
template <typename F>
auto with_kv_type(int kv_type, F &&f) { return kv_type == T_F32 ? f(float()) : f(__half()); }

// tensor-parallel helpers (tp.cuh).  spread: the embedding row every rank computed for itself -> the X exchange buffer's unit form (stamp 0);
// collect: the gathered logits units -> the plain f32 logits array the host reads; bump: the token is complete, the epoch moves on.
__global__ void __launch_bounds__(256) tp_spread_kernel(const float *__restrict__ x, int n) {
    const TpCtx &T = c_tp;
    pdl_wait();
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    uint2 *dst = (uint2 *)(T.peer[T.rank] + T.off[TPB_X]) + i;
    *dst = make_uint2(__float_as_uint(__ldcg(x + i)), tp_tag(T, 0));
}
__global__ void __launch_bounds__(256) tp_collect_kernel(float *__restrict__ logits, int n) {
    const TpCtx &T = c_tp;
    pdl_wait();
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) logits[i] = tp_get_f32(T, TPB_LOGITS, i, tp_tag(T, 0));
}
__global__ void tp_bump_kernel() {
    const TpCtx &T = c_tp;
    pdl_wait();
    if (threadIdx.x == 0) *T.epoch = *(volatile unsigned *)T.epoch + 1;
}

// the qkv mat-vec with the RoPE + KV store epilogue for the session's cache (an f32 cache: single GPU only)
template <int TYPE, bool TP>
const MmvPlan &qkv_plan(bool kv32, const QWeight &w, const CtaFootprint &succ) {
    if constexpr (!TP) if (kv32) return mmv_plan<TYPE, EPI_QKV_F32, false>(w, succ);
    return mmv_plan<TYPE, EPI_QKV, TP>(w, succ);
}
template <int TYPE, bool TP>
void launch_qkv(bool kv32, const QWeight &w, const MmvArgs &A, const MmvPlan &plan, cudaStream_t st) {
    if constexpr (!TP) if (kv32) { launch_mmv<TYPE, EPI_QKV_F32>(w, A, plan, st); return; }
    launch_mmv<TYPE, EPI_QKV, TP>(w, A, plan, st);
}

template <int TYPE, bool TP>
void decode_ops_t(const DecodeParams &P, const std::vector<DecodeLayer> &layers, int n_kv_bucket, int4 *xpack_a, cudaStream_t st, int *launches) {
    const int q81 = has_min(TYPE) ? 1 : 0, off = TYPE == T_Q5_0 ? 16 : 0, s16 = TYPE == T_Q4_0 ? 1 : 0;
    const int e = P.e, f = P.f;
    const TpCtx &T = P.tp;
    constexpr bool tp = TP;
    B200_ASSERT(tp == (T.world > 1));
    const int e_loc = tp ? P.e_loc : e;
    // layer stamps (tp.cuh): X carries stamp il when it enters layer il (0 = the embedding), il + 1 when layer il leaves it; FF / XD / XF of layer il carry il + 1
    auto ts = [&](int in_buf, unsigned in_v, int add_buf, unsigned add_v, int out_buf, unsigned out_v) {
        TpSync S;
        if (tp) { S.in_buf = in_buf; S.in_v = in_v; S.add_buf = add_buf; S.add_v = add_v; S.out_buf = out_buf; S.out_v = out_v; }
        return S;
    };
    int n = 0;
    auto pr = [&]() -> unsigned long long * { return P.prof && n < B200_PROF_SLOTS ? P.prof + n : nullptr; };   // timeline slot of the next launch
    // rms_norm * gain -> records of the next mat-vec; with `normed` (the final norm of a single-GPU token) also the f32 row
    auto launch_norm = [&](const float *x, const float *gain, const TpSync &S, float *normed = nullptr) {
        const dim3 grid((e / QK + 31) / 32), block(256);
        if constexpr (TP) launch_k(norm_pack_tp_kernel, grid, block, 0, st, x, gain, xpack_a, e, P.eps, q81, off, s16, pr(), S);
        else if (normed) launch_k(norm_pack_store_kernel, grid, block, 0, st, x, gain, xpack_a, e, P.eps, q81, off, s16, pr(), normed);
        else { (void)S; launch_k(norm_pack_kernel, grid, block, 0, st, x, gain, xpack_a, e, P.eps, q81, off, s16, pr()); }
        n++;
    };
    // the token boundary: a plain launch (no programmatic attribute), so nothing of this token starts before the previous token has completed --
    // attn_fused_kernel reads n_past and the older KV cache ahead of its griddepcontrol.wait on that guarantee
    get_rows_q(P.wte, P.token, P.x, 1, st); n++;
    if (tp) { launch_k(tp_spread_kernel, dim3((e + 255) / 256), dim3(256), 0, st, (const float *)P.x, e); n++; }
    // attention: one cluster launch per layer, or the two-kernel variant for head sizes a cluster cannot cover and for buckets whose scores
    // and V rows do not fit one CTA's shared memory (an f32 cache: past 1664 positions)
    const bool kv32 = !TP && P.kv_type == T_F32;                // sessions of a tensor-parallel model keep an f16 cache
    const int kv_type = kv32 ? T_F32 : T_F16;
    const size_t fa_smem = attn_fused_smem(n_kv_bucket, P.hd, P.kv_type);
    const bool fused_attn = P.hd % 32 == 0 && P.hd <= 128 && P.n_ctx % 8 == 0 && attn_fused_fits(n_kv_bucket, P.hd, P.kv_type);
    B200_ASSERT(fused_attn || !tp);                              // the tensor-parallel exchange lives in the fused attention kernel's epilogue (start_session_tp checks the size)
    const size_t sv_smem = attn_sv_smem(P.n_ctx, kv_type);
    attn_sv_reserve(sv_smem);
    // the two-kernel attention's KQ instance for the cache's element type (heads of 64 or 128)
    auto attn_kq_of = [&](auto kt) { return P.hd == 128 ? attn_kq_kernel<128, decltype(kt)> : attn_kq_kernel<64, decltype(kt)>; };
    // mat-vec plans, each leaving room for what follows it (planned from the successor backwards; every layer has the same shapes): the norm
    // kernels release their dependents at entry, so beside wo and w2 there has to be room for the norm AND the next mat-vec
    const CtaFootprint f_norm = TP ? footprint_of(norm_pack_tp_kernel, 256, 0) : footprint_of(norm_pack_kernel, 256, 0);
    const CtaFootprint f_attn = fused_attn ? attn_fused_footprint(TP, P.hd, false, kv_type, fa_smem)
                                           : with_kv_type(kv_type, [&](auto kt) { return footprint_of(attn_kq_of(kt), 128, 0); });
    const MmvPlan &p_qkv = qkv_plan<TYPE, TP>(kv32, layers[0].wqkv, f_attn);
    const MmvPlan &p_w2 = mmv_plan<TYPE, EPI_RES, TP>(layers[0].w2, f_norm + p_qkv.cta);
    const MmvPlan &p_w13 = mmv_plan<TYPE, EPI_SILU, TP>(layers[0].w13, p_w2.cta);
    const MmvPlan &p_wo = mmv_plan<TYPE, EPI_RES, TP>(layers[0].wo, f_norm + p_w13.cta);
    const bool kq_out = !TP && is_kquant(P.output.type);       // a K-quant lm_head (per-tensor types): not a mat-vec of this schedule's TYPE
    const MmvPlan *p_out = kq_out ? nullptr : &mmv_plan<TYPE, EPI_LOGITS, TP>(P.output, CtaFootprint{});
    for (int il = 0; il < P.n_layer; il++) {
        const DecodeLayer &L = layers[il];
        const unsigned v = (unsigned)il + 1;                     // flag value of this layer's exchanges (tp.cuh)
        launch_norm(P.x, L.attn_norm, ts(TPB_X, (unsigned)il, -1, 0, -1, 0));
        MmvArgs A{}; A.xpack = xpack_a; A.q = P.q; A.K = L.K; A.V = L.V; A.rope_cs = P.rope_cs; A.rope_half = P.rope_half; A.hd = P.hd; A.e = e_loc; A.gqa = P.gqa;
        A.n_ctx = P.n_ctx; A.n_past = P.n_past;
        A.prof = pr(); launch_qkv<TYPE, TP>(kv32, L.wqkv, A, p_qkv, st); n++;
        if (fused_attn) {
            launch_attn_fused(st, TP, P.q, L.K, L.V, P.xpack_d, P.n_past, P.lut_exp, P.kq_scale, P.hd, P.n_head, P.n_head_kv, P.gqa, P.n_ctx, n_kv_bucket, q81, off, s16, pr(),
                              ts(-1, 0, -1, 0, TPB_XD, v), tp ? P.head0 : 0, nullptr, kv_type);
            n++;
        } else with_kv_type(kv_type, [&](auto kt) {
            using KT = decltype(kt);
            launch_k(attn_kq_of(kt), dim3((n_kv_bucket + 63) / 64, P.n_head), dim3(128), 0, st,
                     P.q, (const KT *)L.K, P.kq, P.n_past, P.gqa, P.n_head, P.n_head_kv, P.n_ctx, pr());
            n++;
            launch_k(attn_sv_kernel<KT>, dim3(P.n_head * (P.hd / 32)), dim3(128), sv_smem, st, P.kq, (const KT *)L.V, P.xpack_d, P.n_past, P.lut_exp, P.kq_scale,
                     P.hd, P.n_head, P.n_head_kv, P.n_ctx, q81, off, s16, pr()); n++;
        });
        MmvArgs Bo{}; Bo.xpack = P.xpack_d; Bo.dst = P.ff; Bo.addend = P.x;
        Bo.ts = ts(TPB_XD, v, TPB_X, (unsigned)il, TPB_FF, v); Bo.row0 = tp ? P.row0_e : 0;
        Bo.prof = pr(); launch_mmv<TYPE, EPI_RES, TP>(L.wo, Bo, p_wo, st); n++;
        launch_norm(P.ff, L.ffn_norm, ts(TPB_FF, v, -1, 0, -1, 0));
        MmvArgs C{}; C.xpack = xpack_a; C.xpack_out = P.xpack_f; C.lut_silu = P.lut_silu; C.q81 = q81; C.off = off; C.scale16 = s16;
        C.ts = ts(-1, 0, -1, 0, TPB_XF, v); C.row0 = tp ? P.row0_w13 : 0;
        C.prof = pr(); launch_mmv<TYPE, EPI_SILU, TP>(L.w13, C, p_w13, st); n++;
        MmvArgs D{}; D.xpack = P.xpack_f; D.dst = P.x; D.addend = P.ff;
        D.ts = ts(TPB_XF, v, TPB_FF, v, TPB_X, v); D.row0 = tp ? P.row0_e : 0;
        D.prof = pr(); launch_mmv<TYPE, EPI_RES, TP>(L.w2, D, p_w2, st); n++;
    }
    launch_norm(P.x, P.norm, ts(TPB_X, (unsigned)P.n_layer, -1, 0, -1, 0), P.normed);
    if (kq_out) {
        // ggml_mul_mat(output, cur) on the f32 row the final norm stored: quantize_row_q8_K, then the K-quant mat-vec, whose launch also advances n_past
        quantize_act_q8k(P.normed, P.e, P.xq8k, P.e, 1, st); n++;
        mul_mat_kq_exact(P.output.type, P.output.qs, P.xq8k, P.logits, P.n_vocab, P.e, P.n_vocab, 1, nullptr, 0, st, P.n_past); n++;
    } else {
        MmvArgs Z{}; Z.xpack = xpack_a; Z.dst = P.logits; Z.addend = nullptr; Z.n_past_inc = P.n_past;
        Z.ts = ts(-1, 0, -1, 0, TPB_LOGITS, 0); Z.row0 = tp ? P.row0_v : 0;
        Z.prof = pr(); launch_mmv<TYPE, EPI_LOGITS, TP>(P.output, Z, *p_out, st); n++;
    }
    if (tp) {                                                    // gathered logits -> the plain array the host reads; then the epoch moves on
        launch_k(tp_collect_kernel, dim3((P.n_vocab_full + 255) / 256), dim3(256), 0, st, P.logits, P.n_vocab_full); n++;
        launch_k(tp_bump_kernel, dim3(1), dim3(32), 0, st); n++;
    }
    B200_CHECK(cudaGetLastError());
    (void)f;
    if (launches) *launches = n;
}

// ---- GPT-NeoX --------------------------------------------------------------------------------------------------------------------------------
// LayerNorm (ggml_compute_forward_norm_f32, LC/ggml.c:10063-10111) * gain + bias -> Q8 records.  Same shape as norm_pack_kernel: every CTA reduces
// the whole row from registers (two passes: mean, then the variance of the centred values) and packs its own 32 blocks.
// BIAS false (MPT): norm * gain only -- no add node, so a -0 stays -0.
// STORE (the token's final norm only): each CTA also stores its own float4s of the f32 row to `normed`, the embeddings of OutputRequest.
template <bool BIAS, bool STORE = false>
__device__ __forceinline__ void ln_pack_body(const float *__restrict__ x, const float *__restrict__ gain, const float *__restrict__ bias, int4 *__restrict__ pack,
                                             int e, int q81, int off, int scale16, float *__restrict__ normed = nullptr) {
    __shared__ double shd[16];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_trigger();
    pdl_wait();
    constexpr int MAXV = 8;                                     // n_embd <= 8192
    const int nv = e / 4, mine = blockIdx.x * 256 + tid;
    float4 v[MAXV];
#pragma unroll
    for (int k = 0; k < MAXV; k++) { const int i = tid + k * 256; v[k] = i < nv ? __ldcg((const float4 *)x + i) : make_float4(0.f, 0.f, 0.f, 0.f); }
    const bool active = mine < nv;
    const float4 gv = active ? __ldg((const float4 *)gain + mine) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 bv = BIAS && active ? __ldg((const float4 *)bias + mine) : make_float4(0.f, 0.f, 0.f, 0.f);
    auto tree = [&](int k) { return ((shd[k] + shd[k + 1]) + (shd[k + 2] + shd[k + 3])) + ((shd[k + 4] + shd[k + 5]) + (shd[k + 6] + shd[k + 7])); };
    // the mean: sum x and, for row_sum_settled, sum |x|
    double s = 0.0, a = 0.0;
#pragma unroll
    for (int k = 0; k < MAXV; k++) if (tid + k * 256 < nv) {
        s += (double)v[k].x; s += (double)v[k].y; s += (double)v[k].z; s += (double)v[k].w;
        a += fabs((double)v[k].x); a += fabs((double)v[k].y); a += fabs((double)v[k].z); a += fabs((double)v[k].w);
    }
    s = warp_sum(s); a = warp_sum(a);
    if (lane == 0) { shd[warp] = s; shd[8 + warp] = a; }
    __syncthreads();
    double sum = tree(0);
    const double abs_sum = tree(8);                             // the same in every CTA, and so is each decision below
    if (!row_sum_settled(sum, abs_sum, e)) {
        if (!row_sum_within(sum, row_sum_prefix_bound(prefix_abs_sum(x, e), abs_sum, e, 4 * MAXV + 8), e))
            sum = row_sum_in_order(e, [=](int64_t i) { return (double)__ldcg(x + i); });
#pragma unroll                                                  // the row again: the calls above need not keep it in registers
        for (int k = 0; k < MAXV; k++) { const int i = tid + k * 256; v[k] = i < nv ? __ldcg((const float4 *)x + i) : make_float4(0.f, 0.f, 0.f, 0.f); }
    }
    const float mean = (float)(sum / (double)e);
    double s2 = 0.0;
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < MAXV; k++) if (tid + k * 256 < nv) {
        float4 c;
        c.x = __fsub_rn(v[k].x, mean); c.y = __fsub_rn(v[k].y, mean); c.z = __fsub_rn(v[k].z, mean); c.w = __fsub_rn(v[k].w, mean);
        s2 += (double)__fmul_rn(c.x, c.x); s2 += (double)__fmul_rn(c.y, c.y); s2 += (double)__fmul_rn(c.z, c.z); s2 += (double)__fmul_rn(c.w, c.w);
        if (k == (int)blockIdx.x) xv = c;                       // float4 index tid + k * 256 == mine
    }
    s2 = warp_sum(s2);
    __syncthreads();                                            // every thread has read shd
    if (lane == 0) shd[warp] = s2;
    __syncthreads();
    double sum2 = tree(0);
    if (!row_sum_settled(sum2, sum2, e))
        sum2 = row_sum_in_order(e, [=](int64_t i) { const float c = __fsub_rn(__ldcg(x + i), mean); return (double)__fmul_rn(c, c); });
    const float variance = (float)(sum2 / (double)e);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(variance, 1e-5f)));
    float4 y;
    if (BIAS) {
        y.x = __fadd_rn(__fmul_rn(__fmul_rn(xv.x, scale), gv.x), bv.x); y.y = __fadd_rn(__fmul_rn(__fmul_rn(xv.y, scale), gv.y), bv.y);
        y.z = __fadd_rn(__fmul_rn(__fmul_rn(xv.z, scale), gv.z), bv.z); y.w = __fadd_rn(__fmul_rn(__fmul_rn(xv.w, scale), gv.w), bv.w);
    } else {
        y.x = __fmul_rn(__fmul_rn(xv.x, scale), gv.x); y.y = __fmul_rn(__fmul_rn(xv.y, scale), gv.y);
        y.z = __fmul_rn(__fmul_rn(xv.z, scale), gv.z); y.w = __fmul_rn(__fmul_rn(xv.w, scale), gv.w);
    }
    if constexpr (STORE) if (active) ((float4 *)normed)[mine] = y;
    pack_quad(y, pack + (active ? mine >> 3 : 0) * 4, lane, active, q81, off, scale16);
}
__global__ void __launch_bounds__(256) ln_pack_kernel(const float *__restrict__ x, const float *__restrict__ gain, const float *__restrict__ bias, int4 *__restrict__ pack,
                                                      int e, int q81, int off, int scale16) {
    ln_pack_body<true>(x, gain, bias, pack, e, q81, off, scale16);
}
__global__ void __launch_bounds__(256) ln_pack_nobias_kernel(const float *__restrict__ x, const float *__restrict__ gain, const float *__restrict__ bias, int4 *__restrict__ pack,
                                                             int e, int q81, int off, int scale16) {
    ln_pack_body<false>(x, gain, bias, pack, e, q81, off, scale16);
}
// the final LayerNorm of a token (gptneox lib.rs:333-337, gpt2 :311-317, mpt :236-239, bloom :317-324, gptj :286-289): the records, and the f32 row in `normed`
__global__ void __launch_bounds__(256) ln_pack_store_kernel(const float *__restrict__ x, const float *__restrict__ gain, const float *__restrict__ bias, int4 *__restrict__ pack,
                                                            int e, int q81, int off, int scale16, float *__restrict__ normed) {
    ln_pack_body<true, true>(x, gain, bias, pack, e, q81, off, scale16, normed);
}
__global__ void __launch_bounds__(256) ln_pack_nobias_store_kernel(const float *__restrict__ x, const float *__restrict__ gain, const float *__restrict__ bias,
                                                                   int4 *__restrict__ pack, int e, int q81, int off, int scale16, float *__restrict__ normed) {
    ln_pack_body<false, true>(x, gain, bias, pack, e, q81, off, scale16, normed);
}

// qkv [3e] (bias added) -> q [e], k -> f16 cache row n_past, v -> f16 cache column n_past.  GPT-NeoX (gptneox lib.rs:205-247): rows per head are q | k | v
// (head stride 3 hd) and q, k get RoPE mode 2 -- the ggml neox branch (LC/ggml.c:11876-11897) rotates EVERY block of n_rot dims of the head, pairs
// (c, c + n_rot/2).  GPT-2 (gpt2 lib.rs:190-210): the three thirds of the row, no rotation (n_rot = 0).  One thread per channel.
// KT: the cache's element type (float: K and V stored as they are)
template <typename KT>
__global__ void __launch_bounds__(256) neox_rope_store_kernel(const float *__restrict__ qkv, float *__restrict__ q, KT *__restrict__ Kl, KT *__restrict__ Vl,
                                                              const int *__restrict__ n_past, const float2 *__restrict__ rope_cs, int rope_half, int n_rot, int hd, int e, int n_ctx,
                                                              int head_stride, int k_off, int v_off) {
    pdl_trigger();
    pdl_wait();
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= e) return;
    const int p = __ldcg(n_past);
    const int h = i / hd, c = i - h * hd;
    const float *base = qkv + (int64_t)h * head_stride;
    float qo = __ldcg(base + c), ko = __ldcg(base + k_off + c);
    if (n_rot > 0) {
        const int hb = n_rot / 2, ib = c / n_rot, r = c - ib * n_rot;
        if (ib < hd / n_rot) {
            const bool lo = r < hb;
            const int partner = lo ? c + hb : c - hb;
            const float2 cs = __ldg(rope_cs + (int64_t)p * rope_half + ib * hb + (lo ? r : r - hb));
            const float qp = __ldcg(base + partner), kp = __ldcg(base + k_off + partner);
            // x0 = element of the lower half, x1 = upper: out0 = fma(x0, cos, -(x1 sin)), out1 = fma(x0, sin, x1 cos)  (rowops.cu::rope_kernel)
            qo = lo ? __fmaf_rn(qo, cs.x, -__fmul_rn(qp, cs.y)) : __fmaf_rn(qp, cs.y, __fmul_rn(qo, cs.x));
            ko = lo ? __fmaf_rn(ko, cs.x, -__fmul_rn(kp, cs.y)) : __fmaf_rn(kp, cs.y, __fmul_rn(ko, cs.x));
        }
    }
    q[i] = qo;
    Kl[(int64_t)p * e + i] = kv_cast<KT>(ko);
    Vl[(int64_t)i * n_ctx + p] = kv_cast<KT>(__ldcg(base + v_off + c));
}

// GPT-2: inpL = wte[token] + wpe[n_past]  (gpt2 lib.rs:164-172), position read from device memory
__global__ void __launch_bounds__(256) gpt2_add_pos_kernel(float *__restrict__ x, const float *__restrict__ wpe, const int *__restrict__ n_past, int e) {
    pdl_wait();
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < e) x[i] = __fadd_rn(x[i], __ldg(wpe + (int64_t)__ldcg(n_past) * e + i));
}

template <int TYPE>
void neox_ops_t(const NeoxParams &P, const std::vector<NeoxLayer> &layers, int n_kv_bucket, cudaStream_t st, int *launches) {
    const int q81 = has_min(TYPE) ? 1 : 0, off = TYPE == T_Q5_0 ? 16 : 0, s16 = TYPE == T_Q4_0 ? 1 : 0;
    const int e = P.e;
    int n = 0;
    // the token boundary: a plain launch (no programmatic attribute), so nothing of this token starts before the previous token has completed --
    // attn_fused_kernel reads n_past and the older KV cache ahead of its griddepcontrol.wait on that guarantee
    if (P.emb_g) {                                                // BLOOM (bloom lib.rs:139-144): the row, then LayerNorm -> the residual stream
        get_rows_q(P.wte, P.token, P.qkv, 1, st); n++;
        layer_norm(P.qkv, P.x, P.emb_g, P.emb_b, e, 1, st); n++;
    } else {
        get_rows_q(P.wte, P.token, P.x, 1, st); n++;
    }
    if (P.wpe) { launch_k(gpt2_add_pos_kernel, dim3((e + 255) / 256), dim3(256), 0, st, P.x, P.wpe, (const int *)P.n_past, e); n++; }
    B200_ASSERT(neox_decode_fits(P, n_kv_bucket));
    const size_t fa_smem = attn_fused_smem(n_kv_bucket, P.hd, P.kv_type);
    const dim3 ln_grid((e / 4 + 255) / 256);
    const TpSync S{};
    // MPT has no biases: its norms take ln_pack_nobias_kernel and its up-projection the gelu epilogue without a bias node
    const bool biased = layers[0].ln1_b != nullptr, fc_bias = layers[0].bfc != nullptr;
    auto ln_kernel = biased ? ln_pack_kernel : ln_pack_nobias_kernel;
    auto ln_final = biased ? ln_pack_store_kernel : ln_pack_nobias_store_kernel;     // + the f32 row (NeoxParams::normed)
    const CtaFootprint f_ln = footprint_of(ln_kernel, 256, 0);
    const CtaFootprint f_attn = attn_fused_footprint(false, P.hd, P.alibi != nullptr, P.kv_type, fa_smem);
    const CtaFootprint f_store = with_kv_type(P.kv_type, [](auto kt) { return footprint_of(neox_rope_store_kernel<decltype(kt)>, 256, 0); });
    const MmvPlan &p_qkv = mmv_plan<TYPE, EPI_BIAS, false>(layers[0].wqkv, f_store + f_attn);
    const MmvPlan &p_proj = mmv_plan<TYPE, EPI_BIAS, false>(layers[0].wproj, f_ln + p_qkv.cta);
    const MmvPlan &p_fc = fc_bias ? mmv_plan<TYPE, EPI_GELU, false>(layers[0].wfc, p_proj.cta) : mmv_plan<TYPE, EPI_GELU_NB, false>(layers[0].wfc, p_proj.cta);
    const MmvPlan &p_dense = mmv_plan<TYPE, EPI_BIAS, false>(layers[0].wdense, f_ln + p_fc.cta);
    const MmvPlan &p_head = mmv_plan<TYPE, EPI_BIAS, false>(P.lm_head, CtaFootprint{});
    for (int il = 0; il < P.n_layer; il++) {
        const NeoxLayer &L = layers[il];
        launch_k(ln_kernel, ln_grid, dim3(256), 0, st, (const float *)P.x, L.ln1_g, L.ln1_b, P.xpack_a, e, q81, off, s16); n++;               // :192-196
        MmvArgs A{}; A.xpack = P.xpack_a; A.dst = P.qkv; A.bias = L.bqkv;
        launch_mmv<TYPE, EPI_BIAS>(L.wqkv, A, p_qkv, st); n++;                                                                                      // :199-200
        with_kv_type(P.kv_type, [&](auto kt) {
            using KT = decltype(kt);
            launch_k(neox_rope_store_kernel<KT>, dim3((e + 255) / 256), dim3(256), 0, st, (const float *)P.qkv, P.q, (KT *)L.K, (KT *)L.V, (const int *)P.n_past,
                     P.rope_cs, P.rope_half, P.n_rot, P.hd, e, P.n_ctx, P.qkv_layout.head_stride, P.qkv_layout.k_off, P.qkv_layout.v_off);
        });
        n++;                                                                                                                                  // :205-247
        launch_attn_fused(st, false, P.q, L.K, L.V, P.xpack_d, P.n_past, P.lut_exp, P.kq_scale, P.hd, P.n_head, P.n_head, e, P.n_ctx, n_kv_bucket, q81, off, s16,
                          nullptr, S, 0, P.alibi, P.kv_type); n++;                                                                        // :250-298
        // attention.dense (+bias); sequential residual: ff_in = that + inpL                                                                    :301-312
        MmvArgs Bo{}; Bo.xpack = P.xpack_d; Bo.dst = P.attn_out; Bo.bias = L.bdense; Bo.add1 = P.parallel_residual ? nullptr : P.x;
        launch_mmv<TYPE, EPI_BIAS>(L.wdense, Bo, p_dense, st); n++;
        // mlp: LayerNorm of inpL (parallel residual) or of ff_in                                                                                :313-316 / ffn
        launch_k(ln_kernel, ln_grid, dim3(256), 0, st, (const float *)(P.parallel_residual ? P.x : P.attn_out), L.ln2_g, L.ln2_b, P.xpack_a, e, q81, off, s16); n++;
        MmvArgs C{}; C.xpack = P.xpack_a; C.xpack_out = P.xpack_f; C.bias = L.bfc; C.lut_gelu = P.lut_gelu; C.q81 = q81; C.off = off; C.scale16 = s16;
        if (fc_bias) launch_mmv<TYPE, EPI_GELU>(L.wfc, C, p_fc, st); else launch_mmv<TYPE, EPI_GELU_NB>(L.wfc, C, p_fc, st);
        n++;
        // parallel: inpL = ((proj + bias) + attn) + inpL; sequential: inpL = (proj + bias) + ff_in                                              :317-325
        MmvArgs D{}; D.xpack = P.xpack_f; D.dst = P.x; D.bias = L.bproj; D.add1 = P.attn_out; D.add2 = P.parallel_residual ? P.x : nullptr;
        launch_mmv<TYPE, EPI_BIAS>(L.wproj, D, p_proj, st); n++;
    }
    launch_k(ln_final, ln_grid, dim3(256), 0, st, (const float *)P.x, P.lnf_g, P.lnf_b, P.xpack_a, e, q81, off, s16, P.normed); n++;                 // :332-334
    MmvArgs Z{}; Z.xpack = P.xpack_a; Z.dst = P.logits; Z.n_past_inc = P.n_past;
    launch_mmv<TYPE, EPI_BIAS>(P.lm_head, Z, p_head, st); n++;                                                                                        // :342
    B200_CHECK(cudaGetLastError());
    if (launches) *launches = n;
}

// ---- GPT-J (crates/models/gptj/src/lib.rs:153-305): 6 kernels per layer + 3 ------------------------------------------------------------------
//   ln_pack(ln_1) -> xpack_a;  qkv [q|k|v thirds] with the LLaMA epilogue (RoPE mode 0 over the whole head on q, k; K by row, V by column);
//   cluster attention -> xpack_d;  out_proj (no bias) -> attn_out;  fc_in + bias, gelu, quantized, reading the SAME xpack_a records (one LayerNorm feeds
//   attention and MLP, :174, :270);  fc_out: ((W h + b_out) + attn_out) + x -> x (:276-282).  Then ln_f and the lm_head + lm_head.bias (:286-296).
template <int TYPE>
void gptj_ops_t(const NeoxParams &P, const std::vector<NeoxLayer> &layers, int n_kv_bucket, cudaStream_t st, int *launches) {
    const int q81 = has_min(TYPE) ? 1 : 0, off = TYPE == T_Q5_0 ? 16 : 0, s16 = TYPE == T_Q4_0 ? 1 : 0;
    const int e = P.e;
    int n = 0;
    // the token boundary: a plain launch (no programmatic attribute), see neox_ops_t
    get_rows_q(P.wte, P.token, P.x, 1, st); n++;                                                                                                     // :161
    B200_ASSERT(neox_decode_fits(P, n_kv_bucket));
    const bool kv32 = P.kv_type == T_F32;
    const size_t fa_smem = attn_fused_smem(n_kv_bucket, P.hd, P.kv_type);
    const dim3 ln_grid((e / 4 + 255) / 256);
    const TpSync S{};
    const CtaFootprint f_ln = footprint_of(ln_pack_kernel, 256, 0);
    const CtaFootprint f_attn = attn_fused_footprint(false, P.hd, false, P.kv_type, fa_smem);
    // each ring planned against the node launched after it: qkv -> attention, out_proj -> fc_in, fc_in -> fc_out, fc_out -> next layer's ln_1 + qkv
    const MmvPlan &p_qkv = qkv_plan<TYPE, false>(kv32, layers[0].wqkv, f_attn);
    const MmvPlan &p_proj = mmv_plan<TYPE, EPI_BIAS, false>(layers[0].wproj, f_ln + p_qkv.cta);
    const MmvPlan &p_fc = mmv_plan<TYPE, EPI_GELU, false>(layers[0].wfc, p_proj.cta);
    const MmvPlan &p_dense = mmv_plan<TYPE, EPI_BIAS, false>(layers[0].wdense, p_fc.cta);
    const MmvPlan &p_head = mmv_plan<TYPE, EPI_BIAS, false>(P.lm_head, CtaFootprint{});
    for (int il = 0; il < P.n_layer; il++) {
        const NeoxLayer &L = layers[il];
        launch_k(ln_pack_kernel, ln_grid, dim3(256), 0, st, (const float *)P.x, L.ln1_g, L.ln1_b, P.xpack_a, e, q81, off, s16); n++;                 // :168-174
        MmvArgs A{}; A.xpack = P.xpack_a; A.q = P.q; A.K = L.K; A.V = L.V; A.rope_cs = P.rope_cs; A.rope_half = P.rope_half; A.hd = P.hd; A.e = e; A.gqa = e;
        A.n_ctx = P.n_ctx; A.n_past = P.n_past;
        launch_qkv<TYPE, false>(kv32, L.wqkv, A, p_qkv, st); n++;                                                                                     // :178-220
        launch_attn_fused(st, false, P.q, L.K, L.V, P.xpack_d, P.n_past, P.lut_exp, P.kq_scale, P.hd, P.n_head, P.n_head, e, P.n_ctx, n_kv_bucket, q81, off, s16,
                          nullptr, S, 0, nullptr, P.kv_type); n++;                                                                                      // :222-262
        MmvArgs Bo{}; Bo.xpack = P.xpack_d; Bo.dst = P.attn_out;
        launch_mmv<TYPE, EPI_BIAS>(L.wdense, Bo, p_dense, st); n++;                                                                                    // :265
        MmvArgs C{}; C.xpack = P.xpack_a; C.xpack_out = P.xpack_f; C.bias = L.bfc; C.lut_gelu = P.lut_gelu; C.q81 = q81; C.off = off; C.scale16 = s16;
        launch_mmv<TYPE, EPI_GELU>(L.wfc, C, p_fc, st); n++;                                                                                           // :270-273
        MmvArgs D{}; D.xpack = P.xpack_f; D.dst = P.x; D.bias = L.bproj; D.add1 = P.attn_out; D.add2 = P.x;
        launch_mmv<TYPE, EPI_BIAS>(L.wproj, D, p_proj, st); n++;                                                                                       // :276-282
    }
    launch_k(ln_pack_store_kernel, ln_grid, dim3(256), 0, st, (const float *)P.x, P.lnf_g, P.lnf_b, P.xpack_a, e, q81, off, s16, P.normed); n++;         // :286-287
    MmvArgs Z{}; Z.xpack = P.xpack_a; Z.dst = P.logits; Z.bias = P.lm_head_b; Z.n_past_inc = P.n_past;
    launch_mmv<TYPE, EPI_BIAS>(P.lm_head, Z, p_head, st); n++;                                                                                        // :292-296
    B200_CHECK(cudaGetLastError());
    if (launches) *launches = n;
}

}  // namespace

// The cluster attention takes heads of up to 128 (GPT-J's wide form: up to 256) in 32-wide slices and the bucket's scores and V rows in shared
// memory (an f32 cache: up to 1664 positions); ln_pack_body holds rows of up to 8192; the mat-vecs stream rows of n_embd and 4 n_embd.
bool neox_decode_fits(const NeoxParams &P, int n_kv_bucket) {
    QWeight k_e, k_4e;
    k_e.nb = P.e / QK; k_4e.nb = 4 * P.e / QK;
    return P.hd % 32 == 0 && P.hd <= (P.gptj ? 256 : 128) && P.e % 128 == 0 && P.e <= 8192 && P.n_ctx % 8 == 0 &&
           mmv_exact_stream_supported(k_e) && mmv_exact_stream_supported(k_4e) && attn_fused_fits(n_kv_bucket, P.hd, P.kv_type);
}

void neox_decode_enqueue(const NeoxParams &P, const std::vector<NeoxLayer> &layers, int wtype, int n_kv_bucket, cudaStream_t st, int *launches) {
    switch (wtype) {
        case T_Q4_0: if (P.gptj) gptj_ops_t<T_Q4_0>(P, layers, n_kv_bucket, st, launches); else neox_ops_t<T_Q4_0>(P, layers, n_kv_bucket, st, launches); break;
        case T_Q4_1: if (P.gptj) gptj_ops_t<T_Q4_1>(P, layers, n_kv_bucket, st, launches); else neox_ops_t<T_Q4_1>(P, layers, n_kv_bucket, st, launches); break;
        case T_Q5_0: if (P.gptj) gptj_ops_t<T_Q5_0>(P, layers, n_kv_bucket, st, launches); else neox_ops_t<T_Q5_0>(P, layers, n_kv_bucket, st, launches); break;
        case T_Q5_1: if (P.gptj) gptj_ops_t<T_Q5_1>(P, layers, n_kv_bucket, st, launches); else neox_ops_t<T_Q5_1>(P, layers, n_kv_bucket, st, launches); break;
        case T_Q8_0: if (P.gptj) gptj_ops_t<T_Q8_0>(P, layers, n_kv_bucket, st, launches); else neox_ops_t<T_Q8_0>(P, layers, n_kv_bucket, st, launches); break;
        default: B200_ASSERT(!"neox_decode_enqueue: unsupported weight type");
    }
}

// the process's tensor-parallel context (session.cu calls it after the slabs are connected and when the measurement switch flips); not inside a stream capture
void decode_set_tp(const TpCtx &T, cudaStream_t st) {
    B200_CHECK(cudaStreamSynchronize(st));
    B200_CHECK(cudaMemcpyToSymbol(c_tp, &T, sizeof(TpCtx)));
    B200_CHECK(cudaDeviceSynchronize());
}

// Enqueue one decode step (position read from *P.n_past on the device) on `st`.  n_kv_bucket >= n_past + 1 sizes the KQ grid.
void decode_ops_enqueue(const DecodeParams &P, const std::vector<DecodeLayer> &layers, int wtype, int n_kv_bucket, int4 *xpack_a, cudaStream_t st, int *launches) {
    const bool tp = P.tp.world > 1;
    switch (wtype) {
        case T_Q4_0: if (tp) decode_ops_t<T_Q4_0, true>(P, layers, n_kv_bucket, xpack_a, st, launches); else decode_ops_t<T_Q4_0, false>(P, layers, n_kv_bucket, xpack_a, st, launches); break;
        case T_Q4_1: if (tp) decode_ops_t<T_Q4_1, true>(P, layers, n_kv_bucket, xpack_a, st, launches); else decode_ops_t<T_Q4_1, false>(P, layers, n_kv_bucket, xpack_a, st, launches); break;
        case T_Q5_0: if (tp) decode_ops_t<T_Q5_0, true>(P, layers, n_kv_bucket, xpack_a, st, launches); else decode_ops_t<T_Q5_0, false>(P, layers, n_kv_bucket, xpack_a, st, launches); break;
        case T_Q5_1: if (tp) decode_ops_t<T_Q5_1, true>(P, layers, n_kv_bucket, xpack_a, st, launches); else decode_ops_t<T_Q5_1, false>(P, layers, n_kv_bucket, xpack_a, st, launches); break;
        case T_Q8_0: if (tp) decode_ops_t<T_Q8_0, true>(P, layers, n_kv_bucket, xpack_a, st, launches); else decode_ops_t<T_Q8_0, false>(P, layers, n_kv_bucket, xpack_a, st, launches); break;
        default: B200_ASSERT(!"decode_ops_enqueue: unsupported weight type");
    }
}

DecodeGraphCache::DecodeGraphCache() {
    B200_CHECK(cudaMalloc(&d_n_past, sizeof(int)));
    B200_CHECK(cudaMallocHost(&h_n_past, sizeof(int)));
}
DecodeGraphCache::~DecodeGraphCache() {
    drop();
    B200_CHECK(cudaFree(d_n_past));
    B200_CHECK(cudaFreeHost(h_n_past));
}

int DecodeGraphCache::bucket(int n_kv, int n_ctx) { return std::min((n_kv + 255) / 256 * 256, n_ctx); }

int DecodeGraphCache::run(int n_kv, int n_ctx, bool replay, const std::function<void(int, cudaStream_t, int *)> &enqueue, cudaStream_t st) {
    if (dev_n_past != n_kv - 1) {
        B200_CHECK(cudaStreamSynchronize(st));      // the pinned staging word may still be in flight
        *h_n_past = n_kv - 1;
        B200_CHECK(cudaMemcpyAsync(d_n_past, h_n_past, sizeof(int), cudaMemcpyHostToDevice, st));
    }
    const int bucket = DecodeGraphCache::bucket(n_kv, n_ctx);
    int nodes = 0;
    if (!warm || !replay) {
        enqueue(bucket, st, &nodes);
        warm = true;
    } else {
        const Graph *g = nullptr;
        for (const Graph &x : graphs) if (x.bucket == bucket) g = &x;
        if (!g) {
            cudaGraph_t graph;
            cudaGraphExec_t exec;
            B200_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            enqueue(bucket, st, &nodes);
            B200_CHECK(cudaStreamEndCapture(st, &graph));
            B200_CHECK(cudaGraphInstantiate(&exec, graph, 0));
            B200_CHECK(cudaGraphDestroy(graph));
            graphs.push_back(Graph{bucket, exec, nodes});
            g = &graphs.back();
        }
        B200_CHECK(cudaGraphLaunch(g->exec, st));
        nodes = g->nodes;
    }
    dev_n_past = n_kv;
    return nodes;
}

void DecodeGraphCache::drop() {
    for (const Graph &g : graphs) cudaGraphExecDestroy(g.exec);
    graphs.clear();
}

}  // namespace b200
