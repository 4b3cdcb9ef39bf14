// llm_b200/csrc/decode.cu -- one decoded token = ONE persistent cooperative kernel (Llama::evaluate with a single token,
// crates/models/llama/src/lib.rs:144-368), bit-exact with the reference's CPU path.
//
// Why: at batch 1 the 7B graph is ~129 weight mat-vecs of a few microseconds each plus ~400 tiny row ops; launched one by one the GPU
// spends more time filling and draining pipelines than streaming weights.  Here every CTA stays resident for the whole token:
//   * its producer warp walks the model's weight matrices in graph order and keeps the shared-memory ring full with cp.async;
//     weights do not depend on activations, so streaming continues while the compute warps wait at a phase boundary or run attention;
//   * its 4 compute warps execute the graph phase by phase, separated by grid-wide barriers (6 per layer):
//       A  pack(rms_norm(x) * attn_norm) -> [wq|wk|wv] mat-vec -> RoPE, K/V rows stored to the f16 cache     (llama lib.rs:183-244)
//       B  KQ = K . f16(Q) for every cached position                                                         (:246-265)
//       C  scale + soft_max (fp16 exp table) + KQV = V^T . f16(P), written in merged [n_embd] order          (:268-307)
//       D  pack(attn) -> wo mat-vec + residual                                                               (:310-314)
//       E  pack(rms_norm(inpFF) * ffn_norm) -> [w1|w3] mat-vec                                               (:318-325)
//       F  pack(silu(w1 x) * (w3 x)) -> w2 mat-vec + residual                                                (:328-334)
//     then final norm -> lm_head.  Every CTA re-derives the (tiny) quantized activation vector it needs on its own; only the
//     mat-vec outputs travel through global memory (L2).
// Arithmetic is exactly that of exact.cu / rowops.cu (AVX2 lane chains, ggml_vec_dot_f16 order, fp16 tables, host-built RoPE table).
#include "decode.h"
#include "stream_core.cuh"

namespace b200 {

using namespace stream;

namespace {

__device__ __forceinline__ float lutf(const uint16_t *t, float x) { return f16_bits_to_f32(__ldg(t + f32_to_f16_bits(x))); }

// all CTAs resident (cooperative launch); only the 128 compute threads of each CTA take part
__device__ __forceinline__ void grid_sync(unsigned int *bar, int tid) {
    compute_sync();
    if (tid == 0) {
        volatile unsigned int *genp = bar + 1;
        const unsigned int gen = *genp;
        __threadfence();
        if (atomicAdd(bar, 1u) == gridDim.x - 1) {
            bar[0] = 0;
            __threadfence();
            atomicAdd(bar + 1, 1u);
        } else {
            while (*genp == gen) __nanosleep(32);
        }
        __threadfence();
    }
    compute_sync();
}

// element i (i < 16: low half, element i and i+16 of the block) of one quant block of a planes matrix (dequantize_row_*, LC/ggml.c:1525-1635)
template <int TYPE>
__device__ __forceinline__ void dequant_pair(const QWeight &w, int64_t blk, int j, float &lo, float &hi) {
    float d, m = 0.f;
    if (has_min(TYPE)) { const __half2 dm = ((const __half2 *)w.dm)[blk]; d = __low2float(dm); m = __high2float(dm); }
    else d = __half2float(((const __half *)w.dm)[blk]);
    if (TYPE == T_Q8_0) { const int8_t *q = (const int8_t *)w.qs + blk * 32; lo = (float)q[j] * d; hi = (float)q[j + 16] * d; return; }
    const int q = w.qs[blk * 16 + j];
    int q0 = q & 0xF, q1 = q >> 4;
    if (has_qh(TYPE)) { const uint32_t qh = w.qh[blk]; q0 |= ((qh >> j) & 1) << 4; q1 |= ((qh >> (j + 16)) & 1) << 4; }
    if (TYPE == T_Q4_0) { lo = (float)(q0 - 8) * d; hi = (float)(q1 - 8) * d; }
    else if (TYPE == T_Q5_0) { lo = (float)(q0 - 16) * d; hi = (float)(q1 - 16) * d; }
    else { lo = __fmaf_rn((float)q0, d, m); hi = __fmaf_rn((float)q1, d, m); }
}

// ggml_vec_dot_f16 reduction tree over a warp (see exact.cu)
__device__ __forceinline__ float f16dot_tree(float s) {
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 16));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 8));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 4));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 1));
    s = __fadd_rn(s, __shfl_down_sync(0xffffffffu, s, 2));
    return s;
}

template <int TYPE>
__global__ void __launch_bounds__(STHREADS) llama_decode_kernel(const DecodeParams P) {
    using T = St<TYPE>;
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int DST = (TYPE == T_Q8_0) ? 5 : 8;              // ring depth: ~80 KB of weights in flight per CTA (2 CTAs / SM)
    Ring R{(uint64_t *)smem, (uint64_t *)smem + SST_MAX, smem + 256, 0u, DST};
    double *shd = (double *)(smem + 128);                      // 8 doubles of reduction scratch (behind the 16 mbarriers)
    uint8_t *scratch = R.base + T::ring_bytes(DST);                 // activation records (mat-vec phases) | attention scratch (phases B, C)
    int4 *sx = (int4 *)scratch;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, ncta = gridDim.x;
    if (tid == 0) ring_init(R.full, R.empty, DST);
    __syncthreads();

    if (tid >= SCOMPUTE) {
        // ===== producer warp: the token's weights, in graph order =====
        for (int il = 0; il < P.n_layer; il++) {
            const DecodeLayer *L = P.layers + il;
            { const QWeight w = L->wqkv; produce_matvec<TYPE>(w, R, cta, ncta, lane); }
            { const QWeight w = L->wo;   produce_matvec<TYPE>(w, R, cta, ncta, lane); }
            { const QWeight w = L->w13;  produce_matvec<TYPE>(w, R, cta, ncta, lane, 2); }
            { const QWeight w = L->w2;   produce_matvec<TYPE>(w, R, cta, ncta, lane); }
        }
        produce_matvec<TYPE>(P.output, R, cta, ncta, lane);
        return;
    }

    // ===== compute warps =====
    const int e = P.e, f = P.f, hd = P.hd, gqa = P.gqa, n_ctx = P.n_ctx;
    const int p = __ldcg(P.n_past), n_kv = p + 1;
    const int tok = __ldcg(P.token);
    int pslot = 0;
    auto mark = [&]() {
        if (P.prof && cta == 0 && tid == 0 && pslot < 127) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); P.prof[pslot] = t; }
        pslot++;
    };
    mark();
    float *sv = (float *)(scratch + (size_t)(e / QK) * 64);     // [e] staged activation vector, right behind the e-sized record array
    float *stash = (float *)(scratch + (size_t)P.scratch_bytes - 256); // 64 floats at the very end of the scratch area

    // rms_norm(src) * gain -> quantize -> records in sx.  The vector and the gain are fetched with ALL loads in flight (registers),
    // the normalised row goes through shared memory, then each warp quantizes every 4th block (ggml_rms_norm + ggml_mul + the
    // INIT-phase quantize_row_q8_* of the following mul_mat; LC/ggml.c:10129-10175, 1217-1300).
    constexpr int MAXV = 12;                                    // float4 per thread: n_embd <= 6144
    auto norm_pack = [&](const float *src, const float *gain) {
        float4 xv[MAXV], gv[MAXV];
        const int nv4 = e / 4;
#pragma unroll
        for (int k = 0; k < MAXV; k++) {
            const int i = tid + k * SCOMPUTE;
            if (i < nv4) { xv[k] = __ldcg((const float4 *)src + i); gv[k] = __ldg((const float4 *)gain + i); }
        }
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < MAXV; k++)
            if (tid + k * SCOMPUTE < nv4) {
                s += (double)__fmul_rn(xv[k].x, xv[k].x); s += (double)__fmul_rn(xv[k].y, xv[k].y);
                s += (double)__fmul_rn(xv[k].z, xv[k].z); s += (double)__fmul_rn(xv[k].w, xv[k].w);
            }
        s = warp_sum(s);
        if (lane == 0) shd[warp] = s;
        compute_sync();
        const double tot = (shd[0] + shd[1]) + (shd[2] + shd[3]);
        const float mean = (float)(tot / (double)e);
        const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, P.eps)));
#pragma unroll
        for (int k = 0; k < MAXV; k++) {
            const int i = tid + k * SCOMPUTE;
            if (i < nv4) {
                float4 y;
                y.x = __fmul_rn(__fmul_rn(xv[k].x, scale), gv[k].x); y.y = __fmul_rn(__fmul_rn(xv[k].y, scale), gv[k].y);
                y.z = __fmul_rn(__fmul_rn(xv[k].z, scale), gv[k].z); y.w = __fmul_rn(__fmul_rn(xv[k].w, scale), gv[k].w);
                ((float4 *)sv)[i] = y;
            }
        }
        compute_sync();
        for (int b0 = warp * 4; b0 < e / QK; b0 += SCOMPUTE / 8) {           // 4 blocks per warp pass (e / 32 is a multiple of 4)
            const int b = b0 + (lane >> 3);
            pack_quad(((const float4 *)sv)[b * 8 + (lane & 7)], sx + b * 4, lane, true, has_min(TYPE) ? 1 : 0, TYPE == T_Q5_0 ? 16 : 0, TYPE == T_Q4_0 ? 1 : 0);
        }
        compute_sync();
    };
    auto load_pack = [&](const int4 *src, int nbk) {           // records produced by an earlier phase (global, L2) -> sx
        for (int i = tid; i < nbk * 4; i += SCOMPUTE) sx[i] = __ldcg(src + i);
        compute_sync();
    };

    // embedding row: get_rows(tok_embeddings, token)                                             llama lib.rs:170
    for (int b = cta; b < e / QK; b += ncta)
        if (tid < 16) {
            float lo, hi;
            dequant_pair<TYPE>(P.wte, (int64_t)tok * (e / QK) + b, tid, lo, hi);
            P.x[b * QK + tid] = lo; P.x[b * QK + tid + 16] = hi;
        }
    grid_sync(P.bar, tid);
    mark();

    for (int il = 0; il < P.n_layer; il++) {
        const DecodeLayer *L = P.layers + il;
        __half *Kl = L->K, *Vl = L->V;
        // ---- A: attention norm -> QKV mat-vec -> RoPE + KV store ----
        {
            norm_pack(P.x, L->attn_norm);
            mark();
            const QWeight w = L->wqkv;
            consume_matvec<TYPE>(w, sx, R, cta, ncta, tid, [&](int64_t row, float v) {
                const float other = __shfl_xor_sync(0xffffffffu, v, 4);          // the rotation partner: rows 2i and 2i+1 sit in adjacent quads
                if ((tid & 3) != 0 || row >= w.N) return;
                if (row < e + gqa) {                                               // Q or K row: ggml_rope mode 0 (LC/ggml.c:11859-11874)
                    const int within = (int)(row < e ? row : row - e);
                    const float2 cs = __ldg(P.rope_cs + (int64_t)p * P.rope_half + (within % hd) / 2);
                    const bool even = (row & 1) == 0;
                    const float x0 = even ? v : other, x1 = even ? other : v;
                    const float out = even ? __fmaf_rn(x0, cs.x, -__fmul_rn(x1, cs.y)) : __fmaf_rn(x0, cs.y, __fmul_rn(x1, cs.x));
                    if (row < e) P.q[row] = out;
                    else Kl[(int64_t)p * gqa + within] = __float2half_rn(out);    // cpy f32 -> f16 into memory_k          (:243)
                } else {
                    Vl[(int64_t)(row - e - gqa) * n_ctx + p] = __float2half_rn(v); // transposed V store                    (:244)
                }
            });
        }
        mark(); grid_sync(P.bar, tid); mark();
        // ---- B: KQ[h][j] = K[j][h] . f16(Q[h])  (ggml_vec_dot_f16 order); work item = 64 cached positions of one head ----
        {
            __half *q16 = (__half *)scratch;
            __half *kt = (__half *)(scratch + 512);                 // [64][hd] staged K rows
            const int chunks = (n_kv + 63) / 64, items = P.n_head * chunks;
            const int vec_per_row = hd / 8;                         // 16-byte vectors per K row
            for (int it = cta; it < items; it += ncta) {
                const int h = it / chunks, j0 = (it - h * chunks) * 64;
                const int hk = h / (P.n_head / P.n_head_kv);
                const int rows = n_kv - j0 < 64 ? n_kv - j0 : 64;
                for (int i = tid; i < hd; i += SCOMPUTE) q16[i] = __float2half_rn(__ldcg(P.q + h * hd + i));
                for (int i = tid; i < rows * vec_per_row; i += SCOMPUTE) {       // all 16-byte loads of the tile in flight at once
                    const int rr = i / vec_per_row, cc = i - rr * vec_per_row;
                    ((int4 *)kt)[rr * vec_per_row + cc] = __ldcg((const int4 *)(Kl + (int64_t)(j0 + rr) * gqa + hk * hd) + cc);
                }
                compute_sync();
                const int np = hd & ~31;
                for (int jj = warp; jj < rows; jj += SCOMPUTE / 32) {
                    const __half *krow = kt + jj * hd;
                    float s = 0.f;
                    for (int k = lane; k < np; k += 32) s = __fmaf_rn(__half2float(krow[k]), __half2float(q16[k]), s);
                    s = f16dot_tree(s);
                    if (lane == 0) {
                        double sumf = (double)s;
                        for (int k = np; k < hd; k++) sumf += (double)__fmul_rn(__half2float(krow[k]), __half2float(q16[k]));
                        P.kq[(int64_t)h * n_ctx + j0 + jj] = (float)sumf;
                    }
                }
                compute_sync();
            }
        }
        mark(); grid_sync(P.bar, tid); mark();
        // ---- C: scale, soft_max, KQV for 32 channels of one head per work item; the 32 outputs are one quant block of wo's input ----
        {
            constexpr int KC = 128;                              // cached positions per staged V tile
            float *sc = (float *)scratch;                        // [n_kv] exp values
            __half *p16 = (__half *)(scratch + (size_t)n_ctx * 4);
            __half *vt = (__half *)(scratch + (size_t)n_ctx * 6);   // [32][KC]
            float *shf = (float *)shd;
            const int per_head = hd / 32, items = P.n_head * per_head;
            for (int it = cta; it < items; it += ncta) {
                const int h = it / per_head, c0 = (it - h * per_head) * 32;
                const int hk = h / (P.n_head / P.n_head_kv);
                float mx = -INFINITY;
                for (int j = tid; j < n_kv; j += SCOMPUTE) { const float v = __fmul_rn(__ldcg(P.kq + (int64_t)h * n_ctx + j), P.kq_scale); sc[j] = v; mx = fmaxf(mx, v); }
                mx = warp_max(mx);
                if (lane == 0) shf[warp] = mx;
                compute_sync();
                mx = fmaxf(fmaxf(shf[0], shf[1]), fmaxf(shf[2], shf[3]));
                double s = 0.0;
                for (int j = tid; j < n_kv; j += SCOMPUTE) { const float ev = lutf(P.lut_exp, __fsub_rn(sc[j], mx)); sc[j] = ev; s += (double)ev; }
                s = warp_sum(s);
                if (lane == 0) shd[4 + warp] = s;
                compute_sync();
                const float inv = (float)(1.0 / ((shd[4] + shd[5]) + (shd[6] + shd[7])));
                for (int j = tid; j < n_kv; j += SCOMPUTE) p16[j] = __float2half_rn(__fmul_rn(sc[j], inv));
                const int np = n_kv & ~31;
                float acc[8];
#pragma unroll
                for (int cc = 0; cc < 8; cc++) acc[cc] = 0.f;
                // leftover columns [np, n_kv) of the 32 V rows, fetched up front (one 16-byte vector per thread)
                __half *vleft = vt + 32 * KC;                     // [32][32]
                if (np < n_kv) {
                    const int rr = tid >> 2, part = tid & 3;
                    ((int4 *)vleft)[tid] = __ldcg((const int4 *)(Vl + (int64_t)(hk * hd + c0 + rr) * n_ctx + np) + part);
                }
                int4 pre[KC / 32];                                 // next V tile, prefetched into registers while the current one is consumed
                auto fetch = [&](int k0) {
#pragma unroll
                    for (int u = 0; u < KC / 32; u++) {
                        const int i = tid + u * SCOMPUTE, rr = i / (KC / 8), cc = i - rr * (KC / 8);
                        pre[u] = __ldcg((const int4 *)(Vl + (int64_t)(hk * hd + c0 + rr) * n_ctx + k0) + cc);
                    }
                };
                if (np > 0) fetch(0);
                for (int k0 = 0; k0 < np; k0 += KC) {
                    compute_sync();                                // p16 complete / previous tile consumed
#pragma unroll
                    for (int u = 0; u < KC / 32; u++) ((int4 *)vt)[tid + u * SCOMPUTE] = pre[u];
                    compute_sync();
                    if (k0 + KC < np) fetch(k0 + KC);
                    const int kend = np - k0 < KC ? np - k0 : KC;
#pragma unroll
                    for (int cc = 0; cc < 8; cc++) {
                        const __half *vrow = vt + (warp * 8 + cc) * KC;
                        for (int k = lane; k < kend; k += 32) acc[cc] = __fmaf_rn(__half2float(vrow[k]), __half2float(p16[k0 + k]), acc[cc]);
                    }
                }
                compute_sync();
#pragma unroll
                for (int cc = 0; cc < 8; cc++) {
                    const float a = f16dot_tree(acc[cc]);
                    if (lane == 0) {
                        const __half *vrow = vleft + (warp * 8 + cc) * 32;
                        double sumf = (double)a;
                        for (int k = np; k < n_kv; k++) sumf += (double)__fmul_rn(__half2float(vrow[k - np]), __half2float(p16[k]));
                        stash[warp * 8 + cc] = (float)sumf;
                    }
                }
                compute_sync();
                if (warp == 0)
                    pack_quad(((const float4 *)stash)[lane & 7], P.xpack_d + (int64_t)((h * hd + c0) / QK) * 4, lane, lane < 8, has_min(TYPE) ? 1 : 0,
                              TYPE == T_Q5_0 ? 16 : 0, TYPE == T_Q4_0 ? 1 : 0);
                compute_sync();
            }
        }
        mark(); grid_sync(P.bar, tid); mark();
        // ---- D: wo + residual ----
        {
            load_pack(P.xpack_d, e / QK);
            mark();
            const QWeight w = L->wo;
            consume_matvec<TYPE>(w, sx, R, cta, ncta, tid, [&](int64_t row, float v) {
                if ((tid & 3) == 0 && row < w.N) P.ff[row] = __fadd_rn(v, __ldcg(P.x + row));
            });
        }
        mark(); grid_sync(P.bar, tid); mark();
        // ---- E: ffn norm -> [w1|w3] (rows interleaved in 32-row chunks: a pair of tiles = w1 x and w3 x for the same 32 channels)
        //         -> silu(w1 x) * (w3 x) quantized right here: one block of w2's input per tile pair ----
        {
            norm_pack(P.ff, L->ffn_norm);
            mark();
            const QWeight w = L->w13;
            consume_matvec<TYPE>(w, sx, R, cta, ncta, tid, [&](int64_t row, float v) {
                if ((tid & 3) == 0) stash[row & 63] = v;
                if (((row >> 5) & 1) == 0) return;                                 // first tile of the pair: keep going
                compute_sync();
                if (warp == 0) {
                    const int w8 = lane & 7;
                    const float4 a = ((const float4 *)stash)[w8], b = ((const float4 *)stash)[8 + w8];
                    float4 hm;                                                     // silu(w1 x) * (w3 x)  (:328-330)
                    hm.x = __fmul_rn(lutf(P.lut_silu, a.x), b.x); hm.y = __fmul_rn(lutf(P.lut_silu, a.y), b.y);
                    hm.z = __fmul_rn(lutf(P.lut_silu, a.z), b.z); hm.w = __fmul_rn(lutf(P.lut_silu, a.w), b.w);
                    pack_quad(hm, P.xpack_f + (row >> 6) * 4, lane, lane < 8, has_min(TYPE) ? 1 : 0, TYPE == T_Q5_0 ? 16 : 0, TYPE == T_Q4_0 ? 1 : 0);
                }
                compute_sync();
            }, 2);
        }
        mark(); grid_sync(P.bar, tid); mark();
        // ---- F: w2 + residual ----
        {
            load_pack(P.xpack_f, f / QK);
            mark();
            const QWeight w = L->w2;
            consume_matvec<TYPE>(w, sx, R, cta, ncta, tid, [&](int64_t row, float v) {
                if ((tid & 3) == 0 && row < w.N) P.x[row] = __fadd_rn(v, __ldcg(P.ff + row));
            });
        }
        mark(); grid_sync(P.bar, tid); mark();
    }
    // ---- final norm -> lm_head ----
    {
        norm_pack(P.x, P.norm);
        consume_matvec<TYPE>(P.output, sx, R, cta, ncta, tid, [&](int64_t row, float v) {
            if ((tid & 3) == 0 && row < P.output.N) P.logits[row] = v;
        });
    }
    if (P.prof && cta == 0 && tid == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); P.prof[127] = t; }
    if (cta == 0 && tid == 0) *P.n_past = p + 1;               // InferenceSession::n_past += 1 (inference_session.rs:288)
}

template <int TYPE>
int decode_smem_bytes(const DecodeParams &P) {
    return (int)(256 + St<TYPE>::ring_bytes(TYPE == T_Q8_0 ? 5 : 8) + P.scratch_bytes);
}

template <int TYPE>
bool launch_decode_t(const DecodeParams &P, cudaStream_t st, int *grid_out) {
    const int smem = decode_smem_bytes<TYPE>(P);
    static int smem_set = 0, grid = 0;
    if (smem > 227 * 1024) return false;
    if (smem != smem_set) {
        B200_CHECK(cudaFuncSetAttribute(llama_decode_kernel<TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        int dev, sms, per_sm;
        B200_CHECK(cudaGetDevice(&dev));
        B200_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        B200_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, llama_decode_kernel<TYPE>, STHREADS, smem));
        if (per_sm < 1) return false;
        grid = sms * per_sm;                                   // every CTA resident: the grid barrier relies on it (cooperative launch checks)
        smem_set = smem;
    }
    void *args[] = {(void *)&P};
    B200_CHECK(cudaLaunchCooperativeKernel((const void *)llama_decode_kernel<TYPE>, dim3(grid), dim3(STHREADS), args, smem, st));
    if (grid_out) *grid_out = grid;
    return true;
}

}  // namespace

int decode_scratch_bytes(int e, int f, int hd, int n_ctx) {
    size_t a = (size_t)(e / QK) * 64 + (size_t)e * 4;        // records + staged vector (phases A, E, final)
    size_t b = (size_t)(f / QK) * 64;                          // records of w2's input (phase F)
    size_t c = 512 + (size_t)64 * hd * 2;                      // q16 + staged K tile (phase B)
    size_t d = (size_t)n_ctx * 6 + 32 * 128 * 2 + 32 * 32 * 2;  // exp values, fp16 probabilities, staged V tile + leftover columns (phase C)
    size_t m = a; if (b > m) m = b; if (c > m) m = c; if (d > m) m = d;
    return (int)(((m + 255) & ~(size_t)255) + 256);            // + 64 floats of epilogue stash at the end
}

bool decode_supported(const DecodeParams &P, int wtype) {
    if (P.e > 6144 || P.e % 128 || P.f % 32 || P.hd % 32 || P.n_ctx % 128 || P.hd > 256) return false;
    QWeight probe; probe.nb = P.e / QK;
    QWeight probe2; probe2.nb = P.f / QK;
    return is_quant(wtype) && mmv_exact_stream_supported(probe) && mmv_exact_stream_supported(probe2) && P.hd % 2 == 0 && P.hd <= 256 && P.e % 64 == 0 &&
           P.gqa % SR == 0 && P.e % SR == 0;
}

bool launch_decode(const DecodeParams &P, int wtype, cudaStream_t st, int *grid_out) {
    switch (wtype) {
        case T_Q4_0: return launch_decode_t<T_Q4_0>(P, st, grid_out);
        case T_Q4_1: return launch_decode_t<T_Q4_1>(P, st, grid_out);
        case T_Q5_0: return launch_decode_t<T_Q5_0>(P, st, grid_out);
        case T_Q5_1: return launch_decode_t<T_Q5_1>(P, st, grid_out);
        case T_Q8_0: return launch_decode_t<T_Q8_0>(P, st, grid_out);
    }
    return false;
}

}  // namespace b200
