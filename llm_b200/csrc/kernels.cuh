// llm_b200/csrc/kernels.cuh -- launchers of the hand-written sm_90a kernels (plain pointers, explicit stream).
// Used by all three front ends: the ggml_cuda_* seam (seam.cu) and the native LLaMA (session.cu) and GPT-NeoX / GPT-2 (neox.cu) sessions.
#pragma once
#include "common.cuh"

namespace b200 {

// ---- quant.cu ------------------------------------------------------------------------------------------------
// Carve the planes of a QWeight out of `base` (allocates nothing); returns bytes needed when base == nullptr.
size_t qweight_layout(QWeight &w, int type, int64_t K, int64_t N, void *base);
// raw: N rows of GGML blocks (device memory, as uploaded from the file/host tensor) -> planes of w
void repack_weights(const QWeight &w, const void *raw, cudaStream_t st);
// inverse (debug / tests): planes -> GGML array-of-blocks
void unpack_weights(const QWeight &w, void *raw, cudaStream_t st);
// Activation quantizer, bit-faithful to the reference's AVX2 quantize_row_q8_0 / q8_1 (LC/ggml.c:1217-1300, 1427-1518).
//   x  : [B] rows of K f32, row stride ldx elements
//   qs : [B][K] int8          ds : [B][K/32] float2 {d, aux}
//   Q8_0: d = f32(fp16(amax/127)), aux = (float)sum(q)   (exact integer; used for the -8/-16 offsets)
//   Q8_1: d = amax/127 (f32),      aux = d * (float)sum(q)  (= block_q8_1.s, LC/ggml.c:1474)
void quantize_act(int vdt, const float *x, int64_t ldx, int8_t *qs, float2 *ds, int64_t K, int64_t B, cudaStream_t st);
// get_rows on a quantized matrix (dequantize_row_*, LC/ggml.c:1525-1635): dst[i][:] = dequant(W[ids[i]][:])
void get_rows_q(const QWeight &w, const int32_t *ids, float *dst, int64_t n, cudaStream_t st);
// same, but source is GGML array-of-blocks in device memory (seam path keeps tok_embeddings in file layout)
void get_rows_raw(int type, const void *raw, int64_t K, const int32_t *ids, float *dst, int64_t n, cudaStream_t st);

// ---- mmvq.cu : decode path, HBM-bound --------------------------------------------------------------------------
// dst[n] = sum_b (d_w d_x) * int_dot + m_w s_x  (+ addend[n]);  one activation row
void mul_mat_vec_q(const QWeight &w, const int8_t *xq, const float2 *xds, float *dst, const float *addend, cudaStream_t st);

// ---- mmq.cu : prefill path, integer-exact tensor-core GEMM ------------------------------------------------------
// dst[b*ldd + n], b < B
void mul_mat_q(const QWeight &w, const int8_t *xq, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);
// cross-check implementation (CUDA cores, dp4a), same contract
void mul_mat_q_simple(const QWeight &w, const int8_t *xq, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);

// ---- exact.cu : bit-exact (AVX2 operation order) versions; the DEFAULT of every front end -----------------------------------------
// same contract as mul_mat_q for any B >= 1; results are bit-identical to ggml_compute_forward_mul_mat on the reference's x86 build
void mul_mat_q_exact(const QWeight &w, const int8_t *xq, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);

// ---- exact_mma.cu : bit-exact batched mat-mul with the block dots on tensor cores (block-diagonal f16 MMA) --------------------------
// xh = fp16 quants in the MMA-fragment tile order of exact_mma.cu (16-token tiles: allocate xh_bytes(K, B))
inline size_t xh_bytes(int64_t K, int64_t B) { return (size_t)((B + 15) / 16 * 16) * (size_t)K * 2; }
void quantize_act_f16(int vdt, const float *x, int64_t ldx, __half *xh, float2 *ds, int64_t K, int64_t B, cudaStream_t st);
void mul_mat_q_exact_mma(const QWeight &w, const __half *xh, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);

// ---- exact_tc5.cu : the same bit-exact batched mat-mul on wgmma tensor cores (TMA-staged activations, register accumulators) ------------
// xh = fp16 quants, plain row-major [B][K] (16-byte aligned; the TMA source); xds as above
void quantize_act_f16_rm(int vdt, const float *x, int64_t ldx, __half *xh, float2 *ds, int64_t K, int64_t B, cudaStream_t st);
int exact_tc5_check_timeout();   // debugging aid of the op-level entry points: non-zero if a pipeline barrier of the kernel ever timed out
void mul_mat_q_exact_tc5(const QWeight &w, const __half *xh, const float2 *xds, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);

// ---- mmq_tc5.cu : order-free (NON-conformant) fused dequant -> wgmma GEMM, f16 operands, f32 accumulation over K in registers --------------------
void cvt_act_f16(const float *x, int64_t ldx, __half *xh, int64_t K, int64_t B, cudaStream_t st);      // f32 rows -> fp16 row-major [B][K]
void mul_mat_q_fast_tc5(const QWeight &w, const __half *xh, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);
int fast_tc5_check_timeout();

// ---- exact_stream.cu : the bit-exact decode mat-vec at HBM speed (TMA bulk-copy ring + AVX2 lane chains) ----------------------------
bool mmv_exact_stream_supported(const QWeight &w);
// bit-faithful activation quantizer emitting 16-byte records per (block, word): see exact_stream.cu
void quantize_act_pack(int wtype, const float *x, int4 *pack, int64_t K, cudaStream_t st);
void mul_mat_vec_q_exact_stream(const QWeight &w, const int4 *xpack, float *dst, const float *addend, cudaStream_t st);

// ---- exact_f16.cu : F16 weights (QWeight type T_F16), ggml_vec_dot_f16 order on fp16-rounded activations (xh: cvt_act_f16 rows) ----------
bool mmv_f16_supported(const QWeight &w);      // the streaming mat-vec's shared memory holds the activation row
void mul_mat_vec_f16(const QWeight &w, const __half *xh, float *dst, const float *addend, cudaStream_t st);                    // one row
void mul_mat_f16_gemm(const QWeight &w, const __half *xh, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda, cudaStream_t st);
void get_rows_f16(const QWeight &w, const int32_t *ids, float *dst, int64_t n, cudaStream_t st);
void f16_to_f32(const void *src, float *dst, int64_t n, cudaStream_t st);          // exact widening (F16 tensors kept as f32)

// ---- mul_mat.cu : the bit-exact ggml_mul_mat of every front end -------------------------------------------------------------------------
bool prefill_gemm_tc5();         // B200_PREFILL_GEMM != "mma" (the default)
// activation buffers for B rows of K: xq [B][K] int8, xds [B][K/32], xpack (K/32) * 64 bytes, xh xh_bytes(K, B)
// xq8k: q8k_bytes(K, B) of Q8_K super-blocks, needed for K-quant weights only
struct ExactActs { int8_t *xq; float2 *xds; int4 *xpack; __half *xh; void *xq8k = nullptr; };
// dst[b*ldd + n] (+ addend[b*lda + n]) for B rows of x (row stride ldx): quantizes x and runs the exact kernel for B -- the streaming mat-vec
// (B == 1), the wgmma GEMM (B >= 96, prefill_gemm_tc5()), the mma.sync GEMM (B >= 16) or exact.cu.  An F16 weight rounds x to fp16 and runs
// exact_f16.cu's mat-vec (B == 1) or GEMM.  A K-quant weight quantizes x to Q8_K and runs kquants.cu.  Returns the number of launches (2).
int mul_mat_exact_auto(const QWeight &w, const float *x, int64_t ldx, int64_t B, float *dst, int64_t ldd, const float *addend, int64_t lda,
                       const ExactActs &a, cudaStream_t st);

// ---- kquants.cu : Q2_K .. Q6_K weights x Q8_K activations, bit-exact with ggml_vec_dot_q*_K_q8_K (AVX2 build) -------------------------
size_t q8k_bytes(int64_t K, int64_t B);
void quantize_act_q8k(const float *x, int64_t ldx, void *y, int64_t K, int64_t B, cudaStream_t st);       // quantize_row_q8_K of every src1 row -> block_q8_K
// w_raw: N rows of K/256 GGML super-blocks, as in the file; n_past_inc (nullable): a word the launch increments once (the decode graph's last node)
void mul_mat_kq_exact(int type, const void *w_raw, const void *xq8k, float *dst, int64_t ldd, int64_t K, int64_t N, int64_t B, const float *addend, int64_t lda,
                      cudaStream_t st, int *n_past_inc = nullptr);
// get_rows on a K-quant matrix in file layout: dequantize_row_q*_K of rows ids[0, n) (w_raw: N rows of K/256 super-blocks)
void get_rows_kq(int type, const void *w_raw, int64_t K, const int32_t *ids, float *dst, int64_t n, cudaStream_t st);

// ---- synth.cu : seeded synthetic tensors generated in HBM (bench / tests) ------------------------------------------------------------
void synth_qweight(const QWeight &w, uint64_t seed, cudaStream_t st);
void synth_gain(float *g, int64_t n, uint64_t seed, cudaStream_t st);                       // 1 + 0.1 N(0,1)
void scale_shift_f32(float *p, int64_t n, float a, float b, cudaStream_t st);                // p = p * a + b

// ---- quantize_file.cu : ggml_quantize_q{4_0,4_1,5_0,5_1,8_0} on the GPU, bit-exact (LC/ggml.c:18083-18208) -------------------------------------
// nblk 32-element blocks of src (src_type T_F32 or T_F16, contiguous) -> nblk GGML blocks of `type` in file layout at dst (16-byte aligned);
// hist (nullable): += the reference's 16-bin histogram of the quants
void quantize_blocks(int type, int src_type, const void *src, int64_t nblk, void *dst, unsigned long long *hist, cudaStream_t st);

// ---- lora.cu : LoRA adapters patched into a weight at load time, bit-exact with the reference's CPU graph (LoraAdapter::patch) ----------------------
// B200_OK, or the LoadError (TensorWrongSize / UnsupportedElementType) for factors A [a_ne0 = r, a_ne1] and B [b_ne0, b_ne1] on a target [K, N] of wtype
int lora_check(int wtype, int64_t K, int64_t N, int a_type, int64_t a_ne0, int64_t a_ne1, int b_type, int64_t b_ne0, int64_t b_ne1);
// in place, on device memory: w (N rows of K in GGML layout, F32 or a 32-element block type) += scaling * (A x B); a: K rows of r (F32 / F16),
// b: nb_rows rows of r f32 (row n of W takes row n % nb_rows).  Arguments checked by lora_check.
void lora_patch(int wtype, void *w, int64_t K, int64_t N, int a_type, const void *a, const float *b, int64_t r, int64_t nb_rows, float scaling, cudaStream_t st);

// ---- ppl.cu : the reference's perplexity arithmetic on logits in HBM, bit-exact (glibc expf / logf restated in libm_f32.h) ---------------------
// terms[r] = -ln(softmax(row r)[targets[r]]) of `rows` rows of n_vocab logits: max, in-order f32 sum of expf(v - max), expf(l[t] - max) / sum
void nll_rows(const float *logits, int64_t rows, int64_t n_vocab, const int32_t *targets, float *terms, cudaStream_t st);
struct PplState { float nll; int64_t count; };        // the running f32 nll and row count of one perplexity call (device memory)
// state += terms[0..n) in order; *ppl = expf(nll / (f32)count)
void nll_fold(const float *terms, int64_t n, PplState *state, float *ppl, cudaStream_t st);

// ---- sample.cu : the reference's default sampler chain (repetition, top-k, top-p, temperature, one draw) on a logits row in HBM -----------
// the draw-th output of SplitMix64 seeded with seed (the draw's uniform is (z >> 40) * 2^-24)
__host__ __device__ inline uint64_t splitmix64(uint64_t seed, uint64_t draw) {
    uint64_t z = seed + (draw + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
struct SampleArgs { float penalty; int last_n, top_k; float top_p, temperature; uint64_t seed, draw; };   // b200_sampler, checked by the caller
struct SampleResult { int32_t id, status, n_cand, n_kept; };      // status 0, or 1: a NaN in the row (the id is then -1)
// device scratch: two key buffers of sample_key_bytes(n_vocab), a zero-initialised fail word, and (nullable) n_vocab floats that receive the
// row when it fails
struct SampleBufs { uint64_t *keys[2]; int *fail; float *backup; };
size_t sample_key_bytes(int n_vocab);
// The chain on row[0, n_vocab) with the penalty window hist[max(0, n_past - last_n), n_past).  The id goes to *tok_dst and *hist_dst, the
// result to *res (mapped host memory: written last, after a system fence); each nullable.  cand_* (nullable): the min(k, n_vocab, 1024)
// candidates in order -- ids, their unpenalized logits row[id], and their top-p probabilities.  Nothing is written to row.
void sample_row(const float *row, int n_vocab, const int32_t *hist, int n_past, const SampleArgs &a, const SampleBufs &b, int32_t *tok_dst, int32_t *hist_dst,
                SampleResult *res, int32_t *cand_ids, float *cand_vals, float *cand_probs, cudaStream_t st);

// ---- rowops.cu : warp/block-reduce kernels ------------------------------------------------------------------------
struct Luts { const uint16_t *silu, *gelu, *exp; };   // 3 x 64 Ki fp16 tables built on the host with libm (LC/ggml.c:4313-4326)
const Luts &luts();                                   // uploaded on first use
// y = x / sqrt(mean(x^2) + eps) [* gain]   (LC/ggml.c:10129-10175 + the following ggml_mul node)
void rms_norm(const float *x, float *y, const float *gain, int64_t n, int64_t rows, float eps, cudaStream_t st);
// y = (x - mean) / sqrt(var + 1e-5) [* gain] [+ bias]   (LC/ggml.c:10063-10111)
void layer_norm(const float *x, float *y, const float *gain, const float *bias, int64_t n, int64_t rows, cudaStream_t st);
// rows of nc: optional scale, optional causal mask (col > n_past + (row % nr) -> -inf), softmax through the fp16 exp table
void soft_max(const float *x, float *y, int64_t nc, int64_t rows, int64_t nr, float scale, bool do_scale, int n_past, bool do_mask, bool do_softmax, cudaStream_t st);
// scale, ALiBi (column i of a row of head row / nr: fma(i, alibi[head], v)), causal mask, softmax -- the MPT / BLOOM attention (alibi: device slopes)
void soft_max_alibi(const float *x, float *y, int64_t nc, int64_t rows, int64_t nr, float scale, int n_past, const float *alibi, cudaStream_t st);
enum { UNARY_SILU = 0, UNARY_GELU = 1 };
void unary_lut(int which, const float *x, float *y, int64_t n, cudaStream_t st);
// y = silu(a) * b  (silu node then mul node, llama lib.rs:328-330)
void silu_mul(const float *a, const float *b, float *y, int64_t n, cudaStream_t st);
// dst = a (op) b with b broadcast modulo its extent (LC/ggml.c:8095-8127, 8852-8886): nb_elems = elements of b
void add_f32(const float *a, const float *b, float *dst, int64_t n, int64_t nb_elems, cudaStream_t st);
void mul_f32(const float *a, const float *b, float *dst, int64_t n, int64_t nb_elems, cudaStream_t st);
void scale_f32(const float *a, float scale, float *dst, int64_t n, cudaStream_t st);
// RoPE through host-built cos/sin tables that follow the reference's f32 recurrence (LC/ggml.c:11832-11897)
struct RopeTable { const float2 *cs; int n_pos; int half; int n_dims; int mode; float freq_base, freq_scale; int ne0; };
const RopeTable &rope_table(int n_dims, int mode, float freq_base, float freq_scale, int ne0, int n_pos_needed);
// x: [ne2 positions][ne1 heads][ne0] f32 with strides (elements) s1, s2; position p = n_past + i2
void rope_f32(const float *x, float *y, int64_t ne0, int64_t ne1, int64_t ne2, int64_t s1, int64_t s2, int64_t ds1, int64_t ds2,
              int n_past, const RopeTable &tab, cudaStream_t st);
// generic strided copy with type conversion f32->f32 / f32->f16 / f16->f16 / f16->f32; shapes may differ, element order is kept
struct StridedDesc { int64_t ne[4]; int64_t nb[4]; };  // nb in BYTES
void cpy_strided(const void *src, int src_type, const StridedDesc &s, void *dst, int dst_type, const StridedDesc &d, cudaStream_t st);

// ---- attn.cu : the two non-weight mat-muls on the f16 KV cache ------------------------------------------------------
// dst[i2][i1][i0] = sum_k f16(src0[i2/(ne12/ne02)][i0][k]) * f16round(src1[i2][i1][k]), f32 accumulate
// (F16 type traits: src1 is rounded to fp16 first, LC/ggml.c:1650-1656, 10504-10520; ggml_vec_dot_f16 :2325-2359)
void mul_mat_f16(const __half *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                 const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                 float *dst, int64_t nbd1, int64_t nbd2, cudaStream_t st);

// ggml_vec_dot_f16 operation order (exact.cu); causal_past >= 0 skips outputs i0 > causal_past + i1 (masked to -inf downstream)
void mul_mat_f16_exact(const __half *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                       const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                       float *dst, int64_t nbd1, int64_t nbd2, int causal_past, cudaStream_t st);
// the same shape contract and causal skip on an f32 cache: ggml_vec_dot_f32 operation order (f32dot.cuh), src1 as it is (F32 type traits: no
// rounding, LC/ggml.c:1646-1648, 10504-10520)
void mul_mat_f32_exact(const float *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                       const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12,
                       float *dst, int64_t nbd1, int64_t nbd2, int causal_past, cudaStream_t st);

}  // namespace b200
