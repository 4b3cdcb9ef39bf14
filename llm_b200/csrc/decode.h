// llm_b200/csrc/decode.h -- parameters of the decode schedules (decode_ops.cu) and the sessions' cache of decode graphs
#pragma once
#include <functional>
#include <utility>
#include <vector>

#include "kernels.cuh"
#include "tp.cuh"

#ifndef B200_PROF_SLOTS
#define B200_PROF_SLOTS 1024
#endif

namespace b200 {

struct DecodeLayer {
    QWeight wqkv, wo, w13, w2;
    const float *attn_norm, *ffn_norm;
    void *K, *V;                        // this layer's slice of memory_k ([n_ctx][gqa]) / memory_v ([gqa][n_ctx], transposed), of DecodeParams::kv_type
};

struct DecodeParams {
    int n_layer;
    QWeight wte, output;
    const float *norm;
    int e, f, hd, gqa, n_head, n_head_kv, n_ctx, n_vocab;
    float kq_scale, eps;
    int kv_type;                        // the KV cache's element type: T_F16 or T_F32 (single GPU only)
    const float2 *rope_cs; int rope_half;
    const uint16_t *lut_silu, *lut_exp;
    const int32_t *token;
    int *n_past;                        // device copy of InferenceSession::n_past; the step's last kernel increments it
    float *x, *q, *kq, *ff, *logits;
    float *normed;                      // single GPU: the final norm's f32 row [e], stored by every step (OutputRequest::embeddings); else null
    int4 *xpack_d, *xpack_f;            // activation records of wo's input (written by the attention kernel) and of w2's input (the w13 epilogue)
    void *xq8k = nullptr;               // single GPU, K-quant lm_head: the Q8_K super-blocks of the final norm's row (q8k_bytes(e, 1))
    // tensor-parallel decode (tp.cuh): dims above are THIS RANK's (n_head, n_head_kv, gqa = local heads / cache width; f = local n_ff / G;
    // n_vocab = local rows of the lm_head) except e = the full n_embd; e_loc = n_embd / G (q rows, rows of wo / w2 owned here)
    TpCtx tp;
    int e_loc = 0, head0 = 0;           // first global head of this rank
    int n_vocab_full = 0;               // rows of the whole lm_head (the gathered logits)
    int64_t row0_e = 0, row0_w13 = 0, row0_v = 0;   // first row of this rank in the full wo / w2 output, the interleaved [w1|w3] rows, the lm_head
    unsigned long long *prof;           // optional (B200_DECODE_PROF): 8 x B200_PROF_SLOTS per-launch %globaltimer slots, see b200_session_decode_timeline
};

// ---- GPT-NeoX (crates/models/gptneox/src/lib.rs:156-350) fused decode schedule: 8 kernels per layer, same mat-vec core -------------------------
struct NeoxLayer {
    QWeight wqkv, wdense, wfc, wproj;   // query_key_value [3e x e] (rows per head: q | k | v), attention.dense, mlp.dense_h_to_4h, mlp.dense_4h_to_h
    const float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *bqkv, *bdense, *bfc, *bproj;
    void *K, *V;                        // [n_ctx][e] by position / [e][n_ctx] transposed, as the reference lays out memory_k / memory_v (:233-247),
                                        // of NeoxParams::kv_type
};
// where q / k / v of head h start inside a row of the fused qkv projection: h * head_stride, + k_off, + v_off.  GPT-NeoX: per head [q | k | v]
// (3 hd, hd, 2 hd); GPT-2, MPT, BLOOM, GPT-J: the three thirds of the row (hd, e, 2 e)
struct QkvLayout { int head_stride, k_off, v_off; };
struct NeoxParams {
    int n_layer, e, hd, n_head, n_ctx, n_vocab, parallel_residual;
    int kv_type;                                // the KV cache's element type: T_F16 or T_F32
    int n_rot;                                  // RoPE mode 2 (GPT-NeoX) on n_rot of every head; 0: no mode-2 rotation
    QkvLayout qkv_layout;
    const float *wpe;                           // GPT-2 (crates/models/gpt2/src/lib.rs:138-329): learned positions [n_ctx][e] f32, else nullptr
    QWeight wte, lm_head;
    const float *lnf_g, *lnf_b;
    float kq_scale;
    const float2 *rope_cs; int rope_half;
    const uint16_t *lut_gelu, *lut_exp;
    const int32_t *token; int *n_past;
    float *x, *qkv, *q, *attn_out, *logits;     // residual stream [e], raw qkv [3e], roped q [e], attention branch output [e]
    float *normed;                              // the final LayerNorm's f32 row [e], stored by every step (OutputRequest::embeddings)
    int4 *xpack_a, *xpack_d, *xpack_f;          // records: layer-norm output (K = e), attention rows (K = e), gelu output (K = 4e)
    // MPT / BLOOM (crates/models/{mpt,bloom}): the GPT-2 row layout (no wpe) plus ALiBi; MPT leaves every bias pointer null
    const float *alibi = nullptr;               // per-head ALiBi slopes [n_head] (alibi_slopes), else nullptr
    const float *emb_g = nullptr, *emb_b = nullptr;   // BLOOM: LayerNorm of the embedding row before layer 0, else nullptr
    // GPT-J (crates/models/gptj): q | k | v thirds with RoPE mode 0 over the whole head (rope_cs: rope_table(n_rot, 0, .., hd, ..)), one LayerNorm per
    // layer feeding attention and MLP (ln2_*, bqkv, bdense null), the 6-kernel schedule of decode_ops.cu::gptj_ops_t
    int gptj = 0;
    const float *lm_head_b = nullptr;           // GPT-J: lm_head.bias [n_vocab], added after the lm_head; else nullptr
};
// ggml_alibi's per-head slopes (LC/ggml.c:11570-11588), computed with the host's libm powf exactly as the reference computes them
std::vector<float> alibi_slopes(int n_head, float max_bias);
void decode_set_tp(const TpCtx &T, cudaStream_t st);   // uploads the tensor-parallel context the decode kernels read (constant memory)
void neox_decode_enqueue(const NeoxParams &P, const std::vector<NeoxLayer> &layers, int wtype, int n_kv_bucket, cudaStream_t st, int *launches);
// whether neox_decode_enqueue takes a session of P's geometry and a step in the context bucket n_kv_bucket; otherwise the step runs per op
bool neox_decode_fits(const NeoxParams &P, int n_kv_bucket);

// whether attn_fused_kernel's shared memory for a context bucket of n_kv_bucket positions (rounded up to 64) and head size hd fits the 227 KB
// opt-in limit: true up to 3264 positions for every hd <= 256 with an f16 cache (kv_type T_F16), up to 1664 with an f32 cache (T_F32: f32
// probabilities and V rows, 136 bytes per position instead of 70), so 256-position buckets up to 1536.  Past it LLaMA decodes with the two-kernel
// attention and the GPT-NeoX family per op.
bool attn_fused_fits(int n_kv_bucket, int hd, int kv_type = T_F16);
// the longest context (27520 positions) whose scores, f32 probabilities and V tiles the two-kernel attention of an f32 cache holds in one CTA's
// shared memory; LLaMA sessions with an f32 cache and a longer context decode per op
int attn_sv_f32_max_ctx();

// default decode schedule: 8 fused kernels per layer on `st` (decode_ops.cu); position read from *P.n_past on the device
void decode_ops_enqueue(const DecodeParams &P, const std::vector<DecodeLayer> &layers, int wtype, int n_kv_bucket, int4 *xpack_a, cudaStream_t st, int *launches);

// A session's decode graphs (decode_ops.cu): one per context bucket of 256 positions, and the device copy of n_past the schedules read.
struct DecodeGraphCache {
    struct Graph { int bucket; cudaGraphExec_t exec; int nodes; };   // nodes: the step's launches (buckets past 3264 positions launch more)
    std::vector<Graph> graphs;
    bool warm = false;                  // the first step runs eagerly (it sets kernel attributes), later ones replay a graph
    int *d_n_past = nullptr, *h_n_past = nullptr;          // device word, pinned staging word
    int dev_n_past = -1;                // value currently held by *d_n_past (-1: unknown)

    DecodeGraphCache();                 // allocates the n_past words
    ~DecodeGraphCache();                // drop() and frees them
    DecodeGraphCache(const DecodeGraphCache &) = delete;
    DecodeGraphCache &operator=(const DecodeGraphCache &) = delete;

    // the context bucket a step at position n_kv - 1 runs in: n_kv rounded up to 256 positions, at most n_ctx
    static int bucket(int n_kv, int n_ctx);
    // one decode step at position n_kv - 1 (its last kernel increments *d_n_past): enqueue(bucket, st, &nodes) enqueues the schedule for up to
    // `bucket` positions.  Uploads n_past first if the device copy is stale (after a prefill, a rewind, or steps that did not run the schedule).
    // Runs it eagerly on the first step or when replay is false, else replays (capturing on first use) the bucket's graph.
    // Returns the step's launch count.
    int run(int n_kv, int n_ctx, bool replay, const std::function<void(int, cudaStream_t, int *)> &enqueue, cudaStream_t st);
    // destroys every graph (they hold kernel arguments that changed)
    void drop();
};

}  // namespace b200
