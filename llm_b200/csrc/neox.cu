// llm_b200/csrc/neox.cu -- native host runtime for GPT-NeoX and GPT-2 (include/llm_b200.h: b200_neox_*): model + InferenceSession on the GPU.
//
// Mirrors   GptNeoX::new / TensorLoader         crates/models/gptneox/src/lib.rs:36-140
//           GptNeoX::evaluate (the graph)       crates/models/gptneox/src/lib.rs:156-350   (feed-forward: :487-515)
//           Gpt2::new / Gpt2::evaluate          crates/models/gpt2/src/lib.rs:43-136, 138-329   (hp.arch == 1: c_attn rows in thirds, no RoPE, learned positions,
//                                                                                               sequential residual, lm_head optional -> tied to wte)
//           GptJ::new / GptJ::evaluate          crates/models/gptj/src/lib.rs:47-122, 134-311   (hp.arch == 4: q_proj | k_proj | v_proj as thirds of one wqkv,
//                                                                                               RoPE mode 0 over the whole head, one LayerNorm feeding attention and
//                                                                                               MLP, lm_head + lm_head.bias; decode: decode_ops.cu::gptj_ops_t)
//           InferenceSession::compute           crates/llm-base/src/inference_session.rs:114-295
// Batches (prefill) run node by node on the bit-exact kernels of this directory (LayerNorm, bias adds, RoPE mode 2 on n_rot of the head size, gelu table,
// exact quantized mat-muls incl. the wgmma GEMM, exact f16 attention mat-muls); single tokens run the fused 8-kernels-per-layer schedule of
// decode_ops.cu::neox_decode_enqueue from one CUDA graph per context bucket.  Logits are bit-identical to the reference's CPU path (tests/test_gpu_neox.py).
#include <math.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/llm_b200.h"
#include "host.h"

using namespace b200;

namespace {

// One tensor of an architecture.  Sizes: E = n_embd, E3 / E4 = 3 / 4 n_embd, VOCAB = n_vocab, CTX_E = context_size x n_embd.
enum Dim : uint8_t { E, E3, E4, VOCAB, CTX_E };
enum Kind : uint8_t {
    MAT,        // quantized K x N matrix
    GAIN,       // f32 vector of K floats, synthesized as 1 + 0.1 N(0,1)
    BIAS,       // f32 vector of K floats, synthesized as 0.01 N(0,1)
    ROWS,       // rows [at n_embd, (at + 1) n_embd) of the matrix q, which another entry carves and draws
};
template <class O> using QRef = QWeight O::*;
template <class O> using FRef = float *O::*;
template <class Owner> struct TensorDef {
    const char *name;           // the model's name, or a layer's suffix under the layer prefix; nullptr: carved and drawn, never loaded by name
    Kind kind;
    QRef<Owner> q;
    FRef<Owner> f;
    Dim K, N = E;
    uint8_t at = 0;
    bool if_lm_head = false;    // present only when hparams.has_lm_head (GPT-2's model/lm_head)
};
template <class O> constexpr TensorDef<O> mat(const char *n, QRef<O> q, Dim K, Dim N) { return {n, MAT, q, nullptr, K, N}; }
template <class O> constexpr TensorDef<O> gain(const char *n, FRef<O> f, Dim K = E) { return {n, GAIN, nullptr, f, K}; }
template <class O> constexpr TensorDef<O> bias(const char *n, FRef<O> f, Dim K = E) { return {n, BIAS, nullptr, f, K}; }
template <class O> constexpr TensorDef<O> rows(const char *n, QRef<O> q, uint8_t at) { return {n, ROWS, q, nullptr, E, E, at}; }
template <class O> constexpr TensorDef<O> if_lm_head(TensorDef<O> d) { d.if_lm_head = true; return d; }

// The activations of a batched step (b200_neox_evaluate_ragged, b200_neox_evaluate_sessions): the rows of n sessions' chunks, grown on demand to
// the largest step seen, freed with the model.
struct NeoxBatch {
    BatchCore core;                     // the row table, the ids, the sampler jobs and the logits (host.h)
    DeviceBuf<float> x, cur, qkv, kq, attn, h4, hact, t;
    DeviceBuf<int8_t> xq; DeviceBuf<float2> xds; DeviceBuf<int4> xpack; DeviceBuf<__half> xh; DeviceBuf<char> xq8k;
};

}  // namespace

struct b200_neox_model : Weights {
    b200_neox_hparams hp;
    int hd = 0;
    QWeight wte, lm_head;
    float *lnf_g = nullptr, *lnf_b = nullptr, *wpe = nullptr;     // wpe: GPT-2 learned positions [n_ctx][e] f32
    float *emb_g = nullptr, *emb_b = nullptr;                     // BLOOM: LayerNorm of the embedding row
    DeviceBuf<float> alibi;                                       // MPT / BLOOM: ALiBi slopes [n_head] (alibi_slopes)
    float *lm_head_b = nullptr;                                   // GPT-J: lm_head.bias [n_vocab]
    const RopeTable *rope = nullptr;                              // GPT-NeoX: mode 2 on n_rot of every head; GPT-J: mode 0 over the whole head; else none
    QkvLayout qkv_layout;
    bool parallel = false;                                        // GPT-NeoX with use_parallel_residual: attention and MLP both read inpL
    float kq_scale = 0.0f;
    bool any_kquant = false;                                      // some matrix is a K-quant (the sessions hold a Q8_K activation buffer)
    bool uniform = true;                                          // every matrix is of hp.wtype, as one fused qkv per layer: the decode graph's layout
    NeoxBatch batch;
    bool neox() const { return hp.arch == 0; }
    bool mpt() const { return hp.arch == 2; }
    bool bloom() const { return hp.arch == 3; }
    bool gptj() const { return hp.arch == 4; }
    // MPT: every bias null; GPT-J: ln2_*, bqkv and bdense null (one LayerNorm per layer, no attention biases).  wv: GPT-J's v_proj of another
    // type than q_proj: then wqkv holds [q_proj | k_proj] and wv is its own matrix writing the same qkv rows (wv.N == 0 otherwise)
    struct Layer { QWeight wqkv, wdense, wfc, wproj; float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *bqkv, *bdense, *bfc, *bproj; QWeight wv; };
    std::vector<Layer> layers;
    template <class F> void each_tensor(F &&f);
    int64_t dim(Dim d) const;
    bool lookup(const char *name, Slot &s, int &id);
};

struct b200_neox_session : SessionCore {   // memory_k [n_layer][n_ctx][e], memory_v [n_layer][e][n_ctx]
    b200_neox_model *m = nullptr;
    DeviceBuf<float> x, cur, qkv, kq, attn, h4, hact, t, logits;
    DeviceBuf<float> qdec;
    DeviceBuf<int8_t> xq; DeviceBuf<float2> xds; DeviceBuf<int4> xpack; DeviceBuf<__half> xh;
    DeviceBuf<int4> xpack_a, xpack_d, xpack_f;
    DeviceBuf<char> xq8k;                                         // Q8_K activations of K-quant weights (models with one)
    std::vector<NeoxLayer> dl;
    NeoxParams dp;
};

namespace {

using Model = b200_neox_model;
using Layer = b200_neox_model::Layer;

// The tensors of each architecture in slab order: the slab is carved and b200_neox_synthesize draws in this order, so it fixes both the slab
// layout and the synthetic weights.  A tensor's slot (the loaded bitmap) is its place among the named entries.
struct ArchTensors {
    std::vector<TensorDef<Model>> globals;
    const char *layer_fmt;      // a per-layer name: the layer prefix, then the suffix
    std::vector<TensorDef<Layer>> layer;
};
const ArchTensors &arch_tensors(int arch) {      // by b200_neox_hparams.arch
    static const ArchTensors tab[] = {
        {   // GPT-NeoX: crates/models/gptneox/src/lib.rs:59-127
            {mat("gpt_neox.embed_in.weight", &Model::wte, E, VOCAB), mat("embed_out.weight", &Model::lm_head, E, VOCAB),
             gain("gpt_neox.final_layer_norm.weight", &Model::lnf_g), bias("gpt_neox.final_layer_norm.bias", &Model::lnf_b)},
            "gpt_neox.layers.%d.%95s",
            {gain("input_layernorm.weight", &Layer::ln1_g), bias("input_layernorm.bias", &Layer::ln1_b),
             gain("post_attention_layernorm.weight", &Layer::ln2_g), bias("post_attention_layernorm.bias", &Layer::ln2_b),
             bias("attention.query_key_value.bias", &Layer::bqkv, E3), bias("attention.dense.bias", &Layer::bdense),
             bias("mlp.dense_h_to_4h.bias", &Layer::bfc, E4), bias("mlp.dense_4h_to_h.bias", &Layer::bproj),
             mat("attention.query_key_value.weight", &Layer::wqkv, E, E3), mat("attention.dense.weight", &Layer::wdense, E, E),
             mat("mlp.dense_h_to_4h.weight", &Layer::wfc, E, E4), mat("mlp.dense_4h_to_h.weight", &Layer::wproj, E4, E)}},
        {   // GPT-2: crates/models/gpt2/src/lib.rs:59-107
            {mat("model/wte", &Model::wte, E, VOCAB), if_lm_head(mat("model/lm_head", &Model::lm_head, E, VOCAB)),
             gain("model/ln_f/g", &Model::lnf_g), bias("model/ln_f/b", &Model::lnf_b), bias("model/wpe", &Model::wpe, CTX_E)},
            "model/h%d/%95s",
            {gain("ln_1/g", &Layer::ln1_g), bias("ln_1/b", &Layer::ln1_b), gain("ln_2/g", &Layer::ln2_g), bias("ln_2/b", &Layer::ln2_b),
             bias("attn/c_attn/b", &Layer::bqkv, E3), bias("attn/c_proj/b", &Layer::bdense), bias("mlp/c_fc/b", &Layer::bfc, E4), bias("mlp/c_proj/b", &Layer::bproj),
             mat("attn/c_attn/w", &Layer::wqkv, E, E3), mat("attn/c_proj/w", &Layer::wdense, E, E),
             mat("mlp/c_fc/w", &Layer::wfc, E, E4), mat("mlp/c_proj/w", &Layer::wproj, E4, E)}},
        {   // MPT: crates/models/mpt/src/lib.rs:49-65, no biases
            {mat("transformer.wte.weight", &Model::wte, E, VOCAB), gain("transformer.norm_f.weight", &Model::lnf_g)},
            "transformer.blocks.%d.%95s",
            {gain("norm_1.weight", &Layer::ln1_g), gain("norm_2.weight", &Layer::ln2_g),
             mat("attn.Wqkv.weight", &Layer::wqkv, E, E3), mat("attn.out_proj.weight", &Layer::wdense, E, E),
             mat("ffn.up_proj.weight", &Layer::wfc, E, E4), mat("ffn.down_proj.weight", &Layer::wproj, E4, E)}},
        {   // BLOOM: crates/models/bloom/src/lib.rs:56-83
            {mat("tok_embeddings.weight", &Model::wte, E, VOCAB), mat("output.weight", &Model::lm_head, E, VOCAB),
             gain("output_norm.weight", &Model::lnf_g), bias("output_norm.bias", &Model::lnf_b), gain("norm.weight", &Model::emb_g), bias("norm.bias", &Model::emb_b)},
            "layers.%d.%95s",
            {gain("attention_norm.weight", &Layer::ln1_g), bias("attention_norm.bias", &Layer::ln1_b),
             gain("ffn_norm.weight", &Layer::ln2_g), bias("ffn_norm.bias", &Layer::ln2_b),
             bias("attention.query_key_value.bias", &Layer::bqkv, E3), bias("attention.wo.bias", &Layer::bdense),
             bias("feed_forward.w1.bias", &Layer::bfc, E4), bias("feed_forward.w2.bias", &Layer::bproj),
             mat("attention.query_key_value.weight", &Layer::wqkv, E, E3), mat("attention.wo.weight", &Layer::wdense, E, E),
             mat("feed_forward.w1.weight", &Layer::wfc, E, E4), mat("feed_forward.w2.weight", &Layer::wproj, E4, E)}},
        {   // GPT-J: crates/models/gptj/src/lib.rs:59-103, no attention biases, one LayerNorm per layer; q_proj / k_proj / v_proj are the thirds of wqkv
            {mat("transformer.wte.weight", &Model::wte, E, VOCAB), mat("lm_head.weight", &Model::lm_head, E, VOCAB),
             gain("transformer.ln_f.weight", &Model::lnf_g), bias("transformer.ln_f.bias", &Model::lnf_b), bias("lm_head.bias", &Model::lm_head_b, VOCAB)},
            "transformer.h.%d.%95s",
            {gain("ln_1.weight", &Layer::ln1_g), bias("ln_1.bias", &Layer::ln1_b), bias("mlp.fc_in.bias", &Layer::bfc, E4), bias("mlp.fc_out.bias", &Layer::bproj),
             mat(nullptr, &Layer::wqkv, E, E3), rows("attn.q_proj.weight", &Layer::wqkv, 0), rows("attn.k_proj.weight", &Layer::wqkv, 1),
             rows("attn.v_proj.weight", &Layer::wqkv, 2), mat("attn.out_proj.weight", &Layer::wdense, E, E),
             mat("mlp.fc_in.weight", &Layer::wfc, E, E4), mat("mlp.fc_out.weight", &Layer::wproj, E4, E)}},
    };
    return tab[arch];
}

}  // namespace

// f(def, owner, il) for every tensor of the model in slab order: the model's own (il = -1, owner = the model), then layer by layer
template <class F> void b200_neox_model::each_tensor(F &&f) {
    const ArchTensors &a = arch_tensors(hp.arch);
    for (const TensorDef<Model> &d : a.globals)
        if (!d.if_lm_head || hp.has_lm_head) f(d, *this, -1);
    for (int il = 0; il < hp.n_layer; il++)
        for (const TensorDef<Layer> &d : a.layer) f(d, layers[il], il);
}

int64_t b200_neox_model::dim(Dim d) const {
    const int64_t e = hp.n_embd;
    switch (d) {
        case E3: return 3 * e;
        case E4: return 4 * e;
        case VOCAB: return hp.n_vocab;
        case CTX_E: return hp.context_size * e;
        default: return e;
    }
}

bool b200_neox_model::lookup(const char *name, Slot &s, int &id) {
    int il = -1; char sub[96];
    if (sscanf(name, arch_tensors(hp.arch).layer_fmt, &il, sub) != 2) il = -1;
    int slot = 0;
    bool found = false;
    each_tensor([&](const auto &d, auto &o, int l) {
        if (found || !d.name) return;
        if (l < 0 ? !strcmp(name, d.name) : l == il && !strcmp(sub, d.name)) {
            s = Slot();
            if (d.kind == MAT) { s.q = o.*d.q; s.is_q = true; }
            else if (d.kind == ROWS) {     // rows past the fused matrix's own: GPT-J's v_proj of its own type
                const QWeight &q = o.*d.q;
                s.q = (d.at + 1) * (int64_t)hp.n_embd > q.N ? layers[l].wv : row_view(q, d.at * (int64_t)hp.n_embd, hp.n_embd);
                s.is_q = true;
            }
            else { s.f = o.*d.f; s.n = dim(d.K); }
            id = slot;
            found = true;
        }
        slot++;
    });
    if (found && wpe && s.f == wpe) s.f16_src = true;      // gpt2 lib.rs:59 loads wpe in the file's type; get_rows of F16 rows is exact in f32
    return found;
}

namespace {

void forward(b200_neox_session *s, int n, bool all_rows) {
    b200_neox_model *m = s->m;
    const b200_neox_hparams &hp = m->hp;
    cudaStream_t st = rt().stream;
    const int e = hp.n_embd, hd = m->hd, n_head = hp.n_head, n_ctx = hp.context_size, n_past = s->n_past, n_kv = n_past + n;
    int L = 0;
    // the graph schedule's attention keeps the whole bucket in shared memory: steps in buckets past 3264 positions run per op below, and the
    // graph cache re-uploads the device n_past when graph steps resume (after a rewind)
    // F16 weights decode per op (exact_f16.cu's mat-vec): the graph schedule is built on Q8 activation records.  So do models with a K-quant
    // matrix or with matrices of more than one type: the graph takes one classic type throughout.
    if (n == 1 && hp.wtype != T_F16 && m->uniform && !m->any_kquant && neox_decode_fits(s->dp, DecodeGraphCache::bucket(n_kv, n_ctx))) {   // f32 cache: up to 1664 positions
        s->last_launches = s->decode.run(n_kv, n_ctx, true, [s, &hp](int bucket, cudaStream_t st, int *nodes) {
            neox_decode_enqueue(s->dp, s->dl, hp.wtype, bucket, st, nodes);
        }, st);
        s->n_past += 1;
        s->last_n = 1;
        return;
    }
    const ExactActs acts{s->xq.get(), s->xds.get(), s->xpack.get(), s->xh.get(), s->xq8k.get()};
    const bool kv32 = s->kv_type == T_F32;
    const int64_t ke = (int64_t)s->kv_elem_bytes();
    const bool gptj = m->gptj(), parallel = m->parallel;
    const RopeTable *rope = m->rope;
    const int64_t ld3 = 3 * (int64_t)e;
    const int64_t hs = m->qkv_layout.head_stride, koff = m->qkv_layout.k_off, voff = m->qkv_layout.v_off;
    if (m->emb_g) {                                                                                                               // bloom lib.rs:139-144
        get_rows_q(m->wte, s->d_tokens.get(), s->t.get(), n, st); L++;
        layer_norm(s->t.get(), s->x.get(), m->emb_g, m->emb_b, e, n, st); L++;
    } else {
        get_rows_q(m->wte, s->d_tokens.get(), s->x.get(), n, st); L++;                                                           // :178
    }
    if (m->wpe) { add_f32(s->x.get(), m->wpe + (size_t)n_past * e, s->x.get(), (int64_t)n * e, (int64_t)n * e, st); L++; }               // gpt2 lib.rs:164-172: + wpe[n_past + i]
    for (int il = 0; il < hp.n_layer; il++) {
        const b200_neox_model::Layer &ly = m->layers[il];
        void *Kl = s->kv_at(0, (size_t)il * n_ctx * e), *Vl = s->kv_at(1, (size_t)il * n_ctx * e);
        layer_norm(s->x.get(), s->cur.get(), ly.ln1_g, ly.ln1_b, e, n, st); L++;                                                  // :192-196
        L += mul_mat_exact_auto(ly.wqkv, s->cur.get(), e, n, s->qkv.get(), ld3, nullptr, 0, acts, st);                                // :199
        if (ly.wv.N) L += mul_mat_exact_auto(ly.wv, s->cur.get(), e, n, s->qkv.get() + voff, ld3, nullptr, 0, acts, st);               // GPT-J v_proj of its own type
        if (ly.bqkv) { add_f32(s->qkv.get(), ly.bqkv, s->qkv.get(), (int64_t)n * ld3, ld3, st); L++; }                            // :200 (MPT: no bias)
        if (rope) {   // RoPE in place on q and k: mode 2 (GPT-NeoX :205-228), mode 0 (GPT-J :178-201)
            rope_f32(s->qkv.get(), s->qkv.get(), hd, n_head, n, hs, ld3, hs, ld3, n_past, *rope, st); L++;
            rope_f32(s->qkv.get() + koff, s->qkv.get() + koff, hd, n_head, n, hs, ld3, hs, ld3, n_past, *rope, st); L++;
        }
        {   // k -> cache rows n_past.., v -> cache columns (transposed; GPT-2's v_trans copy of every evaluate is this layout)       :231-247
            StridedDesc sk{{hd, n_head, n, 1}, {4, hs * 4, ld3 * 4, 0}}, dk{{hd, n_head, n, 1}, {ke, (int64_t)hd * ke, (int64_t)e * ke, 0}};
            cpy_strided(s->qkv.get() + koff, T_F32, sk, (char *)Kl + (size_t)n_past * e * ke, s->kv_type, dk, st); L++;
            StridedDesc dv{{hd, n_head, n, 1}, {(int64_t)n_ctx * ke, (int64_t)hd * n_ctx * ke, ke, 0}};
            cpy_strided(s->qkv.get() + voff, T_F32, sk, (char *)Vl + (size_t)n_past * ke, s->kv_type, dv, st); L++;
        }
        if (kv32) mul_mat_f32_exact((const float *)Kl, hd, n_kv, n_head, (int64_t)e * 4, (int64_t)hd * 4, s->qkv.get(), n, n_head, ld3 * 4, hs * 4,
                                    s->kq.get(), (int64_t)n_kv * 4, (int64_t)n_kv * n * 4, n_past, st);
        else mul_mat_f16_exact((const __half *)Kl, hd, n_kv, n_head, (int64_t)e * 2, (int64_t)hd * 2, s->qkv.get(), n, n_head, ld3 * 4, hs * 4,
                               s->kq.get(), (int64_t)n_kv * 4, (int64_t)n_kv * n * 4, n_past, st);
        L++;                                                                                                                      // :250-267
        if (m->alibi) soft_max_alibi(s->kq.get(), s->kq.get(), n_kv, (int64_t)n_head * n, n, m->kq_scale, n_past, m->alibi.get(), st);   // MPT / BLOOM: + ALiBi
        else soft_max(s->kq.get(), s->kq.get(), n_kv, (int64_t)n_head * n, n, m->kq_scale, true, n_past, true, true, st);                // :270-279
        L++;
        // GPT-J: cur (ln_1's output, input_sa) still feeds fc_in, so the merged KQV goes to t
        float *kqv = gptj ? s->t.get() : s->cur.get();
        if (kv32) mul_mat_f32_exact((const float *)Vl, n_kv, hd, n_head, (int64_t)n_ctx * 4, (int64_t)n_ctx * hd * 4, s->kq.get(), n, n_head, (int64_t)n_kv * 4,
                                    (int64_t)n_kv * n * 4, kqv, (int64_t)e * 4, (int64_t)hd * 4, -1, st);
        else mul_mat_f16_exact((const __half *)Vl, n_kv, hd, n_head, (int64_t)n_ctx * 2, (int64_t)n_ctx * hd * 2, s->kq.get(), n, n_head, (int64_t)n_kv * 4,
                               (int64_t)n_kv * n * 4, kqv, (int64_t)e * 4, (int64_t)hd * 4, -1, st);
        L++;                                                                                                                      // :282-298
        L += mul_mat_exact_auto(ly.wdense, kqv, e, n, s->attn.get(), e, nullptr, 0, acts, st);                                        // :301
        if (gptj) {   // gptj lib.rs:265-282: t = (fc_out gelu(fc_in input_sa + b_in) + b_out) + attn; inpL = t + inpL
            L += mul_mat_exact_auto(ly.wfc, s->cur.get(), e, n, s->h4.get(), 4 * (int64_t)e, nullptr, 0, acts, st);
            add_f32(s->h4.get(), ly.bfc, s->h4.get(), (int64_t)n * 4 * e, 4 * (int64_t)e, st); L++;
            unary_lut(UNARY_GELU, s->h4.get(), s->hact.get(), (int64_t)n * 4 * e, st); L++;
            L += mul_mat_exact_auto(ly.wproj, s->hact.get(), 4 * (int64_t)e, n, s->t.get(), e, nullptr, 0, acts, st);
            add_f32(s->t.get(), ly.bproj, s->t.get(), (int64_t)n * e, e, st); L++;
            add_f32(s->t.get(), s->attn.get(), s->t.get(), (int64_t)n * e, (int64_t)n * e, st); L++;
            add_f32(s->t.get(), s->x.get(), s->x.get(), (int64_t)n * e, (int64_t)n * e, st); L++;
            continue;
        }
        if (ly.bdense) { add_f32(s->attn.get(), ly.bdense, s->attn.get(), (int64_t)n * e, e, st); L++; }                          // :302
        const float *ff_in = s->x.get();
        if (!parallel) { add_f32(s->attn.get(), s->x.get(), s->attn.get(), (int64_t)n * e, (int64_t)n * e, st); L++; ff_in = s->attn.get(); }   // :308-309 / gpt2 :279
        layer_norm(ff_in, s->cur.get(), ly.ln2_g, ly.ln2_b, e, n, st); L++;                                                 // feed_forward :487-493
        L += mul_mat_exact_auto(ly.wfc, s->cur.get(), e, n, s->h4.get(), 4 * (int64_t)e, nullptr, 0, acts, st);
        if (ly.bfc) { add_f32(s->h4.get(), ly.bfc, s->h4.get(), (int64_t)n * 4 * e, 4 * (int64_t)e, st); L++; }
        unary_lut(UNARY_GELU, s->h4.get(), s->hact.get(), (int64_t)n * 4 * e, st); L++;
        L += mul_mat_exact_auto(ly.wproj, s->hact.get(), 4 * (int64_t)e, n, s->t.get(), e, nullptr, 0, acts, st);
        if (ly.bproj) { add_f32(s->t.get(), ly.bproj, s->t.get(), (int64_t)n * e, e, st); L++; }
        add_f32(s->t.get(), s->attn.get(), s->t.get(), (int64_t)n * e, (int64_t)n * e, st); L++;                                        // parallel: ffn + attn; sequential: ffn + ff_in
        if (parallel) { add_f32(s->t.get(), s->x.get(), s->x.get(), (int64_t)n * e, (int64_t)n * e, st); L++; }        // :324
        else { B200_CHECK(cudaMemcpyAsync(s->x.get(), s->t.get(), (size_t)n * e * 4, cudaMemcpyDeviceToDevice, st)); }
    }
    if (all_rows || n == 1) {
        layer_norm(s->x.get(), s->cur.get(), m->lnf_g, m->lnf_b, e, n, st); L++;                                                   // :332-334
        L += mul_mat_exact_auto(m->lm_head, s->cur.get(), e, n, s->logits.get(), hp.n_vocab, nullptr, 0, acts, st);                   // :342
        if (m->lm_head_b) { add_f32(s->logits.get(), m->lm_head_b, s->logits.get(), (int64_t)n * hp.n_vocab, hp.n_vocab, st); L++; }  // gptj lib.rs:296
    } else {
        const size_t last = (size_t)(n - 1);
        float *row = s->logits.get() + last * hp.n_vocab;
        layer_norm(s->x.get() + last * e, s->cur.get() + last * e, m->lnf_g, m->lnf_b, e, 1, st); L++;
        L += mul_mat_exact_auto(m->lm_head, s->cur.get() + last * e, e, 1, row, hp.n_vocab, nullptr, 0, acts, st);
        if (m->lm_head_b) { add_f32(row, m->lm_head_b, row, hp.n_vocab, hp.n_vocab, st); L++; }
    }
    s->last_launches = L;
    s->last_n = n;
    s->n_past += n;
}

// ---- batched steps: one step for n sessions of one model, a chunk each (b200_neox_evaluate_ragged; decode: chunks of one token) ---------------
// forward() over the rows of n sessions' chunks: the weight mat-muls and the row-wise nodes over all rows; the learned positions, RoPE, the cache
// stores and the attention per row on its own session's cache, position and chunk (the step's tables).  Each row's arithmetic is forward()'s on its
// chunk alone, including the final LayerNorm and the lm_head on each chunk's last row only (p.out) unless every row's logits are asked for.
// Returns the launches: the same for every step of one-token chunks.
int forward_rows(b200_neox_model *m, const BatchStep &p, cudaStream_t st) {
    const b200_neox_hparams &hp = m->hp;
    NeoxBatch &w = m->batch;
    const int n = p.n, e = hp.n_embd, hd = m->hd, n_head = hp.n_head, n_ctx = hp.context_size, V = hp.n_vocab;
    const int64_t ld3 = 3 * (int64_t)e, e4 = 4 * (int64_t)e, ne = (int64_t)n * e;
    const QkvLayout lay = m->qkv_layout;
    const BatchRow *rows = p.rows;
    const int kv_type = p.kv_type;
    const ExactActs acts{w.xq.get(), w.xds.get(), w.xpack.get(), w.xh.get(), w.xq8k.get()};
    auto mm = [&](const QWeight &W, const float *x, float *dst, int64_t ldd, int64_t B) { return mul_mat_exact_auto(W, x, W.K, B, dst, ldd, nullptr, 0, acts, st); };
    float *x = w.x.get(), *cur = w.cur.get(), *qkv = w.qkv.get(), *kq = w.kq.get(), *attn = w.attn.get(), *h4 = w.h4.get(), *hact = w.hact.get(),
          *t = w.t.get(), *logits = p.logits;
    int L = 0;
    if (m->emb_g) {
        get_rows_q(m->wte, p.ids, t, n, st); L++;
        layer_norm(t, x, m->emb_g, m->emb_b, e, n, st); L++;
    } else {
        get_rows_q(m->wte, p.ids, x, n, st); L++;
    }
    if (m->wpe) { add_pos_rows(x, m->wpe, rows, n, e, st); L++; }
    for (int il = 0; il < hp.n_layer; il++) {
        const b200_neox_model::Layer &ly = m->layers[il];
        const size_t layer_off = (size_t)il * n_ctx * e;
        layer_norm(x, cur, ly.ln1_g, ly.ln1_b, e, n, st); L++;
        L += mm(ly.wqkv, cur, qkv, ld3, n);
        if (ly.wv.N) L += mm(ly.wv, cur, qkv + lay.v_off, ld3, n);
        if (ly.bqkv) { add_f32(qkv, ly.bqkv, qkv, n * ld3, ld3, st); L++; }
        rope_store_rows(qkv, ld3, lay, hd, n_head, n_head, rows, n, layer_off, n_ctx, kv_type, m->rope, st); L++;
        L += attn_kq_step(p, layer_off, qkv, ld3, lay.head_stride, hd, n_head, n_head, n_ctx, kq, st);
        if (m->alibi) soft_max_alibi_rows(kq, rows, n, n_head, n_ctx, m->kq_scale, m->alibi.get(), st);
        else soft_max_rows(kq, rows, n, n_head, n_ctx, m->kq_scale, st);
        L++;
        float *kqv = m->gptj() ? t : cur;                     // GPT-J: cur still feeds fc_in
        L += attn_kqv_step(p, layer_off, kq, hd, n_head, n_head, n_ctx, kqv, e, st);
        L += mm(ly.wdense, kqv, attn, e, n);
        if (m->gptj()) {
            L += mm(ly.wfc, cur, h4, e4, n);
            add_f32(h4, ly.bfc, h4, n * e4, e4, st); L++;
            unary_lut(UNARY_GELU, h4, hact, n * e4, st); L++;
            L += mm(ly.wproj, hact, t, e, n);
            add_f32(t, ly.bproj, t, ne, e, st); L++;
            add_f32(t, attn, t, ne, ne, st); L++;
            add_f32(t, x, x, ne, ne, st); L++;
            continue;
        }
        if (ly.bdense) { add_f32(attn, ly.bdense, attn, ne, e, st); L++; }
        const float *ff_in = x;
        if (!m->parallel) { add_f32(attn, x, attn, ne, ne, st); L++; ff_in = attn; }
        layer_norm(ff_in, cur, ly.ln2_g, ly.ln2_b, e, n, st); L++;
        L += mm(ly.wfc, cur, h4, e4, n);
        if (ly.bfc) { add_f32(h4, ly.bfc, h4, n * e4, e4, st); L++; }
        unary_lut(UNARY_GELU, h4, hact, n * e4, st); L++;
        L += mm(ly.wproj, hact, t, e, n);
        if (ly.bproj) { add_f32(t, ly.bproj, t, ne, e, st); L++; }
        add_f32(t, attn, t, ne, ne, st); L++;
        if (m->parallel) { add_f32(t, x, x, ne, ne, st); L++; }
        else { B200_CHECK(cudaMemcpyAsync(x, t, (size_t)ne * 4, cudaMemcpyDeviceToDevice, st)); }
    }
    const float *xl = x;
    if (p.out) { gather_rows(x, e, p.out, p.n_out, attn, st); L++; xl = attn; }         // each chunk's last row (attn is free here)
    layer_norm(xl, cur, m->lnf_g, m->lnf_b, e, p.n_out, st); L++;
    L += mm(m->lm_head, cur, logits, V, p.n_out);
    if (m->lm_head_b) { add_f32(logits, m->lm_head_b, logits, (int64_t)p.n_out * V, V, st); L++; }
    return L;
}

// the batched step's activations for B rows (BatchCore::reserve, with the stream idle): b200_neox_start_session's buffers; kq is [B][n_head][n_ctx]
void batch_reserve(b200_neox_model *m, size_t B) {
    NeoxBatch &w = m->batch;
    const b200_neox_hparams &hp = m->hp;
    const size_t e = hp.n_embd, n_ctx = hp.context_size;
    w.x = device_alloc<float>(B * e * 4); w.cur = device_alloc<float>(B * e * 4); w.qkv = device_alloc<float>(B * 3 * e * 4);
    w.kq = device_alloc<float>((size_t)hp.n_head * B * n_ctx * 4); w.attn = device_alloc<float>(B * e * 4);
    w.h4 = device_alloc<float>(B * 4 * e * 4); w.hact = device_alloc<float>(B * 4 * e * 4); w.t = device_alloc<float>(B * e * 4);
    w.xq = device_alloc<int8_t>(B * 4 * e); w.xds = device_alloc<float2>(B * (4 * e / QK) * sizeof(float2));
    w.xpack = device_alloc<int4>((4 * e / QK) * 64); w.xh = device_alloc<__half>(xh_bytes(4 * e, B));
    if (m->any_kquant) w.xq8k = device_alloc<char>(q8k_bytes(4 * e, B));          // the widest K: fc_out's 4 n_embd
}

BatchFront batch_front(b200_neox_model *m) {
    return BatchFront{[m](size_t B) { batch_reserve(m, B); }, [m](const BatchStep &p) { return forward_rows(m, p, rt().stream); },
                      attn_tiles_aligned(m->hd, 3 * (int64_t)m->hp.n_embd, m->qkv_layout.head_stride, m->hp.context_size)};
}

// a tensor's whole name: the model's own, or the layer prefix of layer il (layer_fmt up to its "%95s") followed by the suffix
std::string full_name(const ArchTensors &a, const char *name, int il) {
    if (il < 0) return name;
    const std::string pre(a.layer_fmt, strstr(a.layer_fmt, "%95s") - a.layer_fmt);
    char buf[64];
    snprintf(buf, sizeof(buf), pre.c_str(), il);
    return std::string(buf) + name;
}

// hp->arch 0 .. 4; alibi_bias_max: MPT's header float, 8 for BLOOM (ignored by the others); rope_freq_base / scale <= 0: 10000 / 1.
// GPT-NeoX and GPT-J rotate: n_rot even, positive and at most the head size (the asserts of ggml_rope, LC/ggml.c:11807-11808).
// Every matrix is of hp->wtype unless types[0, n_types) names it (the model file's per-tensor types); every refusal comes before any allocation.
b200_neox_model *neox_new(const b200_neox_hparams *hp, float alibi_bias_max, float rope_freq_base, float rope_freq_scale, const b200_tensor_type *types,
                          int32_t n_types, int *err) {
    int dummy; if (!err) err = &dummy;
    *err = B200_ERR_BAD_ARG;
    if (!hp || hp->arch < 0 || hp->arch > 4 || hp->n_embd % 64 || hp->n_head <= 0 || hp->n_embd % hp->n_head || hp->n_layer <= 0 || hp->context_size <= 0 ||
        ((hp->arch == 0 || hp->arch == 4) && (hp->n_rot <= 0 || hp->n_rot % 2 || hp->n_rot > hp->n_embd / hp->n_head)) || n_types < 0 || (n_types && !types)) return nullptr;
    for (int32_t i = 0; i < n_types; i++) if (!types[i].name) return nullptr;
    b200_neox_model *m = new b200_neox_model();
    m->hp = *hp;
    const int e = hp->n_embd, hd = e / hp->n_head;
    m->hd = hd;
    m->layers.resize(hp->n_layer);
    // the type of every matrix in slab order (mt), and each layer's separate v_proj type (vt, -1: v_proj is the last third of the fused qkv)
    const ArchTensors &arch = arch_tensors(hp->arch);
    std::vector<uint8_t> used((size_t)n_types, 0);
    auto type_of = [&](const std::string &name) {
        int t = hp->wtype;
        for (int32_t i = 0; i < n_types; i++) if (!strcmp(types[i].name, name.c_str())) { t = types[i].type; used[(size_t)i] = 1; }
        return t;
    };
    std::vector<int> mt, vt((size_t)hp->n_layer, -1);
    bool f16 = false, other = false;
    int rc = B200_OK;
    size_t fused = 0;                                   // mt's entry of the layer's nameless fused matrix (GPT-J's wqkv)
    m->each_tensor([&](const auto &d, auto &, int il) {
        if (rc != B200_OK || (d.kind != MAT && d.kind != ROWS)) return;
        if (!d.name) { fused = mt.size(); mt.push_back(-1); return; }      // typed by its rows
        const std::string name = full_name(arch, d.name, il);
        const int t = type_of(name);
        if (!is_qweight_type(t) && !is_kquant(t)) {
            fprintf(stderr, "llm_b200: %s is element type %d; 2-D weights are F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 or Q2_K..Q6_K\n", name.c_str(), t);
            rc = B200_ERR_UNSUPPORTED_ELEMENT_TYPE; return;
        }
        const int64_t ne0 = d.kind == ROWS ? e : m->dim(d.K);
        if (is_kquant(t) && ne0 % 256) {
            fprintf(stderr, "llm_b200: %s: a K-quant row of %lld elements is not whole super-blocks of 256\n", name.c_str(), (long long)ne0);
            rc = B200_ERR_INVARIANT_BROKEN; return;
        }
        (t == T_F16 ? f16 : other) = true;
        if (d.kind == MAT) { mt.push_back(t); return; }
        if (d.at == 0) mt[fused] = t;                   // q_proj types the fused matrix
        else if (d.at == 1 && t != mt[fused]) {         // [q_proj | k_proj] is one matrix: no quantizer the reference ships writes them in two types
            fprintf(stderr, "llm_b200: %s is of another element type than the layer's q_proj\n", name.c_str());
            rc = B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
        } else if (d.at == 2 && t != mt[fused]) vt[(size_t)il] = t;
    });
    for (int32_t i = 0; i < n_types && rc == B200_OK; i++)
        if (!used[(size_t)i]) { fprintf(stderr, "llm_b200: %s is not a matrix of this model\n", types[i].name); rc = B200_ERR_UNKNOWN_TENSOR; }
    // F16 weights come as whole F16 files: an F16 matrix beside block-format ones is refused (as for LLaMA)
    if (rc == B200_OK && f16 && other) { fprintf(stderr, "llm_b200: F16 weights beside weights of other element types: F16 models are F16 throughout\n"); rc = B200_ERR_UNSUPPORTED_ELEMENT_TYPE; }
    if (rc != B200_OK) { *err = rc; delete m; return nullptr; }
    for (int t : mt) { m->uniform &= t == hp->wtype; m->any_kquant |= is_kquant(t); }
    for (int t : vt) { m->uniform &= t < 0; m->any_kquant |= is_kquant(t); }
    rt().ensure_init();
    int n_slots = 0;
    m->each_tensor([&n_slots](const auto &d, auto &, int) { n_slots += d.name != nullptr; });
    // with one type for every matrix this is the layout of a one-type model: same matrices, same order, same bytes
    m->carve(hp->wtype, n_slots, [m, &mt, &vt, e](SlabCarver &c) {
        size_t k = 0;
        m->each_tensor([&](const auto &d, auto &o, int il) {
            if (d.kind == MAT) {
                const bool split = !d.name && vt[(size_t)il] >= 0;
                c.q(o.*d.q, m->dim(d.K), split ? 2 * (int64_t)e : m->dim(d.N), mt[k++]);
                if (split) c.q(m->layers[il].wv, e, e, vt[(size_t)il]);
            }
            else if (d.kind != ROWS) c.f(o.*d.f, m->dim(d.K));
        });
    });
    // no output matrix (GPT-2 without model/lm_head, gpt2 lib.rs:319-320; MPT): the output projection is tied to wte, which is streamed as the lm_head
    // in wte's type
    if (!m->lm_head.qs) m->lm_head = m->wte;
    else m->weight_bytes -= (size_t)hp->n_vocab * m->wte.nb * qweight_block_bytes(m->wte.type);  // the embedding table is gathered from, not streamed
    if (m->mpt() || m->bloom()) {
        const std::vector<float> slopes = alibi_slopes(hp->n_head, alibi_bias_max);
        m->alibi = device_alloc<float>(slopes.size() * 4);
        B200_CHECK(cudaMemcpy(m->alibi.get(), slopes.data(), slopes.size() * 4, cudaMemcpyHostToDevice));
    }
    // GPT-NeoX: mode 2 on n_rot of every head; GPT-J: mode 0 over ALL hd elements of the head with theta_scale base^(-2/n_rot) (gptj lib.rs:178-201,
    // LC/ggml.c:11859-11874 walks ne0, not n_dims).  ModelParameters::rope_overrides: ggml_rope_custom_inplace's base and scale (context.rs:558-590)
    if (m->neox() || m->gptj())
        m->rope = &rope_table(hp->n_rot, m->neox() ? 2 : 0, rope_freq_base > 0.f ? rope_freq_base : 10000.0f, rope_freq_scale > 0.f ? rope_freq_scale : 1.0f,
                              hd, hp->context_size);
    // where q / k / v of head h live inside a row of the fused projection: GPT-NeoX per head [q | k | v], the others the three thirds of the row
    m->qkv_layout = m->neox() ? QkvLayout{3 * hd, hd, 2 * hd} : QkvLayout{hd, e, 2 * e};
    m->parallel = m->neox() && hp->use_parallel_residual;
    m->kq_scale = 1.0f / sqrtf((float)e / (float)hp->n_head);                                                                   // gptneox lib.rs:270-273
    *err = B200_OK;
    return m;
}

}  // namespace

// a 2-D weight a model of architecture `arch` (b200_neox_hparams.arch) and n_layer layers holds: a MAT or ROWS entry of its tensor table
bool b200::neox_matrix_name(int arch, const char *name, int n_layer) {
    if (arch < 0 || arch > 4) return false;
    const ArchTensors &a = arch_tensors(arch);
    auto matrix = [](const auto &d, const char *n) { return d.name && (d.kind == MAT || d.kind == ROWS) && !strcmp(n, d.name); };
    for (const TensorDef<Model> &d : a.globals) if (matrix(d, name)) return true;
    int il = -1, used = 0; char sub[96];
    if (sscanf(name, (std::string(a.layer_fmt) + "%n").c_str(), &il, sub, &used) != 2 || il < 0 || il >= n_layer || name[used]) return false;
    for (const TensorDef<Layer> &d : a.layer) if (matrix(d, sub)) return true;
    return false;
}

// ggml_compute_forward_alibi_f32 (LC/ggml.c:11570-11588), the slope of head k.  libm powf on the host, as the reference's CPU build calls it:
// the same glibc gives the same bits, which CUDA's powf does not promise.
std::vector<float> b200::alibi_slopes(int n_head, float max_bias) {
    const int n_heads_log2_floor = 1 << (int)floor(log2(n_head));
    const float m0 = ::powf(2.0f, -(max_bias) / n_heads_log2_floor);
    const float m1 = ::powf(2.0f, -(max_bias / 2.0f) / n_heads_log2_floor);
    std::vector<float> m(n_head);
    for (int k = 0; k < n_head; k++) m[k] = k < n_heads_log2_floor ? ::powf(m0, k + 1) : ::powf(m1, 2 * (k - n_heads_log2_floor) + 1);
    return m;
}

extern "C" {

// the untyped forms: one classic or F16 type for every matrix, the default RoPE
b200_neox_model *b200_neox_new(const b200_neox_hparams *hp) {
    return hp && (hp->arch == 0 || hp->arch == 1 || hp->arch == 4) && is_qweight_type(hp->wtype) ? neox_new(hp, 0.0f, 0.0f, 0.0f, nullptr, 0, nullptr) : nullptr;
}

b200_neox_model *b200_neox_new_alibi(const b200_neox_hparams *hp, float alibi_bias_max) {   // MPT, BLOOM
    return hp && (hp->arch == 2 || hp->arch == 3) && is_qweight_type(hp->wtype) ? neox_new(hp, alibi_bias_max, 0.0f, 0.0f, nullptr, 0, nullptr) : nullptr;
}

b200_neox_model *b200_neox_new_typed(const b200_neox_hparams *hp, float alibi_bias_max, float rope_freq_base, float rope_freq_scale,
                                     const b200_tensor_type *types, int32_t n, int *err) {
    return neox_new(hp, alibi_bias_max, rope_freq_base, rope_freq_scale, types, n, err);
}

int b200_neox_is_loaded(b200_neox_model *m) { return m && m->all_loaded(); }

size_t b200_neox_weight_bytes(b200_neox_model *m) { return m ? m->weight_bytes : 0; }

int b200_neox_load_tensor(b200_neox_model *m, const char *name, int32_t type, const void *host_data, size_t nbytes) {
    if (!m || !name || !host_data) return B200_ERR_BAD_ARG;
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    const int rc = load_slot(s, type, host_data, nbytes);
    if (rc == B200_OK) m->mark(id);
    return rc;
}

// the loader's dims check (2-D: ne0 = row length, ne1 = rows; an f32 matrix such as GPT-2's wpe is one slot of ne0 * ne1 floats) and the adapters
int b200_neox_load_tensor_lora(b200_neox_model *m, const char *name, int32_t type, int32_t n_dims, int64_t ne0, int64_t ne1, const void *host_data, size_t nbytes,
                               const b200_ggml_file *const *adapters, int32_t n_adapters) {
    if (!m || !name || !host_data || n_adapters < 0 || (n_adapters > 0 && !adapters)) return B200_ERR_BAD_ARG;
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    if (n_dims == 1) ne1 = 1;
    if (n_dims < 1 || n_dims > 2 || (s.is_q ? n_dims != 2 || ne0 != s.q.K || ne1 != s.q_rows() : ne0 * ne1 != s.n)) return B200_ERR_TENSOR_SHAPE;
    const LoraTarget t{name, ne0, ne1, adapters, n_adapters};
    const int rc = load_slot(s, type, host_data, nbytes, n_adapters ? &t : nullptr);
    if (rc == B200_OK) m->mark(id);
    return rc;
}

// seeded synthetic weights generated in HBM (bench): LayerNorm gains 1 + 0.1 N(0,1), biases = gains - 1 (small)
int b200_neox_synthesize(b200_neox_model *m, uint64_t seed) {
    if (!m) return B200_ERR_BAD_ARG;
    m->synthesize(seed, [m](SeedSeq &r) {
        m->each_tensor([&](const auto &d, auto &o, int il) {
            if (d.kind == MAT) { r.q(o.*d.q); if (!d.name && m->layers[il].wv.N) r.q(m->layers[il].wv); }
            else if (d.kind == GAIN) r.gain(o.*d.f, m->dim(d.K));
            else if (d.kind == BIAS) r.bias(o.*d.f, m->dim(d.K));
        });
    });
    return B200_OK;
}

void b200_neox_free(b200_neox_model *m) {
    if (!m) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    delete m;                                           // the slab goes with it
}

b200_neox_session *b200_neox_start_session(b200_neox_model *m, int32_t n_batch) { return b200_neox_start_session_flags(m, n_batch, 0); }

b200_neox_session *b200_neox_start_session_flags(b200_neox_model *m, int32_t n_batch, int32_t flags) {
    if (!m || n_batch < 1 || (flags & ~B200_SESSION_KV_F32)) return nullptr;
    if (!m->all_loaded()) { fprintf(stderr, "llm_b200: neox start_session: %d of %d tensors loaded\n", m->n_loaded, (int)m->loaded.size()); return nullptr; }
    b200_neox_session *s = new b200_neox_session();
    s->m = m;
    const b200_neox_hparams &hp = m->hp;
    const size_t e = hp.n_embd, B = n_batch, n_ctx = hp.context_size, V = hp.n_vocab;
    s->start(n_batch, hp.context_size, hp.n_vocab, (size_t)hp.n_layer * n_ctx * e, (flags & B200_SESSION_KV_F32) ? T_F32 : T_F16);
    s->x = device_alloc<float>(B * e * 4); s->cur = device_alloc<float>(B * e * 4); s->qkv = device_alloc<float>(B * 3 * e * 4);
    s->kq = device_alloc<float>((size_t)hp.n_head * B * n_ctx * 4); s->attn = device_alloc<float>(B * e * 4);
    s->h4 = device_alloc<float>(B * 4 * e * 4); s->hact = device_alloc<float>(B * 4 * e * 4); s->t = device_alloc<float>(B * e * 4);
    s->logits = device_alloc<float>(B * V * 4);
    s->xq = device_alloc<int8_t>(B * 4 * e); s->xds = device_alloc<float2>(B * (4 * e / QK) * sizeof(float2));
    s->xpack = device_alloc<int4>((4 * e / QK) * 64); s->xh = device_alloc<__half>(xh_bytes(4 * e, B));
    s->qdec = device_alloc<float>(e * 4);
    if (m->any_kquant) s->xq8k = device_alloc<char>(q8k_bytes(4 * e, B));           // the widest K: fc_out's 4 n_embd
    s->xpack_a = device_alloc<int4>((e / QK) * 64); s->xpack_d = device_alloc<int4>((e / QK) * 64); s->xpack_f = device_alloc<int4>((4 * e / QK) * 64);
    s->dl.resize(hp.n_layer);
    for (int il = 0; il < hp.n_layer; il++) {
        const b200_neox_model::Layer &L = m->layers[il];
        s->dl[il] = NeoxLayer{L.wqkv, L.wdense, L.wfc, L.wproj, L.ln1_g, L.ln1_b, L.ln2_g, L.ln2_b, L.bqkv, L.bdense, L.bfc, L.bproj,
                              s->kv_at(0, (size_t)il * n_ctx * e), s->kv_at(1, (size_t)il * n_ctx * e)};
    }
    NeoxParams &P = s->dp;
    P.n_layer = hp.n_layer; P.e = (int)e; P.hd = m->hd; P.n_head = hp.n_head; P.n_ctx = (int)n_ctx; P.n_vocab = hp.n_vocab;
    P.kv_type = s->kv_type; P.parallel_residual = m->parallel; P.qkv_layout = m->qkv_layout; P.n_rot = m->rope && m->rope->mode ? m->rope->n_dims : 0; P.wpe = m->wpe;
    P.alibi = m->alibi.get(); P.emb_g = m->emb_g; P.emb_b = m->emb_b; P.wte = m->wte; P.lm_head = m->lm_head; P.lnf_g = m->lnf_g; P.lnf_b = m->lnf_b;
    P.gptj = m->gptj() ? 1 : 0; P.lm_head_b = m->lm_head_b;
    P.kq_scale = m->kq_scale; P.rope_cs = m->rope ? m->rope->cs : nullptr; P.rope_half = m->rope ? m->rope->half : 0;
    P.lut_gelu = luts().gelu; P.lut_exp = luts().exp; P.token = s->d_tokens.get(); P.n_past = s->decode.d_n_past;
    P.x = s->x.get(); P.qkv = s->qkv.get(); P.q = s->qdec.get(); P.attn_out = s->attn.get(); P.logits = s->logits.get();
    P.normed = s->cur.get();                                     // row 0 of cur: where forward()'s final LayerNorm leaves a one-token batch
    P.xpack_a = s->xpack_a.get(); P.xpack_d = s->xpack_d.get(); P.xpack_f = s->xpack_f.get();
    B200_CHECK(cudaDeviceSynchronize());
    return s;
}

int32_t b200_neox_n_past(const b200_neox_session *s) { return s ? s->n_past : -1; }
int b200_neox_set_n_past(b200_neox_session *s, int32_t n_past) { return s ? s->set_n_past(n_past) : B200_ERR_BAD_ARG; }
int b200_neox_read_kv(b200_neox_session *s, int32_t which, void *host_out, size_t nbytes) { return s ? s->read_kv(which, host_out, nbytes) : B200_ERR_BAD_ARG; }
int32_t b200_neox_last_launches(const b200_neox_session *s) { return s ? s->last_launches : 0; }
int b200_neox_sync(b200_neox_session *s) { if (!s) return B200_ERR_BAD_ARG; B200_CHECK(cudaStreamSynchronize(rt().stream)); return B200_OK; }

// tokens already in HBM (left there by the last b200_neox_evaluate), logits stay in HBM
int b200_neox_evaluate_device(b200_neox_session *s, int32_t n) {
    if (!s) return B200_ERR_BAD_ARG;
    if (const int rc = s->admit(n)) return rc;
    s->record_tokens(n);
    forward(s, n, true);
    return B200_OK;
}

// embeddings_out: row n - 1 of the final LayerNorm's output, which forward() leaves in cur (the graph step: its row 0)
int b200_neox_evaluate_output(b200_neox_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits, float *embeddings_out) {
    if (!s || !tokens) return B200_ERR_BAD_ARG;
    if (const int rc = s->admit(n)) return rc;
    if (const int rc = s->stage_tokens(tokens, n)) return rc;
    forward(s, n, all_logits != 0);
    s->copy_logits(logits_out, s->logits.get(), n, all_logits != 0);
    s->copy_row(embeddings_out, s->cur.get() + (size_t)(n - 1) * s->m->hp.n_embd, s->m->hp.n_embd);
    return B200_OK;
}

int b200_neox_evaluate(b200_neox_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits) {
    return b200_neox_evaluate_output(s, tokens, n, logits_out, all_logits, nullptr);
}

int b200_neox_perplexity(b200_neox_session *s, const int32_t *tokens, int64_t n, int32_t bos, float *ppl_out, float *terms_out, int32_t *n_chunk_out) {
    if (!s) return B200_ERR_BAD_ARG;
    return s->perplexity(tokens, n, bos, ppl_out, terms_out, n_chunk_out, s->logits.get(), [s](int rows) { forward(s, rows, true); });
}

int b200_neox_infer_next_token(b200_neox_session *s, const b200_sampler *sampler, int32_t *token_out) {
    SampleArgs a;
    if (!s || !sampler_args(sampler, a)) return B200_ERR_BAD_ARG;
    return s->infer_next_token(a, s->logits.get(), [s]() { forward(s, 1, true); }, token_out);
}

// ---- batched steps over sessions of one model (include/llm_b200.h) ---------------------------------------------------------------------------
int b200_neox_evaluate_ragged(b200_neox_model *m, b200_neox_session *const *sessions, int32_t n, const int32_t *counts, const int32_t *tokens,
                              float *logits_out, int32_t all_logits) {
    BatchSession ss[B200_MAX_SESSIONS];
    if (const int rc = batch_sessions(m, sessions, n, ss)) return rc;
    return m->batch.core.evaluate(ss, n, counts, tokens, logits_out, all_logits != 0, batch_front(m));
}

int b200_neox_evaluate_sessions(b200_neox_model *m, b200_neox_session *const *sessions, int32_t n, const int32_t *tokens, float *logits_out) {
    return b200_neox_evaluate_ragged(m, sessions, n, decode_counts(), tokens, logits_out, 0);
}

int b200_neox_infer_next_tokens(b200_neox_model *m, b200_neox_session *const *sessions, int32_t n, const b200_sampler *samplers, int32_t *tokens_out,
                                int32_t *status_out) {
    BatchSession ss[B200_MAX_SESSIONS];
    if (const int rc = batch_sessions(m, sessions, n, ss)) return rc;
    return m->batch.core.infer(ss, n, samplers, tokens_out, status_out, batch_front(m));
}

int32_t b200_neox_read_tokens(b200_neox_session *s, int32_t *tokens_out, int32_t max) { return s ? s->read_tokens(tokens_out, max) : B200_ERR_BAD_ARG; }
int b200_neox_last_logits(b200_neox_session *s, float *logits_out) { return s ? s->last_logits(s->logits.get(), logits_out) : B200_ERR_BAD_ARG; }

void b200_neox_session_free(b200_neox_session *s) {
    if (!s) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    delete s;                                           // every buffer, the decode graphs and n_past words go with it
}

// ---- snapshots (snapshot.cu): GPT-2, MPT and BLOOM keep V by position in the reference (gpt2 lib.rs:197-211, mpt :139-148, bloom :188-203) ---------
static RefKvLayout ref_layout(const b200_neox_model *m) {
    return RefKvLayout{m->hp.n_layer, m->hp.n_embd, m->hp.n_embd, m->hp.arch == 1 || m->mpt() || m->bloom()};
}

int b200_neox_get_snapshot(b200_neox_session *s, b200_snapshot *snap) {
    return s ? s->get_snapshot(ref_layout(s->m), s->logits.get(), snap) : B200_ERR_BAD_ARG;
}

int b200_neox_write_snapshot(b200_neox_session *s, const char *path) {
    return s ? s->write_snapshot(ref_layout(s->m), s->logits.get(), path) : B200_ERR_BAD_ARG;
}

static b200_neox_session *neox_session_from(b200_neox_model *m, const b200_snapshot *snap, const char *path, int *err) {
    if (!m) { if (err) *err = B200_ERR_BAD_ARG; return nullptr; }
    return session_from_snapshot<b200_neox_session>(snap, path, m->hp.context_size, m->hp.n_vocab, ref_layout(m), err,
        [m](int n_batch, bool kv32, float *&logits) -> b200_neox_session * {
            b200_neox_session *s = b200_neox_start_session_flags(m, n_batch, kv32 ? B200_SESSION_KV_F32 : 0);
            if (s) logits = s->logits.get();
            return s;
        },
        [](b200_neox_session *s) { b200_neox_session_free(s); });
}

b200_neox_session *b200_neox_session_from_snapshot(b200_neox_model *m, const b200_snapshot *snap, int *err) {
    return neox_session_from(m, snap, nullptr, err);
}

b200_neox_session *b200_neox_session_read_snapshot(b200_neox_model *m, const char *path, int *err) {
    if (!path) { if (err) *err = B200_ERR_BAD_ARG; return nullptr; }
    return neox_session_from(m, nullptr, path, err);
}

}  // extern "C"
