// llm_b200/csrc/neox.cu -- native host runtime for GPT-NeoX and GPT-2 (include/llm_b200.h: b200_neox_*): model + InferenceSession on the GPU.
//
// Mirrors   GptNeoX::new / TensorLoader         crates/models/gptneox/src/lib.rs:36-140
//           GptNeoX::evaluate (the graph)       crates/models/gptneox/src/lib.rs:156-350   (feed-forward: :487-515)
//           Gpt2::new / Gpt2::evaluate          crates/models/gpt2/src/lib.rs:43-136, 138-329   (hp.arch == 1: c_attn rows in thirds, no RoPE, learned positions,
//                                                                                               sequential residual, lm_head optional -> tied to wte)
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

struct b200_neox_model : Weights {
    b200_neox_hparams hp;
    int hd = 0;
    QWeight wte, lm_head;
    float *lnf_g = nullptr, *lnf_b = nullptr, *wpe = nullptr;     // wpe: GPT-2 learned positions [n_ctx][e] f32
    float *emb_g = nullptr, *emb_b = nullptr;                     // BLOOM: LayerNorm of the embedding row
    DeviceBuf<float> alibi;                                       // MPT / BLOOM: ALiBi slopes [n_head] (alibi_slopes)
    bool gpt2() const { return hp.arch == 1; }
    bool mpt() const { return hp.arch == 2; }
    bool bloom() const { return hp.arch == 3; }
    bool thirds() const { return hp.arch >= 1; }                  // GPT-2, MPT, BLOOM: q | k | v are the thirds of the fused row, no RoPE
    struct Layer { QWeight wqkv, wdense, wfc, wproj; float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *bqkv, *bdense, *bfc, *bproj; };   // MPT: every bias null
    std::vector<Layer> layers;
    int n_slots() const {
        if (mpt()) return 2 + 6 * hp.n_layer;                                 // wte, norm_f, 6 per block
        if (bloom()) return 6 + 12 * hp.n_layer;                              // wte, norm.{weight,bias}, output_norm.{weight,bias}, output, 12 per layer
        return 4 + 12 * hp.n_layer + (gpt2() && hp.has_lm_head ? 1 : 0);       // GPT-2: slot 3 = wpe, lm_head (if present) last
    }
    bool lookup(const char *name, Slot &s, int &id);
    bool lookup_alibi(const char *name, Slot &s, int &id);
};

struct b200_neox_session : SessionCore {   // memory_k [n_layer][n_ctx][e], memory_v [n_layer][e][n_ctx]
    b200_neox_model *m = nullptr;
    DeviceBuf<float> x, cur, qkv, kq, attn, h4, hact, t, logits;
    DeviceBuf<float> qdec;
    DeviceBuf<int8_t> xq; DeviceBuf<float2> xds; DeviceBuf<int4> xpack; DeviceBuf<__half> xh;
    DeviceBuf<int4> xpack_a, xpack_d, xpack_f;
    bool decode_ok = false;
    std::vector<NeoxLayer> dl;
    NeoxParams dp;
};

// MPT: crates/models/mpt/src/lib.rs:49-65; BLOOM: crates/models/bloom/src/lib.rs:56-83
bool b200_neox_model::lookup_alibi(const char *name, Slot &s, int &id) {
    const int e = hp.n_embd;
    int il = -1; char sub[96];
    struct Entry { const char *n; QWeight *q; float *f; int64_t len; };
    if (mpt()) {
        if (!strcmp(name, "transformer.wte.weight")) { s.q = wte; s.is_q = true; id = 0; return true; }
        if (!strcmp(name, "transformer.norm_f.weight")) { s.f = lnf_g; s.n = e; id = 1; return true; }
        if (sscanf(name, "transformer.blocks.%d.%95s", &il, sub) != 2 || il < 0 || il >= hp.n_layer) return false;
        Layer &L = layers[il];
        const Entry tab[] = {{"norm_1.weight", nullptr, L.ln1_g, e}, {"attn.Wqkv.weight", &L.wqkv, nullptr, 0}, {"attn.out_proj.weight", &L.wdense, nullptr, 0},
                             {"norm_2.weight", nullptr, L.ln2_g, e}, {"ffn.up_proj.weight", &L.wfc, nullptr, 0}, {"ffn.down_proj.weight", &L.wproj, nullptr, 0}};
        for (int k = 0; k < 6; k++)
            if (!strcmp(sub, tab[k].n)) {
                if (tab[k].q) { s.q = *tab[k].q; s.is_q = true; } else { s.f = tab[k].f; s.n = tab[k].len; }
                id = 2 + 6 * il + k;
                return true;
            }
        return false;
    }
    const Entry glob[] = {{"tok_embeddings.weight", &wte, nullptr, 0}, {"norm.weight", nullptr, emb_g, e}, {"norm.bias", nullptr, emb_b, e},
                          {"output_norm.weight", nullptr, lnf_g, e}, {"output_norm.bias", nullptr, lnf_b, e}, {"output.weight", &lm_head, nullptr, 0}};
    for (int k = 0; k < 6; k++)
        if (!strcmp(name, glob[k].n)) {
            if (glob[k].q) { s.q = *glob[k].q; s.is_q = true; } else { s.f = glob[k].f; s.n = glob[k].len; }
            id = k;
            return true;
        }
    if (sscanf(name, "layers.%d.%95s", &il, sub) != 2 || il < 0 || il >= hp.n_layer) return false;
    Layer &L = layers[il];
    const Entry tab[] = {
        {"attention_norm.weight", nullptr, L.ln1_g, e}, {"attention_norm.bias", nullptr, L.ln1_b, e},
        {"attention.query_key_value.weight", &L.wqkv, nullptr, 0}, {"attention.query_key_value.bias", nullptr, L.bqkv, 3 * (int64_t)e},
        {"attention.wo.weight", &L.wdense, nullptr, 0}, {"attention.wo.bias", nullptr, L.bdense, e},
        {"ffn_norm.weight", nullptr, L.ln2_g, e}, {"ffn_norm.bias", nullptr, L.ln2_b, e},
        {"feed_forward.w1.weight", &L.wfc, nullptr, 0}, {"feed_forward.w1.bias", nullptr, L.bfc, 4 * (int64_t)e},
        {"feed_forward.w2.weight", &L.wproj, nullptr, 0}, {"feed_forward.w2.bias", nullptr, L.bproj, e}};
    for (int k = 0; k < 12; k++)
        if (!strcmp(sub, tab[k].n)) {
            if (tab[k].q) { s.q = *tab[k].q; s.is_q = true; } else { s.f = tab[k].f; s.n = tab[k].len; }
            id = 6 + 12 * il + k;
            return true;
        }
    return false;
}

bool b200_neox_model::lookup(const char *name, Slot &s, int &id) {
    const int e = hp.n_embd;
    s = Slot();
    if (hp.arch >= 2) return lookup_alibi(name, s, id);
    if (gpt2()) {                                                         // tensor names of crates/models/gpt2/src/lib.rs:59-107
        if (!strcmp(name, "model/wte")) { s.q = wte; s.is_q = true; id = 0; return true; }
        if (!strcmp(name, "model/ln_f/g")) { s.f = lnf_g; s.n = e; id = 1; return true; }
        if (!strcmp(name, "model/ln_f/b")) { s.f = lnf_b; s.n = e; id = 2; return true; }
        if (!strcmp(name, "model/wpe")) { s.f = wpe; s.n = (int64_t)hp.context_size * e; id = 3; return true; }
        if (!strcmp(name, "model/lm_head")) { if (!hp.has_lm_head) return false; s.q = lm_head; s.is_q = true; id = 4 + 12 * hp.n_layer; return true; }
        int il = -1; char sub[96];
        if (sscanf(name, "model/h%d/%95s", &il, sub) != 2 || il < 0 || il >= hp.n_layer) return false;
        Layer &L = layers[il];
        struct { const char *n; QWeight *q; float *f; int64_t len; } tab[] = {
            {"ln_1/g", nullptr, L.ln1_g, e}, {"ln_1/b", nullptr, L.ln1_b, e}, {"ln_2/g", nullptr, L.ln2_g, e}, {"ln_2/b", nullptr, L.ln2_b, e},
            {"attn/c_attn/w", &L.wqkv, nullptr, 0}, {"attn/c_attn/b", nullptr, L.bqkv, 3 * (int64_t)e}, {"attn/c_proj/w", &L.wdense, nullptr, 0}, {"attn/c_proj/b", nullptr, L.bdense, e},
            {"mlp/c_fc/w", &L.wfc, nullptr, 0}, {"mlp/c_fc/b", nullptr, L.bfc, 4 * (int64_t)e}, {"mlp/c_proj/w", &L.wproj, nullptr, 0}, {"mlp/c_proj/b", nullptr, L.bproj, e}};
        for (int k = 0; k < 12; k++)
            if (!strcmp(sub, tab[k].n)) {
                if (tab[k].q) { s.q = *tab[k].q; s.is_q = true; } else { s.f = tab[k].f; s.n = tab[k].len; }
                id = 4 + 12 * il + k;
                return true;
            }
        return false;
    }
    if (!strcmp(name, "gpt_neox.embed_in.weight")) { s.q = wte; s.is_q = true; id = 0; return true; }
    if (!strcmp(name, "gpt_neox.final_layer_norm.weight")) { s.f = lnf_g; s.n = e; id = 1; return true; }
    if (!strcmp(name, "gpt_neox.final_layer_norm.bias")) { s.f = lnf_b; s.n = e; id = 2; return true; }
    if (!strcmp(name, "embed_out.weight")) { s.q = lm_head; s.is_q = true; id = 3; return true; }
    int il = -1; char sub[96];
    if (sscanf(name, "gpt_neox.layers.%d.%95s", &il, sub) != 2 || il < 0 || il >= hp.n_layer) return false;
    Layer &L = layers[il];
    const int base = 4 + 12 * il;
    struct { const char *n; QWeight *q; float *f; int64_t len; } tab[] = {
        {"input_layernorm.weight", nullptr, L.ln1_g, e}, {"input_layernorm.bias", nullptr, L.ln1_b, e},
        {"post_attention_layernorm.weight", nullptr, L.ln2_g, e}, {"post_attention_layernorm.bias", nullptr, L.ln2_b, e},
        {"attention.query_key_value.weight", &L.wqkv, nullptr, 0}, {"attention.query_key_value.bias", nullptr, L.bqkv, 3 * (int64_t)e},
        {"attention.dense.weight", &L.wdense, nullptr, 0}, {"attention.dense.bias", nullptr, L.bdense, e},
        {"mlp.dense_h_to_4h.weight", &L.wfc, nullptr, 0}, {"mlp.dense_h_to_4h.bias", nullptr, L.bfc, 4 * (int64_t)e},
        {"mlp.dense_4h_to_h.weight", &L.wproj, nullptr, 0}, {"mlp.dense_4h_to_h.bias", nullptr, L.bproj, e}};
    for (int k = 0; k < 12; k++)
        if (!strcmp(sub, tab[k].n)) {
            if (tab[k].q) { s.q = *tab[k].q; s.is_q = true; } else { s.f = tab[k].f; s.n = tab[k].len; }
            id = base + k;
            return true;
        }
    return false;
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
    if (n == 1 && s->decode_ok && attn_fused_fits((DecodeGraphCache::bucket(n_kv, n_ctx) + 63) / 64 * 64, hd)) {
        s->last_launches = s->decode.run(n_kv, n_ctx, true, [s, &hp](int bucket, cudaStream_t st, int *nodes) {
            neox_decode_enqueue(s->dp, s->dl, hp.wtype, bucket, st, nodes);
        }, st);
        s->n_past += 1;
        return;
    }
    const ExactActs acts{s->xq.get(), s->xds.get(), s->xpack.get(), s->xh.get()};
    const float kq_scale = 1.0f / sqrtf((float)e / (float)n_head);                                                  // :270-273
    const bool g2 = m->thirds(), parallel = !g2 && hp.use_parallel_residual;
    const RopeTable *rope = g2 ? nullptr : &rope_table(hp.n_rot, 2, 10000.0f, 1.0f, hd, n_ctx);
    const int64_t ld3 = 3 * (int64_t)e;
    // where q / k / v of head h live inside a row of the fused projection: NeoX per head [q | k | v], GPT-2 / MPT / BLOOM the three thirds of the row
    const int64_t hs = g2 ? hd : 3 * hd, koff = g2 ? e : hd, voff = g2 ? 2 * (int64_t)e : 2 * hd;
    if (m->bloom()) {                                                                                                             // bloom lib.rs:139-144
        get_rows_q(m->wte, s->d_tokens.get(), s->t.get(), n, st); L++;
        layer_norm(s->t.get(), s->x.get(), m->emb_g, m->emb_b, e, n, st); L++;
    } else {
        get_rows_q(m->wte, s->d_tokens.get(), s->x.get(), n, st); L++;                                                           // :178
    }
    if (m->gpt2()) { add_f32(s->x.get(), m->wpe + (size_t)n_past * e, s->x.get(), (int64_t)n * e, (int64_t)n * e, st); L++; }             // gpt2 lib.rs:164-172: + wpe[n_past + i]
    for (int il = 0; il < hp.n_layer; il++) {
        const b200_neox_model::Layer &ly = m->layers[il];
        __half *Kl = s->memory_k.get() + (size_t)il * n_ctx * e, *Vl = s->memory_v.get() + (size_t)il * n_ctx * e;
        layer_norm(s->x.get(), s->cur.get(), ly.ln1_g, ly.ln1_b, e, n, st); L++;                                                  // :192-196
        L += mul_mat_exact_auto(ly.wqkv, s->cur.get(), e, n, s->qkv.get(), ld3, nullptr, 0, acts, st);                                // :199
        if (ly.bqkv) { add_f32(s->qkv.get(), ly.bqkv, s->qkv.get(), (int64_t)n * ld3, ld3, st); L++; }                            // :200 (MPT: no bias)
        if (!g2) {   // RoPE mode 2 in place on q and k                                                                       :205-228
            rope_f32(s->qkv.get(), s->qkv.get(), hd, n_head, n, hs, ld3, hs, ld3, n_past, *rope, st); L++;
            rope_f32(s->qkv.get() + koff, s->qkv.get() + koff, hd, n_head, n, hs, ld3, hs, ld3, n_past, *rope, st); L++;
        }
        {   // k -> cache rows n_past.., v -> cache columns (transposed; GPT-2's v_trans copy of every evaluate is this layout)       :231-247
            StridedDesc sk{{hd, n_head, n, 1}, {4, hs * 4, ld3 * 4, 0}}, dk{{hd, n_head, n, 1}, {2, (int64_t)hd * 2, (int64_t)e * 2, 0}};
            cpy_strided(s->qkv.get() + koff, T_F32, sk, Kl + (size_t)n_past * e, T_F16, dk, st); L++;
            StridedDesc dv{{hd, n_head, n, 1}, {(int64_t)n_ctx * 2, (int64_t)hd * n_ctx * 2, 2, 0}};
            cpy_strided(s->qkv.get() + voff, T_F32, sk, Vl + n_past, T_F16, dv, st); L++;
        }
        mul_mat_f16_exact(Kl, hd, n_kv, n_head, (int64_t)e * 2, (int64_t)hd * 2, s->qkv.get(), n, n_head, ld3 * 4, hs * 4,
                          s->kq.get(), (int64_t)n_kv * 4, (int64_t)n_kv * n * 4, n_past, st); L++;                          // :250-267
        if (m->alibi) soft_max_alibi(s->kq.get(), s->kq.get(), n_kv, (int64_t)n_head * n, n, kq_scale, n_past, m->alibi.get(), st);   // MPT / BLOOM: + ALiBi
        else soft_max(s->kq.get(), s->kq.get(), n_kv, (int64_t)n_head * n, n, kq_scale, true, n_past, true, true, st);                // :270-279
        L++;
        mul_mat_f16_exact(Vl, n_kv, hd, n_head, (int64_t)n_ctx * 2, (int64_t)n_ctx * hd * 2, s->kq.get(), n, n_head, (int64_t)n_kv * 4, (int64_t)n_kv * n * 4,
                          s->cur.get(), (int64_t)e * 4, (int64_t)hd * 4, -1, st); L++;                                      // :282-298
        L += mul_mat_exact_auto(ly.wdense, s->cur.get(), e, n, s->attn.get(), e, nullptr, 0, acts, st);                               // :301
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
    } else {
        const size_t last = (size_t)(n - 1);
        layer_norm(s->x.get() + last * e, s->cur.get() + last * e, m->lnf_g, m->lnf_b, e, 1, st); L++;
        L += mul_mat_exact_auto(m->lm_head, s->cur.get() + last * e, e, 1, s->logits.get() + last * hp.n_vocab, hp.n_vocab, nullptr, 0, acts, st);
    }
    s->last_launches = L;
    s->n_past += n;
}

// hp->arch 0 / 1 (b200_neox_new) or 2 / 3 (b200_neox_new_alibi, alibi_bias_max: the ALiBi bias of MPT's header, 8 for BLOOM)
b200_neox_model *neox_new(const b200_neox_hparams *hp, float alibi_bias_max) {
    if (!hp || !is_quant(hp->wtype) || hp->n_embd % 64 || hp->n_head <= 0 || hp->n_embd % hp->n_head || hp->n_layer <= 0 || hp->context_size <= 0 ||
        (hp->arch == 0 && (hp->n_rot <= 0 || hp->n_rot % 2 || hp->n_rot > hp->n_embd / hp->n_head))) return nullptr;
    rt().ensure_init();
    b200_neox_model *m = new b200_neox_model();
    m->hp = *hp;
    const int e = hp->n_embd, v = hp->n_vocab, t = hp->wtype;
    m->hd = e / hp->n_head;
    m->layers.resize(hp->n_layer);
    if (m->mpt()) {                                                       // no biases (mpt lib.rs:49-65)
        m->carve(t, m->n_slots(), [m, e, v](SlabCarver &c) {
            c.q(m->wte, e, v); c.f(m->lnf_g, e);
            for (auto &L : m->layers) { c.f(L.ln1_g, e); c.f(L.ln2_g, e); c.q(L.wqkv, e, 3 * e); c.q(L.wdense, e, e); c.q(L.wfc, e, 4 * e); c.q(L.wproj, 4 * e, e); }
        });
    } else {
        m->carve(t, m->n_slots(), [m, hp, e, v](SlabCarver &c) {
            c.q(m->wte, e, v);
            if (!m->gpt2() || hp->has_lm_head) c.q(m->lm_head, e, v);
            c.f(m->lnf_g, e); c.f(m->lnf_b, e);
            if (m->gpt2()) c.f(m->wpe, (int64_t)hp->context_size * e);
            if (m->bloom()) { c.f(m->emb_g, e); c.f(m->emb_b, e); }
            for (auto &L : m->layers) {
                c.f(L.ln1_g, e); c.f(L.ln1_b, e); c.f(L.ln2_g, e); c.f(L.ln2_b, e); c.f(L.bqkv, 3 * e); c.f(L.bdense, e); c.f(L.bfc, 4 * e); c.f(L.bproj, e);
                c.q(L.wqkv, e, 3 * e); c.q(L.wdense, e, e); c.q(L.wfc, e, 4 * e); c.q(L.wproj, 4 * e, e);
            }
        });
    }
    // tied output projection (gpt2 lib.rs:319-320, MPT always): wte is streamed as the lm_head
    if ((m->gpt2() && !hp->has_lm_head) || m->mpt()) m->lm_head = m->wte;
    else m->weight_bytes -= (size_t)v * (e / QK) * ggml_block_bytes(t);  // the embedding table is gathered from, not streamed
    if (hp->arch >= 2) {
        const std::vector<float> slopes = alibi_slopes(hp->n_head, alibi_bias_max);
        m->alibi = device_alloc<float>(slopes.size() * 4);
        B200_CHECK(cudaMemcpy(m->alibi.get(), slopes.data(), slopes.size() * 4, cudaMemcpyHostToDevice));
    }
    return m;
}

}  // namespace

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

b200_neox_model *b200_neox_new(const b200_neox_hparams *hp) { return hp && (hp->arch == 0 || hp->arch == 1) ? neox_new(hp, 0.0f) : nullptr; }

b200_neox_model *b200_neox_new_alibi(const b200_neox_hparams *hp, float alibi_bias_max) {
    return hp && (hp->arch == 2 || hp->arch == 3) ? neox_new(hp, alibi_bias_max) : nullptr;   // MPT, BLOOM
}

size_t b200_neox_weight_bytes(b200_neox_model *m) { return m ? m->weight_bytes : 0; }

int b200_neox_load_tensor(b200_neox_model *m, const char *name, int32_t type, const void *host_data, size_t nbytes) {
    if (!m || !name || !host_data) return B200_ERR_BAD_ARG;
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    const int rc = load_slot(s, type, host_data, nbytes);
    if (rc == B200_OK) m->mark(id);
    return rc;
}

// seeded synthetic weights generated in HBM (bench): LayerNorm gains 1 + 0.1 N(0,1), biases = gains - 1 (small)
int b200_neox_synthesize(b200_neox_model *m, uint64_t seed) {
    if (!m) return B200_ERR_BAD_ARG;
    const int64_t e = m->hp.n_embd;
    m->synthesize(seed, [m, e](SeedSeq &r) {
        if (m->mpt()) {
            r.q(m->wte); r.gain(m->lnf_g, e);
            for (auto &L : m->layers) { r.gain(L.ln1_g, e); r.gain(L.ln2_g, e); r.q(L.wqkv); r.q(L.wdense); r.q(L.wfc); r.q(L.wproj); }
            return;
        }
        r.q(m->wte); if (!m->gpt2() || m->hp.has_lm_head) r.q(m->lm_head); r.gain(m->lnf_g, e); r.bias(m->lnf_b, e);
        if (m->gpt2()) r.bias(m->wpe, (int64_t)m->hp.context_size * e);
        if (m->bloom()) { r.gain(m->emb_g, e); r.bias(m->emb_b, e); }
        for (auto &L : m->layers) {
            r.gain(L.ln1_g, e); r.bias(L.ln1_b, e); r.gain(L.ln2_g, e); r.bias(L.ln2_b, e); r.bias(L.bqkv, 3 * e); r.bias(L.bdense, e); r.bias(L.bfc, 4 * e); r.bias(L.bproj, e);
            r.q(L.wqkv); r.q(L.wdense); r.q(L.wfc); r.q(L.wproj);
        }
    });
    return B200_OK;
}

void b200_neox_free(b200_neox_model *m) {
    if (!m) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    delete m;                                           // the slab goes with it
}

b200_neox_session *b200_neox_start_session(b200_neox_model *m, int32_t n_batch) {
    if (!m || n_batch < 1) return nullptr;
    if (!m->all_loaded()) { fprintf(stderr, "llm_b200: neox start_session: %d of %d tensors loaded\n", m->n_loaded, m->n_slots()); return nullptr; }
    b200_neox_session *s = new b200_neox_session();
    s->m = m;
    const b200_neox_hparams &hp = m->hp;
    const size_t e = hp.n_embd, B = n_batch, n_ctx = hp.context_size, V = hp.n_vocab;
    s->start(n_batch, hp.context_size, hp.n_vocab, (size_t)hp.n_layer * n_ctx * e);
    s->x = device_alloc<float>(B * e * 4); s->cur = device_alloc<float>(B * e * 4); s->qkv = device_alloc<float>(B * 3 * e * 4);
    s->kq = device_alloc<float>((size_t)hp.n_head * B * n_ctx * 4); s->attn = device_alloc<float>(B * e * 4);
    s->h4 = device_alloc<float>(B * 4 * e * 4); s->hact = device_alloc<float>(B * 4 * e * 4); s->t = device_alloc<float>(B * e * 4);
    s->logits = device_alloc<float>(B * V * 4);
    s->xq = device_alloc<int8_t>(B * 4 * e); s->xds = device_alloc<float2>(B * (4 * e / QK) * sizeof(float2));
    s->xpack = device_alloc<int4>((4 * e / QK) * 64); s->xh = device_alloc<__half>(xh_bytes(4 * e, B));
    s->qdec = device_alloc<float>(e * 4);
    s->xpack_a = device_alloc<int4>((e / QK) * 64); s->xpack_d = device_alloc<int4>((e / QK) * 64); s->xpack_f = device_alloc<int4>((4 * e / QK) * 64);
    const RopeTable *rt_ = m->thirds() ? nullptr : &rope_table(hp.n_rot, 2, 10000.0f, 1.0f, m->hd, (int)n_ctx);
    s->dl.resize(hp.n_layer);
    for (int il = 0; il < hp.n_layer; il++) {
        const b200_neox_model::Layer &L = m->layers[il];
        s->dl[il] = NeoxLayer{L.wqkv, L.wdense, L.wfc, L.wproj, L.ln1_g, L.ln1_b, L.ln2_g, L.ln2_b, L.bqkv, L.bdense, L.bfc, L.bproj,
                              s->memory_k.get() + (size_t)il * n_ctx * e, s->memory_v.get() + (size_t)il * n_ctx * e};
    }
    NeoxParams &P = s->dp;
    P.n_layer = hp.n_layer; P.e = (int)e; P.hd = m->hd; P.n_head = hp.n_head; P.n_ctx = (int)n_ctx; P.n_vocab = hp.n_vocab; P.n_rot = hp.n_rot;
    P.parallel_residual = !m->thirds() && hp.use_parallel_residual; P.gpt2 = m->thirds() ? 1 : 0; P.wpe = m->wpe;
    P.alibi = m->alibi.get(); P.emb_g = m->emb_g; P.emb_b = m->emb_b; P.wte = m->wte; P.lm_head = m->lm_head; P.lnf_g = m->lnf_g; P.lnf_b = m->lnf_b;
    P.kq_scale = 1.0f / sqrtf((float)e / (float)hp.n_head); P.rope_cs = rt_ ? rt_->cs : nullptr; P.rope_half = rt_ ? rt_->half : 0;
    P.lut_gelu = luts().gelu; P.lut_exp = luts().exp; P.token = s->d_tokens.get(); P.n_past = s->decode.d_n_past;
    P.x = s->x.get(); P.qkv = s->qkv.get(); P.q = s->qdec.get(); P.attn_out = s->attn.get(); P.logits = s->logits.get();
    P.xpack_a = s->xpack_a.get(); P.xpack_d = s->xpack_d.get(); P.xpack_f = s->xpack_f.get();
    QWeight p1; p1.nb = (int64_t)e / QK; QWeight p2; p2.nb = 4 * (int64_t)e / QK;
    s->decode_ok = m->hd % 32 == 0 && m->hd <= 128 && e % 128 == 0 && e <= 8192 && n_ctx % 8 == 0 && mmv_exact_stream_supported(p1) && mmv_exact_stream_supported(p2) &&
                   !getenv("B200_NEOX_UNFUSED");
    B200_CHECK(cudaDeviceSynchronize());
    return s;
}

int32_t b200_neox_n_past(const b200_neox_session *s) { return s ? s->n_past : -1; }
int b200_neox_set_n_past(b200_neox_session *s, int32_t n_past) { return s ? s->set_n_past(n_past) : B200_ERR_BAD_ARG; }
int b200_neox_read_kv(b200_neox_session *s, int32_t which, void *host_out, size_t nbytes) {
    if (!s || !host_out) return B200_ERR_BAD_ARG;
    const size_t kv_bytes = (size_t)s->m->hp.n_layer * s->m->hp.context_size * s->m->hp.n_embd * 2;
    if (nbytes != kv_bytes) return B200_ERR_TENSOR_SHAPE;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    B200_CHECK(cudaMemcpy(host_out, which ? s->memory_v.get() : s->memory_k.get(), kv_bytes, cudaMemcpyDeviceToHost));
    return B200_OK;
}
int32_t b200_neox_last_launches(const b200_neox_session *s) { return s ? s->last_launches : 0; }
int b200_neox_sync(b200_neox_session *s) { if (!s) return B200_ERR_BAD_ARG; B200_CHECK(cudaStreamSynchronize(rt().stream)); return B200_OK; }

// tokens already in HBM (left there by the last b200_neox_evaluate), logits stay in HBM
int b200_neox_evaluate_device(b200_neox_session *s, int32_t n) {
    if (!s) return B200_ERR_BAD_ARG;
    if (const int rc = s->admit(n)) return rc;
    forward(s, n, true);
    return B200_OK;
}

int b200_neox_evaluate(b200_neox_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits) {
    if (!s || !tokens) return B200_ERR_BAD_ARG;
    if (const int rc = s->admit(n)) return rc;
    if (const int rc = s->stage_tokens(tokens, n)) return rc;
    forward(s, n, all_logits != 0);
    s->copy_logits(logits_out, s->logits.get(), n, all_logits != 0);
    return B200_OK;
}

void b200_neox_session_free(b200_neox_session *s) {
    if (!s) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    delete s;                                           // every buffer, the decode graphs and n_past words go with it
}

}  // extern "C"
