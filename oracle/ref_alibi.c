/*
 * oracle/ref_alibi.c -- TEST INFRASTRUCTURE (see ref_harness.c): the reference's MPT and BLOOM models driven through the UNMODIFIED ggml C API.
 *
 * Restates node for node:
 *   Mpt::new / Mpt::evaluate       crates/models/mpt/src/lib.rs:40-258     (arch 2) LayerNorm = norm, mul gain (no bias anywhere), fused Wqkv split
 *                                                                          in thirds of the row, scale -> alibi(alibi_bias_max) -> diag_mask_inf ->
 *                                                                          soft_max, gelu MLP, residual x + attn then + ffn, lm_head tied to wte
 *   Bloom::new / Bloom::evaluate   crates/models/bloom/src/lib.rs:48-345   (arch 3) embedding row -> norm * norm.weight + norm.bias, then the GPT-2
 *                                                                          block with biases on qkv / wo / w1 / w2 and alibi(8); output_norm, output
 *   InferenceSession::new / ::compute   crates/llm-base/src/inference_session.rs:114-295   f16 KV cache, both K and V stored by position
 * CPU build only: GGML_OP_ALIBI has no ggml_cuda_* entry point, so the reference runs these graphs on the host.
 */
#include "ggml.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define RA_MAX_LAYERS 64

typedef struct {
    int32_t n_vocab, n_ctx, n_embd, n_head, n_layer;
    int32_t wtype;      /* enum ggml_type of the 2-D weights */
    int32_t n_threads, n_batch;
    int32_t arch;       /* 2 MPT, 3 BLOOM */
    float alibi_bias_max;   /* MPT: from the file header; BLOOM: 8 (bloom lib.rs:240) */
} ra_params;

typedef struct {
    struct ggml_tensor *ln_1_g, *ln_1_b, *ln_2_g, *ln_2_b, *wqkv, *bqkv, *wo, *bo, *w1, *b1, *w2, *b2;   /* MPT: every bias NULL */
} ra_layer;

typedef struct {
    ra_params hp;
    struct ggml_context *model_ctx, *session_ctx, *ctx0;
    struct ggml_tensor *wte, *norm_g, *norm_b, *out_g, *out_b, *output;   /* norm_*: BLOOM's embedding norm; out_b, output: BLOOM only */
    ra_layer layers[RA_MAX_LAYERS];
    struct ggml_tensor *memory_k, *memory_v;
    void *eval_buf; size_t eval_size;
    void *scratch[2]; size_t scratch_size;
    int n_past, finalized;
} ra_model;

static size_t ra_bytes(enum ggml_type t, int64_t ne0, int64_t ne1) { return (size_t)(ne0 / ggml_blck_size(t)) * ggml_type_size(t) * (size_t)ne1; }

static void ra_use_scratch(ra_model *m, int idx) {
    struct ggml_scratch s = {0, 0, NULL};
    if (idx >= 0) { s.size = m->scratch_size; s.data = m->scratch[idx]; }
    ggml_set_scratch(m->ctx0, s);
}

ra_model *ra_new(const ra_params *p) {
    if (p->n_layer > RA_MAX_LAYERS || (p->arch != 2 && p->arch != 3)) return NULL;
    ra_model *m = calloc(1, sizeof(*m));
    m->hp = *p;
    const enum ggml_type wt = (enum ggml_type)p->wtype;
    const int64_t e = p->n_embd;
    const int bloom = p->arch == 3;
    size_t wbytes = ra_bytes(wt, e, p->n_vocab) * 2 + (size_t)e * 4 * 4;
    wbytes += (size_t)p->n_layer * (ra_bytes(wt, e, 3 * e) + ra_bytes(wt, e, e) + ra_bytes(wt, e, 4 * e) + ra_bytes(wt, 4 * e, e) + (size_t)e * 4 * 13);
    wbytes += (size_t)(6 + 12 * p->n_layer) * 512 + (1u << 20);
    struct ggml_init_params ip = { wbytes, NULL, false };
    m->model_ctx = ggml_init(ip);
    struct ggml_context *c = m->model_ctx;
    m->wte = ggml_new_tensor_2d(c, wt, e, p->n_vocab);
    m->out_g = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
    if (bloom) {
        m->norm_g = ggml_new_tensor_1d(c, GGML_TYPE_F32, e); m->norm_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
        m->out_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
        m->output = ggml_new_tensor_2d(c, wt, e, p->n_vocab);
    }
    for (int i = 0; i < p->n_layer; i++) {
        ra_layer *L = &m->layers[i];
        L->ln_1_g = ggml_new_tensor_1d(c, GGML_TYPE_F32, e); L->ln_2_g = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
        L->wqkv = ggml_new_tensor_2d(c, wt, e, 3 * e); L->wo = ggml_new_tensor_2d(c, wt, e, e);
        L->w1 = ggml_new_tensor_2d(c, wt, e, 4 * e);   L->w2 = ggml_new_tensor_2d(c, wt, 4 * e, e);
        if (bloom) {
            L->ln_1_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e); L->ln_2_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
            L->bqkv = ggml_new_tensor_1d(c, GGML_TYPE_F32, 3 * e); L->bo = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
            L->b1 = ggml_new_tensor_1d(c, GGML_TYPE_F32, 4 * e);   L->b2 = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
        }
    }
    return m;
}

void *ra_tensor(ra_model *m, const char *name, size_t *nbytes) {     /* loader names: mpt lib.rs:50-65, bloom lib.rs:56-83 */
    struct ggml_tensor *t = NULL;
    int il = -1; char sub[96];
    if (m->hp.arch == 2) {
        if (!strcmp(name, "transformer.wte.weight")) t = m->wte;
        else if (!strcmp(name, "transformer.norm_f.weight")) t = m->out_g;
        else if (sscanf(name, "transformer.blocks.%d.%95s", &il, sub) == 2 && il >= 0 && il < m->hp.n_layer) {
            ra_layer *L = &m->layers[il];
            if      (!strcmp(sub, "norm_1.weight")) t = L->ln_1_g;
            else if (!strcmp(sub, "attn.Wqkv.weight")) t = L->wqkv;
            else if (!strcmp(sub, "attn.out_proj.weight")) t = L->wo;
            else if (!strcmp(sub, "norm_2.weight")) t = L->ln_2_g;
            else if (!strcmp(sub, "ffn.up_proj.weight")) t = L->w1;
            else if (!strcmp(sub, "ffn.down_proj.weight")) t = L->w2;
        }
    } else {
        if (!strcmp(name, "tok_embeddings.weight")) t = m->wte;
        else if (!strcmp(name, "norm.weight")) t = m->norm_g;
        else if (!strcmp(name, "norm.bias")) t = m->norm_b;
        else if (!strcmp(name, "output_norm.weight")) t = m->out_g;
        else if (!strcmp(name, "output_norm.bias")) t = m->out_b;
        else if (!strcmp(name, "output.weight")) t = m->output;
        else if (sscanf(name, "layers.%d.%95s", &il, sub) == 2 && il >= 0 && il < m->hp.n_layer) {
            ra_layer *L = &m->layers[il];
            if      (!strcmp(sub, "attention_norm.weight")) t = L->ln_1_g;
            else if (!strcmp(sub, "attention_norm.bias")) t = L->ln_1_b;
            else if (!strcmp(sub, "attention.query_key_value.weight")) t = L->wqkv;
            else if (!strcmp(sub, "attention.query_key_value.bias")) t = L->bqkv;
            else if (!strcmp(sub, "attention.wo.weight")) t = L->wo;
            else if (!strcmp(sub, "attention.wo.bias")) t = L->bo;
            else if (!strcmp(sub, "ffn_norm.weight")) t = L->ln_2_g;
            else if (!strcmp(sub, "ffn_norm.bias")) t = L->ln_2_b;
            else if (!strcmp(sub, "feed_forward.w1.weight")) t = L->w1;
            else if (!strcmp(sub, "feed_forward.w1.bias")) t = L->b1;
            else if (!strcmp(sub, "feed_forward.w2.weight")) t = L->w2;
            else if (!strcmp(sub, "feed_forward.w2.bias")) t = L->b2;
        }
    }
    if (!t) return NULL;
    if (nbytes) *nbytes = ggml_nbytes(t);
    return t->data;
}

int ra_finalize(ra_model *m) {
    const ra_params *p = &m->hp;
    const size_t n_elements = (size_t)p->n_embd * p->n_layer * p->n_ctx;     /* inference_session.rs:127-160 */
    struct ggml_init_params ip = { n_elements * 2 * 2 + 8192, NULL, false };
    m->session_ctx = ggml_init(ip);
    m->memory_k = ggml_new_tensor_1d(m->session_ctx, GGML_TYPE_F16, n_elements);
    m->memory_v = ggml_new_tensor_1d(m->session_ctx, GGML_TYPE_F16, n_elements);
    memset(m->memory_k->data, 0, ggml_nbytes(m->memory_k));
    memset(m->memory_v->data, 0, ggml_nbytes(m->memory_v));
    const size_t B = (size_t)p->n_batch;
    size_t per = B * p->n_embd * 4 * (4 * 3 + 16) + (size_t)p->n_head * B * p->n_ctx * 4 * 2 + (size_t)p->n_ctx * p->n_embd * 2 * 2 + (64u << 20);
    m->scratch_size = per;
    m->scratch[0] = malloc(per); m->scratch[1] = malloc(per);
    m->eval_size = B * p->n_vocab * 4 + B * p->n_embd * 64 + (size_t)p->n_layer * 96 * 512 + B * p->n_embd * 4 * 40 + ggml_graph_overhead() + (64u << 20);
    m->eval_buf = malloc(m->eval_size);
    m->finalized = 1;
    return 0;
}

void ra_reset(ra_model *m) { m->n_past = 0; }

/* norm, mul by the gain, add the bias if there is one (MPT has none: no add node at all, which would turn -0 into +0) */
static struct ggml_tensor *ra_ln(struct ggml_context *ctx0, struct ggml_tensor *x, struct ggml_tensor *g, struct ggml_tensor *b) {
    struct ggml_tensor *cur = ggml_mul(ctx0, ggml_norm(ctx0, x), g);
    return b ? ggml_add(ctx0, cur, b) : cur;
}
static struct ggml_tensor *ra_bias(struct ggml_context *ctx0, struct ggml_tensor *x, struct ggml_tensor *b) { return b ? ggml_add(ctx0, x, b) : x; }

int ra_eval(ra_model *m, const int32_t *tokens, int n, float *logits_out) {
    const ra_params *p = &m->hp;
    if (!m->finalized || n < 1 || n > p->n_batch || m->n_past + n > p->n_ctx) return -1;
    const int n_embd = p->n_embd, n_head = p->n_head, ctx_size = p->n_ctx, session_len = m->n_past;
    const int mpt = p->arch == 2;
    const size_t ksz = 2, vsz = 2, f32sz = 4;

    if (m->ctx0) ggml_free(m->ctx0);
    struct ggml_init_params ip = { m->eval_size, m->eval_buf, false };
    m->ctx0 = ggml_init(ip);
    struct ggml_context *ctx0 = m->ctx0;

    struct ggml_tensor *embd = ggml_new_tensor_1d(ctx0, GGML_TYPE_I32, n);
    struct ggml_tensor *inpL = ggml_get_rows(ctx0, m->wte, embd);
    if (!mpt) inpL = ra_ln(ctx0, inpL, m->norm_g, m->norm_b);
    struct ggml_cgraph *gf = ggml_new_graph(ctx0);

    for (int il = 0; il < p->n_layer; il++) {
        const ra_layer *L = &m->layers[il];
        ra_use_scratch(m, 0);
        struct ggml_tensor *cur = ra_ln(ctx0, inpL, L->ln_1_g, L->ln_1_b);
        cur = ra_bias(ctx0, ggml_mul_mat(ctx0, L->wqkv, cur), L->bqkv);
        const size_t nb = cur->nb[1];
        struct ggml_tensor *qcur = ggml_view_2d(ctx0, cur, n_embd, n, nb, 0);
        struct ggml_tensor *kcur = ggml_view_2d(ctx0, cur, n_embd, n, nb, f32sz * n_embd);
        struct ggml_tensor *vcur = ggml_view_2d(ctx0, cur, n_embd, n, nb, f32sz * n_embd * 2);
        struct ggml_tensor *k = ggml_view_1d(ctx0, m->memory_k, (int64_t)n * n_embd, (ksz * n_embd) * ((size_t)il * ctx_size + session_len));
        struct ggml_tensor *v = ggml_view_1d(ctx0, m->memory_v, (int64_t)n * n_embd, (vsz * n_embd) * ((size_t)il * ctx_size + session_len));
        ggml_build_forward_expand(gf, ggml_cpy(ctx0, kcur, k));
        ggml_build_forward_expand(gf, ggml_cpy(ctx0, vcur, v));
        struct ggml_tensor *q = ggml_permute(ctx0, ggml_cpy(ctx0, qcur, ggml_new_tensor_3d(ctx0, GGML_TYPE_F32, n_embd / n_head, n_head, n)), 0, 2, 1, 3);
        struct ggml_tensor *kk = ggml_permute(ctx0,
            ggml_reshape_3d(ctx0, ggml_view_1d(ctx0, m->memory_k, (int64_t)(session_len + n) * n_embd, (size_t)il * ctx_size * ksz * n_embd),
                            n_embd / n_head, n_head, session_len + n), 0, 2, 1, 3);
        struct ggml_tensor *kq = ggml_mul_mat(ctx0, kk, q);
        struct ggml_tensor *kq_scaled = ggml_scale(ctx0, kq, ggml_new_f32(ctx0, 1.0f / sqrtf((float)n_embd / (float)n_head)));
        struct ggml_tensor *kq_alibi = ggml_alibi(ctx0, kq_scaled, session_len, n_head, p->alibi_bias_max);
        struct ggml_tensor *kq_masked = ggml_diag_mask_inf(ctx0, kq_alibi, session_len);
        struct ggml_tensor *kq_softmax = ggml_soft_max(ctx0, kq_masked);
        struct ggml_tensor *v_trans = ggml_cpy(ctx0,
            ggml_permute(ctx0,
                ggml_reshape_3d(ctx0, ggml_view_1d(ctx0, m->memory_v, (int64_t)(session_len + n) * n_embd, (size_t)il * ctx_size * vsz * n_embd),
                                n_embd / n_head, n_head, session_len + n), 1, 2, 0, 3),
            ggml_new_tensor_3d(ctx0, m->memory_v->type, session_len + n, n_embd / n_head, n_head));
        struct ggml_tensor *kqv = ggml_mul_mat(ctx0, v_trans, kq_softmax);
        struct ggml_tensor *kqv_merged = ggml_permute(ctx0, kqv, 0, 2, 1, 3);
        cur = ggml_cpy(ctx0, kqv_merged, ggml_new_tensor_2d(ctx0, GGML_TYPE_F32, n_embd, n));
        cur = ra_bias(ctx0, ggml_mul_mat(ctx0, L->wo, cur), L->bo);
        struct ggml_tensor *ff_in = mpt ? ggml_add(ctx0, inpL, cur) : ggml_add(ctx0, cur, inpL);
        ra_use_scratch(m, 1);
        cur = ra_ln(ctx0, ff_in, L->ln_2_g, L->ln_2_b);
        cur = ra_bias(ctx0, ggml_mul_mat(ctx0, L->w1, cur), L->b1);
        cur = ggml_gelu(ctx0, cur);
        cur = ra_bias(ctx0, ggml_mul_mat(ctx0, L->w2, cur), L->b2);
        inpL = mpt ? ggml_add(ctx0, ff_in, cur) : ggml_add(ctx0, cur, ff_in);
    }
    ra_use_scratch(m, 0);
    inpL = ra_ln(ctx0, inpL, m->out_g, m->out_b);
    ra_use_scratch(m, -1);
    inpL = ggml_mul_mat(ctx0, mpt ? m->wte : m->output, inpL);

    memcpy(embd->data, tokens, (size_t)n * 4);
    ggml_build_forward_expand(gf, inpL);
    struct ggml_cplan plan = ggml_graph_plan(gf, p->n_threads);
    struct ggml_tensor *work = ggml_new_tensor_1d(ctx0, GGML_TYPE_I8, plan.work_size ? plan.work_size : 1);
    plan.work_data = work->data;
    ggml_graph_compute(gf, &plan);
    m->n_past += n;
    if (logits_out) memcpy(logits_out, inpL->data, (size_t)n * p->n_vocab * 4);
    return 0;
}

/* memory_k (which = 0) / memory_v (1): [n_layer][n_ctx][n_embd] f16, both by position */
void *ra_kv(ra_model *m, int which, size_t *nbytes) {
    struct ggml_tensor *t = which ? m->memory_v : m->memory_k;
    if (nbytes) *nbytes = ggml_nbytes(t);
    return t->data;
}

void ra_free(ra_model *m) {
    if (!m) return;
    if (m->ctx0) ggml_free(m->ctx0);
    if (m->session_ctx) ggml_free(m->session_ctx);
    if (m->model_ctx) ggml_free(m->model_ctx);
    free(m->eval_buf); free(m->scratch[0]); free(m->scratch[1]);
    free(m);
}
