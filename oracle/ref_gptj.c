/*
 * oracle/ref_gptj.c -- TEST INFRASTRUCTURE (see ref_harness.c): the reference's GPT-J model driven through the UNMODIFIED ggml C API.
 *
 * Restates node for node:
 *   GptJ::new / GptJ::evaluate          crates/models/gptj/src/lib.rs:47-311   one LayerNorm per layer (input_sa) feeding q/k/v AND fc_in, q_proj /
 *                                                                               k_proj / v_proj as three mat-muls, ggml_rope_inplace mode 0 on q and k,
 *                                                                               K stored by position, V transposed (by channel), scale -> diag_mask_inf ->
 *                                                                               soft_max, out_proj (no bias); ((fc_out gelu(fc_in input_sa + b) + b) + attn)
 *                                                                               + inpL; ln_f, lm_head, + lm_head.bias
 *   InferenceSession::new / ::compute   crates/llm-base/src/inference_session.rs:114-295   f16 KV cache, no rope overrides
 * No scratch buffers: every node gets its own memory in the evaluation context (the values do not depend on where they live).
 */
#include "ggml.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define RJ_MAX_LAYERS 64

typedef struct {
    int32_t n_vocab, n_ctx, n_embd, n_head, n_layer, n_rot;
    int32_t wtype;      /* enum ggml_type of the 2-D weights */
    int32_t n_threads, n_batch;
} rj_params;

typedef struct {
    struct ggml_tensor *ln_1_g, *ln_1_b, *wq, *wk, *wv, *wo, *fc_in_w, *fc_in_b, *fc_out_w, *fc_out_b;
} rj_layer;

typedef struct {
    rj_params hp;
    struct ggml_context *model_ctx, *session_ctx, *ctx0;
    struct ggml_tensor *wte, *ln_f_g, *ln_f_b, *lmh_g, *lmh_b;
    rj_layer layers[RJ_MAX_LAYERS];
    struct ggml_tensor *memory_k, *memory_v;
    void *eval_buf; size_t eval_size;
    int n_past, finalized;
} rj_model;

static size_t rj_bytes(enum ggml_type t, int64_t ne0, int64_t ne1) { return (size_t)(ne0 / ggml_blck_size(t)) * ggml_type_size(t) * (size_t)ne1; }

rj_model *rj_new(const rj_params *p) {
    if (p->n_layer > RJ_MAX_LAYERS || p->n_layer < 1) return NULL;
    rj_model *m = calloc(1, sizeof(*m));
    m->hp = *p;
    const enum ggml_type wt = (enum ggml_type)p->wtype;
    const int64_t e = p->n_embd, v = p->n_vocab;
    size_t wbytes = rj_bytes(wt, e, v) * 2 + (size_t)e * 4 * 2 + (size_t)v * 4;
    wbytes += (size_t)p->n_layer * (rj_bytes(wt, e, e) * 4 + rj_bytes(wt, e, 4 * e) + rj_bytes(wt, 4 * e, e) + (size_t)e * 4 * 7);
    wbytes += (size_t)(5 + 10 * p->n_layer) * 512 + (1u << 20);
    struct ggml_init_params ip = { wbytes, NULL, false };
    m->model_ctx = ggml_init(ip);
    struct ggml_context *c = m->model_ctx;
    m->wte = ggml_new_tensor_2d(c, wt, e, v);
    m->ln_f_g = ggml_new_tensor_1d(c, GGML_TYPE_F32, e); m->ln_f_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
    m->lmh_g = ggml_new_tensor_2d(c, wt, e, v);          m->lmh_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, v);
    for (int i = 0; i < p->n_layer; i++) {
        rj_layer *L = &m->layers[i];
        L->ln_1_g = ggml_new_tensor_1d(c, GGML_TYPE_F32, e); L->ln_1_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
        L->wq = ggml_new_tensor_2d(c, wt, e, e); L->wk = ggml_new_tensor_2d(c, wt, e, e); L->wv = ggml_new_tensor_2d(c, wt, e, e);
        L->wo = ggml_new_tensor_2d(c, wt, e, e);
        L->fc_in_w = ggml_new_tensor_2d(c, wt, e, 4 * e);  L->fc_in_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, 4 * e);
        L->fc_out_w = ggml_new_tensor_2d(c, wt, 4 * e, e); L->fc_out_b = ggml_new_tensor_1d(c, GGML_TYPE_F32, e);
    }
    return m;
}

void *rj_tensor(rj_model *m, const char *name, size_t *nbytes) {     /* loader names: gptj lib.rs:59-103 */
    struct ggml_tensor *t = NULL;
    int il = -1; char sub[96];
    if (!strcmp(name, "transformer.wte.weight")) t = m->wte;
    else if (!strcmp(name, "transformer.ln_f.weight")) t = m->ln_f_g;
    else if (!strcmp(name, "transformer.ln_f.bias")) t = m->ln_f_b;
    else if (!strcmp(name, "lm_head.weight")) t = m->lmh_g;
    else if (!strcmp(name, "lm_head.bias")) t = m->lmh_b;
    else if (sscanf(name, "transformer.h.%d.%95s", &il, sub) == 2 && il >= 0 && il < m->hp.n_layer) {
        rj_layer *L = &m->layers[il];
        if      (!strcmp(sub, "ln_1.weight")) t = L->ln_1_g;
        else if (!strcmp(sub, "ln_1.bias")) t = L->ln_1_b;
        else if (!strcmp(sub, "attn.q_proj.weight")) t = L->wq;
        else if (!strcmp(sub, "attn.k_proj.weight")) t = L->wk;
        else if (!strcmp(sub, "attn.v_proj.weight")) t = L->wv;
        else if (!strcmp(sub, "attn.out_proj.weight")) t = L->wo;
        else if (!strcmp(sub, "mlp.fc_in.weight")) t = L->fc_in_w;
        else if (!strcmp(sub, "mlp.fc_in.bias")) t = L->fc_in_b;
        else if (!strcmp(sub, "mlp.fc_out.weight")) t = L->fc_out_w;
        else if (!strcmp(sub, "mlp.fc_out.bias")) t = L->fc_out_b;
    }
    if (!t) return NULL;
    if (nbytes) *nbytes = ggml_nbytes(t);
    return t->data;
}

int rj_finalize(rj_model *m) {
    const rj_params *p = &m->hp;
    const size_t n_elements = (size_t)p->n_embd * p->n_layer * p->n_ctx;     /* inference_session.rs:127-160 */
    struct ggml_init_params ip = { n_elements * 2 * 2 + 8192, NULL, false };
    m->session_ctx = ggml_init(ip);
    m->memory_k = ggml_new_tensor_1d(m->session_ctx, GGML_TYPE_F16, n_elements);
    m->memory_v = ggml_new_tensor_1d(m->session_ctx, GGML_TYPE_F16, n_elements);
    memset(m->memory_k->data, 0, ggml_nbytes(m->memory_k));
    memset(m->memory_v->data, 0, ggml_nbytes(m->memory_v));
    const size_t B = (size_t)p->n_batch, e = (size_t)p->n_embd;
    const size_t per_layer = B * e * 4 * 16 + B * 4 * e * 4 * 4 + (size_t)p->n_head * B * p->n_ctx * 4 * 2 + (64u << 10);
    m->eval_size = (size_t)p->n_layer * per_layer + B * p->n_vocab * 4 * 3 + B * e * 4 * 8 + ggml_graph_overhead() + (64u << 20);
    m->eval_buf = malloc(m->eval_size);
    m->finalized = m->eval_buf != NULL;
    return m->finalized ? 0 : -1;
}

void rj_reset(rj_model *m) { m->n_past = 0; }

int rj_eval(rj_model *m, const int32_t *tokens, int n, float *logits_out) {
    const rj_params *p = &m->hp;
    if (!m->finalized || n < 1 || n > p->n_batch || m->n_past + n > p->n_ctx) return -1;
    const int n_embd = p->n_embd, n_head = p->n_head, n_rot = p->n_rot, ctx_size = p->n_ctx, session_len = m->n_past, hd = n_embd / n_head;
    const size_t ksz = ggml_element_size(m->memory_k), vsz = ggml_element_size(m->memory_v);

    if (m->ctx0) ggml_free(m->ctx0);
    struct ggml_init_params ip = { m->eval_size, m->eval_buf, false };
    m->ctx0 = ggml_init(ip);
    struct ggml_context *ctx0 = m->ctx0;

    struct ggml_tensor *embd = ggml_new_tensor_1d(ctx0, GGML_TYPE_I32, n);
    struct ggml_tensor *inpL = ggml_get_rows(ctx0, m->wte, embd);
    struct ggml_cgraph *gf = ggml_new_graph(ctx0);

    for (int il = 0; il < p->n_layer; il++) {
        const rj_layer *L = &m->layers[il];
        struct ggml_tensor *cur = ggml_add(ctx0, ggml_mul(ctx0, ggml_norm(ctx0, inpL), L->ln_1_g), L->ln_1_b);
        struct ggml_tensor *input_sa = cur;
        struct ggml_tensor *qcur = ggml_rope_inplace(ctx0, ggml_reshape_3d(ctx0, ggml_mul_mat(ctx0, L->wq, cur), hd, n_head, n), session_len, n_rot, 0, 0);
        struct ggml_tensor *kcur = ggml_rope_inplace(ctx0, ggml_reshape_3d(ctx0, ggml_mul_mat(ctx0, L->wk, cur), hd, n_head, n), session_len, n_rot, 0, 0);
        struct ggml_tensor *vcur = ggml_transpose(ctx0, ggml_mul_mat(ctx0, L->wv, cur));
        struct ggml_tensor *k = ggml_view_1d(ctx0, m->memory_k, (int64_t)n * n_embd, (ksz * n_embd) * ((size_t)il * ctx_size + session_len));
        struct ggml_tensor *v = ggml_view_2d(ctx0, m->memory_v, n, n_embd, (size_t)ctx_size * vsz,
                                             (size_t)il * ctx_size * vsz * n_embd + (size_t)session_len * vsz);
        ggml_build_forward_expand(gf, ggml_cpy(ctx0, kcur, k));
        ggml_build_forward_expand(gf, ggml_cpy(ctx0, vcur, v));
        struct ggml_tensor *q = ggml_permute(ctx0, qcur, 0, 2, 1, 3);
        struct ggml_tensor *big_k = ggml_permute(ctx0,
            ggml_reshape_3d(ctx0, ggml_view_1d(ctx0, m->memory_k, (int64_t)(session_len + n) * n_embd, (size_t)il * ctx_size * ksz * n_embd),
                            hd, n_head, session_len + n), 0, 2, 1, 3);
        struct ggml_tensor *kq = ggml_mul_mat(ctx0, big_k, q);
        struct ggml_tensor *kq_scaled = ggml_scale_inplace(ctx0, kq, ggml_new_f32(ctx0, 1.0f / sqrtf((float)n_embd / (float)n_head)));
        struct ggml_tensor *kq_masked = ggml_diag_mask_inf_inplace(ctx0, kq_scaled, session_len);
        struct ggml_tensor *kq_softmax = ggml_soft_max_inplace(ctx0, kq_masked);
        struct ggml_tensor *big_v = ggml_view_3d(ctx0, m->memory_v, session_len + n, hd, n_head, (size_t)ctx_size * vsz, (size_t)ctx_size * vsz * hd,
                                                 (size_t)il * ctx_size * vsz * n_embd);
        struct ggml_tensor *kqv = ggml_mul_mat(ctx0, big_v, kq_softmax);
        struct ggml_tensor *kqv_merged = ggml_permute(ctx0, kqv, 0, 2, 1, 3);
        cur = ggml_cpy(ctx0, kqv_merged, ggml_new_tensor_2d(ctx0, GGML_TYPE_F32, n_embd, n));
        cur = ggml_mul_mat(ctx0, L->wo, cur);
        struct ggml_tensor *ff_in = cur;
        cur = ggml_add(ctx0, ggml_mul_mat(ctx0, L->fc_in_w, input_sa), L->fc_in_b);
        cur = ggml_gelu(ctx0, cur);
        cur = ggml_add(ctx0, ggml_mul_mat(ctx0, L->fc_out_w, cur), L->fc_out_b);
        cur = ggml_add(ctx0, cur, ff_in);
        inpL = ggml_add(ctx0, cur, inpL);
    }
    inpL = ggml_add(ctx0, ggml_mul(ctx0, ggml_norm(ctx0, inpL), m->ln_f_g), m->ln_f_b);
    inpL = ggml_mul_mat(ctx0, m->lmh_g, inpL);
    inpL = ggml_add(ctx0, inpL, m->lmh_b);

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

/* memory_k (which = 0): [n_layer][n_ctx][n_embd]; memory_v (1): [n_layer][n_embd][n_ctx] (V transposed, gptj lib.rs:212-217); both f16 */
void *rj_kv(rj_model *m, int which, size_t *nbytes) {
    struct ggml_tensor *t = which ? m->memory_v : m->memory_k;
    if (nbytes) *nbytes = ggml_nbytes(t);
    return t->data;
}

void rj_free(rj_model *m) {
    if (!m) return;
    if (m->ctx0) ggml_free(m->ctx0);
    if (m->session_ctx) ggml_free(m->session_ctx);
    if (m->model_ctx) ggml_free(m->model_ctx);
    free(m->eval_buf);
    free(m);
}
