/*
 * oracle/ref_lora.c -- TEST INFRASTRUCTURE (see ref_harness.c): the reference's LoRA patch driven through the UNMODIFIED ggml C API.
 *
 * Restates LoraAdapter::patch (crates/llm-base/src/lora.rs:71-140) for one adapter and one target tensor W [ne0 = K, ne1 = N]:
 *   ba = ggml_mul_mat(A [r, K], B [r, NB])          f32 [K, NB]
 *   ba = ggml_scale(ba, scaling)                     only when scaling != 1
 *   W  = ggml_add(W, ba)                             add_q_f32 for the block types, add_f32 (rows of ba repeated) for F32
 *   computed with 8 threads (GraphExecutionPlan::new(&mut gf, 8)), the result copied over W.
 */
#include "ggml.h"

#include <stdlib.h>
#include <string.h>

static size_t rl_bytes(enum ggml_type t, int64_t ne0, int64_t ne1) { return (size_t)(ne0 / ggml_blck_size(t)) * ggml_type_size(t) * (size_t)ne1; }

/* w_inout: N rows of the target in GGML layout; a: K rows of r elements (F32 or F16); b: NB rows of r floats.  Returns 0, or -1 if ggml_init fails. */
int rl_patch(int32_t wtype, void *w_inout, int64_t K, int64_t N, int32_t a_type, const void *a, const float *b, int64_t r, int64_t nb_rows, float scaling,
             int32_t n_threads) {
    const enum ggml_type wt = (enum ggml_type)wtype, at = (enum ggml_type)a_type;
    const size_t wbytes = rl_bytes(wt, K, N), abytes = rl_bytes(at, r, K), bbytes = rl_bytes(GGML_TYPE_F32, r, nb_rows);
    const size_t ctx_bytes = wbytes * 2 + abytes + bbytes + (size_t)K * nb_rows * 4 * 2 + (1u << 20);   /* + the graph and the tensor headers */
    struct ggml_init_params ip = { ctx_bytes, NULL, false };
    struct ggml_context *ctx = ggml_init(ip);
    if (!ctx) return -1;
    struct ggml_tensor *w = ggml_new_tensor_2d(ctx, wt, K, N);
    struct ggml_tensor *ta = ggml_new_tensor_2d(ctx, at, r, K);
    struct ggml_tensor *tb = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, r, nb_rows);
    memcpy(w->data, w_inout, wbytes);
    memcpy(ta->data, a, abytes);
    memcpy(tb->data, b, bbytes);

    struct ggml_cgraph *gf = ggml_new_graph(ctx);
    struct ggml_tensor *ba = ggml_mul_mat(ctx, ta, tb);
    if (scaling != 1.0f) ba = ggml_scale(ctx, ba, ggml_new_f32(ctx, scaling));
    struct ggml_tensor *out = ggml_add(ctx, w, ba);
    ggml_build_forward_expand(gf, out);
    struct ggml_cplan plan = ggml_graph_plan(gf, n_threads);
    void *work = malloc(plan.work_size ? plan.work_size : 1);
    plan.work_data = work;
    ggml_graph_compute(gf, &plan);
    memcpy(w_inout, out->data, wbytes);
    free(work);
    ggml_free(ctx);
    return 0;
}
