// llm_b200/csrc/ops.cu -- single-op entry points on host buffers (include/llm_b200.h: b200_op_*): one kernel family per call, for tests and
// kernel benchmarks
#include <string.h>

#include <vector>

#include "../../include/llm_b200.h"
#include "host.h"
#include "kernels.cuh"
#include "runtime.h"

using namespace b200;

namespace {

// The activation operand of the batched mat-mul implementations: the tensor-core GEMMs read f16 rows (EXACT_TC5 / EXACT_MMA with the Q8 block
// scales in xds), every other implementation reads Q8 blocks (xq, xds).
struct Acts { int8_t *xq; float2 *xds; __half *xh; };

void prepare(int32_t impl, int32_t wtype, const float *dx, int64_t K, int64_t B, const Acts &a, cudaStream_t st) {
    if (impl == B200_MM_FAST_TC5) cvt_act_f16(dx, K, a.xh, K, B, st);
    else if (impl == B200_MM_EXACT_TC5) quantize_act_f16_rm(vec_dot_type(wtype), dx, K, a.xh, a.xds, K, B, st);
    else if (impl == B200_MM_EXACT_MMA) quantize_act_f16(vec_dot_type(wtype), dx, K, a.xh, a.xds, K, B, st);
    else quantize_act(vec_dot_type(wtype), dx, K, a.xq, a.xds, K, B, st);
}

// FAST_TC5, EXACT_TC5, EXACT_MMA, or else the Q8 GEMM (mmq.cu)
void run(int32_t impl, const QWeight &w, const Acts &a, float *dd, int64_t N, int64_t B, cudaStream_t st) {
    if (impl == B200_MM_FAST_TC5) mul_mat_q_fast_tc5(w, a.xh, dd, N, B, nullptr, 0, st);
    else if (impl == B200_MM_EXACT_TC5) mul_mat_q_exact_tc5(w, a.xh, a.xds, dd, N, B, nullptr, 0, st);
    else if (impl == B200_MM_EXACT_MMA) mul_mat_q_exact_mma(w, a.xh, a.xds, dd, N, B, nullptr, 0, st);
    else mul_mat_q(w, a.xq, a.xds, dd, N, B, nullptr, 0, st);
}

// F16 weight rows: AUTO = the sessions' dispatch (exact_f16.cu), EXACT = exact.cu's mul_mat_f16_exact (the attention mat-mul kernel) on the same rows
void run_f16(int32_t impl, const QWeight &w, const float *dx, __half *xh, float *dd, int64_t B, cudaStream_t st) {
    if (impl == B200_MM_AUTO) mul_mat_exact_auto(w, dx, w.K, B, dd, w.N, nullptr, 0, {nullptr, nullptr, nullptr, xh}, st);
    else mul_mat_f16_exact((const __half *)w.qs, w.K, w.N, 1, w.K * 2, w.N * w.K * 2, dx, B, 1, w.K * 4, B * w.K * 4, dd, w.N * 4, B * w.N * 4, -1, st);
}

// B200_ERR_IO if a pipeline barrier of the wgmma kernel `impl` ever timed out (call after the stream is synchronized)
int check_timeout(int32_t impl) {
    if (impl == B200_MM_EXACT_TC5 && exact_tc5_check_timeout() != 0) return B200_ERR_IO;
    if (impl == B200_MM_FAST_TC5 && fast_tc5_check_timeout() != 0) return B200_ERR_IO;
    return B200_OK;
}

}  // namespace

extern "C" {

int b200_op_norm_device(int32_t op, const float *d_x, float *d_y, int64_t n, int64_t rows, float eps) {
    if ((op != 1 && op != 2) || !d_x || !d_y || n <= 0 || rows < 0 || rows > INT32_MAX) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init();
    if (op == 1) rms_norm(d_x, d_y, nullptr, n, rows, eps, R.stream);
    else layer_norm(d_x, d_y, nullptr, nullptr, n, rows, R.stream);
    return B200_OK;
}

int b200_op_quantize_act(int32_t vdt, const float *x, int64_t K, int64_t B, int8_t *qs_out, float *d_out, float *aux_out) {
    if (!x || K % QK || (vdt != T_Q8_0 && vdt != T_Q8_1)) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    const size_t nblk = (size_t)B * (K / QK);
    float *dx = (float *)R.op_arena.get((size_t)B * K * 4, st);
    int8_t *dq = (int8_t *)R.op_arena.get((size_t)B * K, st);
    float2 *dds = (float2 *)R.op_arena.get(nblk * sizeof(float2), st);
    B200_CHECK(cudaMemcpyAsync(dx, x, (size_t)B * K * 4, cudaMemcpyHostToDevice, st));
    quantize_act(vdt, dx, K, dq, dds, K, B, st);
    std::vector<float2> h(nblk);
    B200_CHECK(cudaMemcpyAsync(qs_out, dq, (size_t)B * K, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaMemcpyAsync(h.data(), dds, nblk * sizeof(float2), cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    for (size_t i = 0; i < nblk; i++) { if (d_out) d_out[i] = h[i].x; if (aux_out) aux_out[i] = h[i].y; }
    return B200_OK;
}

int b200_op_quantize_q8_K(const float *x, int64_t K, int64_t B, void *blocks_out) {      // quantize_row_q8_K of B rows -> B * K/256 block_q8_K (292 bytes each)
    if (!x || !blocks_out || K % 256) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    float *dx = (float *)R.op_arena.get((size_t)B * K * 4, st);
    void *xq = R.op_arena.get(q8k_bytes(K, B), st);
    B200_CHECK(cudaMemcpyAsync(dx, x, (size_t)B * K * 4, cudaMemcpyHostToDevice, st));
    quantize_act_q8k(dx, K, xq, K, B, st);
    B200_CHECK(cudaMemcpyAsync(blocks_out, xq, q8k_bytes(K, B), cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

int b200_op_mul_mat(int32_t wtype, const void *w_ggml, int64_t K, int64_t N, const float *x, int64_t B, float *dst, int32_t impl) {
    if (is_kquant(wtype)) {                              // Q2_K .. Q6_K: one exact kernel (kquants.cu); `impl` must be AUTO or EXACT
        if (!w_ggml || !x || !dst || K % 256 || (impl != B200_MM_AUTO && impl != B200_MM_EXACT)) return B200_ERR_BAD_ARG;
        Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
        cudaStream_t st = R.stream;
        const size_t raw_bytes = (size_t)N * (K / 256) * kquant_block_bytes(wtype);
        void *raw = R.op_arena.get(raw_bytes, st);
        float *dx = (float *)R.op_arena.get((size_t)B * K * 4, st);
        float *dd = (float *)R.op_arena.get((size_t)B * N * 4, st);
        void *xq = R.op_arena.get(q8k_bytes(K, B), st);
        B200_CHECK(cudaMemcpyAsync(raw, w_ggml, raw_bytes, cudaMemcpyHostToDevice, st));
        B200_CHECK(cudaMemcpyAsync(dx, x, (size_t)B * K * 4, cudaMemcpyHostToDevice, st));
        quantize_act_q8k(dx, K, xq, K, B, st);
        mul_mat_kq_exact(wtype, raw, xq, dd, N, K, N, B, nullptr, 0, st);
        B200_CHECK(cudaMemcpyAsync(dst, dd, (size_t)B * N * 4, cudaMemcpyDeviceToHost, st));
        B200_CHECK(cudaStreamSynchronize(st));
        return B200_OK;
    }
    if (wtype == T_F16) {                                // ggml_vec_dot_f16 order; `impl` must be AUTO or EXACT
        if (!w_ggml || !x || !dst || K % 64 || K < 64 || N < 1 || B < 1 || B > 65535 || (impl != B200_MM_AUTO && impl != B200_MM_EXACT)) return B200_ERR_BAD_ARG;
        Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
        cudaStream_t st = R.stream;
        QWeight w;
        qweight_layout(w, T_F16, K, N, R.op_arena.get(qweight_layout(w, T_F16, K, N, nullptr), st));
        float *dx = (float *)R.op_arena.get((size_t)B * K * 4, st);
        float *dd = (float *)R.op_arena.get((size_t)B * N * 4, st);
        __half *xh = (__half *)R.op_arena.get((size_t)B * K * 2, st);
        B200_CHECK(cudaMemcpyAsync((void *)w.qs, w_ggml, (size_t)N * K * 2, cudaMemcpyHostToDevice, st));
        B200_CHECK(cudaMemcpyAsync(dx, x, (size_t)B * K * 4, cudaMemcpyHostToDevice, st));
        run_f16(impl, w, dx, xh, dd, B, st);
        B200_CHECK(cudaMemcpyAsync(dst, dd, (size_t)B * N * 4, cudaMemcpyDeviceToHost, st));
        B200_CHECK(cudaStreamSynchronize(st));
        return B200_OK;
    }
    if (!is_quant(wtype) || !w_ggml || !x || !dst || K % 64) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    const size_t raw_bytes = (size_t)N * (K / QK) * ggml_block_bytes(wtype);
    void *raw = R.op_arena.get(raw_bytes, st);
    B200_CHECK(cudaMemcpyAsync(raw, w_ggml, raw_bytes, cudaMemcpyHostToDevice, st));
    QWeight w;
    const size_t pb = qweight_layout(w, wtype, K, N, nullptr);
    qweight_layout(w, wtype, K, N, R.op_arena.get(pb, st));
    repack_weights(w, raw, st);
    float *dx = (float *)R.op_arena.get((size_t)B * K * 4, st);
    float *dd = (float *)R.op_arena.get((size_t)B * N * 4, st);
    Acts a{};
    a.xq = (int8_t *)R.op_arena.get((size_t)B * K, st);
    a.xds = (float2 *)R.op_arena.get((size_t)B * (K / QK) * sizeof(float2), st);
    if (impl == B200_MM_EXACT_MMA) a.xh = (__half *)R.op_arena.get(xh_bytes(K, B), st);
    else if (impl == B200_MM_EXACT_TC5 || impl == B200_MM_FAST_TC5) a.xh = (__half *)R.op_arena.get((size_t)B * K * 2 + 16, st);
    else if (impl == B200_MM_AUTO) a.xh = (__half *)R.op_arena.get(xh_bytes(K, B) + 16, st);       // the larger of the two above
    B200_CHECK(cudaMemcpyAsync(dx, x, (size_t)B * K * 4, cudaMemcpyHostToDevice, st));
    if (impl != B200_MM_AUTO) prepare(impl, wtype, dx, K, B, a, st);
    if (impl == B200_MM_AUTO) {                          // the exact dispatch of the sessions and the seam (mul_mat.cu): the kernel follows from B and K
        int4 *pack = (int4 *)R.op_arena.get((size_t)(K / QK) * 64, st);
        mul_mat_exact_auto(w, dx, K, B, dd, N, nullptr, 0, {a.xq, a.xds, pack, a.xh}, st);
        B200_CHECK(cudaStreamSynchronize(st));
        if (const int rc = check_timeout(B200_MM_EXACT_TC5)) return rc;
    } else if (impl == B200_MM_EXACT_STREAM) {
        if (!mmv_exact_stream_supported(w)) return B200_ERR_BAD_ARG;
        int4 *pack = (int4 *)R.op_arena.get((size_t)(K / QK) * 64, st);
        for (int64_t b = 0; b < B; b++) { quantize_act_pack(wtype, dx + b * K, pack, K, st); mul_mat_vec_q_exact_stream(w, pack, dd + b * N, nullptr, st); }
    } else if (impl == B200_MM_EXACT) mul_mat_q_exact(w, a.xq, a.xds, dd, N, B, nullptr, 0, st);
    else if (impl == B200_MM_VEC) { for (int64_t b = 0; b < B; b++) mul_mat_vec_q(w, a.xq + b * K, a.xds + b * (K / QK), dd + b * N, nullptr, st); }
    else if (impl == B200_MM_SIMPLE) mul_mat_q_simple(w, a.xq, a.xds, dd, N, B, nullptr, 0, st);
    else {
        run(impl, w, a, dd, N, B, st);
        B200_CHECK(cudaStreamSynchronize(st));
        if (const int rc = check_timeout(impl)) return rc;
    }
    B200_CHECK(cudaMemcpyAsync(dst, dd, (size_t)B * N * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

// the sessions' KQ / KQV (exact.cu: mul_mat_f16_exact / mul_mat_f32_exact) on host buffers with ggml_mul_mat's shapes and byte strides.  dst is
// uploaded too, so the outputs the causal skip leaves alone come back as the caller's values.
int b200_op_mul_mat_kv(int32_t src0_type, const void *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                       const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12, float *dst, int64_t nbd1, int64_t nbd2, int32_t causal_past) {
    const int64_t es = src0_type == T_F16 ? 2 : 4;
    if ((src0_type != T_F16 && src0_type != T_F32) || !src0 || !src1 || !dst || ne00 < 1 || ne01 < 1 || ne02 < 1 || ne11 < 1 || ne12 < 1 ||
        ne12 % ne02 || ne11 > 65535 || ne12 > 65535 || nb01 < ne00 * es || nb02 < 0 || nb11 < ne00 * 4 || nb12 < 0 || nbd1 < ne01 * 4 || nbd2 < 0 ||
        nb01 % es || nb02 % es || nb11 % 4 || nb12 % 4 || nbd1 % 4 || nbd2 % 4)
        return B200_ERR_BAD_ARG;
    const size_t b0 = (size_t)((ne02 - 1) * nb02 + (ne01 - 1) * nb01 + ne00 * es);          // one past the last byte each operand touches
    const size_t b1 = (size_t)((ne12 - 1) * nb12 + (ne11 - 1) * nb11 + ne00 * 4);
    const size_t bd = (size_t)((ne12 - 1) * nbd2 + (ne11 - 1) * nbd1 + ne01 * 4);
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    void *d0 = R.op_arena.get(b0, st);
    float *d1 = (float *)R.op_arena.get(b1, st), *dd = (float *)R.op_arena.get(bd, st);
    B200_CHECK(cudaMemcpyAsync(d0, src0, b0, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(d1, src1, b1, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(dd, dst, bd, cudaMemcpyHostToDevice, st));
    if (src0_type == T_F16) mul_mat_f16_exact((const __half *)d0, ne00, ne01, ne02, nb01, nb02, d1, ne11, ne12, nb11, nb12, dd, nbd1, nbd2, causal_past, st);
    else mul_mat_f32_exact((const float *)d0, ne00, ne01, ne02, nb01, nb02, d1, ne11, ne12, nb11, nb12, dd, nbd1, nbd2, causal_past, st);
    B200_CHECK(cudaMemcpyAsync(dst, dd, bd, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

// ggml_quantize_q{4_0,4_1,5_0,5_1,8_0} on the GPU (crates/llm-base/src/quantize.rs:320-414 calls them per tensor): f32 rows in, GGML blocks out,
// through the kernel of b200_quantize_file
int b200_op_quantize_weights(int32_t wtype, const float *w_host, int64_t K, int64_t N, void *ggml_blocks_out) {
    if (!is_quant(wtype) || !w_host || !ggml_blocks_out || K % QK) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    float *dw = (float *)R.op_arena.get((size_t)N * K * 4, st);
    B200_CHECK(cudaMemcpyAsync(dw, w_host, (size_t)N * K * 4, cudaMemcpyHostToDevice, st));
    const size_t raw_bytes = (size_t)N * (K / QK) * ggml_block_bytes(wtype);
    void *raw = R.op_arena.get(raw_bytes, st);
    quantize_blocks(wtype, T_F32, dw, N * (K / QK), raw, nullptr, st);
    B200_CHECK(cudaMemcpyAsync(ggml_blocks_out, raw, raw_bytes, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

// the same kernel on device buffers, enqueued on the backend's stream without a sync (kernel timing with b200_timing_begin / end_ms)
int b200_op_quantize_blocks_device(int32_t target, int32_t src_type, const void *d_src, int64_t nblk, void *d_dst, void *d_hist) {
    if (!is_quant(target) || (src_type != T_F32 && src_type != T_F16) || !d_src || !d_dst || nblk < 0 || ((uintptr_t)d_dst & 15)) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init();
    quantize_blocks(target, src_type, d_src, nblk, d_dst, (unsigned long long *)d_hist, R.stream);
    return B200_OK;
}

// LoraAdapter::patch of one adapter on host buffers: w (N rows of K, GGML layout) += scaling * (A [r, K] x B [r, N])
int b200_op_lora_patch(int32_t wtype, void *w_ggml_inout, int64_t K, int64_t N, int32_t a_type, const void *a, const float *b, int64_t r, float scaling) {
    if (!w_ggml_inout || !a || !b || K < 1 || N < 1 || r < 0) return B200_ERR_BAD_ARG;
    const int rc = lora_check(wtype, K, N, a_type, r, K, T_F32, r, N);
    if (rc != B200_OK) return rc;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    const size_t wb = (size_t)N * (wtype == T_F32 ? (size_t)K * 4 : wtype == T_F16 ? (size_t)K * 2 : (size_t)(K / QK) * ggml_block_bytes(wtype));
    const size_t ab = (size_t)K * r * (a_type == T_F16 ? 2 : 4), bb = (size_t)N * r * 4;
    void *dw = R.op_arena.get(wb, st), *da = R.op_arena.get(ab ? ab : 1, st);
    float *db = (float *)R.op_arena.get(bb ? bb : 4, st);
    B200_CHECK(cudaMemcpyAsync(dw, w_ggml_inout, wb, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(da, a, ab, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(db, b, bb, cudaMemcpyHostToDevice, st));
    lora_patch(wtype, dw, K, N, a_type, da, db, r, N, scaling, st);
    B200_CHECK(cudaMemcpyAsync(w_ggml_inout, dw, wb, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

int b200_op_nll_rows(const float *logits, int64_t rows, int64_t n_vocab, const int32_t *targets, float *terms_out) {
    if (!logits || !targets || !terms_out || rows < 1 || rows > INT32_MAX || n_vocab < 1) return B200_ERR_BAD_ARG;
    for (int64_t r = 0; r < rows; r++) if (targets[r] < 0 || targets[r] >= n_vocab) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    float *dl = (float *)R.op_arena.get((size_t)rows * n_vocab * 4, st), *dt = (float *)R.op_arena.get((size_t)rows * 4, st);
    int32_t *dtg = (int32_t *)R.op_arena.get((size_t)rows * 4, st);
    B200_CHECK(cudaMemcpyAsync(dl, logits, (size_t)rows * n_vocab * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(dtg, targets, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    nll_rows(dl, rows, n_vocab, dtg, dt, st);
    B200_CHECK(cudaMemcpyAsync(terms_out, dt, (size_t)rows * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

int b200_op_sample(const float *logits, int64_t n_vocab, const int32_t *history, int32_t n_past, const b200_sampler *sampler, int32_t *id_out,
                   int32_t *n_kept_out, int32_t *cand_ids_out, float *cand_probs_out) {
    SampleArgs a;
    if (!logits || !id_out || n_vocab < 1 || n_vocab > INT32_MAX / 2 || n_past < 0 || (n_past > 0 && !history) || !sampler_args(sampler, a)) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    const int V = (int)n_vocab, kk = a.top_k < V ? (a.top_k < 1024 ? a.top_k : 1024) : (V < 1024 ? V : 1024);
    float *dl = (float *)R.op_arena.get((size_t)V * 4, st);
    int32_t *dh = (int32_t *)R.op_arena.get((size_t)(n_past > 0 ? n_past : 1) * 4, st);
    int32_t *dids = (int32_t *)R.op_arena.get((size_t)kk * 4, st);
    float *dprobs = (float *)R.op_arena.get((size_t)kk * 4, st);
    SampleResult *dres = (SampleResult *)R.op_arena.get(sizeof(SampleResult), st);
    SampleBufs b{{(uint64_t *)R.op_arena.get(sample_key_bytes(V), st), (uint64_t *)R.op_arena.get(sample_key_bytes(V), st)},
                 (int *)R.op_arena.get(sizeof(int), st), nullptr};
    B200_CHECK(cudaMemcpyAsync(dl, logits, (size_t)V * 4, cudaMemcpyHostToDevice, st));
    if (n_past > 0) B200_CHECK(cudaMemcpyAsync(dh, history, (size_t)n_past * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemsetAsync(b.fail, 0, sizeof(int), st));
    sample_row(dl, V, dh, n_past, a, b, nullptr, nullptr, dres, dids, nullptr, dprobs, st);
    SampleResult r;
    std::vector<int32_t> ids(kk);
    std::vector<float> probs(kk);
    B200_CHECK(cudaMemcpyAsync(&r, dres, sizeof(r), cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaMemcpyAsync(ids.data(), dids, (size_t)kk * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaMemcpyAsync(probs.data(), dprobs, (size_t)kk * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    if (r.status != 0) return B200_ERR_SAMPLER_FAILURE;
    *id_out = r.id;
    if (n_kept_out) *n_kept_out = r.n_kept;
    if (cand_ids_out) memcpy(cand_ids_out, ids.data(), (size_t)kk * 4);
    if (cand_probs_out) memcpy(cand_probs_out, probs.data(), (size_t)kk * 4);
    return B200_OK;
}

// Kernel-only timing of one weight mat-mul on device-resident synthetic operands (seeded random weights and activations): used by
// tools/prefill_gemm_bench.py and bench.py's prefill roofline; impl = B200_MM_EXACT_MMA / B200_MM_EXACT_TC5 / B200_MM_TENSOR
int b200_op_bench_mul_mat(int32_t wtype, int64_t K, int64_t N, int64_t B, int32_t impl, int32_t iters, float *ms_out) {
    if (!is_qweight_type(wtype) || K % 64 || !ms_out || iters < 1) return B200_ERR_BAD_ARG;
    if (wtype == T_F16 && ((impl != B200_MM_AUTO && impl != B200_MM_EXACT) || B < 1 || B > 65535)) return B200_ERR_BAD_ARG;
    Runtime &R = rt(); R.ensure_init(); R.op_arena.reset();
    cudaStream_t st = R.stream;
    QWeight w;
    const size_t pb = qweight_layout(w, wtype, K, N, nullptr);
    void *base = R.op_arena.get(pb, st);
    qweight_layout(w, wtype, K, N, base);
    synth_qweight(w, 777u, st);
    float *dx = (float *)R.op_arena.get((size_t)B * K * 4, st);
    float *dd = (float *)R.op_arena.get((size_t)B * N * 4, st);
    if (wtype == T_F16) {                                // the whole mat-mul as a session runs it: the activation rounding included
        __half *xh = (__half *)R.op_arena.get((size_t)B * K * 2, st);
        synth_gain(dx, B * K, 12345u, st);
        for (int i = 0; i < 2; i++) run_f16(impl, w, dx, xh, dd, B, st);
        cudaEvent_t e0, e1;
        B200_CHECK(cudaEventCreate(&e0)); B200_CHECK(cudaEventCreate(&e1));
        B200_CHECK(cudaEventRecord(e0, st));
        for (int i = 0; i < iters; i++) run_f16(impl, w, dx, xh, dd, B, st);
        B200_CHECK(cudaEventRecord(e1, st));
        B200_CHECK(cudaEventSynchronize(e1));
        float ms = 0.f;
        B200_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        *ms_out = ms / iters;
        B200_CHECK(cudaEventDestroy(e0)); B200_CHECK(cudaEventDestroy(e1));
        return B200_OK;
    }
    Acts a;
    a.xds = (float2 *)R.op_arena.get((size_t)B * (K / QK) * sizeof(float2), st);
    a.xh = (__half *)R.op_arena.get(xh_bytes(K, B) + 16, st);
    a.xq = (int8_t *)R.op_arena.get((size_t)B * K, st);
    synth_gain(dx, B * K, 12345u, st);
    prepare(impl, wtype, dx, K, B, a, st);
    for (int i = 0; i < 2; i++) run(impl, w, a, dd, N, B, st);
    cudaEvent_t e0, e1;
    B200_CHECK(cudaEventCreate(&e0)); B200_CHECK(cudaEventCreate(&e1));
    B200_CHECK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; i++) run(impl, w, a, dd, N, B, st);
    B200_CHECK(cudaEventRecord(e1, st));
    B200_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    B200_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    *ms_out = ms / iters;
    B200_CHECK(cudaEventDestroy(e0)); B200_CHECK(cudaEventDestroy(e1));
    return check_timeout(impl);
}

}  // extern "C"
