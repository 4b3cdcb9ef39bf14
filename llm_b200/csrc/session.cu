// llm_b200/csrc/session.cu -- native host runtime (include/llm_b200.h): Llama model + InferenceSession on the GPU.
//
// Mirrors, in C++ over the kernels of this directory, what the reference does in Rust over ggml:
//   Llama::new / TensorLoader          crates/models/llama/src/lib.rs:43-140
//   InferenceSession::new / compute    crates/llm-base/src/inference_session.rs:114-295
//   Llama::evaluate (the graph)        crates/models/llama/src/lib.rs:144-368
// The forward pass below is that graph, node for node in arithmetic, but scheduled statically: no per-eval graph
// construction, no arena reset, weights resident in HBM in the planes layout, wq|wk|wv and w1|w3 stored as single matrices
// so one activation quantization and one mat-mul launch serve them.
#include <string.h>

#include <string>
#include <vector>

#include "../../include/llm_b200.h"
#include "host.h"

using namespace b200;

namespace {

struct Layer {
    float *attention_norm = nullptr, *ffn_norm = nullptr;
    QWeight wqkv, wo, w13, w2;          // wqkv rows: [wq | wk | wv]; w13 rows: [w1 | w3]
    QWeight wv;                         // wv of a type other than wq's: then wqkv rows are [wq | wk] and wv is this matrix (wv.N == 0 otherwise)
};

}  // namespace

struct b200_model : Weights {
    b200_llama_hparams hp;
    int gqa = 0, hd = 0;
    // tensor parallelism (b200_llama_new_tp): this rank holds 1/tp_world of the ROWS of every weight matrix (tp.cuh); *_loc = local row counts
    int tp_rank = 0, tp_world = 1;
    int e_loc = 0, gqa_loc = 0, f_loc = 0, v_loc = 0;
    QWeight wte, output;
    float *norm = nullptr;
    std::vector<Layer> layers;
    bool any_kquant = false, any_f16 = false;       // some 2-D weight is a K-quant / F16
    bool uniform_layers = true;                     // every layer matrix is of hp.wtype (the layout and decode graph of a one-type file)

    bool lookup(const char *name, Slot &s, int &slot_id);
    int n_slots() const { return 3 + 9 * hp.n_layer; }
};

struct b200_session : SessionCore {     // memory_k [n_layer][n_ctx][gqa], memory_v [n_layer][gqa][n_ctx] (V transposed)
    b200_model *m = nullptr;
    b200_session_config cfg;
    // activations (sized for n_batch rows)
    DeviceBuf<float> x, cur, ff, qkv, kq, h13, hmul, logits;
    DeviceBuf<int8_t> xq; DeviceBuf<float2> xds; DeviceBuf<int4> xpack; DeviceBuf<__half> xh;
    DeviceBuf<char> xq8k;               // Q8_K activations of K-quant weights (models with one)
    // the graph decode schedule (decode_ops.cu)
    DeviceBuf<unsigned long long> d_prof;
    DeviceBuf<float> qbuf; DeviceBuf<int4> xpack_d, xpack_f;
    bool graph_ok = false;                             // the session's geometry decodes through the graph schedule
    std::vector<DecodeLayer> h_layers;                 // the layer table (kernel arguments of the decode graph)
    DeviceBuf<int4> xpack_a;
    DecodeParams dp;
    // debug taps (tests): copy one intermediate buffer of (layer, stage) aside during forward()
    int tap_layer = -2, tap_stage = 0;
    DeviceBuf<float> tap; size_t tap_cap = 0, tap_count = 0;
    // tensor parallelism: the exchange slab (x | ff | records | logits | flags), [epoch, timeouts, CTA-arrival counters], peers' slabs mapped through CUDA IPC
    DeviceBuf<char> tp_slab; size_t tp_slab_bytes = 0; DeviceBuf<unsigned> tp_state;
    void *tp_peer_map[TP_MAX] = {};
    bool tp_connected = false;
};

bool b200_model::lookup(const char *name, Slot &s, int &slot_id) {
    const int e = hp.n_embd;
    const int eq = e_loc, f = f_loc;          // local row counts (== n_embd, n_ff on a single GPU)
    const int gqa = gqa_loc;
    s = Slot();
    if (!strcmp(name, "tok_embeddings.weight")) { s.q = wte; s.is_q = true; slot_id = 0; return true; }
    if (!strcmp(name, "norm.weight")) { s.f = norm; s.n = e; slot_id = 1; return true; }
    if (!strcmp(name, "output.weight")) { s.q = output; s.is_q = true; slot_id = 2; return true; }
    int il = -1; char sub[64];
    if (sscanf(name, "layers.%d.%63s", &il, sub) != 2 || il < 0 || il >= hp.n_layer) return false;
    Layer &L = layers[il];
    const int base = 3 + 9 * il;
    if (!strcmp(sub, "attention_norm.weight")) { s.f = L.attention_norm; s.n = e; slot_id = base + 0; return true; }
    if (!strcmp(sub, "ffn_norm.weight"))       { s.f = L.ffn_norm; s.n = e; slot_id = base + 1; return true; }
    s.is_q = true;
    if (!strcmp(sub, "attention.wq.weight")) { s.q = row_view(L.wqkv, 0, eq); slot_id = base + 2; return true; }
    if (!strcmp(sub, "attention.wk.weight")) { s.q = row_view(L.wqkv, eq, gqa); slot_id = base + 3; return true; }
    if (!strcmp(sub, "attention.wv.weight")) { s.q = L.wv.N ? L.wv : row_view(L.wqkv, eq + gqa, gqa); slot_id = base + 4; return true; }
    if (!strcmp(sub, "attention.wo.weight")) { s.q = L.wo; slot_id = base + 5; return true; }
    if (!strcmp(sub, "feed_forward.w1.weight")) { s.q = L.w13; s.chunk = 32; s.row0 = 0;  s.stride = 64; s.rows = f; slot_id = base + 6; return true; }
    if (!strcmp(sub, "feed_forward.w3.weight")) { s.q = L.w13; s.chunk = 32; s.row0 = 32; s.stride = 64; s.rows = f; slot_id = base + 7; return true; }
    if (!strcmp(sub, "feed_forward.w2.weight")) { s.q = L.w2; slot_id = base + 8; return true; }
    return false;
}

// the 2-D weights a LLaMA model holds: tok_embeddings, output, and layers.<il>.{attention.w[qkvo], feed_forward.w[123]}.weight
bool b200::llama_matrix_name(const char *name, int n_layer) {
    if (!strcmp(name, "tok_embeddings.weight") || !strcmp(name, "output.weight")) return true;
    int il = -1, used = 0; char sub[64];
    if (sscanf(name, "layers.%d.%63s%n", &il, sub, &used) != 2 || il < 0 || il >= n_layer || name[used]) return false;
    static const char *const mats[] = {"attention.wq.weight", "attention.wk.weight", "attention.wv.weight", "attention.wo.weight",
                                       "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight"};
    for (const char *m : mats) if (!strcmp(sub, m)) return true;
    return false;
}

namespace {

}  // namespace
void silu_mul_rows(const float *h13, float *out, int64_t f, int64_t n, cudaStream_t st);

namespace {

// ---- the forward pass (crates/models/llama/src/lib.rs:166-362) ---------------------------------------------------------------
// ggml_mul_mat(w, x): quantize the f32 activation rows (the INIT phase of ggml_compute_forward_mul_mat) and multiply; returns the launches
int matmul(b200_session *s, const QWeight &w, const float *x, float *dst, int64_t ldd, int64_t B, const float *addend, int64_t lda,
           cudaStream_t st, bool fast) {
    if (!fast || is_kquant(w.type))      // the order-free kernels take the five block formats: K-quants run their exact kernels in FAST sessions too
        return mul_mat_exact_auto(w, x, w.K, B, dst, ldd, addend, lda, {s->xq.get(), s->xds.get(), s->xpack.get(), s->xh.get(), s->xq8k.get()}, st);
    quantize_act(vec_dot_type(w.type), x, w.K, s->xq.get(), s->xds.get(), w.K, B, st);
    if (B == 1)      mul_mat_vec_q(w, s->xq.get(), s->xds.get(), dst, addend, st);
    else if (B < 16) mul_mat_q_simple(w, s->xq.get(), s->xds.get(), dst, ldd, B, addend, lda, st);
    else if (prefill_gemm_tc5() && B >= 64) { cvt_act_f16(x, w.K, s->xh.get(), w.K, B, st); mul_mat_q_fast_tc5(w, s->xh.get(), dst, ldd, B, addend, lda, st); }   // fused dequant -> wgmma GEMM
    else             mul_mat_q(w, s->xq.get(), s->xds.get(), dst, ldd, B, addend, lda, st);
    return 2;
}

// all_rows == false: only the last row goes through the final norm and the lm_head (OutputRequest without all_logits reads nothing else:
// model/common.rs:6-39); rows are independent, so that row is bit-identical to the all-rows pass.
void forward(b200_session *s, int n, bool all_rows = true) {
    b200_model *m = s->m;
    const b200_llama_hparams &hp = m->hp;
    cudaStream_t st = rt().stream;
    const int e = hp.n_embd, f = hp.n_ff, hd = m->hd, gqa = m->gqa, n_head = hp.n_head, n_head_kv = hp.n_head_kv;
    const int n_ctx = hp.context_size, n_past = s->n_past, n_kv = n_past + n;
    const int qkv_ld = e + 2 * gqa;
    const float kq_scale = 1.0f / sqrtf((float)e / (float)n_head);                           // llama lib.rs:268-270
    const RopeTable &rope = rope_table(hp.n_rot, 0, hp.rope_freq_base, hp.rope_freq_scale, hd, n_ctx);
    int L = 0;
    const bool tp = m->tp_world > 1;
    const bool fast = !tp && (s->cfg.flags & B200_SESSION_FAST) != 0;
    const bool kv32 = s->kv_type == T_F32;                                                   // InferenceSessionConfig::memory_k_type / memory_v_type
    const int64_t ke = (int64_t)s->kv_elem_bytes();
    if (tp && (n != 1 || !s->tp_connected)) { fprintf(stderr, "llm_b200: tensor-parallel sessions decode one token per step, after b200_session_tp_connect\n"); exit(1); }
    if (n == 1 && s->graph_ok && !fast && (tp || (!(s->cfg.flags & B200_SESSION_UNFUSED) && s->tap_layer == -2))) {
        // 7 fused kernels per layer, replayed from one CUDA graph per token (decode_ops.cu)
        s->last_launches = s->decode.run(n_kv, n_ctx, !(s->cfg.flags & B200_SESSION_NO_GRAPH), [s, &hp](int bucket, cudaStream_t st, int *nodes) {
            decode_ops_enqueue(s->dp, s->h_layers, hp.wtype, bucket, s->xpack_a.get(), st, nodes);
        }, st);
        s->last_n = 1; s->n_past += 1;
        return;
    }
    int il = -1;
    auto TAP = [&](int stage, const float *buf, size_t count) {
        if (s->tap_layer != il || s->tap_stage != stage) return;
        if (count > s->tap_cap) { s->tap.reset(); s->tap = device_alloc<float>(count * 4); s->tap_cap = count; }
        B200_CHECK(cudaMemcpyAsync(s->tap.get(), buf, count * 4, cudaMemcpyDeviceToDevice, st));
        s->tap_count = count;
    };

    get_rows_q(m->wte, s->d_tokens.get(), s->x.get(), n, st); L++;                                      // :170
    for (il = 0; il < hp.n_layer; il++) {
        const Layer &ly = m->layers[il];
        void *Kl = s->kv_at(0, (size_t)il * n_ctx * gqa);                                          // :227-231
        void *Vl = s->kv_at(1, (size_t)il * n_ctx * gqa);                                          // :233-239
        rms_norm(s->x.get(), s->cur.get(), ly.attention_norm, e, n, 5e-6f, st); L++;                    // :183,186
        TAP(1, s->cur.get(), (size_t)n * e);
        L += matmul(s, ly.wqkv, s->cur.get(), s->qkv.get(), qkv_ld, n, nullptr, 0, st, fast);                // :194,208,223
        if (ly.wv.N) L += matmul(s, ly.wv, s->cur.get(), s->qkv.get() + e + gqa, qkv_ld, n, nullptr, 0, st, fast);   // wv of its own type, into the same rows
        TAP(2, s->qkv.get(), (size_t)n * qkv_ld);
        // RoPE on Q and K heads in place: [hd, n_head + n_head_kv, n] with row stride qkv_ld    :190-217
        rope_f32(s->qkv.get(), s->qkv.get(), hd, n_head + n_head_kv, n, hd, qkv_ld, hd, qkv_ld, n_past, rope, st); L++;
        TAP(3, s->qkv.get(), (size_t)n * qkv_ld);
        {   // store K (row per position) and V (transposed) into the cache (f16, or f32 as it is)   :243-244
            StridedDesc sk{{gqa, n, 1, 1}, {4, (int64_t)qkv_ld * 4, 0, 0}}, dk{{gqa, n, 1, 1}, {ke, (int64_t)gqa * ke, 0, 0}};
            cpy_strided(s->qkv.get() + e, T_F32, sk, (char *)Kl + (size_t)n_past * gqa * ke, s->kv_type, dk, st); L++;
            StridedDesc sv{{n, gqa, 1, 1}, {(int64_t)qkv_ld * 4, 4, 0, 0}}, dv{{n, gqa, 1, 1}, {ke, (int64_t)n_ctx * ke, 0, 0}};
            cpy_strided(s->qkv.get() + e + gqa, T_F32, sv, (char *)Vl + (size_t)n_past * ke, s->kv_type, dv, st); L++;
        }
        // KQ[h][i][j] = K[j][h] . f16(Q[i][h])  (f32 cache: K[j][h] . Q[i][h], also in FAST sessions)        :246-265
        if (kv32) mul_mat_f32_exact((const float *)Kl, hd, n_kv, n_head_kv, (int64_t)gqa * 4, (int64_t)hd * 4,
                                    s->qkv.get(), n, n_head, (int64_t)qkv_ld * 4, (int64_t)hd * 4,
                                    s->kq.get(), (int64_t)n_kv * 4, (int64_t)n_kv * n * 4, n_past, st);
        else if (fast) mul_mat_f16((const __half *)Kl, hd, n_kv, n_head_kv, (int64_t)gqa * 2, (int64_t)hd * 2,
                                   s->qkv.get(), n, n_head, (int64_t)qkv_ld * 4, (int64_t)hd * 4,
                                   s->kq.get(), (int64_t)n_kv * 4, (int64_t)n_kv * n * 4, st);
        else mul_mat_f16_exact((const __half *)Kl, hd, n_kv, n_head_kv, (int64_t)gqa * 2, (int64_t)hd * 2,
                               s->qkv.get(), n, n_head, (int64_t)qkv_ld * 4, (int64_t)hd * 4,
                               s->kq.get(), (int64_t)n_kv * 4, (int64_t)n_kv * n * 4, n_past, st);
        L++;
        TAP(4, s->kq.get(), (size_t)n_head * n * n_kv);
        soft_max(s->kq.get(), s->kq.get(), n_kv, (int64_t)n_head * n, n, kq_scale, true, n_past, true, true, st); L++;   // :268-281
        TAP(5, s->kq.get(), (size_t)n_head * n * n_kv);
        // KQV[h][i][c] = V[h][c][:] . f16(P[h][i][:]) (f32 cache: . P[h][i][:]) written straight into the merged [n][e] layout     :284-307
        if (kv32) mul_mat_f32_exact((const float *)Vl, n_kv, hd, n_head_kv, (int64_t)n_ctx * 4, (int64_t)n_ctx * hd * 4,
                                    s->kq.get(), n, n_head, (int64_t)n_kv * 4, (int64_t)n_kv * n * 4,
                                    s->cur.get(), (int64_t)e * 4, (int64_t)hd * 4, -1, st);
        else if (fast) mul_mat_f16((const __half *)Vl, n_kv, hd, n_head_kv, (int64_t)n_ctx * 2, (int64_t)n_ctx * hd * 2,
                                   s->kq.get(), n, n_head, (int64_t)n_kv * 4, (int64_t)n_kv * n * 4,
                                   s->cur.get(), (int64_t)e * 4, (int64_t)hd * 4, st);
        else mul_mat_f16_exact((const __half *)Vl, n_kv, hd, n_head_kv, (int64_t)n_ctx * 2, (int64_t)n_ctx * hd * 2,
                               s->kq.get(), n, n_head, (int64_t)n_kv * 4, (int64_t)n_kv * n * 4,
                               s->cur.get(), (int64_t)e * 4, (int64_t)hd * 4, -1, st);
        L++;
        TAP(6, s->cur.get(), (size_t)n * e);
        L += matmul(s, ly.wo, s->cur.get(), s->ff.get(), e, n, s->x.get(), e, st, fast);                           // :310,314  (inpFF = wo.cur + inpSA)
        TAP(7, s->ff.get(), (size_t)n * e);
        rms_norm(s->ff.get(), s->cur.get(), ly.ffn_norm, e, n, 5e-6f, st); L++;                         // :318,321
        TAP(8, s->cur.get(), (size_t)n * e);
        L += matmul(s, ly.w13, s->cur.get(), s->h13.get(), 2 * f, n, nullptr, 0, st, fast);                  // :323,325
        TAP(9, s->h13.get(), (size_t)n * 2 * f);
        silu_mul_rows(s->h13.get(), s->hmul.get(), f, n, st); L++;                                      // :328,330  silu(w1 x) * (w3 x)
        TAP(10, s->hmul.get(), (size_t)n * f);
        L += matmul(s, ly.w2, s->hmul.get(), s->x.get(), e, n, s->ff.get(), e, st, fast);                          // :332,334
        TAP(11, s->x.get(), (size_t)n * e);
    }
    il = -1;
    if (all_rows || n == 1 || s->tap_layer != -2) {
        rms_norm(s->x.get(), s->cur.get(), m->norm, e, n, 5e-6f, st); L++;                              // :343,346
        L += matmul(s, m->output, s->cur.get(), s->logits.get(), hp.n_vocab, n, nullptr, 0, st, fast);       // :352
    } else {
        const size_t last = (size_t)(n - 1);
        rms_norm(s->x.get() + last * e, s->cur.get() + last * e, m->norm, e, 1, 5e-6f, st); L++;
        L += matmul(s, m->output, s->cur.get() + last * e, s->logits.get() + last * hp.n_vocab, hp.n_vocab, 1, nullptr, 0, st, fast);
    }
    s->last_launches = L;
    s->last_n = n;
    s->n_past += n;                                                                           // inference_session.rs:288
}

}  // namespace

// silu(a)*b over rows of [w1 x | w3 x] interleaved in 32-column pieces: h1[c] at (c/32)*64 + c%32, h3[c] 32 further
__global__ void silu_mul_rows_kernel(const uint16_t *__restrict__ t, const float *__restrict__ h13, float *__restrict__ out, int64_t f, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int64_t r = i / f, c = i - r * f;
    const int64_t o = r * 2 * f + (c >> 5) * 64 + (c & 31);
    const float a = h13[o], b = h13[o + 32];
    out[i] = __fmul_rn(f16_bits_to_f32(__ldg(t + f32_to_f16_bits(a))), b);
}
void silu_mul_rows(const float *h13, float *out, int64_t f, int64_t n, cudaStream_t st) {
    const int64_t total = f * n;
    if (total == 0) return;
    silu_mul_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(luts().silu, h13, out, f, total);
    B200_CHECK(cudaGetLastError());
}

// ==== exported C ABI ==========================================================================================================
extern "C" {

int b200_init(int device) {
    Runtime &R = rt();
    if (!R.inited) R.device = device;
    R.ensure_init();
    return R.device == device ? B200_OK : B200_ERR_BAD_ARG;
}

int b200_device_info(int32_t *sm_count, size_t *free_bytes, size_t *total_bytes) {
    rt().ensure_init();
    if (sm_count) *sm_count = rt().sm_count;
    size_t fr = 0, tot = 0;
    B200_CHECK(cudaMemGetInfo(&fr, &tot));
    if (free_bytes) *free_bytes = fr;
    if (total_bytes) *total_bytes = tot;
    return B200_OK;
}

void *b200_stream(void) { rt().ensure_init(); return (void *)rt().stream; }

static cudaEvent_t g_ev0 = nullptr, g_ev1 = nullptr;
int b200_timing_begin(void) {
    rt().ensure_init();
    if (!g_ev0) { B200_CHECK(cudaEventCreate(&g_ev0)); B200_CHECK(cudaEventCreate(&g_ev1)); }
    B200_CHECK(cudaEventRecord(g_ev0, rt().stream));
    return B200_OK;
}
float b200_timing_end_ms(void) {
    B200_CHECK(cudaEventRecord(g_ev1, rt().stream));
    B200_CHECK(cudaEventSynchronize(g_ev1));
    float ms = 0.f;
    B200_CHECK(cudaEventElapsedTime(&ms, g_ev0, g_ev1));
    return ms;
}

float b200_session_probe_matvec(b200_session *s, int32_t reps, int64_t *launches, double *bytes) {
    if (!s || reps < 1 || s->m->tp_world > 1) return -1.f;
    b200_model *m = s->m;
    cudaStream_t st = rt().stream;
    const int e = m->hp.n_embd, f = m->hp.n_ff;
    // a valid quantized activation row for both K = n_embd and K = n_ff
    const bool fast = (s->cfg.flags & B200_SESSION_FAST) != 0;
    B200_CHECK(cudaMemsetAsync(s->hmul.get(), 0, (size_t)f * 4, st));
    if (!is_kquant(m->hp.wtype)) {
        quantize_act(vec_dot_type(m->hp.wtype), s->hmul.get(), f, s->xq.get(), s->xds.get(), f, 1, st);
        quantize_act_pack(m->hp.wtype, s->hmul.get(), s->xpack.get(), f, st);
    }
    cvt_act_f16(s->hmul.get(), f, s->xh.get(), f, 1, st);
    if (m->any_kquant) quantize_act_q8k(s->hmul.get(), f, s->xq8k.get(), f / 256 * 256, 1, st);
    (void)e;
    int64_t n = 0;
    auto mv = [&](const QWeight &w, float *out) {
        if (w.type == T_F16) {
            if (mmv_f16_supported(w)) mul_mat_vec_f16(w, s->xh.get(), out, nullptr, st);
            else mul_mat_f16_gemm(w, s->xh.get(), out, w.N, 1, nullptr, 0, st);
        }
        else if (is_kquant(w.type)) mul_mat_kq_exact(w.type, w.qs, s->xq8k.get(), out, w.N, w.K, w.N, 1, nullptr, 0, st);
        else if (fast) mul_mat_vec_q(w, s->xq.get(), s->xds.get(), out, nullptr, st);
        else if (mmv_exact_stream_supported(w)) mul_mat_vec_q_exact_stream(w, s->xpack.get(), out, nullptr, st);
        else mul_mat_q_exact(w, s->xq.get(), s->xds.get(), out, w.N, 1, nullptr, 0, st);
        n++;
    };
    auto pass = [&]() {
        for (auto &L : m->layers) {
            mv(L.wqkv, s->qkv.get());
            if (L.wv.N) mv(L.wv, s->qkv.get());
            mv(L.wo, s->ff.get()); mv(L.w13, s->h13.get()); mv(L.w2, s->cur.get());
        }
        mv(m->output, s->logits.get());
    };
    pass();                      // warm-up (also first-touch of every page)
    n = 0;
    b200_timing_begin();
    for (int r = 0; r < reps; r++) pass();
    const float ms = b200_timing_end_ms();
    if (launches) *launches = n;
    if (bytes) *bytes = (double)m->weight_bytes * reps;
    return ms;
}

// the element type of each 2-D weight of one layer (wq and wk share one, w1 and w3 share one)
struct LayerTypes { int qk, v, o, ff13, w2; };

static b200_model *llama_new_impl(const b200_llama_hparams *hp, int tp_rank, int tp_world, const b200_tensor_type *types = nullptr, int32_t n_types = 0,
                                  int *err = nullptr) {
    int dummy; if (!err) err = &dummy;
    *err = B200_ERR_BAD_ARG;
    if (!hp || hp->n_embd % 64 || hp->n_ff % 64 || hp->n_head <= 0 || hp->n_head_kv <= 0 ||
        hp->n_head % hp->n_head_kv || hp->n_embd % hp->n_head || hp->n_layer <= 0 || hp->context_size <= 0 || n_types < 0 || (n_types && !types)) return nullptr;
    if (!is_qweight_type(hp->wtype) && !is_kquant(hp->wtype)) { *err = B200_ERR_UNSUPPORTED_ELEMENT_TYPE; return nullptr; }
    const int G = tp_world;
    if (G < 1 || G > TP_MAX || tp_rank < 0 || tp_rank >= G) return nullptr;
    if (G > 1 && hp->wtype == T_F16) return nullptr;      // shards decode through the fused schedule only, which is built on Q8 activation records
    // every 2-D weight's type: the table's entry, else hp->wtype; refused before anything is allocated
    auto type_of = [&](const char *name) { int t = hp->wtype; for (int32_t i = 0; i < n_types; i++) if (types[i].name && !strcmp(types[i].name, name)) t = types[i].type; return t; };
    for (int32_t i = 0; i < n_types; i++) {
        if (!types[i].name) return nullptr;
        if (!llama_matrix_name(types[i].name, hp->n_layer)) { *err = B200_ERR_UNKNOWN_TENSOR; return nullptr; }
    }
    auto check = [&](const char *name, int t, int64_t ne0) -> int {
        if (!is_qweight_type(t) && !is_kquant(t)) {
            fprintf(stderr, "llm_b200: %s is element type %d; 2-D weights are F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 or Q2_K..Q6_K\n", name, t);
            return B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
        }
        if (is_kquant(t) && ne0 % 256) { fprintf(stderr, "llm_b200: %s: a K-quant row of %lld elements is not whole super-blocks of 256\n", name, (long long)ne0); return B200_ERR_INVARIANT_BROKEN; }
        if (is_kquant(t) && G > 1) { fprintf(stderr, "llm_b200: %s: K-quant weights are not offered on tensor-parallel shards\n", name); return B200_ERR_BAD_ARG; }
        return B200_OK;
    };
    const int t_wte = type_of("tok_embeddings.weight"), t_out = type_of("output.weight");
    if ((*err = check("tok_embeddings.weight", t_wte, hp->n_embd)) != B200_OK || (*err = check("output.weight", t_out, hp->n_embd)) != B200_OK) return nullptr;
    std::vector<LayerTypes> lt((size_t)hp->n_layer);
    for (int il = 0; il < hp->n_layer; il++) {
        char nm[7][64];
        static const char *const sfx[7] = {"attention.wq", "attention.wk", "attention.wv", "attention.wo", "feed_forward.w1", "feed_forward.w3", "feed_forward.w2"};
        int t[7];
        for (int k = 0; k < 7; k++) {
            snprintf(nm[k], sizeof(nm[k]), "layers.%d.%s.weight", il, sfx[k]);
            t[k] = type_of(nm[k]);
            if ((*err = check(nm[k], t[k], k == 6 ? hp->n_ff : hp->n_embd)) != B200_OK) return nullptr;
        }
        // [wq | wk] and [w1 | w3] are one matrix each: no quantizer the reference ships writes their halves in different types
        if (t[1] != t[0] || t[5] != t[4]) {
            fprintf(stderr, "llm_b200: %s is of another element type than %s\n", t[1] != t[0] ? nm[1] : nm[5], t[1] != t[0] ? nm[0] : nm[4]);
            *err = B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
            return nullptr;
        }
        lt[il] = LayerTypes{t[0], t[2], t[3], t[4], t[6]};
    }
    // F16 weights come as whole F16 files: an F16 matrix beside block-format ones is refused (as before per-tensor types)
    bool f16 = t_wte == T_F16 || t_out == T_F16, other = t_wte != T_F16 || t_out != T_F16;
    for (const LayerTypes &x : lt)
        for (int y : {x.qk, x.v, x.o, x.ff13, x.w2}) { f16 |= y == T_F16; other |= y != T_F16; }
    if (f16 && other) {
        fprintf(stderr, "llm_b200: F16 weights beside weights of other element types: F16 models are F16 throughout\n");
        *err = B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
        return nullptr;
    }
    const int gqa_full = hp->n_embd / (hp->n_head / hp->n_head_kv);
    // row split: whole heads per rank, 32-row pieces of w1|w3 and of the lm_head, 32-element blocks of wo / w2's output slices
    if (G > 1 && (hp->n_head % G || hp->n_head_kv % G || (hp->n_ff / G) % 32 || hp->n_ff % G || (hp->n_embd / G) % 32 || hp->n_vocab % G || (hp->n_vocab / G) % 32)) return nullptr;
    rt().ensure_init();
    b200_model *m = new b200_model();
    m->hp = *hp;
    if (m->hp.rope_freq_base == 0.f) m->hp.rope_freq_base = 10000.0f;
    if (m->hp.rope_freq_scale == 0.f) m->hp.rope_freq_scale = 1.0f;
    const int e = hp->n_embd, v = hp->n_vocab, t = hp->wtype;
    m->hd = e / hp->n_head;
    m->gqa = gqa_full;
    m->tp_rank = tp_rank; m->tp_world = G;
    m->e_loc = e / G; m->gqa_loc = gqa_full / G; m->f_loc = hp->n_ff / G; m->v_loc = v / G;
    m->layers.resize(hp->n_layer);
    for (const LayerTypes &x : lt) m->uniform_layers &= x.qk == t && x.v == t && x.o == t && x.ff13 == t && x.w2 == t;
    // with one type for every weight this is the layout of a one-type model: same matrices, same order, same bytes
    m->carve(t, m->n_slots(), [m, hp, e, v, &lt, t_wte, t_out](SlabCarver &c) {
        c.q(m->wte, e, v, t_wte); c.q(m->output, e, m->v_loc, t_out); c.f(m->norm, e);
        for (int il = 0; il < hp->n_layer; il++) {
            Layer &L = m->layers[il];
            const LayerTypes &y = lt[il];
            c.f(L.attention_norm, e); c.f(L.ffn_norm, e);
            if (y.v == y.qk) c.q(L.wqkv, e, m->e_loc + 2 * m->gqa_loc, y.qk);
            else { c.q(L.wqkv, e, m->e_loc + m->gqa_loc, y.qk); c.q(L.wv, e, m->gqa_loc, y.v); }
            c.q(L.wo, e, m->e_loc, y.o); c.q(L.w13, e, 2 * m->f_loc, y.ff13); c.q(L.w2, hp->n_ff, m->e_loc, y.w2);
        }
    });
    auto note = [m](const QWeight &w) { m->any_kquant |= is_kquant(w.type); m->any_f16 |= w.type == T_F16; };
    note(m->wte); note(m->output);
    for (const Layer &L : m->layers) { note(L.wqkv); note(L.wo); note(L.w13); note(L.w2); if (L.wv.N) note(L.wv); }
    m->weight_bytes -= (size_t)v * m->wte.nb * qweight_block_bytes(m->wte.type);   // tok_embeddings is only gathered from, never streamed
    *err = B200_OK;
    return m;
}

b200_model *b200_llama_new(const b200_llama_hparams *hp) { return llama_new_impl(hp, 0, 1); }

// A model whose 2-D weights each have their own element type: types[0, n) name tensors (tok_embeddings.weight, output.weight,
// layers.<i>.attention.w{q,k,v,o}.weight, layers.<i>.feed_forward.w{1,2,3}.weight); the others are of hp->wtype.
b200_model *b200_llama_new_typed(const b200_llama_hparams *hp, const b200_tensor_type *types, int32_t n, int *err) {
    return llama_new_impl(hp, 0, 1, types, n, err);
}

// Tensor-parallel shard `tp_rank` of `tp_world` (one process per GPU): the model's tensors keep their names, but every 2-D weight except
// tok_embeddings holds only this rank's rows -- wq / wk / wv: its heads; w1 / w3: rows [rank * n_ff/G, +n_ff/G); wo / w2: rows
// [rank * n_embd/G, +n_embd/G); output: rows [rank * n_vocab/G, +n_vocab/G) -- and b200_model_load_tensor expects exactly those rows.
b200_model *b200_llama_new_tp(const b200_llama_hparams *hp, int32_t tp_rank, int32_t tp_world) { return llama_new_impl(hp, tp_rank, tp_world); }

size_t b200_model_weight_bytes(b200_model *m) { return m ? m->weight_bytes : 0; }

size_t b200_model_tensor_nbytes(b200_model *m, const char *name) {
    Slot s; int id;
    if (!m || !m->lookup(name, s, id)) return 0;
    return s.bytes();
}

int b200_model_load_tensor(b200_model *m, const char *name, int32_t type, const void *host_data, size_t nbytes) {
    if (!m || !name || !host_data) return B200_ERR_BAD_ARG;
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    const int rc = load_slot(s, type, host_data, nbytes);
    if (rc == B200_OK) m->mark(id);
    return rc;
}

// TensorLoader::load checks the dims too (TensorWrongSize): a file whose tensor has the right byte count but swapped / wrong dims must not load
int b200_model_load_tensor_shaped(b200_model *m, const char *name, int32_t type, int32_t n_dims, int64_t ne0, int64_t ne1, const void *host_data, size_t nbytes) {
    if (!m || !name) return B200_ERR_BAD_ARG;
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    if (s.is_q) { if (n_dims != 2 || ne0 != s.q.K || ne1 != s.q_rows()) return B200_ERR_TENSOR_SHAPE; }
    else if (n_dims != 1 || ne0 != s.n) return B200_ERR_TENSOR_SHAPE;
    return b200_model_load_tensor(m, name, type, host_data, nbytes);
}

int b200_model_load_tensor_lora(b200_model *m, const char *name, int32_t type, int32_t n_dims, int64_t ne0, int64_t ne1, const void *host_data, size_t nbytes,
                                const b200_ggml_file *const *adapters, int32_t n_adapters) {
    if (n_adapters == 0) return b200_model_load_tensor_shaped(m, name, type, n_dims, ne0, ne1, host_data, nbytes);
    if (!m || !name || !host_data || !adapters || n_adapters < 0 || m->tp_world > 1) return B200_ERR_BAD_ARG;   // shards: out of scope
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    if (s.is_q) { if (n_dims != 2 || ne0 != s.q.K || ne1 != s.q_rows()) return B200_ERR_TENSOR_SHAPE; }
    else if (n_dims != 1 || ne0 != s.n) return B200_ERR_TENSOR_SHAPE;
    const LoraTarget t{name, ne0, s.is_q ? ne1 : 1, adapters, n_adapters};
    const int rc = load_slot(s, type, host_data, nbytes, &t);
    if (rc == B200_OK) m->mark(id);
    return rc;
}

int b200_model_read_tensor(b200_model *m, const char *name, void *host_out, size_t nbytes) {
    if (!m || !name || !host_out) return B200_ERR_BAD_ARG;
    Slot s; int id;
    if (!m->lookup(name, s, id)) return B200_ERR_UNKNOWN_TENSOR;
    return read_slot(s, host_out, nbytes);
}

int b200_model_synthesize(b200_model *m, uint64_t seed) {
    if (!m || m->tp_world > 1) return B200_ERR_BAD_ARG;       // shards are cut from a full model's tensors by the host (llm_b200/tp.py)
    const int64_t e = m->hp.n_embd;
    m->synthesize(seed, [m, e](SeedSeq &r) {
        r.q(m->wte); r.gain(m->norm, e); r.q(m->output);
        for (auto &L : m->layers) {
            r.gain(L.attention_norm, e); r.gain(L.ffn_norm, e); r.q(L.wqkv);
            if (L.wv.N) r.q(L.wv);
            r.q(L.wo); r.q(L.w13); r.q(L.w2);
        }
    });
    return B200_OK;
}

int b200_model_is_loaded(b200_model *m) { return m && m->all_loaded(); }

void b200_model_free(b200_model *m) {
    if (!m) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    delete m;                                           // the slab goes with it
}

// the layer table of the decode schedules: each layer's weights and its slice of the KV cache (gqa_loc: this rank's cache width, all of it on one GPU)
static std::vector<DecodeLayer> decode_layers(const b200_session *s) {
    const b200_model *m = s->m;
    const size_t slice = (size_t)m->hp.context_size * m->gqa_loc;
    std::vector<DecodeLayer> hl(m->hp.n_layer);
    for (int il = 0; il < m->hp.n_layer; il++) {
        const Layer &L = m->layers[il];
        hl[il] = DecodeLayer{L.wqkv, L.wo, L.w13, L.w2, L.attention_norm, L.ffn_norm, s->kv_at(0, il * slice), s->kv_at(1, il * slice)};
    }
    return hl;
}

// what single-GPU and tensor-parallel sessions both allocate: the KV cache (this rank's heads), token and logits staging, the sampler's
// buffers, and the decode schedules' q vector, activation records and timeline slots
static void start_common(b200_session *s) {
    const b200_model *m = s->m;
    const b200_llama_hparams &hp = m->hp;
    s->start(s->cfg.n_batch, hp.context_size, hp.n_vocab, (size_t)hp.n_layer * hp.context_size * m->gqa_loc, (s->cfg.flags & B200_SESSION_KV_F32) ? T_F32 : T_F16);
    s->qbuf = device_alloc<float>((size_t)m->e_loc * 4);
    s->xpack_a = device_alloc<int4>((size_t)(hp.n_embd / QK) * 64);
    s->d_prof = device_zeros<unsigned long long>(B200_PROF_SLOTS * 8 * sizeof(unsigned long long));
}

// ---- tensor-parallel session: decode only (prompts are fed token by token), activations that cross GPUs live in ONE exchange slab -------------
static b200_session *start_session_tp(b200_session *s) {
    b200_model *m = s->m;
    const b200_llama_hparams &hp = m->hp;
    const int G = m->tp_world, r = m->tp_rank;
    const size_t e = hp.n_embd, f = hp.n_ff, n_ctx = hp.context_size, V = hp.n_vocab;
    // the exchange lives in the fused attention kernel, whose shared memory holds the whole context bucket
    if (!attn_fused_fits(hp.context_size, m->hd)) {
        fprintf(stderr, "llm_b200: tensor-parallel session: context_size %d is more than the fused attention kernel holds (3264 positions)\n", hp.context_size);
        b200_session_free(s);
        return nullptr;
    }
    start_common(s);
    // the exchange slab: arrays of 8-byte {word, tag} units (tp.cuh) -- x | ff | attention records | ffn records | logits, 256-byte aligned pieces
    TpCtx &T = s->dp.tp;
    T = TpCtx();
    T.world = G; T.rank = r; T.vmul = (unsigned)hp.n_layer + 1;
    { const char *e = getenv("B200_TP_RELAX"); T.relax = e ? atoi(e) : 0; }
    size_t off = 0;
    auto piece = [&](size_t units) { const size_t o = off; off += (units * 8 + 255) & ~(size_t)255; return (uint32_t)o; };
    T.off[TPB_X] = piece(e); T.off[TPB_FF] = piece(e); T.off[TPB_XD] = piece((e / QK) * 16); T.off[TPB_XF] = piece((f / QK) * 16); T.off[TPB_LOGITS] = piece(V);
    s->tp_slab_bytes = off;
    s->tp_slab = device_zeros<char>(off);                                 // tag 0 never matches
    s->tp_state = device_zeros<unsigned>(2 * sizeof(unsigned));
    T.epoch = s->tp_state.get();
    for (int p = 0; p < TP_MAX; p++) T.peer[p] = nullptr;
    T.peer[r] = s->tp_slab.get();                                        // peers are mapped by b200_session_tp_connect
    s->x = device_alloc<float>(e * 4);                                    // the embedding row (plain f32) before it is spread into the X units
    s->logits = device_alloc<float>(V * 4);                               // the gathered logits, plain f32 for the host
    const RopeTable &rt_ = rope_table(hp.n_rot, 0, hp.rope_freq_base, hp.rope_freq_scale, m->hd, (int)n_ctx);
    s->h_layers = decode_layers(s);
    DecodeParams &P = s->dp;
    P.n_layer = hp.n_layer; P.wte = m->wte; P.output = m->output; P.norm = m->norm;
    P.e = (int)e; P.f = m->f_loc; P.hd = m->hd; P.gqa = m->gqa_loc; P.n_head = hp.n_head / G; P.n_head_kv = hp.n_head_kv / G; P.n_ctx = (int)n_ctx; P.n_vocab = m->v_loc;
    P.kq_scale = 1.0f / sqrtf((float)hp.n_embd / (float)hp.n_head); P.eps = 5e-6f; P.kv_type = s->kv_type;
    P.rope_cs = rt_.cs; P.rope_half = rt_.half;
    P.lut_silu = luts().silu; P.lut_exp = luts().exp;
    P.token = s->d_tokens.get(); P.n_past = s->decode.d_n_past;
    P.x = s->x.get(); P.q = s->qbuf.get(); P.kq = nullptr; P.ff = nullptr; P.logits = s->logits.get();
    P.xpack_d = nullptr; P.xpack_f = nullptr; P.normed = nullptr;        // embeddings are not offered on tensor-parallel sessions
    P.e_loc = m->e_loc; P.head0 = r * (hp.n_head / G); P.n_vocab_full = hp.n_vocab;
    P.row0_e = (int64_t)r * m->e_loc; P.row0_w13 = (int64_t)r * 2 * m->f_loc; P.row0_v = (int64_t)r * m->v_loc;
    P.prof = nullptr;
    QWeight probe; probe.nb = (int64_t)e / QK;
    QWeight probe2; probe2.nb = (int64_t)f / QK;
    s->graph_ok = hp.n_rot == m->hd && (m->hd == 64 || m->hd == 128) && mmv_exact_stream_supported(probe) && mmv_exact_stream_supported(probe2) &&
                  m->gqa_loc % 32 == 0 && m->e_loc % 32 == 0 && hp.context_size % 8 == 0;
    B200_CHECK(cudaDeviceSynchronize());
    if (!s->graph_ok) { fprintf(stderr, "llm_b200: tensor-parallel session: geometry not supported by the fused decode schedule\n"); b200_session_free(s); return nullptr; }
    return s;
}

b200_session *b200_model_start_session(b200_model *m, const b200_session_config *cfg) {
    if (!m || !cfg || cfg->n_batch < 1) return nullptr;
    if (!m->all_loaded()) { fprintf(stderr, "llm_b200: start_session: %d of %d tensors loaded\n", m->n_loaded, m->n_slots()); return nullptr; }
    // the tensor-parallel attention lives in the fused f16 kernel's epilogue: an f32 cache there is not offered
    if (m->tp_world > 1 && (cfg->flags & B200_SESSION_KV_F32)) { fprintf(stderr, "llm_b200: start_session: B200_SESSION_KV_F32 on a tensor-parallel model\n"); return nullptr; }
    b200_session *s = new b200_session();
    s->m = m; s->cfg = *cfg;
    if (m->tp_world > 1) return start_session_tp(s);
    const b200_llama_hparams &hp = m->hp;
    if (m->any_f16 && (cfg->flags & B200_SESSION_FAST)) {   // the order-free kernels take the five block formats only (K-quants run exact)
        fprintf(stderr, "llm_b200: start_session: B200_SESSION_FAST has no kernels for F16 weights\n");
        b200_session_free(s);
        return nullptr;
    }
    const size_t e = hp.n_embd, f = hp.n_ff, B = cfg->n_batch, n_ctx = hp.context_size, gqa = m->gqa;
    start_common(s);
    const size_t kmax = e > f ? e : f;
    s->x = device_alloc<float>(B * e * 4);
    s->cur = device_alloc<float>(B * e * 4);
    s->ff = device_alloc<float>(B * e * 4);
    s->qkv = device_alloc<float>(B * (e + 2 * gqa) * 4);
    s->kq = device_alloc<float>((size_t)hp.n_head * B * n_ctx * 4);
    s->h13 = device_alloc<float>(B * 2 * f * 4);
    s->hmul = device_alloc<float>(B * f * 4);
    s->logits = device_alloc<float>(B * (size_t)hp.n_vocab * 4);
    s->xq = device_alloc<int8_t>(B * kmax);
    s->xds = device_alloc<float2>(B * (kmax / QK) * sizeof(float2));
    s->xpack = device_alloc<int4>((kmax / QK) * 64);
    s->xh = device_alloc<__half>(xh_bytes(kmax, B));
    if (m->any_kquant) s->xq8k = device_alloc<char>(q8k_bytes(kmax / 256 * 256, B));
    const RopeTable &rt_ = rope_table(hp.n_rot, 0, hp.rope_freq_base, hp.rope_freq_scale, m->hd, (int)n_ctx);
    // decode kernel parameters
    s->h_layers = decode_layers(s);
    DecodeParams &P = s->dp;
    P.n_layer = hp.n_layer; P.wte = m->wte; P.output = m->output; P.norm = m->norm;
    P.e = (int)e; P.f = (int)f; P.hd = m->hd; P.gqa = m->gqa; P.n_head = hp.n_head; P.n_head_kv = hp.n_head_kv; P.n_ctx = (int)n_ctx; P.n_vocab = hp.n_vocab;
    P.kq_scale = 1.0f / sqrtf((float)hp.n_embd / (float)hp.n_head); P.eps = 5e-6f; P.kv_type = s->kv_type;
    P.rope_cs = rt_.cs; P.rope_half = rt_.half;
    P.lut_silu = luts().silu; P.lut_exp = luts().exp;
    P.token = s->d_tokens.get(); P.n_past = s->decode.d_n_past;
    P.x = s->x.get(); P.q = s->qbuf.get(); P.kq = s->kq.get(); P.ff = s->ff.get(); P.logits = s->logits.get();
    P.normed = s->cur.get();                                     // row 0 of cur: where forward()'s final rms_norm leaves a one-token batch
    P.xq8k = s->xq8k.get();                                      // a K-quant lm_head's activation row
    s->xpack_d = device_alloc<int4>((e / QK) * 64);
    s->xpack_f = device_alloc<int4>((f / QK) * 64);
    P.xpack_d = s->xpack_d.get(); P.xpack_f = s->xpack_f.get();
    P.prof = getenv("B200_DECODE_PROF") ? s->d_prof.get() : nullptr;
    // The graph schedule takes RoPE over whole heads of 64 or 128 channels and mat-vecs whose K (n_embd, n_ff) the streaming core takes, a multiple
    // of 256.  With what llama_new_impl checks, that covers the rest: a classic weight type, a K/V width n_head_kv * hd of whole 32-row tiles.
    // n_embd <= 6144 and context_size % 128 == 0 are limits of the removed one-kernel decode, kept so that the same geometries decode through the graph.
    QWeight probe; probe.nb = (int64_t)e / QK;
    QWeight probe2; probe2.nb = (int64_t)f / QK;
    // F16 weights decode through the per-op path (exact_f16.cu's mat-vec): the fused schedule is built on Q8 activation records.  So does an f32
    // cache whose context is longer than its two-kernel attention holds (the schedule's attention past 1664 positions).  Per-tensor types: every
    // layer matrix must be of the model's classic type; the lm_head may also be a K-quant (the quantizer's Q6_K output.weight), which the graph
    // runs as quantize_row_q8_K + the K-quant mat-vec.  Layers with a K-quant or another type decode per op.
    s->graph_ok = hp.n_rot == m->hd && (m->hd == 64 || m->hd == 128) && mmv_exact_stream_supported(probe) && mmv_exact_stream_supported(probe2) &&
                  e <= 6144 && n_ctx % 128 == 0 && hp.wtype != T_F16 && (s->kv_type != T_F32 || (int)n_ctx <= attn_sv_f32_max_ctx()) &&
                  !is_kquant(hp.wtype) && m->uniform_layers && (m->output.type == hp.wtype || is_kquant(m->output.type));
    B200_CHECK(cudaDeviceSynchronize());   // the memsets / copies above ran on the legacy stream: order them before anything on the backend's non-blocking stream
    return s;
}

int32_t b200_session_n_past(const b200_session *s) { return s ? s->n_past : -1; }
int b200_session_set_n_past(b200_session *s, int32_t n_past) { return s ? s->set_n_past(n_past) : B200_ERR_BAD_ARG; }
int32_t b200_session_last_launches(const b200_session *s) { return s ? s->last_launches : 0; }

int b200_session_evaluate_device(b200_session *s, const int32_t *d_tokens, int32_t n) {
    if (!s) return B200_ERR_BAD_ARG;
    if (const int rc = s->admit(n)) return rc;
    if (d_tokens && d_tokens != s->d_tokens.get())
        B200_CHECK(cudaMemcpyAsync(s->d_tokens.get(), d_tokens, (size_t)n * 4, cudaMemcpyDeviceToDevice, rt().stream));
    s->record_tokens(n);
    forward(s, n);
    return B200_OK;
}
const float *b200_session_device_logits(b200_session *s) { return s ? s->logits.get() : nullptr; }

// embeddings_out: row n - 1 of the final norm's output, which forward() leaves in cur (the graph step: its row 0)
int b200_session_evaluate_output(b200_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits, float *embeddings_out) {
    if (!s || !tokens || (embeddings_out && s->m->tp_world > 1)) return B200_ERR_BAD_ARG;
    if (const int rc = s->admit(n)) return rc;
    if (s->m->tp_world > 1 && n > 1) {                  // tensor-parallel sessions have the decode schedule only: a batch is fed token by token
        const size_t V = s->m->hp.n_vocab;
        for (int i = 0; i < n; i++) {
            float *out = !logits_out ? nullptr : all_logits ? logits_out + (size_t)i * V : (i == n - 1 ? logits_out : nullptr);
            const int rc = b200_session_evaluate_output(s, tokens + i, 1, out, 0, nullptr);
            if (rc != B200_OK) return rc;
        }
        return B200_OK;
    }
    if (const int rc = s->stage_tokens(tokens, n)) return rc;
    forward(s, n, all_logits != 0);
    s->copy_logits(logits_out, s->logits.get(), n, all_logits != 0);
    s->copy_row(embeddings_out, s->cur.get() + (size_t)(n - 1) * s->m->hp.n_embd, s->m->hp.n_embd);
    return B200_OK;
}

int b200_session_evaluate(b200_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits) {
    return b200_session_evaluate_output(s, tokens, n, logits_out, all_logits, nullptr);
}

// InferenceSession::perplexity (SessionCore::perplexity): tensor-parallel sessions are refused, FAST sessions run (their logits are not the reference's)
int b200_session_perplexity(b200_session *s, const int32_t *tokens, int64_t n, int32_t bos, float *ppl_out, float *terms_out, int32_t *n_chunk_out) {
    if (!s || s->m->tp_world > 1) return B200_ERR_BAD_ARG;
    return s->perplexity(tokens, n, bos, ppl_out, terms_out, n_chunk_out, s->logits.get(), [s](int rows) { forward(s, rows); });
}

// Sampler hand-off (SURVEY.md §8f-3): the k largest logits of the last evaluated row, selected on the device (the sampler's top-k stage, sample.cu);
// 8 k bytes cross PCIe instead of n_vocab floats.  Order = descending logit, ties by ascending token id (what a stable descending sort of
// (id, logit) pairs yields: llm-samplers top-k).
int b200_session_top_k(b200_session *s, int32_t k, int32_t *ids_out, float *logits_out) {
    return s ? s->top_k(s->logits.get(), k, ids_out, logits_out) : B200_ERR_BAD_ARG;
}

// InferenceSession::infer_next_token (SessionCore::infer_next_token): tensor-parallel sessions are refused, FAST sessions run
int b200_session_infer_next_token(b200_session *s, const b200_sampler *sampler, int32_t *token_out) {
    SampleArgs a;
    if (!s || s->m->tp_world > 1 || !sampler_args(sampler, a)) return B200_ERR_BAD_ARG;
    return s->infer_next_token(a, s->logits.get(), [s]() { forward(s, 1); }, token_out);
}

int32_t b200_session_read_tokens(b200_session *s, int32_t *tokens_out, int32_t max) { return s ? s->read_tokens(tokens_out, max) : B200_ERR_BAD_ARG; }
int b200_session_last_logits(b200_session *s, float *logits_out) { return s ? s->last_logits(s->logits.get(), logits_out) : B200_ERR_BAD_ARG; }

// every chunk gets the same request in the reference (:317), so what it leaves behind is the last chunk's: only that one is copied out
int b200_session_feed_prompt_output(b200_session *s, const int32_t *tokens, int32_t n, float *last_logits_out, float *embeddings_out) {
    if (!s || !tokens || n < 0 || (embeddings_out && s->m->tp_world > 1)) return B200_ERR_BAD_ARG;
    if (s->n_past + n > s->m->hp.context_size) return B200_ERR_CONTEXT_FULL;          // inference_session.rs:311-313
    for (int i = 0; i < n; i += s->cfg.n_batch) {                                     // :315-316 chunks(n_batch)
        const int c = (n - i) < s->cfg.n_batch ? (n - i) : s->cfg.n_batch;
        const bool last = i + c >= n;
        const int rc = b200_session_evaluate_output(s, tokens + i, c, last ? last_logits_out : nullptr, 0, last ? embeddings_out : nullptr);
        if (rc != B200_OK) return rc;
    }
    return B200_OK;
}

int b200_session_feed_prompt(b200_session *s, const int32_t *tokens, int32_t n, float *last_logits_out) {
    return b200_session_feed_prompt_output(s, tokens, n, last_logits_out, nullptr);
}

// n_layer x context_size x the cache width (tensor-parallel: this rank's heads) elements of the cache's type
int b200_session_read_kv(b200_session *s, int32_t which, void *host_out, size_t nbytes) {
    return s ? s->read_kv(which, host_out, nbytes) : B200_ERR_BAD_ARG;
}

// ---- snapshots (snapshot.cu): the reference sizes LLaMA's cache by n_embd and uses n_embd_gqa of it per position, V by channel as here ------------
static RefKvLayout ref_layout(const b200_model *m) { return RefKvLayout{m->hp.n_layer, m->gqa, m->hp.n_embd, false}; }

int b200_session_get_snapshot(b200_session *s, b200_snapshot *snap) {
    if (!s || s->m->tp_world > 1) return B200_ERR_BAD_ARG;
    return s->get_snapshot(ref_layout(s->m), s->logits.get(), snap);
}

int b200_session_write_snapshot(b200_session *s, const char *path) {
    if (!s || s->m->tp_world > 1) return B200_ERR_BAD_ARG;
    return s->write_snapshot(ref_layout(s->m), s->logits.get(), path);
}

static b200_session *session_from(b200_model *m, const b200_snapshot *snap, const char *path, int32_t flags, int *err) {
    if (!m || m->tp_world > 1 || (flags & ~(B200_SESSION_NO_GRAPH | B200_SESSION_UNFUSED | B200_SESSION_FAST | B200_SESSION_KV_F32))) {
        if (err) *err = B200_ERR_BAD_ARG;
        return nullptr;
    }
    return session_from_snapshot<b200_session>(snap, path, m->hp.context_size, m->hp.n_vocab, ref_layout(m), err,
        [m, flags](int n_batch, bool kv32, float *&logits) -> b200_session * {
            if ((flags & B200_SESSION_KV_F32) && !kv32) return nullptr;            // the cache type is the snapshot's
            const b200_session_config cfg{n_batch, flags | (kv32 ? B200_SESSION_KV_F32 : 0)};
            b200_session *s = b200_model_start_session(m, &cfg);
            if (s) logits = s->logits.get();
            return s;
        },
        [](b200_session *s) { b200_session_free(s); });
}

b200_session *b200_model_session_from_snapshot(b200_model *m, const b200_snapshot *snap, int32_t flags, int *err) {
    return session_from(m, snap, nullptr, flags, err);
}

b200_session *b200_model_session_read_snapshot(b200_model *m, const char *path, int32_t flags, int *err) {
    if (!path) { if (err) *err = B200_ERR_BAD_ARG; return nullptr; }
    return session_from(m, nullptr, path, flags, err);
}

int b200_session_set_tap(b200_session *s, int32_t layer, int32_t stage) {
    if (!s || s->m->tp_world > 1) return B200_ERR_BAD_ARG;
    s->tap_layer = layer; s->tap_stage = stage; s->tap_count = 0;
    return B200_OK;
}
int64_t b200_session_read_tap(b200_session *s, float *host_out, int64_t max_count) {
    if (!s || !host_out) return B200_ERR_BAD_ARG;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    const size_t c = s->tap_count < (size_t)max_count ? s->tap_count : (size_t)max_count;
    if (c) B200_CHECK(cudaMemcpy(host_out, s->tap.get(), c * 4, cudaMemcpyDeviceToHost));
    return (int64_t)c;
}

// Per-kernel timeline of the graph decode schedule (B200_DECODE_PROF=1): slot i = the i-th launch of the token;
// out = 8 arrays of n (%globaltimer, ns): CTA begin min, CTA end max, prologue-done min, begin max, prologue-done max, first stage landed min / max,
// last stage landed max (mat-vec kernels only for the last three).  reset != 0 re-arms the slots.
int b200_session_decode_timeline(b200_session *s, unsigned long long *out, int n, int reset) {
    if (!s || n < 0 || n > B200_PROF_SLOTS) return B200_ERR_BAD_ARG;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    if (out && n) {
        for (int k = 0; k < 8; k++)
            B200_CHECK(cudaMemcpy(out + (size_t)k * n, s->d_prof.get() + (size_t)k * B200_PROF_SLOTS, (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    }
    if (reset) {                                                  // arrays 0, 2, 5 hold minima, the others maxima
        for (int k = 0; k < 8; k++)
            B200_CHECK(cudaMemset(s->d_prof.get() + (size_t)k * B200_PROF_SLOTS, (k == 0 || k == 2 || k == 5) ? 0xFF : 0, B200_PROF_SLOTS * sizeof(unsigned long long)));
        B200_CHECK(cudaDeviceSynchronize());
    }
    return B200_OK;
}

int b200_session_sync(b200_session *s) { (void)s; B200_CHECK(cudaStreamSynchronize(rt().stream)); return B200_OK; }

// ---- tensor-parallel plumbing: exchange-slab handles (CUDA IPC; one process per GPU, handles travel over the host's own channel) --------
int b200_session_tp_handle(b200_session *s, void *handle_out64) {
    if (!s || !s->tp_slab.get() || !handle_out64) return B200_ERR_BAD_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t h;
    B200_CHECK(cudaIpcGetMemHandle(&h, s->tp_slab.get()));
    memcpy(handle_out64, &h, 64);
    return B200_OK;
}
int b200_session_tp_connect(b200_session *s, const void *handles_by_rank) {
    if (!s || !s->tp_slab.get() || !handles_by_rank) return B200_ERR_BAD_ARG;
    TpCtx &T = s->dp.tp;
    for (int p = 0; p < T.world; p++) {
        if (p == T.rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char *)handles_by_rank + (size_t)p * 64, 64);
        void *ptr = nullptr;
        const cudaError_t err = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
        if (err != cudaSuccess) { fprintf(stderr, "llm_b200: cudaIpcOpenMemHandle(rank %d): %s\n", p, cudaGetErrorString(err)); return B200_ERR_IO; }
        s->tp_peer_map[p] = ptr;
        T.peer[p] = (char *)ptr;
    }
    s->tp_connected = true;
    decode_set_tp(T, rt().stream);
    return B200_OK;
}
int b200_session_tp_set_nowait(b200_session *s, int32_t nowait) {     // measurement aid: the captured graphs carry the flag, so they are dropped
    if (!s || !s->tp_slab.get()) return B200_ERR_BAD_ARG;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    s->dp.tp.nowait = nowait < 0 ? 0 : nowait > 2 ? 2 : nowait;
    decode_set_tp(s->dp.tp, rt().stream);
    s->decode.drop();
    return B200_OK;
}
int32_t b200_session_tp_timeouts(b200_session *s) {      // number of flag waits that gave up (a peer stopped): must be 0
    if (!s || !s->tp_state.get()) return -1;
    unsigned v[2] = {0, 0};
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    B200_CHECK(cudaMemcpy(v, s->tp_state.get(), sizeof(v), cudaMemcpyDeviceToHost));
    return (int32_t)v[1];
}

void b200_session_free(b200_session *s) {
    if (!s) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    for (int p = 0; p < TP_MAX; p++) if (s->tp_peer_map[p]) cudaIpcCloseMemHandle(s->tp_peer_map[p]);   // tensor-parallel session: the peers' slabs
    delete s;                                           // every buffer, the decode graphs and n_past words go with it
}

}  // extern "C"
