// llm_b200/csrc/host.cu -- tensor slots and session state shared by the LLaMA and GPT-NeoX / GPT-2 runtimes (host.h)
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/llm_b200.h"
#include "host.h"

namespace b200 {

// loraA / loraB of `name` in one adapter (UnknownTensor if either is missing), checked against the target [K, N] of wtype
static int lora_factors(const b200_ggml_file *f, const char *name, int wtype, int64_t K, int64_t N, int64_t idx[2], b200_ggml_tensor_info info[2]) {
    const std::string base(name);
    idx[0] = ggml_find_tensor(f, (base + ".loraA").c_str());
    idx[1] = ggml_find_tensor(f, (base + ".loraB").c_str());
    if (idx[0] < 0 || idx[1] < 0) return B200_ERR_UNKNOWN_TENSOR;
    b200_ggml_tensor(f, idx[0], &info[0]);
    b200_ggml_tensor(f, idx[1], &info[1]);
    return lora_check(wtype, K, N, info[0].type, info[0].ne[0], info[0].ne[1], info[1].type, info[1].ne[0], info[1].ne[1]);
}

// LoraAdapter::patch of every adapter in order on w (device, file layout); check = true only validates, so that a bad adapter changes nothing
static int lora_apply(const LoraTarget &t, int wtype, int64_t K, int64_t N, void *w, bool check) {
    Runtime &R = rt();
    for (int i = 0; i < t.n; i++) {
        const b200_ggml_file *f = t.adapters[i];
        if (!f) return B200_ERR_BAD_ARG;
        if (!lora_in_patch_set(f, t.name)) continue;
        int64_t idx[2]; b200_ggml_tensor_info info[2];
        const int rc = lora_factors(f, t.name, wtype, K, N, idx, info);
        if (rc != B200_OK) return rc;
        if (check) continue;
        void *a = R.op_arena.get(info[0].nbytes ? info[0].nbytes : 1, R.stream);
        float *b = (float *)R.op_arena.get(info[1].nbytes ? info[1].nbytes : 4, R.stream);
        B200_CHECK(cudaMemcpyAsync(a, b200_ggml_tensor_data(f, idx[0]), info[0].nbytes, cudaMemcpyHostToDevice, R.stream));
        B200_CHECK(cudaMemcpyAsync(b, b200_ggml_tensor_data(f, idx[1]), info[1].nbytes, cudaMemcpyHostToDevice, R.stream));
        lora_patch(wtype, w, K, N, info[0].type, a, b, info[0].ne[0], info[1].ne[1], lora_scaling(f), R.stream);
    }
    return B200_OK;
}

QWeight row_view(const QWeight &w, int64_t row0, int64_t nrows) {
    QWeight v = w;
    v.N = nrows;
    v.qs = w.qs + (size_t)row0 * w.nb * (w.type == T_F16 || is_kquant(w.type) ? qweight_block_bytes(w.type) : qs_bytes(w.type));
    if (w.qh) v.qh = w.qh + (size_t)row0 * w.nb;
    if (w.dm) v.dm = (const uint8_t *)w.dm + (size_t)row0 * w.nb * (has_min(w.type) ? 4 : 2);
    v.base = nullptr;
    return v;
}

int load_slot(const Slot &s, int32_t type, const void *host, size_t nbytes, const LoraTarget *lora) {
    Runtime &R = rt();
    // the target as the adapters see it: the tensor in file row order (a vector is one row)
    const int64_t K = s.is_q ? s.q.K : lora ? lora->ne0 : 0, N = s.is_q ? s.q_rows() : lora ? lora->ne1 : 0;
    if (lora) {
        if (!s.is_q && K * N != s.n) return B200_ERR_TENSOR_SHAPE;
        if (type == (s.is_q ? s.q.type : T_F32) && nbytes == s.bytes()) {
            const int rc = lora_apply(*lora, type, K, N, nullptr, true);
            if (rc != B200_OK) return rc;
        }
    }
    if (s.is_q) {
        if (type != s.q.type || nbytes != s.bytes()) return B200_ERR_TENSOR_SHAPE;
        R.op_arena.reset();
        void *raw = R.op_arena.get(nbytes, R.stream);
        B200_CHECK(cudaMemcpyAsync(raw, host, nbytes, cudaMemcpyHostToDevice, R.stream));
        if (lora) lora_apply(*lora, type, K, N, raw, false);
        if (!s.chunk) repack_weights(s.q, raw, R.stream);
        else {
            const size_t piece = (size_t)s.chunk * s.q.nb * qweight_block_bytes(type);
            for (int64_t c = 0; c * s.chunk < s.rows; c++)
                repack_weights(row_view(s.q, c * s.stride + s.row0, s.chunk), (const char *)raw + c * piece, R.stream);
        }
        B200_CHECK(cudaStreamSynchronize(R.stream));
    } else if (type == T_F16 && s.f16_src && nbytes == (size_t)s.n * 2) {
        if (lora)                                    // the reference would patch the F16 tensor before it is widened
            for (int i = 0; i < lora->n; i++) if (lora->adapters[i] && lora_in_patch_set(lora->adapters[i], lora->name)) return B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
        R.op_arena.reset();
        void *raw = R.op_arena.get(nbytes, R.stream);
        B200_CHECK(cudaMemcpyAsync(raw, host, nbytes, cudaMemcpyHostToDevice, R.stream));
        f16_to_f32(raw, s.f, s.n, R.stream);
        B200_CHECK(cudaStreamSynchronize(R.stream));
    } else {
        if (type != T_F32 || nbytes != s.bytes()) return B200_ERR_TENSOR_SHAPE;
        B200_CHECK(cudaMemcpy(s.f, host, nbytes, cudaMemcpyHostToDevice));
        B200_CHECK(cudaDeviceSynchronize());   // legacy-stream copy/memset: not ordered with our non-blocking stream, and a pageable H2D cudaMemcpy may return before its DMA lands
        if (lora) {
            R.op_arena.reset();
            lora_apply(*lora, type, K, N, s.f, false);
            B200_CHECK(cudaStreamSynchronize(R.stream));
        }
    }
    return B200_OK;
}

int read_slot(const Slot &s, void *host, size_t nbytes) {
    Runtime &R = rt();
    if (nbytes != s.bytes()) return B200_ERR_TENSOR_SHAPE;
    if (s.is_q) {
        R.op_arena.reset();
        void *raw = R.op_arena.get(nbytes, R.stream);
        if (!s.chunk) unpack_weights(s.q, raw, R.stream);
        else {
            const size_t piece = (size_t)s.chunk * s.q.nb * qweight_block_bytes(s.q.type);
            for (int64_t c = 0; c * s.chunk < s.rows; c++)
                unpack_weights(row_view(s.q, c * s.stride + s.row0, s.chunk), (char *)raw + c * piece, R.stream);
        }
        B200_CHECK(cudaMemcpyAsync(host, raw, nbytes, cudaMemcpyDeviceToHost, R.stream));
        B200_CHECK(cudaStreamSynchronize(R.stream));
    } else {
        B200_CHECK(cudaStreamSynchronize(R.stream));
        B200_CHECK(cudaMemcpy(host, s.f, nbytes, cudaMemcpyDeviceToHost));
    }
    return B200_OK;
}

StreamRing::StreamRing(int n, size_t host_bytes, size_t dev_bytes) : slots((size_t)n) {
    rt().ensure_init();
    for (Slot &s : slots) {
        B200_CHECK(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
        B200_CHECK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
        B200_CHECK(cudaHostAlloc((void **)&s.h, host_bytes, cudaHostAllocDefault));
        if (dev_bytes) B200_CHECK(cudaMalloc((void **)&s.d, dev_bytes));
    }
}

StreamRing::~StreamRing() {                 // no exit() here: it also runs while an exception unwinds
    for (Slot &s : slots) {
        cudaStreamSynchronize(s.st); cudaStreamDestroy(s.st); cudaEventDestroy(s.done);
        cudaFreeHost(s.h); if (s.d) cudaFree(s.d);
    }
}

void StreamRing::after(cudaStream_t st) {
    cudaEvent_t ev;
    B200_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    B200_CHECK(cudaEventRecord(ev, st));
    for (Slot &s : slots) B200_CHECK(cudaStreamWaitEvent(s.st, ev, 0));
    B200_CHECK(cudaEventDestroy(ev));        // released once the waits it feeds have completed
}

void SessionCore::start(int n_batch_, int n_ctx_, int n_vocab_, size_t kv_elems_, int kv_type_) {
    n_batch = n_batch_; n_ctx = n_ctx_; n_vocab = n_vocab_;
    kv_type = kv_type_; kv_elems = kv_elems_;
    memory_k = device_zeros<char>(kv_bytes());                  // offload_no_scratch zero-fills (LC/ggml-cuda.cu:3967-3973)
    memory_v = device_zeros<char>(kv_bytes());
    d_tokens = device_alloc<int32_t>((size_t)n_batch * 4);
    h_tokens = pinned_alloc<int32_t>((size_t)n_batch * 4);
    h_logits = pinned_alloc<float>((size_t)n_batch * n_vocab * 4);
    cudaEvent_t ev;
    B200_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    tokens_uploaded.reset(ev);
    B200_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    sampled.reset(ev);
    history = device_zeros<int32_t>((size_t)n_ctx * 4);
    sample_keys = device_alloc<uint64_t>(2 * sample_key_bytes(n_vocab));
    sample_fail = device_zeros<int>(sizeof(int));
    sample_backup = device_alloc<float>((size_t)n_vocab * 4);
    topk = device_alloc<int32_t>(2048 * 4);
    h_topk = pinned_alloc<int32_t>(2048 * 4);
    void *p = nullptr;
    B200_CHECK(cudaHostAlloc(&p, sizeof(SampleResult), cudaHostAllocMapped));    // the kernel writes the result straight into host memory
    h_sample.reset((SampleResult *)p);
    memset(p, 0, sizeof(SampleResult));
    B200_CHECK(cudaHostGetDevicePointer((void **)&d_sample, p, 0));
}

bool sampler_args(const b200_sampler *s, SampleArgs &a) {
    if (!s || s->top_k < 1 || s->repetition_last_n < 0 || !(s->temperature > 0.0f) || !(s->repetition_penalty > 0.0f) || s->top_p != s->top_p) return false;
    a = SampleArgs{s->repetition_penalty, s->repetition_last_n, s->top_k, s->top_p, s->temperature, s->seed, s->draw};
    return true;
}

// inference_session.rs:381-419.  The sampler's event is recorded before the step is enqueued, so the host learns the id while the step runs
// and the next call's sampler queues right behind it.
int SessionCore::infer_next_token(const SampleArgs &a, float *logits, const std::function<void()> &forward1, int32_t *token) {
    if (!token || last_n < 1) return B200_ERR_BAD_ARG;
    if (n_past + 1 >= n_ctx) return B200_ERR_CONTEXT_FULL;                                         // :388-390
    cudaStream_t st = rt().stream;
    const int row_n = last_n;
    float *row = logits + (size_t)(row_n - 1) * n_vocab;
    const SampleBufs b{{sample_keys.get(), sample_keys.get() + sample_key_bytes(n_vocab) / 8}, sample_fail.get(), sample_backup.get()};
    sample_row(row, n_vocab, history.get(), n_past, a, b, d_tokens.get(), history.get() + n_past, d_sample, nullptr, nullptr, nullptr, st);
    B200_CHECK(cudaEventRecord(sampled.get(), st));
    forward1();                                                                                    // :400 model.evaluate(self, &[next_token])
    B200_CHECK(cudaEventSynchronize(sampled.get()));
    const volatile SampleResult *r = h_sample.get();
    if (r->status != 0) {                                                                          // :392-397 SamplerFailure: undo the step
        B200_CHECK(cudaStreamSynchronize(st));
        n_past -= 1;                                                                               // the decode graphs re-upload their n_past
        last_n = row_n;
        B200_CHECK(cudaMemcpyAsync(row, sample_backup.get(), (size_t)n_vocab * 4, cudaMemcpyDeviceToDevice, st));
        B200_CHECK(cudaStreamSynchronize(st));
        return B200_ERR_SAMPLER_FAILURE;
    }
    *token = r->id;
    return B200_OK;
}

int SessionCore::top_k(const float *logits, int k, int32_t *ids_out, float *vals_out) {
    if (!ids_out || !vals_out || k < 1 || k > 1024 || k > n_vocab || last_n < 1) return B200_ERR_BAD_ARG;
    cudaStream_t st = rt().stream;
    const SampleArgs a{1.0f, 0, k, 1.0f, 1.0f, 0, 0};                                              // the top-k stage alone
    const SampleBufs b{{sample_keys.get(), sample_keys.get() + sample_key_bytes(n_vocab) / 8}, sample_fail.get(), nullptr};
    int32_t *d_ids = topk.get();
    float *d_vals = (float *)(topk.get() + 1024);
    sample_row(logits + (size_t)(last_n - 1) * n_vocab, n_vocab, nullptr, n_past, a, b, nullptr, nullptr, nullptr, d_ids, d_vals, nullptr, st);
    B200_CHECK(cudaMemcpyAsync(h_topk.get(), d_ids, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaMemcpyAsync(h_topk.get() + 1024, d_vals, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    memcpy(ids_out, h_topk.get(), (size_t)k * 4);
    memcpy(vals_out, h_topk.get() + 1024, (size_t)k * 4);
    return B200_OK;
}

int32_t SessionCore::read_tokens(int32_t *out, int32_t max) {
    if (max < 0 || (!out && max > 0)) return B200_ERR_BAD_ARG;
    const int32_t n = n_past < max ? n_past : max;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    if (n > 0) B200_CHECK(cudaMemcpy(out, history.get(), (size_t)n * 4, cudaMemcpyDeviceToHost));
    return n_past;
}

int SessionCore::last_logits(const float *logits, float *out) {
    if (!out || last_n < 1) return B200_ERR_BAD_ARG;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    B200_CHECK(cudaMemcpy(out, logits + (size_t)(last_n - 1) * n_vocab, (size_t)n_vocab * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
}

int SessionCore::read_kv(int which, void *host_out, size_t nbytes) {
    if (!host_out) return B200_ERR_BAD_ARG;
    if (nbytes != kv_bytes()) return B200_ERR_TENSOR_SHAPE;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    B200_CHECK(cudaMemcpy(host_out, which ? memory_v.get() : memory_k.get(), nbytes, cudaMemcpyDeviceToHost));
    return B200_OK;
}

int SessionCore::admit(int n) const {
    if (n < 1 || n > n_batch) return B200_ERR_BAD_ARG;
    if (n_past + n > n_ctx) return B200_ERR_CONTEXT_FULL;
    return B200_OK;
}

int SessionCore::stage_tokens(const int32_t *tokens, int n) {
    for (int i = 0; i < n; i++) if (tokens[i] < 0 || tokens[i] >= n_vocab) return B200_ERR_BAD_ARG;
    cudaStream_t st = rt().stream;
    B200_CHECK(cudaEventSynchronize(tokens_uploaded.get()));   // the previous (feed-only) call may still be reading the staging buffer
    memcpy(h_tokens.get(), tokens, (size_t)n * 4);
    B200_CHECK(cudaMemcpyAsync(d_tokens.get(), h_tokens.get(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(history.get() + n_past, h_tokens.get(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaEventRecord(tokens_uploaded.get(), st));
    return B200_OK;
}

void SessionCore::record_tokens(int n) {
    B200_CHECK(cudaMemcpyAsync(history.get() + n_past, d_tokens.get(), (size_t)n * 4, cudaMemcpyDeviceToDevice, rt().stream));
}

void SessionCore::copy_logits(float *out, const float *logits, int n, bool all_rows) {
    if (!out) return;
    cudaStream_t st = rt().stream;
    const size_t V = n_vocab, rows = all_rows ? n : 1;
    const float *src = all_rows ? logits : logits + (size_t)(n - 1) * V;
    B200_CHECK(cudaMemcpyAsync(h_logits.get(), src, rows * V * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    memcpy(out, h_logits.get(), rows * V * 4);
}

void SessionCore::copy_row(float *out, const float *row, int n) {
    if (!out) return;
    cudaStream_t st = rt().stream;
    B200_CHECK(cudaMemcpyAsync(out, row, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
}

void SessionCore::commit_step(int n, int launches) {
    n_past += n;
    last_n = n;
    last_launches = launches;
    decode.dev_n_past = -1;                     // the next graph step uploads n_past
}

// ---- batched steps (host.h: BatchCore) ---------------------------------------------------------------------------------------------------
// the device half of committing a batched step: row r's id to its session's history at its position, and (when the step computed them) its
// logits to its session's row
__global__ void commit_rows_kernel(const BatchRow *__restrict__ rows, const int32_t *__restrict__ ids, const float *__restrict__ logits, int n_vocab) {
    const BatchRow &r = rows[blockIdx.y];
    if (r.logits) {
        const float *src = logits + (size_t)r.lrow * n_vocab;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_vocab; i += gridDim.x * blockDim.x) r.logits[i] = src[i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) r.hist[r.pos] = ids[blockIdx.y];
}

const int32_t *decode_counts() {
    static const std::vector<int32_t> ones(B200_MAX_SESSIONS, 1);
    return ones.data();
}

// the step's tables for `rows` rows, packed in this order, each 16-byte aligned: BatchRow rows, int32 ids, warp rows, out rows, int2 tiles (at
// most one per row), then the chunks
static size_t tab_bytes(int rows) {
    auto a = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t R = rows;
    return a(R * sizeof(BatchRow)) + 3 * a(R * 4) + a(R * sizeof(int2)) + a(B200_MAX_SESSIONS * sizeof(BatchChunk));
}

void BatchCore::reserve(int n, int n_vocab, const BatchFront &f) {
    if (n <= cap) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));                  // the buffers being replaced may still be in use
    const size_t B = n;
    f.reserve(B);
    logits = device_alloc<float>(B * (size_t)n_vocab * 4);
    tab = device_alloc<char>(tab_bytes(n)); h_tab = pinned_alloc<char>(tab_bytes(n));
    if (!jobs) { jobs = device_alloc<SampleJob>(B200_MAX_SESSIONS * sizeof(SampleJob)); h_jobs = pinned_alloc<SampleJob>(B200_MAX_SESSIONS * sizeof(SampleJob)); }
    if (!staged) { cudaEvent_t ev; B200_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); staged.reset(ev); }
    cap = n;
}

// one batched step of sessions ss[0, n), session i on tokens [sum counts[0, i), + counts[i]) (checked by the caller): stage the tables, run
// forward_rows, commit every row.  Only each chunk's last row reaches the final norm and the lm_head unless all_logits (as in the single
// evaluate), through a gather when some chunk has more than one row.  logits_out (nullable): every row (all_logits), else each chunk's last.
void BatchCore::step(const BatchSession *ss, int n, const int32_t *counts, const int32_t *tokens, float *logits_out, bool all_logits, const BatchFront &f) {
    cudaStream_t st = rt().stream;
    const int V = ss[0].s->n_vocab;
    int rows_n = 0;
    bool ones = true;
    for (int i = 0; i < n; i++) { rows_n += counts[i]; ones &= counts[i] == 1; }
    reserve(rows_n, V, f);
    B200_CHECK(cudaEventSynchronize(staged.get()));
    size_t off = 0;
    auto carve = [&](size_t bytes) { const size_t o = off; off += (bytes + 15) & ~(size_t)15; return o; };
    const size_t o_rows = carve(rows_n * sizeof(BatchRow)), o_ids = carve(rows_n * 4), o_warp = carve(rows_n * 4), o_out = carve(rows_n * 4),
                 o_tiles = carve(rows_n * sizeof(int2)), o_chunks = carve(n * sizeof(BatchChunk));
    char *h = h_tab.get();
    BatchRow *hr = (BatchRow *)(h + o_rows);
    int32_t *hid = (int32_t *)(h + o_ids), *hw = (int32_t *)(h + o_warp), *ho = (int32_t *)(h + o_out);
    int2 *ht = (int2 *)(h + o_tiles);
    BatchChunk *hc = (BatchChunk *)(h + o_chunks);
    const bool gather = !all_logits && !ones;
    int n_warp = 0, max_warp = 0, n_tiles = 0, max_tiles = 0, n_chunks = 0;
    for (int i = 0, r = 0; i < n; i++) {
        SessionCore *s = ss[i].s;
        const int c = counts[i], n_kv = s->n_past + c;
        const bool tiled = f.tiled && c >= ATTN_TILED_MIN_ROWS;                         // mul_mat_attn's choice for the chunk's single evaluate
        if (tiled) {
            hc[n_chunks] = BatchChunk{s->memory_k.get(), s->memory_v.get(), r, c, s->n_past};
            for (int t = 0; t * ATTN_TILE_ROWS < c; t++) ht[n_tiles++] = make_int2(n_chunks, t);
            n_chunks++;
            max_tiles = std::max(max_tiles, n_kv);
        } else {
            max_warp = std::max(max_warp, n_kv);
        }
        for (int j = 0; j < c; j++, r++) {
            const bool out = all_logits || j == c - 1;
            hr[r] = BatchRow{s->memory_k.get(), s->memory_v.get(), out ? ss[i].logits + (size_t)j * V : nullptr, s->history.get(), s->n_past + j, n_kv,
                             out ? (all_logits ? r : i) : -1};
            hid[r] = tokens[r];
            if (!tiled) hw[n_warp++] = r;
            if (gather && j == c - 1) ho[i] = r;
        }
    }
    B200_CHECK(cudaMemcpyAsync(tab.get(), h, off, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaEventRecord(staged.get(), st));
    const char *d = tab.get();
    const int n_out = all_logits ? rows_n : n;
    const BatchStep p{rows_n, ss[0].s->kv_type, (const BatchRow *)(d + o_rows), (const int32_t *)(d + o_ids),
                      (const int32_t *)(d + o_warp), n_warp, max_warp, (const BatchChunk *)(d + o_chunks), (const int2 *)(d + o_tiles), n_tiles, max_tiles,
                      gather ? (const int32_t *)(d + o_out) : nullptr, n_out, logits.get()};
    int L = f.forward_rows(p);
    commit_rows_kernel<<<dim3((unsigned)std::min((V + 255) / 256, 64), (unsigned)rows_n), 256, 0, st>>>(p.rows, p.ids, logits.get(), V); L++;
    B200_CHECK(cudaGetLastError());
    for (int i = 0; i < n; i++) ss[i].s->commit_step(counts[i], L);
    if (logits_out) {
        B200_CHECK(cudaMemcpyAsync(logits_out, logits.get(), (size_t)n_out * V * 4, cudaMemcpyDeviceToHost, st));
        B200_CHECK(cudaStreamSynchronize(st));
    }
}

int BatchCore::evaluate(const BatchSession *ss, int n, const int32_t *counts, const int32_t *tokens, float *logits_out, bool all_logits,
                        const BatchFront &f) {
    if (!counts || !tokens) return B200_ERR_BAD_ARG;
    int64_t rows = 0;
    for (int i = 0; i < n; i++) {
        if (counts[i] < 1 || counts[i] > ss[i].s->n_batch) return B200_ERR_BAD_ARG;          // the single-session evaluate's rule (admit)
        rows += counts[i];
    }
    if (rows > B200_MAX_BATCH_ROWS) return B200_ERR_BAD_ARG;
    for (int64_t r = 0; r < rows; r++) if (tokens[r] < 0 || tokens[r] >= ss[0].s->n_vocab) return B200_ERR_BAD_ARG;
    for (int i = 0; i < n; i++) if (const int rc = ss[i].s->admit(counts[i])) return rc;
    step(ss, n, counts, tokens, logits_out, all_logits, f);
    return B200_OK;
}

// infer_next_token for n sessions: the batched sampler on each session's last row, then (once its results are in) one batched step over the
// sessions whose sampler succeeded.  A failed session is not stepped at all, so its state is what it was.
int BatchCore::infer(const BatchSession *ss, int n, const b200_sampler *samplers, int32_t *tokens_out, int32_t *status_out, const BatchFront &f) {
    if (!samplers || !tokens_out || !status_out) return B200_ERR_BAD_ARG;
    SampleArgs a[B200_MAX_SESSIONS];
    for (int i = 0; i < n; i++) if (!sampler_args(&samplers[i], a[i]) || ss[i].s->last_n < 1) return B200_ERR_BAD_ARG;
    for (int i = 0; i < n; i++) if (ss[i].s->n_past + 1 >= ss[i].s->n_ctx) return B200_ERR_CONTEXT_FULL;   // the single-session infer's rule
    cudaStream_t st = rt().stream;
    const int V = ss[0].s->n_vocab;
    reserve(n, V, f);
    B200_CHECK(cudaEventSynchronize(staged.get()));
    int max_kk = 1;
    for (int i = 0; i < n; i++) {
        SessionCore *s = ss[i].s;
        const SampleBufs b{{s->sample_keys.get(), s->sample_keys.get() + sample_key_bytes(V) / 8}, s->sample_fail.get(), nullptr};
        h_jobs.get()[i] = SampleJob{ss[i].logits + (size_t)(s->last_n - 1) * V, s->history.get(), V, s->n_past, a[i], b, nullptr, nullptr, s->d_sample};
        max_kk = std::max(max_kk, sample_kk(a[i].top_k, V));
    }
    B200_CHECK(cudaMemcpyAsync(jobs.get(), h_jobs.get(), (size_t)n * sizeof(SampleJob), cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaEventRecord(staged.get(), st));
    sample_rows(jobs.get(), n, V, max_kk, st);
    B200_CHECK(cudaStreamSynchronize(st));
    BatchSession ok[B200_MAX_SESSIONS];
    int32_t ids_ok[B200_MAX_SESSIONS];
    int k = 0;
    for (int i = 0; i < n; i++) {
        const volatile SampleResult *r = ss[i].s->h_sample.get();
        if (r->status != 0) { status_out[i] = B200_ERR_SAMPLER_FAILURE; tokens_out[i] = -1; continue; }
        status_out[i] = B200_OK; tokens_out[i] = r->id;
        ok[k] = ss[i]; ids_ok[k++] = r->id;
    }
    if (k) step(ok, k, decode_counts(), ids_ok, nullptr, false, f);
    return B200_OK;
}

int SessionCore::set_n_past(int v) {
    if (v < 0 || v > n_past) return B200_ERR_BAD_ARG;
    n_past = v;
    return B200_OK;
}

// inference_session.rs:514-589, except that every chunk starts at n_past 0 (the reference never rewinds, so its chunk 1 would run past the end of
// the KV cache); chunk 0 is exactly the reference's loop on a fresh session
int SessionCore::perplexity(const int32_t *tokens, int64_t n, int32_t bos, float *ppl_out, float *terms_out, int32_t *n_chunk_out, const float *logits,
                            const std::function<void(int)> &forward) {
    if ((!tokens && n > 0) || n < 0 || !n_chunk_out || bos < 0 || bos >= n_vocab) return B200_ERR_BAD_ARG;
    for (int64_t i = 0; i < n; i++) if (tokens[i] < 0 || tokens[i] >= n_vocab) return B200_ERR_BAD_ARG;
    const int64_t C = n_ctx, n_chunk = n / C;
    if (n_chunk > INT32_MAX || (n_chunk > 0 && !ppl_out)) return B200_ERR_BAD_ARG;
    *n_chunk_out = (int32_t)n_chunk;
    if (n_chunk == 0) return B200_OK;
    const int64_t first = C / 2 < 512 ? C / 2 : 512, scored = C - 1 > first ? C - 1 - first : 0;
    cudaStream_t st = rt().stream;
    DeviceBuf<int32_t> d_tok = device_alloc<int32_t>((size_t)n_chunk * C * 4);                    // the targets t[iC + j + 1]
    DeviceBuf<float> d_terms = device_alloc<float>(((size_t)n_chunk * scored + 1) * 4), d_ppl = device_alloc<float>((size_t)n_chunk * 4);
    DeviceBuf<PplState> state = device_alloc<PplState>(sizeof(PplState));
    B200_CHECK(cudaMemcpyAsync(d_tok.get(), tokens, (size_t)n_chunk * C * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemsetAsync(state.get(), 0, sizeof(PplState), st));                             // nll = 0.0f, count = 0
    std::vector<int32_t> batch(n_batch);
    for (int64_t i = 0; i < n_chunk; i++) {
        const int64_t start = i * C;
        n_past = 0;
        for (int64_t b0 = 0; b0 < C; b0 += n_batch) {
            const int nb = (int)(C - b0 < n_batch ? C - b0 : n_batch);
            memcpy(batch.data(), tokens + start + b0, (size_t)nb * 4);
            if (b0 == 0) batch[0] = bos;                                                          // the chunk's first token, not each batch's
            stage_tokens(batch.data(), nb);                                                       // ids checked above
            forward(nb);
            const int64_t r0 = b0 > first ? b0 : first, r1 = b0 + nb < C - 1 ? b0 + nb : C - 1;   // scored rows of this batch
            if (r1 > r0) nll_rows(logits + (size_t)(r0 - b0) * n_vocab, r1 - r0, n_vocab, d_tok.get() + start + r0 + 1, d_terms.get() + i * scored + (r0 - first), st);
        }
        nll_fold(d_terms.get() + i * scored, scored, state.get(), d_ppl.get() + i, st);
    }
    B200_CHECK(cudaMemcpyAsync(ppl_out, d_ppl.get(), (size_t)n_chunk * 4, cudaMemcpyDeviceToHost, st));
    if (terms_out && scored) B200_CHECK(cudaMemcpyAsync(terms_out, d_terms.get(), (size_t)n_chunk * scored * 4, cudaMemcpyDeviceToHost, st));
    B200_CHECK(cudaStreamSynchronize(st));
    return B200_OK;
}

}  // namespace b200
