// llm_b200/csrc/host.h -- host plumbing shared by the LLaMA (session.cu) and GPT-NeoX / GPT-2 (neox.cu) runtimes: owned device and pinned
// buffers, the weight slab and its named tensor slots, seeded synthesis, and the state every session keeps (KV cache, token / logits staging).
#pragma once
#include <string.h>

#include <functional>
#include <memory>
#include <type_traits>
#include <vector>

#include "../../include/llm_b200.h"
#include "decode.h"
#include "kernels.cuh"
#include "runtime.h"

namespace b200 {

// ---- owned allocations: one cudaMalloc / cudaMallocHost / event each, released with the struct that holds the handle ---------------
struct DeviceFree { void operator()(void *p) const { B200_CHECK(cudaFree(p)); } };
struct PinnedFree { void operator()(void *p) const { B200_CHECK(cudaFreeHost(p)); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { B200_CHECK(cudaEventDestroy(e)); } };
template <class T> using DeviceBuf = std::unique_ptr<T, DeviceFree>;
template <class T> using PinnedBuf = std::unique_ptr<T, PinnedFree>;
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;

template <class T> DeviceBuf<T> device_alloc(size_t bytes) { void *p = nullptr; B200_CHECK(cudaMalloc(&p, bytes)); return DeviceBuf<T>((T *)p); }
// the memset runs on the legacy stream: the caller orders it before the backend's non-blocking stream (cudaDeviceSynchronize)
template <class T> DeviceBuf<T> device_zeros(size_t bytes) { DeviceBuf<T> b = device_alloc<T>(bytes); B200_CHECK(cudaMemset(b.get(), 0, bytes)); return b; }
template <class T> PinnedBuf<T> pinned_alloc(size_t bytes) { void *p = nullptr; B200_CHECK(cudaMallocHost(&p, bytes)); return PinnedBuf<T>((T *)p); }

QWeight row_view(const QWeight &w, int64_t row0, int64_t nrows);   // rows [row0, row0+nrows) of a planes matrix

// ---- the weights of one model -------------------------------------------------------------------------------------------------
// One pass over a model's tensors in slab order: the sizing pass (base == nullptr) only advances `off`, the placing pass also points each tensor
// into the slab. Quantized matrices take qweight_layout's bytes, f32 vectors are padded to 256 bytes.  A matrix is of `wtype` unless the layout
// passes its own type (a per-tensor type of the model file).
struct SlabCarver {
    int wtype; char *base;
    size_t off = 0, streamed = 0;       // streamed: GGML bytes of every matrix carved
    void q(QWeight &w, int64_t K, int64_t N, int type = -1) {
        off += qweight_layout(w, type < 0 ? wtype : type, K, N, base ? base + off : nullptr);
        streamed += (size_t)N * w.nb * qweight_block_bytes(w.type);
    }
    void f(float *&p, int64_t n) { if (base) p = (float *)(base + off); off += ((size_t)n * 4 + 255) & ~(size_t)255; }
};

// The k-th tensor drawn gets seed + 0x1000003 * k, so a model's synthetic weights depend on the order of the draws.
struct SeedSeq {
    uint64_t seed; cudaStream_t st; uint64_t id = 0;
    uint64_t next() { return seed + 0x1000003ull * (++id); }
    void q(const QWeight &w) { synth_qweight(w, next(), st); }                       // N(0, 1/K) quantized by the reference's rule
    void gain(float *p, int64_t n) { synth_gain(p, n, next(), st); }                 // 1 + 0.1 N(0,1)
    void bias(float *p, int64_t n) { synth_gain(p, n, next(), st); scale_shift_f32(p, n, 0.1f, -0.1f, st); }   // 0.01 N(0,1)
};

// One HBM slab holding every weight, and which of the model's named tensors have been loaded into it.
struct Weights {
    DeviceBuf<char> slab;
    size_t slab_bytes = 0, weight_bytes = 0;    // weight_bytes: what one forward pass streams (the front end takes out the gathered-only embedding)
    std::vector<uint8_t> loaded;                // per tensor slot
    int n_loaded = 0;

    // layout(SlabCarver &) carves the tensors: run once to size the slab, then once more to place them in it
    template <class Layout> void carve(int wtype, int n_slots, Layout &&layout) {
        SlabCarver size{wtype, nullptr};
        layout(size);
        slab_bytes = size.off;
        slab = device_alloc<char>(slab_bytes);
        SlabCarver place{wtype, slab.get()};
        layout(place);
        weight_bytes = place.streamed;
        loaded.assign(n_slots, 0);
    }
    void mark(int id) { if (!loaded[id]) { loaded[id] = 1; n_loaded++; } }
    bool all_loaded() const { return n_loaded == (int)loaded.size(); }
    // seeded synthetic weights generated in HBM (bench): draw(SeedSeq &) fills every tensor
    template <class Draw> void synthesize(uint64_t seed, Draw &&draw) {
        SeedSeq seq{seed, rt().stream};
        draw(seq);
        B200_CHECK(cudaStreamSynchronize(rt().stream));
        loaded.assign(loaded.size(), 1);
        n_loaded = (int)loaded.size();
    }
};

// Where a named tensor lives in the slab: a quantized matrix `q` or `n` floats at `f`.
// chunk > 0: the tensor's rows live in `chunk`-row pieces, piece c at rows [c * stride + row0, + chunk) of the matrix `q`
// (LLaMA's w1 / w3 are interleaved in 32-row pieces inside w13 so that 64 consecutive rows hold both factors of 32 silu*mul outputs)
struct Slot {
    QWeight q; float *f = nullptr; int64_t n = 0; bool is_q = false; int chunk = 0; int64_t row0 = 0, stride = 0, rows = 0;
    bool f16_src = false;     // f32 slot that also takes F16 bytes, widened (exactly) to f32 on upload
    int64_t q_rows() const { return chunk ? rows : q.N; }
    size_t bytes() const { return is_q ? (size_t)q_rows() * q.nb * qweight_block_bytes(q.type) : (size_t)n * 4; }
};
// The LoRA adapters of one tensor load: the tensor's name and shape [ne0, ne1] (ne1 = 1 for a vector) and the adapter files, applied in order
struct LoraTarget { const char *name; int64_t ne0, ne1; const b200_ggml_file *const *adapters; int n; };
// GGML blocks (repacked on the GPU) or f32; B200_OK / B200_ERR_TENSOR_SHAPE, or the adapters' LoadError.  With `lora`, every adapter whose patch set
// names the tensor patches its bytes in file layout after the upload and before they are placed (lora.cu).
int load_slot(const Slot &s, int32_t type, const void *host, size_t nbytes, const LoraTarget *lora = nullptr);
int read_slot(const Slot &s, void *host, size_t nbytes);                       // the inverse: GGML blocks or f32 back to the host

// a 2-D weight of a LLaMA model of n_layer layers: tok_embeddings / output / layers.<i>.attention.w[qkvo] / layers.<i>.feed_forward.w[123] (session.cu)
bool llama_matrix_name(const char *name, int n_layer);
// a 2-D weight of a GPT-NeoX-family model (b200_neox_hparams.arch) of n_layer layers: a matrix, or one of GPT-J's q_proj / k_proj / v_proj (neox.cu)
bool neox_matrix_name(int arch, const char *name, int n_layer);

// ---- adapter files (ggml_file.cu) ----
int64_t ggml_find_tensor(const b200_ggml_file *f, const char *name);        // index in the tensor table, -1 if absent
bool lora_in_patch_set(const b200_ggml_file *f, const char *name);          // some tensor of the adapter is `name` + "." + a last component
float lora_scaling(const b200_ggml_file *f);                                // (f32)alpha / (f32)r
// ---- model files written by b200_ggml_write and the quantizer (ggml_file.cu) ----
const char *ggml_tensor_name(const b200_ggml_file *f, int64_t i, size_t *len);     // tensor i's whole name (not NUL-terminated)
// a tensor record: header, name and (GGJT) the zero padding to the next 32-byte offset of the file; false on a write error
bool ggml_write_record(FILE *fp, const char *name, size_t name_len, int32_t n_dims, int32_t type, const int64_t *ne, bool align);

// ---- streaming between host files and HBM in bounded memory (the model quantizer, session snapshots) ------------------------------------
// `n` slots, each with its own stream, a completion event and a pinned and a device buffer.  Chunk c uses slot c % n: the caller waits for the
// slot's previous chunk (retire) before refilling it, so chunk c's copies overlap the host work on chunks c - n + 1 .. c - 1.
struct StreamRing {
    struct Slot {
        cudaStream_t st = nullptr; cudaEvent_t done = nullptr;
        char *h = nullptr, *d = nullptr;
        size_t bytes = 0;               // the chunk's payload (the caller's bookkeeping)
        bool busy = false;              // work recorded on `done` has not been retired
    };
    std::vector<Slot> slots;
    StreamRing(int n, size_t host_bytes, size_t dev_bytes);
    ~StreamRing();                      // waits for every slot, then frees
    StreamRing(const StreamRing &) = delete;
    StreamRing &operator=(const StreamRing &) = delete;
    Slot &at(int64_t chunk) { return slots[(size_t)(chunk % (int64_t)slots.size())]; }
    void after(cudaStream_t st);        // every slot's later work is ordered after what `st` has queued so far
    static void wait(Slot &s) { if (s.busy) { B200_CHECK(cudaEventSynchronize(s.done)); s.busy = false; } }
    void drain() { for (Slot &s : slots) wait(s); }
};

// ---- session snapshots (snapshot.cu): the reference's cache layout, which a front end describes ----------------------------------------
// The reference sizes memory_k / memory_v as n_layer x n_ctx x ref_width values and uses the first n_layer x n_ctx x width of them: K as
// [n_layer][n_ctx][width], V as [n_layer][width][n_ctx], or [n_layer][n_ctx][width] when v_by_position (GPT-2, MPT, BLOOM).  The native cache is
// [n_layer][n_ctx][width] and [n_layer][width][n_ctx] for every architecture.
struct RefKvLayout { int n_layer; int64_t width, ref_width; bool v_by_position; };
// one source of snapshot bytes (a caller's buffer or a session file), read in order; false on a read error
using SnapshotSource = std::function<bool(void *dst, size_t n)>;

// ---- what every session keeps: the KV cache, the position, token and logits staging, the decode graphs -------------------------------
struct SessionCore {
    int n_batch = 0, n_ctx = 0, n_vocab = 0;
    int n_past = 0, last_launches = 0;
    int last_n = 0;                     // rows of the last evaluate: its last row (last_n - 1) is InferenceSession::last_logits
    // memory_k / memory_v of InferenceSessionConfig::memory_k_type / memory_v_type (one type for both): T_F16 (the default) or T_F32
    int kv_type = T_F16;
    size_t kv_elems = 0;                // elements of each
    DeviceBuf<char> memory_k, memory_v;
    DeviceBuf<int32_t> d_tokens; PinnedBuf<int32_t> h_tokens;
    PinnedBuf<float> h_logits;          // n_batch rows of n_vocab
    Event tokens_uploaded;              // guards reuse of h_tokens by the next evaluate()
    DecodeGraphCache decode;            // the decode graphs and the device copy of n_past they read
    DeviceBuf<int32_t> history;         // InferenceSession::tokens: the ids at positions [0, n_past) (n_ctx slots; a rewind truncates implicitly)
    // the sampler (sample.cu): key buffers, fail word, the row kept on a failure, top-k output; its result word in mapped pinned memory
    DeviceBuf<uint64_t> sample_keys; DeviceBuf<int> sample_fail; DeviceBuf<float> sample_backup;
    DeviceBuf<int32_t> topk; PinnedBuf<int32_t> h_topk;                 // 1024 ids + 1024 logits each (top_k)
    PinnedBuf<SampleResult> h_sample; SampleResult *d_sample = nullptr;
    Event sampled;                      // recorded after the sampler, before the step it feeds

    // zero-filled KV cache of kv_elems values of kv_type (T_F16 / T_F32) each for K and V
    void start(int n_batch, int n_ctx, int n_vocab, size_t kv_elems, int kv_type);
    size_t kv_elem_bytes() const { return kv_type == T_F32 ? 4 : 2; }
    size_t kv_bytes() const { return kv_elems * kv_elem_bytes(); }      // of each of memory_k, memory_v
    // element offset `elems` into memory_k (which = 0) or memory_v (1), in bytes of the cache's type
    void *kv_at(int which, size_t elems) const { return (which ? memory_v : memory_k).get() + elems * kv_elem_bytes(); }
    int read_kv(int which, void *host_out, size_t nbytes);            // the raw cache bytes; B200_ERR_TENSOR_SHAPE unless nbytes == kv_bytes()
    int admit(int n) const;             // B200_ERR_BAD_ARG unless 1 <= n <= n_batch, B200_ERR_CONTEXT_FULL if n more positions do not fit
    int stage_tokens(const int32_t *tokens, int n);   // validates the ids and uploads them to d_tokens (and to the history at n_past)
    void record_tokens(int n);          // d_tokens[0, n) -> history at n_past (evaluate entry points whose ids are already in HBM)
    void copy_logits(float *out, const float *logits, int n, bool all_rows);   // rows [0, n) of logits, or only row n - 1, to out (if not null)
    void copy_row(float *out, const float *row, int n);                        // n floats of a device row to out (if not null), after the queued work
    int set_n_past(int v);
    // the host half of committing a batched step of n tokens to this session (its device half, history[n_past, n_past + n) and the logits rows, is
    // the step's commit kernel): n_past + n, last_n n, the step's launches, and the decode graphs' device n_past stale
    void commit_step(int n, int launches);
    // InferenceSession::perplexity over tokens[0, n) with C = n_ctx: chunk i = [iC, (i+1)C) is evaluated from n_past 0 in batches of n_batch, its
    // first token replaced by bos; rows [min(512, C/2), C - 1) are scored on the device (ppl.cu).  forward(rows) runs one batch of the staged
    // tokens at n_past and leaves every row's logits in `logits`.  Each batch's terms are computed on the stream before the next batch overwrites
    // them.  ppl_out: n_chunk values; terms_out (nullable): n_chunk x scored rows.  n_past ends at C (unchanged when n < C).
    int perplexity(const int32_t *tokens, int64_t n, int32_t bos, float *ppl_out, float *terms_out, int32_t *n_chunk_out, const float *logits,
                   const std::function<void(int)> &forward);
    // InferenceSession::infer_next_token: the sampler on the last row of `logits` writes the id into d_tokens[0] and the history, then
    // forward1() enqueues the one-token step (it reads d_tokens and advances n_past); the host waits on the sampler's event only.
    // B200_ERR_CONTEXT_FULL (nothing enqueued), B200_ERR_SAMPLER_FAILURE (n_past, history and the row restored), B200_ERR_BAD_ARG.
    int infer_next_token(const SampleArgs &a, float *logits, const std::function<void()> &forward1, int32_t *token);
    // the k (<= 1024, <= n_vocab) largest logits of the last row, descending, ties by ascending id
    int top_k(const float *logits, int k, int32_t *ids_out, float *vals_out);
    int32_t read_tokens(int32_t *out, int32_t max);                    // min(n_past, max) ids of the history; returns n_past
    int last_logits(const float *logits, float *out);                 // the last evaluated row, n_vocab floats

    // InferenceSession::get_snapshot (snapshot.cu): the scalars and counts always; with the four pointers set, their contents (the counts must be
    // the session's), ordered after the work queued on the backend stream.  last_logits: the last row of `logits`, zeros before any evaluate.
    int get_snapshot(const RefKvLayout &L, const float *logits, b200_snapshot *snap);
    int write_snapshot(const RefKvLayout &L, const float *logits, const char *path);   // the same as a session file, streamed
    // the second half of InferenceSession::from_snapshot on a fresh session whose type and n_batch are the snapshot's (checked by
    // snapshot_check): the cache from k / v (the reference's bytes, in order), n_past, the history and the last row (row 0 of `logits`, last_n 1)
    int restore_snapshot(const RefKvLayout &L, float *logits, const b200_snapshot &h, const SnapshotSource &k, const SnapshotSource &v);
};

// ---- InferenceSession::from_snapshot for a front end (snapshot.cu) ------------------------------------------------------------------------
// A parsed session file: its scalars and counts in `h` (tokens / last_logits point into the vectors below, the memory pointers are null), and
// the cache bytes, read on demand.
struct SnapshotFile {
    b200_snapshot h{};
    std::vector<uint32_t> tokens; std::vector<float> last_logits;
    std::shared_ptr<void> reader;       // the zstd frame reader, positioned at memory_k's bytes
    SnapshotSource k, v;
};
int snapshot_read_file(const char *path, SnapshotFile &f, bool with_data);    // B200_OK, B200_ERR_IO, B200_ERR_SNAPSHOT_FORMAT
// every refusal of from_snapshot for a model of context n_ctx, n_vocab ids and cache layout L: BAD_ARG, SNAPSHOT_SIZE_MISMATCH
int snapshot_check(const b200_snapshot &h, int n_ctx, int n_vocab, const RefKvLayout &L);
// start(n_batch, kv_f32, logits) starts the front end's session (nullptr: refused) and sets `logits` to its logits buffer; release(s) frees it
// when a session file fails to read after it was started.  snap (in memory) or path (a session file) is checked before the session is started.
template <class Sess, class Start, class Release>
Sess *session_from_snapshot(const b200_snapshot *snap, const char *path, int n_ctx, int n_vocab, const RefKvLayout &L, int *err, Start &&start,
                            Release &&release) {
    SnapshotFile file;
    int rc = B200_OK;
    if (path) rc = snapshot_read_file(path, file, true);
    else if (!snap) rc = B200_ERR_BAD_ARG;
    const b200_snapshot &h = path ? file.h : *snap;
    if (rc == B200_OK) rc = snapshot_check(h, n_ctx, n_vocab, L);
    if (rc == B200_OK && !path && (!h.memory_k || !h.memory_v)) rc = B200_ERR_BAD_ARG;
    Sess *s = nullptr;
    float *logits = nullptr;
    if (rc == B200_OK && !(s = start((int)h.n_batch, h.memory_k_type == 1, logits))) rc = B200_ERR_BAD_ARG;
    if (rc == B200_OK) {
        size_t ko = 0, vo = 0;
        const SnapshotSource mk = [&](void *d, size_t n) { memcpy(d, (const char *)h.memory_k + ko, n); ko += n; return true; };
        const SnapshotSource mv = [&](void *d, size_t n) { memcpy(d, (const char *)h.memory_v + vo, n); vo += n; return true; };
        rc = s->restore_snapshot(L, logits, h, path ? file.k : mk, path ? file.v : mv);
        if (rc != B200_OK) { release(s); s = nullptr; }
    }
    if (err) *err = rc;
    return rc == B200_OK ? s : nullptr;
}
// a b200_sampler as the kernels take it; false if it is out of range (top_k < 1, temperature or penalty <= 0 or NaN, last_n < 0, top_p NaN)
bool sampler_args(const b200_sampler *s, SampleArgs &a);

// ---- batched steps: one step for n sessions of one model, each evaluating a chunk of its own (b200_model_evaluate_ragged,
// b200_neox_evaluate_ragged; the decode steps b200_*_evaluate_sessions / b200_*_infer_next_tokens are the steps whose chunks are one token) -----
// One session of a batched call: its core and its logits buffer (row j takes the row of its chunk's token j).
struct BatchSession { SessionCore *s; float *logits; };
// The refusals of a batched call that depend only on its sessions (B200_ERR_BAD_ARG or B200_OK): n outside [1, B200_MAX_SESSIONS], a null
// entry, a session whose model is not m, the same session twice, sessions whose KV cache types differ.  Fills out[0, n) when it accepts.
template <class M, class S> int batch_sessions(const M *m, S *const *ss, int n, BatchSession *out) {
    if (!m || !ss || n < 1 || n > B200_MAX_SESSIONS) return B200_ERR_BAD_ARG;
    for (int i = 0; i < n; i++) {
        S *s = ss[i];
        if (!s || s->m != m || s->kv_type != ss[0]->kv_type) return B200_ERR_BAD_ARG;
        for (int j = 0; j < i; j++) if (ss[j] == s) return B200_ERR_BAD_ARG;
        out[i] = BatchSession{s, s->logits.get()};
    }
    return B200_OK;
}
// the counts of a decode step: B200_MAX_SESSIONS ones
const int32_t *decode_counts();
// The front end's half of a batched step.  reserve(n): grow its activations to n rows (the stream is idle when it is called).
// forward_rows(p): enqueue the forward pass of the step's p.n staged rows into p.logits, every row's arithmetic that of its chunk's single-session
// forward, and return its launches.  tiled: the tiled attention takes the front end's strides (attn_tiles_aligned).
struct BatchFront {
    std::function<void(size_t n)> reserve;
    std::function<int(const BatchStep &p)> forward_rows;
    bool tiled;
};
// What a model keeps for its batched steps: the step's tables (rows, ids, the attention plan, the logits rows) in one pinned and one device
// buffer, the sampler jobs, and the logits of up to `cap` rows, grown on demand to the largest step seen and freed with the model.
struct BatchCore {
    int cap = 0;
    DeviceBuf<float> logits;
    DeviceBuf<char> tab; PinnedBuf<char> h_tab;
    DeviceBuf<SampleJob> jobs; PinnedBuf<SampleJob> h_jobs;
    Event staged;                       // recorded after the uploads: the pinned tables are not rewritten before they have been read

    // b200_model_evaluate_ragged over sessions ss[0, n) that batch_sessions accepted: the counts, the ids and the context checked, then one step
    int evaluate(const BatchSession *ss, int n, const int32_t *counts, const int32_t *tokens, float *logits_out, bool all_logits, const BatchFront &f);
    // b200_model_infer_next_tokens over accepted sessions: the samplers checked, every row sampled, then one step of the sessions that sampled
    int infer(const BatchSession *ss, int n, const b200_sampler *samplers, int32_t *tokens_out, int32_t *status_out, const BatchFront &f);

private:
    void reserve(int rows, int n_vocab, const BatchFront &f);
    void step(const BatchSession *ss, int n, const int32_t *counts, const int32_t *tokens, float *logits_out, bool all_logits, const BatchFront &f);
};

}  // namespace b200
