/*
 * include/llm_b200.h -- native host runtime of libllm_b200.so: the reference's model/session interface for the
 * LLaMA graph, as a C ABI (the reference's own host layer is Rust; no Rust toolchain exists here, so the same interface
 * is offered to C / ctypes callers -- see INTEGRATION.md for the Rust `extern "C"` block that binds it).
 *
 * Names, argument meaning and error behaviour mirror:
 *   Hyperparameters                 crates/models/llama/src/lib.rs:403-447
 *   ModelParameters                 crates/llm-base/src/model/mod.rs:197-229   (context_size, rope overrides)
 *   KnownModel::new / TensorLoader  crates/models/llama/src/lib.rs:43-140      (tensor names "layers.N.attention.wq.weight", ...)
 *   KnownModel::start_session       crates/models/llama/src/lib.rs:130-141  -> InferenceSession::new (inference_session.rs:114-217)
 *   InferenceSessionConfig          crates/llm-base/src/inference_session.rs:799-841 (n_batch; memory_k_type / memory_v_type: f16, or f32 with
 *                                   B200_SESSION_KV_F32 -- the CLI's --no-float16)
 *   Model::evaluate + OutputRequest crates/models/llama/src/lib.rs:144-368, crates/llm-base/src/model/common.rs:6-39
 *   InferenceSession::feed_prompt   crates/llm-base/src/inference_session.rs:299-350 (chunks of n_batch, ContextFull)
 *
 * Where the per-node seam (ggml_b200.h) replays the reference's graph one node per call, this front end owns the whole
 * forward pass: a static schedule of fused sm_90a kernels (captured as a CUDA graph for decode), weights and KV cache
 * resident in HBM.  Both front ends run the same kernels and are held to the same parity bar.
 *
 * Threading / device contract: one process drives ONE device (b200_init picks it; multi-GPU = one process per GPU, see b200_llama_new_tp), and
 * the entry points of this header are to be called from one host thread at a time -- the launch code keeps per-process caches (kernel attributes,
 * occupancy tables, the RoPE / LUT tables) that are not synchronised.  Everything is ordered on the backend's single non-blocking stream.
 * b200_session_evaluate validates token ids; b200_session_evaluate_device takes them from HBM unchecked: ids in [0, n_vocab) are its precondition.
 */
#ifndef LLM_B200_H
#define LLM_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_model b200_model;
typedef struct b200_session b200_session;

typedef struct {
    int32_t n_vocab, n_embd, n_head, n_head_kv, n_layer, n_rot, n_ff;
    int32_t wtype;            /* enum ggml_type of the 2-D weights: 1 F16, 2 Q4_0, 3 Q4_1, 6 Q5_0, 7 Q5_1, 8 Q8_0, 10..14 Q2_K..Q6_K
                                 (b200_llama_new_typed: of the weights its table does not name) */
    int32_t context_size;     /* ModelParameters::context_size (default 2048) */
    float   rope_freq_base;   /* RoPEOverrides::frequency_base (10000) */
    float   rope_freq_scale;  /* RoPEOverrides::frequency_scale (1) */
} b200_llama_hparams;

typedef struct {
    int32_t n_batch;          /* InferenceSessionConfig::n_batch: largest evaluate() batch; reference default 8, prefill@512 uses 512 */
    int32_t flags;            /* B200_SESSION_* */
} b200_session_config;

enum {
    B200_SESSION_NO_GRAPH = 1,     /* launch the decode kernels one by one instead of replaying the captured CUDA graph (debug) */
    B200_SESSION_UNFUSED  = 2,     /* decode with the prefill schedule (one kernel per reference graph node, the seam's kernels) */
    B200_SESSION_FAST     = 4,     /* order-free kernels: integer-exact block dots but a different f32 summation order than the
                                      reference's AVX2 build.  NOT conformant: the reference graph amplifies 1e-7 differences to ~1e-2
                                      in the logits (DESIGN.md "chaos").  Default (flag clear) = bit-exact kernels.  The attention on an
                                      f32 cache stays exact: only the weight mat-muls go order-free. */
    B200_SESSION_KV_F32   = 8,     /* memory_k and memory_v are GGML_TYPE_F32 (InferenceSessionConfig::memory_k_type = memory_v_type = Float32,
                                      the reference CLI's --no-float16): twice the bytes, no fp16 rounding of K, V, Q or the probabilities;
                                      the attention is ggml_vec_dot_f32, bit-exact.  Clear (or a zero-initialised config): f16.
                                      NULL from start_session on a tensor-parallel model. */
};

enum {                            /* return codes (0 = ok).  CUDA failures print and exit(1) like the reference backend. */
    B200_OK = 0,
    B200_ERR_CONTEXT_FULL = -1,   /* InferenceError::ContextFull (inference_session.rs:311-313, 388-390) */
    B200_ERR_BAD_ARG = -2,
    B200_ERR_UNKNOWN_TENSOR = -3, /* LoadError::UnknownTensor */
    B200_ERR_TENSOR_SHAPE = -4,   /* LoadError::TensorWrongSize */
    B200_ERR_NOT_LOADED = -5,
    B200_ERR_SAMPLER_FAILURE = -6,/* InferenceError::SamplerFailure: the logits row holds a NaN (Logits::try_from_iter) */
    /* file loading (ggml::format::LoadError, crates/ggml/src/format/loader.rs:38-70; llm_base::LoadError) */
    B200_ERR_IO = -10,
    B200_ERR_INVALID_MAGIC = -11,
    B200_ERR_INVALID_FORMAT_VERSION = -12,
    B200_ERR_INVARIANT_BROKEN = -13,        /* n_dims > 2, negative sizes, Q4_0/Q4_1 rows with ne0 % 64 != 0 */
    B200_ERR_UNSUPPORTED_ELEMENT_TYPE = -14,
    B200_ERR_QUANTIZATION_VERSION = -15,    /* quantized tensors need quantization version 2 (llm-base loader.rs:481-484) */
    /* model quantization (llm_base::QuantizeError, crates/llm-base/src/quantize.rs:69-121) */
    B200_ERR_INVALID_QUANTIZATION_TARGET = -16,         /* InvalidQuantizationTarget: a target other than Q4_0 / Q4_1 / Q5_0 / Q5_1 / Q8_0 */
    B200_ERR_VOCABULARY_SCORING_NOT_SUPPORTED = -17,    /* VocabularyScoringNotSupported: the GGML container with a non-zero token score */
    /* session snapshots (b200_snapshot below) */
    B200_ERR_SNAPSHOT_SIZE_MISMATCH = -18,  /* SnapshotError::MemorySizeMismatch: another model geometry, context size or KV type */
    B200_ERR_SNAPSHOT_FORMAT = -19,         /* a session file this library cannot read (see b200_snapshot) */
};

/* The reference's default sampler chain (crates/llm-base/src/samplers.rs:97-211, ensure_default_slots), run on the device in this order:
 *   repetition   penalty on each distinct id of the last `repetition_last_n` tokens of the session's history: l <= 0 ? l * penalty : l / penalty
 *                (penalty 1.0 or last_n 0: off); the logits row itself is not modified
 *   top-k        value descending, ties by ascending token id; k capped at min(top_k, n_vocab, 1024)
 *   top-p        p_i = expf(l_i - l_0) / S over the k candidates (S summed in f32 in order); the shortest prefix whose running sum is >= top_p
 *   temperature  l_i / temperature
 *   draw         one uniform u = (z >> 40) * 2^-24, z = the `draw`-th SplitMix64 output of `seed`; weights expf(l_i - l_0), the first candidate
 *                whose running weight sum is > u * (sum of the weights)
 * All f32 with glibc's expf (oracle/sampler_oracle.c restates it in plain C).  The caller owns the draw counter, so a rewind can replay the same
 * draws.  top_k = 1 is greedy decoding.  The random stream is this project's, not the reference's StdRng: only greedy decoding matches it. */
typedef struct {
    float    repetition_penalty;   /* 1.30 */
    int32_t  repetition_last_n;    /* 64 */
    int32_t  top_k;                /* 40; >= 1 */
    float    top_p;                /* 0.95 */
    float    temperature;          /* 0.80; > 0 */
    uint64_t seed;
    uint64_t draw;                 /* index of this step's uniform in the seed's stream */
} b200_sampler;

int  b200_init(int device);                                   /* accelerator::initialize(device), accelerator/mod.rs:68-77 */
int  b200_device_info(int32_t *sm_count, size_t *free_bytes, size_t *total_bytes);

b200_model *b200_llama_new(const b200_llama_hparams *hp);
/* Per-tensor weight types (mixed-type files: the quantizer writes output.weight as Q6_K whenever both its dimensions are multiples of 256, and the
 * K_M mixes give wv / w2 / wo other types than the rest).  Each entry names one 2-D weight -- tok_embeddings.weight, output.weight,
 * layers.<i>.attention.w{q,k,v,o}.weight, layers.<i>.feed_forward.w{1,2,3}.weight -- and gives its enum ggml_type: F16, Q4_0..Q8_0 or Q2_K..Q6_K;
 * weights the table does not name are of hp->wtype.  Refused with NULL and *err (nullable), before anything is allocated:
 *   B200_ERR_UNKNOWN_TENSOR            a name that is not a 2-D weight of this model
 *   B200_ERR_UNSUPPORTED_ELEMENT_TYPE  any other type (F32 2-D weights included), wk / w3 of another type than wq / w1 of the same layer, or F16
 *                                      weights beside weights of other types (an F16 model is F16 throughout)
 *   B200_ERR_INVARIANT_BROKEN          a K-quant tensor whose rows are not whole 256-element super-blocks (ne0 % 256 != 0)
 *   B200_ERR_BAD_ARG                   hyperparameters b200_llama_new refuses
 * K-quant matrices keep the file's super-blocks and run kquants.cu's kernels (bit-exact with ggml_vec_dot_q*_K_q8_K).  A model whose layer matrices
 * are all of one classic type decodes through the decode graph, with a K-quant lm_head as two more launches in place of its mat-vec; layers with
 * a K-quant or a wv of its own type decode per op.  K-quants are refused on tensor-parallel shards (b200_llama_new_tp). */
typedef struct { const char *name; int32_t type; } b200_tensor_type;
b200_model *b200_llama_new_typed(const b200_llama_hparams *hp, const b200_tensor_type *types, int32_t n, int *err);
/* Tensor-parallel shard tp_rank of tp_world (one process per GPU, <= 8; the north star's "weight rows shard across the 8 GPUs"): every 2-D weight but
 * tok_embeddings holds only this rank's OUTPUT ROWS -- wq/wk/wv: its heads, w1/w3: rows [rank*n_ff/G, +n_ff/G), wo/w2: rows [rank*n_embd/G, +n_embd/G),
 * output: rows [rank*n_vocab/G, +n_vocab/G) -- and b200_model_load_tensor takes exactly those rows.  Contrast: LC/ggml-cuda.cu:3355-3583 (row split by
 * g_tensor_split + a gather per mat-mul).  Sessions of such a model decode one token per step (b200_session_evaluate loops over a batch). */
b200_model *b200_llama_new_tp(const b200_llama_hparams *hp, int32_t tp_rank, int32_t tp_world);
/* TensorLoader::load(name) + Tensor::transfer_to(Backend::Gpu): host bytes in GGML layout (block arrays for quantized types) */
int  b200_model_load_tensor(b200_model *m, const char *name, int32_t type, const void *host_data, size_t nbytes);
/* fill every tensor with seeded synthetic weights generated ON the device (N(0,1/K) -> the reference's quantizer rule);
 * used by bench.py / smoke: there are no model files in this environment */
int  b200_model_synthesize(b200_model *m, uint64_t seed);
/* copy a tensor back in GGML layout (tests; lets the CPU oracle run on device-generated weights) */
int  b200_model_read_tensor(b200_model *m, const char *name, void *host_out, size_t nbytes);
size_t b200_model_tensor_nbytes(b200_model *m, const char *name);
size_t b200_model_weight_bytes(b200_model *m);                /* bytes of all 2-D weights resident in HBM */
int  b200_model_is_loaded(b200_model *m);                     /* every tensor of the architecture has been loaded */
void b200_model_free(b200_model *m);

/* ---- GGML / GGMF / GGJT model files (SURVEY.md §8f-2): ggml::format::load / save, llm::load::<Llama> -------------------------
 * The parser is host-only (mmap; usable without a GPU).  Offsets are from the start of the file; GGJT tensor data is 32-byte aligned. */
typedef struct b200_ggml_file b200_ggml_file;
typedef struct {
    char     name[96];
    int32_t  type, n_dims;        /* enum ggml_type; n_dims <= 2 */
    int64_t  ne[2];               /* ne[0] = row length */
    uint64_t offset, nbytes;      /* TensorLoadInfo::start_offset, calc_size() */
} b200_ggml_tensor_info;

enum { B200_ARCH_LLAMA = 0, B200_ARCH_GPT2 = 1, B200_ARCH_GPTNEOX = 2, B200_ARCH_MPT = 3, B200_ARCH_BLOOM = 4, B200_ARCH_GPTJ = 5,
       B200_ARCH_LORA = 6 };   /* whose Hyperparameters::read_ggml lays out the header; LORA: a LoRA adapter (LoraParameters, crates/llm-base/src/lora.rs) */
b200_ggml_file *b200_ggml_open(const char *path, int *err);                     /* LLaMA header; NULL + *err on LoadError */
b200_ggml_file *b200_ggml_open_arch(const char *path, int32_t arch, int *err);
/* the header words in file order: llama n_vocab n_embd n_mult n_head n_layer n_rot file_type | gpt2 n_vocab n_ctx n_embd n_head n_layer file_type n_vocab |
 * gptneox n_vocab n_ctx n_embd n_head n_layer n_rot use_parallel_residual file_type |
 * mpt n_embd max_seq_len n_head n_layer n_vocab alibi_bias_max(f32 bits) clip_kqv(f32 bits) file_type (mpt lib.rs:317-330; the vocabulary count is word 4) |
 * bloom n_vocab n_embd n_mult n_head n_layer file_type |
 * gptj n_vocab n_ctx n_embd n_head n_layer n_rot file_type n_vocab (gptj lib.rs:366-401; the repeated n_vocab must match the first: InvariantBroken) |
 * lora r alpha (no vocabulary; r <= 0 is InvariantBroken, where the reference would divide by it) */
int     b200_ggml_hparams(const b200_ggml_file *f, int32_t *arch, int32_t *words8, int32_t *n_words);
void    b200_ggml_close(b200_ggml_file *f);
int     b200_ggml_container(const b200_ggml_file *f, uint32_t *magic, uint32_t *version);      /* ContainerType */
int64_t b200_ggml_n_tensors(const b200_ggml_file *f);
int     b200_ggml_tensor(const b200_ggml_file *f, int64_t i, b200_ggml_tensor_info *out);
const void *b200_ggml_tensor_data(const b200_ggml_file *f, int64_t i);          /* into the mapping */
int64_t b200_ggml_n_vocab(const b200_ggml_file *f);
int     b200_ggml_token(const b200_ggml_file *f, int64_t i, const uint8_t **bytes, uint32_t *len, float *score);
/* llama Hyperparameters::read_ggml + FileType + the quantization-version rule; n_ff / wtype are taken from the tensor table */
int     b200_ggml_llama_hparams(const b200_ggml_file *f, b200_llama_hparams *out, int32_t *n_mult, int32_t *llama_ftype, int32_t *quantization_version);
/* ggml::format::save (GGJT v3): header words verbatim (any architecture), or the LLaMA convenience form */
int     b200_ggml_write(const char *path, const int32_t *hparam_words, int32_t n_words, int32_t n_vocab, const uint8_t *const *token_bytes, const uint32_t *token_len,
                        const float *token_score, const b200_ggml_tensor_info *tensors, const void *const *data, int64_t n_tensors);
int     b200_ggml_write_llama(const char *path, const b200_llama_hparams *hp, int32_t n_mult, int32_t file_type, const uint8_t *const *token_bytes, const uint32_t *token_len,
                              const float *token_score, const b200_ggml_tensor_info *tensors, const void *const *data, int64_t n_tensors);
/* llm::load::<Llama>(path, ModelParameters): parse + b200_llama_new_typed with every 2-D tensor's type from the file + one b200_model_load_tensor per
 * tensor, straight from the mapping; context_size / rope_* <= 0 keep the defaults (2048, 10000, 1).  Its refusals come before anything is uploaded;
 * B200_ERR_UNSUPPORTED_ELEMENT_TYPE also for a LoRA adapter (the _lora form) that targets a K-quant tensor. */
b200_model *b200_llama_load_file(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int *err);
/* same with ModelParameters::n_gqa (grouped-query attention: n_head_kv = n_head / n_gqa, e.g. 8 for 70B files) */
b200_model *b200_llama_load_file_gqa(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int32_t n_gqa, int *err);
/* b200_model_load_tensor + the loader's dims check (LoadError::TensorWrongSize on a dims mismatch even when the byte count matches) */
int  b200_model_load_tensor_shaped(b200_model *m, const char *name, int32_t type, int32_t n_dims, int64_t ne0, int64_t ne1, const void *host_data, size_t nbytes);
/* ---- LoRA adapters (ModelParameters::lora_adapters, crates/llm-base/src/model/mod.rs:205-206): each adapter is a file opened with B200_ARCH_LORA.
 * For a tensor named in an adapter's patch set (its tensor names without the last "."-component), every adapter in the order given applies
 * W = W + (alpha / r) * (loraA x loraB) on the GPU before the tensor is placed -- LoraAdapter::patch (crates/llm-base/src/lora.rs:71-140), bit-exact
 * with the reference's CPU graph.  loraA [r, ne0] F32 or F16, loraB [r, ne1] F32 (else UnsupportedElementType); a missing .loraA / .loraB is
 * UnknownTensor, shapes that do not fit are TensorWrongSize.  n_adapters == 0 is the shaped load; tensor-parallel models take no adapters (BadArgument). */
int  b200_model_load_tensor_lora(b200_model *m, const char *name, int32_t type, int32_t n_dims, int64_t ne0, int64_t ne1, const void *host_data, size_t nbytes,
                                 const b200_ggml_file *const *adapters, int32_t n_adapters);
/* b200_llama_load_file_gqa with the adapter files lora_paths[0..n_lora), opened and closed here */
b200_model *b200_llama_load_file_lora(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int32_t n_gqa,
                                      const char *const *lora_paths, int32_t n_lora, int *err);

/* ---- model quantization: llm_base::quantize (crates/llm-base/src/quantize.rs:139-414) + ggml::format::save (saver.rs:86-163) --------------------
 * src_path (an F16 / F32 file of architecture `arch`, B200_ARCH_LLAMA .. B200_ARCH_GPTJ) -> dst_path with every selected tensor quantized to
 * target_type (2 Q4_0, 3 Q4_1, 6 Q5_0, 7 Q5_1, 8 Q8_0) on the GPU, byte-identical with the reference given the same tensor order.  Selected: n_dims == 2
 * and a name matching the architecture's quantize_tensors() (".*weight"; GPT-2: model/wte, model/lm_head and the c_attn, c_proj, c_fc and mlp c_proj
 * weights of each layer), unanchored.
 * Every other tensor is copied byte for byte.  Tensors are written in the source file's order; the header words are the source's except the file
 * type, 2000 + llama_ftype(target); the vocabulary is the source's.  container: 0 GGJT v3 (scores, 32-byte aligned data), 1 unversioned GGML (no
 * scores, no padding; B200_ERR_VOCABULARY_SCORING_NOT_SUPPORTED if a score is non-zero).
 * Everything is checked before dst_path is created: B200_ERR_INVALID_QUANTIZATION_TARGET; B200_ERR_UNSUPPORTED_ELEMENT_TYPE for a selected tensor that
 * is not F32 / F16; B200_ERR_INVARIANT_BROKEN for a selected tensor with ne0 % 32 != 0, or ne0 % 64 != 0 for a Q4_0 / Q4_1 target; B200_ERR_BAD_ARG
 * for B200_ARCH_LORA, another container, or a destination that is the source file; the source's LoadError.  On a write error (B200_ERR_IO) the
 * partial output is removed.  cb (nullable) runs once per tensor, in file order, after the tensor's bytes are written.  The totals and the sum of
 * the histograms go to the nullable *_out pointers (hist_out: 16 values). */
typedef struct {
    char    name[96];
    int32_t n_dims, src_type, dst_type;    /* dst_type == src_type: copied, not quantized */
    int64_t ne[2], n_elements, original_size, reduced_size;
    int64_t hist[16];                      /* ggml_quantize_* histogram; zero when copied */
} b200_quantize_report;
typedef void (*b200_quantize_callback)(void *user, const b200_quantize_report *r);
int  b200_quantize_file(const char *src_path, const char *dst_path, int32_t arch, int32_t target_type,
                        int32_t container /* 0 GGJT v3, 1 GGML */, b200_quantize_callback cb, void *user,
                        int64_t *original_size_out, int64_t *reduced_size_out, int64_t *hist_out /* [16] */);

b200_session *b200_model_start_session(b200_model *m, const b200_session_config *cfg);
/* One forward pass over `n` tokens appended at n_past (InferenceSession::compute + Llama::evaluate).  tokens: HOST int32.
 * logits_out: HOST f32, n rows of n_vocab when all_logits (OutputRequest::all_logits), else the last row (read_last_token).
 * May be NULL (feed only).  n must be <= n_batch. */
int  b200_session_evaluate(b200_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits);
/* feed_prompt: evaluate in chunks of n_batch; last row of logits returned */
/* sampler hand-off (SURVEY.md 8f-3): the k (<= 1024) largest logits of the last evaluated row, selected on the device -- descending logit,
 * ties by ascending token id -- so that 8 k bytes cross PCIe instead of n_vocab floats (the top-k stage of b200_session_infer_next_token's
 * sampler, penalty off) */
int  b200_session_top_k(b200_session *s, int32_t k, int32_t *ids_out, float *logits_out);
int  b200_session_feed_prompt(b200_session *s, const int32_t *tokens, int32_t n, float *last_logits_out);
/* Model::evaluate with OutputRequest::embeddings (crates/llm-base/src/model/mod.rs:257-266, model/common.rs:40-59): b200_session_evaluate, and when
 * embeddings_out (HOST, nullable) is set, the n_embd f32 of row n - 1 of the final norm's output -- rms_norm, then * norm.weight (llama lib.rs:343-348),
 * the tensor the lm_head reads -- bit-identical to the reference's CPU graph (B200_SESSION_FAST sessions: from their own order-free numbers).
 * The request changes nothing else: logits, both caches, n_past, the history, last_logits and last_launches are the same with and without it.
 * Every session form serves it (NO_GRAPH, UNFUSED, FAST, both KV types, F16 weights, LoRA-patched models); a tensor-parallel session returns
 * B200_ERR_BAD_ARG when embeddings_out is set.  b200_session_evaluate is this with embeddings_out NULL. */
int  b200_session_evaluate_output(b200_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits, float *embeddings_out);
/* InferenceSession::feed_prompt with an OutputRequest (inference_session.rs:299-350): every chunk is evaluated with the request, so embeddings_out
 * (nullable) receives the last row of the last chunk; an empty prompt (n = 0) leaves it untouched.  Refusals as b200_session_evaluate_output.
 * b200_session_feed_prompt is this with embeddings_out NULL. */
int  b200_session_feed_prompt_output(b200_session *s, const int32_t *tokens, int32_t n, float *last_logits_out, float *embeddings_out);
/* InferenceSession::infer_next_token (inference_session.rs:381-419): sample a token from the last evaluated row with the chain of b200_sampler
 * (history window: the session's tokens), append it to the history and evaluate it as a one-token step.  The id is returned as soon as the
 * sampler has run, while the step is still on the device; only the id crosses PCIe, and the next call queues behind the step.  End of text is
 * the caller's test on *token_out: that token has been evaluated, as in the reference.
 * B200_ERR_CONTEXT_FULL if n_past + 1 >= context_size (the reference's check, one slot stricter than evaluate's), with nothing enqueued;
 * B200_ERR_SAMPLER_FAILURE on a NaN in the row: n_past, the history and the last row are restored; B200_ERR_BAD_ARG: no row evaluated yet,
 * top_k < 1, temperature <= 0, penalty <= 0, a negative last_n, null pointers, a tensor-parallel session.  B200_SESSION_FAST sessions run. */
int  b200_session_infer_next_token(b200_session *s, const b200_sampler *sampler, int32_t *token_out);
/* the token ids at positions [0, n_past) -- what every evaluate fed and infer_next_token sampled (InferenceSession::tokens); a rewind truncates
 * them.  Copies min(n_past, max) ids and returns n_past, or a negative error code. */
int32_t b200_session_read_tokens(b200_session *s, int32_t *tokens_out, int32_t max);
/* the last evaluated row of logits (InferenceSession::last_logits), n_vocab f32; B200_ERR_BAD_ARG before the first evaluate */
int  b200_session_last_logits(b200_session *s, float *logits_out);
/* InferenceSession::perplexity (crates/llm-base/src/inference_session.rs:514-589) over HOST token ids tokens[0, n), computed on the device.
 * With C = context_size, chunk i covers [iC, (i+1)C) for i < n_chunk = n / C (n < C: zero chunks).  Each chunk is evaluated in batches of n_batch
 * with all logits, its first token replaced by `bos` (the model's bot_token_id, else 1); rows j in [min(512, C/2), C - 1) are scored as
 * -ln(softmax(row j)[t[iC + j + 1]]), the reference's f32 arithmetic with glibc's expf / logf, bit-exact.  The logits never leave HBM; nll (f32)
 * runs over all chunks and ppl_out[i] = expf(nll / count) after chunk i.  terms_out (nullable): the n_chunk x (C - 1 - min(512, C/2)) terms.
 * Deviation: every chunk starts at n_past 0 (the reference never rewinds, so its chunk 1 would run past the end of the KV cache); chunk 0 is exactly
 * the reference's loop on a fresh session.  Afterwards n_past = C (unchanged when there are zero chunks) and the cache holds the last chunk.
 * B200_ERR_BAD_ARG: null pointers, n < 0, bos or a token id outside [0, n_vocab), a tensor-parallel session.  B200_SESSION_FAST sessions run. */
int  b200_session_perplexity(b200_session *s, const int32_t *tokens, int64_t n, int32_t bos, float *ppl_out, float *terms_out, int32_t *n_chunk_out);
/* Device-resident variant for measurements: tokens already in HBM, logits stay in HBM (no host copies, no sync) */
int  b200_session_evaluate_device(b200_session *s, const int32_t *d_tokens, int32_t n);
const float *b200_session_device_logits(b200_session *s);    /* [n][n_vocab] of the last evaluate */
int32_t b200_session_n_past(const b200_session *s);
int  b200_session_set_n_past(b200_session *s, int32_t n_past);   /* rewind (supports_rewind, llama lib.rs:396-398) */
/* raw KV cache bytes (get_snapshot, inference_session.rs:599-646): which = 0 memory_k, 1 memory_v; 2 bytes per element (f16), 4 with
 * B200_SESSION_KV_F32 (f32), same layout */
int  b200_session_read_kv(b200_session *s, int32_t which, void *host_out, size_t nbytes);
int  b200_session_sync(b200_session *s);
/* tuning aid (B200_DECODE_PROF=1): per-launch %globaltimer stamps of the graph decode schedule; out = 8*n values, see session.cu */
int  b200_session_decode_timeline(b200_session *s, unsigned long long *out, int n, int reset);
/* debug taps for parity work: keep a copy of one intermediate buffer of (layer, stage) during the next evaluate.
 * stages: 1 attn-norm out [n][e], 2 qkv before rope [n][e+2gqa], 3 qkv after rope, 4 KQ raw [h][n][n_kv], 5 KQ softmax, 6 merged
 * KQV [n][e], 7 inpFF, 8 ffn-norm out, 9 [w1x | w3x] [n][2f], 10 silu*mul [n][f], 11 layer output [n][e] */
int  b200_session_set_tap(b200_session *s, int32_t layer, int32_t stage);
int64_t b200_session_read_tap(b200_session *s, float *host_out, int64_t max_count);
/* kernels launched by the last evaluate (for bench.py's gpu_launches) and whether it replayed a CUDA graph */
int32_t b200_session_last_launches(const b200_session *s);
void b200_session_free(b200_session *s);
/* Tensor-parallel sessions: each rank exports the CUDA IPC handle (64 bytes) of its exchange slab, the host layer gathers the handles of all ranks
 * (any channel: torch.distributed, MPI, a pipe) and hands the table [tp_world][64] back; after that the decode kernels store their output slices
 * straight into every peer's slab over NVLink (llm_b200/csrc/tp.cuh).  Every rank must call evaluate with the same tokens in the same order.
 * ONE tensor-parallel session per process: the exchange context (peer pointers, epoch) lives in constant memory of the decode kernels' module
 * (one process per GPU, like the reference's one-session-per-process global state, LC/ggml-cuda.cu:2598-2686). */
int  b200_session_tp_handle(b200_session *s, void *handle_out64);
int  b200_session_tp_connect(b200_session *s, const void *handles_by_rank);
int32_t b200_session_tp_timeouts(b200_session *s);
/* measurement aid: nowait 1 skips the tag waits (garbage results; time = compute + peer stores), 2 also keeps every store local (time = compute alone):
 * sizes the exchange's share of a token */
int  b200_session_tp_set_nowait(b200_session *s, int32_t nowait);

/* stream handle (cudaStream_t) on which everything above is ordered -- for CUDA-event timing from the host side */
void *b200_stream(void);
/* CUDA-event stopwatch on that stream: begin records an event; end records a second one, waits for it and returns ms */
int   b200_timing_begin(void);
float b200_timing_end_ms(void);
/* Roofline probe for the dominant decode kernel: `reps` passes over EVERY weight mat-vec of the model (wqkv, wo, w13, w2 per
 * layer + output; 3.7 GB for 7B Q4_0, far larger than L2) on the session's current quantized activations, timed with CUDA
 * events.  Returns total ms; *launches = kernels launched, *bytes = algorithmic weight bytes streamed (all reps). */
float b200_session_probe_matvec(b200_session *s, int32_t reps, int64_t *launches, double *bytes);

/* ---- GPT-NeoX (crates/models/gptneox): KnownModel + InferenceSession, same conventions as the LLaMA entry points above --------------------------
 * Hyperparameters (gptneox lib.rs:403-447 region): tensor names are the loader's ("gpt_neox.embed_in.weight", "gpt_neox.layers.N.attention.
 * query_key_value.weight" [3e x e, rows per head: q | k | v], ..., "embed_out.weight"); every 2-D ".weight" is of wtype (1 = F16 or a block format), biases / LayerNorm f32;
 * GPT-2's "model/wpe" may also be F16. */
typedef struct b200_neox_hparams {
    int32_t n_vocab, n_embd, n_head, n_layer, n_rot, use_parallel_residual, wtype, context_size;
    int32_t arch;          /* 0 = GPT-NeoX; 1 = GPT-2 (crates/models/gpt2): tensor names "model/wte", "model/wpe" (f32 [n_ctx][n_embd]), "model/hN/attn/c_attn/w" ...,
                              c_attn rows in thirds, no RoPE (n_rot ignored), sequential residual; context_size = the model's n_ctx (rows of wpe);
                              4 = GPT-J (crates/models/gptj): "transformer.wte.weight", "transformer.ln_f.{weight,bias}", "lm_head.{weight,bias}",
                              "transformer.h.N.{ln_1.{weight,bias}, attn.{q_proj,k_proj,v_proj,out_proj}.weight, mlp.{fc_in,fc_out}.{weight,bias}}"; one LayerNorm
                              per layer feeds attention and MLP, RoPE mode 0 over the whole head (n_rot sets the angle step; even, 0 < n_rot <= head size),
                              out = x + ((fc_out gelu(fc_in ln_1(x) + b) + b) + out_proj attn), logits = lm_head x + lm_head.bias; heads up to 256 wide */
    int32_t has_lm_head;   /* GPT-2: "model/lm_head" present; 0 = output projection tied to model/wte (gpt2 lib.rs:319-320) */
} b200_neox_hparams;
typedef struct b200_neox_model b200_neox_model;
typedef struct b200_neox_session b200_neox_session;
b200_neox_model *b200_neox_new(const b200_neox_hparams *hp);
/* MPT (crates/models/mpt) and BLOOM (crates/models/bloom) on the same runtime: the GPT-2 block (qkv rows in thirds, no RoPE, sequential residual,
 * gelu FFN of width 4 n_embd) with ALiBi on the scaled scores (ggml_alibi: + key position x per-head slope, before the causal mask).
 *   arch 2 = MPT: "transformer.wte.weight" (also the output projection), "transformer.norm_f.weight", "transformer.blocks.N.{norm_1.weight,
 *            attn.Wqkv.weight, attn.out_proj.weight, norm_2.weight, ffn.up_proj.weight, ffn.down_proj.weight}"; no biases; alibi_bias_max from the header
 *   arch 3 = BLOOM: "tok_embeddings.weight", "norm.{weight,bias}" (LayerNorm of the embedding row), "output_norm.{weight,bias}", "output.weight",
 *            "layers.N.{attention_norm,ffn_norm}.{weight,bias}", "layers.N.attention.{query_key_value,wo}.{weight,bias}",
 *            "layers.N.feed_forward.{w1,w2}.{weight,bias}"; alibi_bias_max 8 (bloom lib.rs:240)
 * n_rot, use_parallel_residual and has_lm_head are ignored.  NULL for any other arch (and b200_neox_new returns NULL for 2 and 3).  Every other
 * b200_neox_* entry point serves these models unchanged. */
b200_neox_model *b200_neox_new_alibi(const b200_neox_hparams *hp, float alibi_bias_max);
/* Any of the five architectures (hp->arch 0 .. 4) with a per-tensor element type for its 2-D weights: types[0, n) name matrices by the model's
 * tensor names (GPT-J: attn.q_proj / k_proj / v_proj), the others are of hp->wtype.  Types: F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 and Q2_K..Q6_K (K-quant
 * matrices keep the file's 256-element super-blocks).  A tied output (GPT-2 without model/lm_head, MPT) streams wte in wte's type.  GPT-J's q_proj and
 * k_proj share a type; a v_proj of another type becomes its own matrix writing the same qkv rows.  alibi_bias_max: MPT / BLOOM (ignored by the
 * others); rope_freq_base / rope_freq_scale (<= 0: 10000 / 1): ModelParameters::rope_overrides of GPT-NeoX and GPT-J (ignored by the others).
 * Refused before anything is allocated, with *err: B200_ERR_UNSUPPORTED_ELEMENT_TYPE for F32 2-D weights, F16 weights beside other types, GPT-J
 * q_proj and k_proj of different types; B200_ERR_INVARIANT_BROKEN for a K-quant row that is not whole super-blocks; B200_ERR_UNKNOWN_TENSOR for a
 * name the model does not hold; B200_ERR_BAD_ARG for hyperparameters the untyped forms refuse.  A model whose matrices all share one classic type
 * has the untyped form's layout and decode graph; a model with a K-quant matrix or with mixed types decodes per op.  b200_neox_new and
 * b200_neox_new_alibi are this with no table and the default RoPE. */
b200_neox_model *b200_neox_new_typed(const b200_neox_hparams *hp, float alibi_bias_max, float rope_freq_base, float rope_freq_scale,
                                     const b200_tensor_type *types, int32_t n, int *err);
int  b200_neox_is_loaded(b200_neox_model *m);                          /* every tensor of the model has been loaded */
/* llm::load_dynamic for the GPT-NeoX-family architectures: arch B200_ARCH_GPT2 / GPTNEOX / MPT / BLOOM / GPTJ.  The header maps to
 * b200_neox_hparams as the reference's KnownModel::new reads it (b200_ggml_neox_hparams), every 2-D weight's type comes from the file
 * (b200_neox_new_typed), and each tensor is uploaded from the mapping through b200_neox_load_tensor_lora with the adapters lora_paths[0, n_lora).
 * context_size <= 0: 2048 (ModelParameters::default); GPT-2's context is the header's n_ctx whatever is asked, as its learned positions (model/wpe)
 * have that many rows.  rope_freq_base / rope_freq_scale <= 0: 10000 / 1.  The quantization-version rule of the LLaMA loader applies; an adapter that
 * targets a K-quant tensor is B200_ERR_UNSUPPORTED_ELEMENT_TYPE, before the model is created; a missing tensor is B200_ERR_NOT_LOADED. */
b200_neox_model *b200_neox_load_file(const char *path, int32_t arch, int32_t context_size, float rope_freq_base, float rope_freq_scale,
                                     const char *const *lora_paths, int32_t n_lora, int *err);
/* the GPT-NeoX-family view of a header (a file opened as B200_ARCH_GPT2 .. B200_ARCH_GPTJ): n_vocab, n_embd, n_head, n_layer, n_rot (GPT-NeoX, GPT-J),
 * use_parallel_residual (GPT-NeoX), arch (0 GPT-NeoX, 1 GPT-2, 2 MPT, 3 BLOOM, 4 GPT-J), has_lm_head (GPT-2: model/lm_head present), wtype (the type
 * of the file's first 2-D weight), context_size (GPT-2: the header's n_ctx; the others 2048, the default the loader starts from); *alibi_bias_max:
 * MPT's header float, 8 for BLOOM, 0 otherwise; the quantization version and its rule (B200_ERR_QUANTIZATION_VERSION) as b200_ggml_llama_hparams */
int     b200_ggml_neox_hparams(const b200_ggml_file *f, b200_neox_hparams *out, float *alibi_bias_max, int32_t *quantization_version);
/* the type table the loaders build: every 2-D weight of the file that a model of the file's architecture and n_layer holds, in file order.
 * The names point into the file handle (valid until b200_ggml_close).  Returns the count (at most max entries are written), or a negative error. */
int64_t b200_ggml_weight_types(const b200_ggml_file *f, b200_tensor_type *out, int64_t max);
int  b200_neox_load_tensor(b200_neox_model *m, const char *name, int32_t type, const void *host_data, size_t nbytes);
/* shaped load (2-D: ne0 = row length, ne1 = rows; 1-D: ne1 = 1) with the LoRA adapters of b200_model_load_tensor_lora */
int  b200_neox_load_tensor_lora(b200_neox_model *m, const char *name, int32_t type, int32_t n_dims, int64_t ne0, int64_t ne1, const void *host_data, size_t nbytes,
                                const b200_ggml_file *const *adapters, int32_t n_adapters);
int  b200_neox_synthesize(b200_neox_model *m, uint64_t seed);          /* seeded weights generated in HBM (bench) */
size_t b200_neox_weight_bytes(b200_neox_model *m);                     /* bytes streamed per decoded token */
void b200_neox_free(b200_neox_model *m);
b200_neox_session *b200_neox_start_session(b200_neox_model *m, int32_t n_batch);                     /* the flags = 0 form of the next */
/* flags: 0 (f16 KV cache) or B200_SESSION_KV_F32 (f32 cache, bit-exact with the reference's F32 memory_k / memory_v); NULL for any other flag */
b200_neox_session *b200_neox_start_session_flags(b200_neox_model *m, int32_t n_batch, int32_t flags);
int  b200_neox_evaluate(b200_neox_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits);
/* b200_session_evaluate_output for every architecture of this runtime: embeddings_out (nullable) receives row n - 1 of the final LayerNorm's output,
 * norm * gain + bias -- GPT-NeoX ln_f (gptneox lib.rs:333-337), GPT-2 ln_f (gpt2 :311-317), BLOOM output_norm (bloom :317-324), GPT-J ln_f
 * (gptj :286-289) -- or norm * gain with no add node for MPT's norm_f (mpt :236-239, so a -0 stays -0).  b200_neox_evaluate is this with NULL. */
int  b200_neox_evaluate_output(b200_neox_session *s, const int32_t *tokens, int32_t n, float *logits_out, int32_t all_logits, float *embeddings_out);
int  b200_neox_evaluate_device(b200_neox_session *s, int32_t n);       /* tokens of the last evaluate stay in HBM, logits stay in HBM */
int32_t b200_neox_n_past(const b200_neox_session *s);
int  b200_neox_set_n_past(b200_neox_session *s, int32_t n_past);
/* raw KV cache bytes (2 per element for f16, 4 for an f32 cache), which = 0 memory_k [n_layer][n_ctx][n_embd], 1 memory_v [n_layer][n_embd][n_ctx]
 * (V by channel, also for GPT-2) */
int  b200_neox_read_kv(b200_neox_session *s, int32_t which, void *host_out, size_t nbytes);
int32_t b200_neox_last_launches(const b200_neox_session *s);
int  b200_neox_sync(b200_neox_session *s);
/* b200_session_perplexity for every architecture of this runtime (bos: 1 for GPT-NeoX, GPT-2 and GPT-J; BLOOM's "<s>", MPT's "<|padding|>") */
int  b200_neox_perplexity(b200_neox_session *s, const int32_t *tokens, int64_t n, int32_t bos, float *ppl_out, float *terms_out, int32_t *n_chunk_out);
/* b200_session_infer_next_token / read_tokens / last_logits for every architecture of this runtime */
int  b200_neox_infer_next_token(b200_neox_session *s, const b200_sampler *sampler, int32_t *token_out);
int32_t b200_neox_read_tokens(b200_neox_session *s, int32_t *tokens_out, int32_t max);
int  b200_neox_last_logits(b200_neox_session *s, float *logits_out);
void b200_neox_session_free(b200_neox_session *s);

/* ---- session snapshots: InferenceSession::get_snapshot / from_snapshot (crates/llm-base/src/inference_session.rs:591-646, types :733-792) and the
 * CLI's session files (--save-session / --load-session / --persist-session, binaries/llm-cli/src/snapshot.rs) ------------------------------------
 * memory_k / memory_v are the reference's bytes: n_layer x context_size x n_embd values of the cache's type each (for LLaMA with grouped-query
 * attention the reference sizes them by n_embd and uses the first n_layer x context_size x n_embd_gqa values; the rest is written as zeros and
 * ignored when read).  K is [n_layer][context_size][width]; V is [n_layer][width][context_size] for LLaMA, GPT-NeoX and GPT-J, and
 * [n_layer][context_size][n_embd] (by position) for GPT-2, MPT and BLOOM, whose native cache keeps V by channel: those are transposed on the GPU
 * on the way out and back in.  The cache slots past npast are part of the bytes and are kept.
 *
 * Session file: bincode 1.3.3 (default options: little-endian, fixed-width integers, usize as u64, enum variant as u32, Vec / bytes as a u64
 * count and the elements) of InferenceSnapshotRef -- npast u64, memory_k_type u32, memory_v_type u32, n_batch u64, n_threads u64, tokens (u64 +
 * u32 each), last_logits (u64 + f32 each), memory_k (u64 + bytes), memory_v (u64 + bytes) -- inside one zstd frame.  Written: magic 28 B5 2F FD,
 * frame header descriptor 0xC0 (8-byte content size, not single-segment, no checksum, no dictionary), window descriptor 0x38 (128 KiB), the
 * content size, then 128 KiB raw (stored) blocks, the last one flagged: no compressor is needed and every zstd decoder reads it.  Read: one zstd
 * frame whose blocks are raw or RLE (its checksum, if any, is not verified).  This library has no zstd decoder, so compressed blocks -- what the
 * reference CLI writes at level 1 -- are refused with B200_ERR_SNAPSHOT_FORMAT, as are a truncated file, a bad magic, a reserved bit, a block
 * larger than the window or 128 KiB, a content size that is not the blocks', a length field that overruns the content, content after
 * memory_v, and bytes after the frame.  The cache streams between HBM and the file through a ring of a few 8 MiB pinned and device buffers: the
 * host never holds a copy of the cache.  A failed write removes the partial file.
 *
 * from_snapshot starts a session with the snapshot's n_batch and KV type, then writes the cache, n_past, the history and the last row, which the
 * next infer_next_token samples from (even when it is the reference's initial zeros).  Refusals, all checked before anything is allocated:
 * B200_ERR_SNAPSHOT_SIZE_MISMATCH when memory_k or memory_v is not the bytes this model's cache has with the snapshot's KV type; B200_ERR_BAD_ARG for
 * KV types other than 0 / 1 or unequal ones, npast < 0 or > context_size, n_tokens != npast, a token id outside [0, n_vocab), n_logits !=
 * n_vocab, n_batch outside [1, 65536], null pointers, and tensor-parallel sessions and models.
 * Deviations: tokens must hold exactly npast ids (the reference does not check it, and its direct evaluate calls push no tokens; here the history
 * is positional and every evaluate records it); compressed zstd blocks are refused; a GPT-2 model's context is its n_ctx, so a reference GPT-2
 * session at another context_size is a size mismatch. */
typedef struct {
    int64_t  npast;
    int32_t  memory_k_type, memory_v_type;   /* ModelKVMemoryType variant index: 0 Float16, 1 Float32 (not enum ggml_type) */
    int64_t  n_batch, n_threads;             /* n_threads: written as 8 (the reference default), ignored when read */
    int64_t  n_tokens;  uint32_t *tokens;
    int64_t  n_logits;  float    *last_logits;
    uint64_t memory_k_bytes, memory_v_bytes; void *memory_k, *memory_v;   /* the reference's layout and size */
} b200_snapshot;
/* get_snapshot: with tokens, last_logits, memory_k and memory_v all NULL it fills in the scalars, counts and sizes only; with all four set it also
 * copies into them, and the counts and sizes must be the session's (B200_ERR_BAD_ARG otherwise).  Ordered after the work queued on the stream. */
int  b200_session_get_snapshot(b200_session *s, b200_snapshot *snap);
/* from_snapshot on model m; flags may add B200_SESSION_NO_GRAPH / UNFUSED / FAST, the KV bit comes from the snapshot (a conflicting
 * B200_SESSION_KV_F32 is B200_ERR_BAD_ARG).  NULL and *err (nullable) on a refusal. */
b200_session *b200_model_session_from_snapshot(b200_model *m, const b200_snapshot *snap, int32_t flags, int *err);
int  b200_session_write_snapshot(b200_session *s, const char *path);          /* get_snapshot as a session file; B200_ERR_IO on a write error */
b200_session *b200_model_session_read_snapshot(b200_model *m, const char *path, int32_t flags, int *err);   /* from_snapshot of a session file */
/* the scalars, counts and sizes of a session file (the pointers are set to NULL); B200_ERR_IO, B200_ERR_SNAPSHOT_FORMAT */
int  b200_snapshot_read_header(const char *path, b200_snapshot *snap);
/* the same for every architecture of the GPT-NeoX / GPT-2 runtime (no flags, as b200_neox_start_session_flags) */
int  b200_neox_get_snapshot(b200_neox_session *s, b200_snapshot *snap);
b200_neox_session *b200_neox_session_from_snapshot(b200_neox_model *m, const b200_snapshot *snap, int *err);
int  b200_neox_write_snapshot(b200_neox_session *s, const char *path);
b200_neox_session *b200_neox_session_read_snapshot(b200_neox_model *m, const char *path, int *err);

/* ---- single-op entry points on HOST buffers (unit tests, INTEGRATION examples).  Each uploads, runs the kernel, downloads. */
int  b200_op_quantize_act(int32_t vec_dot_type, const float *x, int64_t K, int64_t B, int8_t *qs_out, float *d_out, float *aux_out);
/* ggml_quantize_q{4_0,4_1,5_0,5_1,8_0} (LC/ggml.c:18083-18230) on the GPU: w_host f32 [N][K] -> N rows of GGML blocks, bit-exact with the reference */
int  b200_op_quantize_weights(int32_t wtype, const float *w_host, int64_t K, int64_t N, void *ggml_blocks_out);
/* the kernel of b200_quantize_file on DEVICE buffers, enqueued on b200_stream() without a sync (for kernel timing): nblk 32-element blocks of
 * d_src (src_type 0 F32 / 1 F16) -> GGML blocks of target at d_dst (16-byte aligned); d_hist (nullable): 16 uint64 counters, added to */
int  b200_op_quantize_blocks_device(int32_t target, int32_t src_type, const void *d_src, int64_t nblk, void *d_dst, void *d_hist);
/* the snapshot's transpose kernel on DEVICE buffers, enqueued on b200_stream() without a sync (for kernel timing): d_dst[c][r] = d_src[r][c] for
 * r < rows, c < cols, elements of elem_bytes (2 or 4) bytes, row strides src_ld / dst_ld elements; bit patterns are copied as they are */
int  b200_op_transpose_device(int32_t elem_bytes, const void *d_src, int64_t src_ld, void *d_dst, int64_t dst_ld, int64_t rows, int64_t cols);
/* the seam's row norms on DEVICE buffers, enqueued on b200_stream() without a sync (for kernel timing): op 1 = ggml_rms_norm (eps), op 2 = ggml_norm;
 * rows rows of n f32 at d_x -> d_y */
int  b200_op_norm_device(int32_t op, const float *d_x, float *d_y, int64_t n, int64_t rows, float eps);
/* wtype: GGML_TYPE_F16 (1; K % 64 == 0, impl AUTO or EXACT = mul_mat_f16_exact), GGML_TYPE_Q4_0/Q4_1/Q5_0/Q5_1/Q8_0 (2,3,6,7,8; K % 64 == 0), or the K-quants Q2_K..Q6_K (10..14; K % 256 == 0, impl AUTO or EXACT:
 * ggml_vec_dot_q{2,3,4,5,6}_K_q8_K of LC/k_quants.c:1240,1763,2492,3023,3592 on quantize_row_q8_K activations, bit-exact with the reference's AVX2 build) */
int  b200_op_mul_mat(int32_t wtype, const void *w_ggml, int64_t K, int64_t N, const float *x, int64_t B, float *dst, int32_t impl);
/* the attention mat-muls of the sessions (KQ on the K cache, KQV on the V cache) on host buffers: ggml_mul_mat(src0, src1) with src0 of
 * src0_type GGML_TYPE_F16 (1: ggml_vec_dot_f16 on src1 rounded to fp16) or GGML_TYPE_F32 (0: ggml_vec_dot_f32), bit-exact with the reference's AVX2 build.
 * dst[i2][i1][i0] = dot(src0[i2 / (ne12 / ne02)] row i0, src1[i2] row i1) over ne00 elements; every stride is in bytes (src0 rows nb01, matrices nb02;
 * src1 f32 rows nb11, matrices nb12; dst f32 rows nbd1, matrices nbd2).  causal_past >= 0 skips i0 > causal_past + i1: those elements of dst keep
 * the values the caller passed in.  ne12 % ne02 == 0, ne11 and ne12 at most 65535. */
int  b200_op_mul_mat_kv(int32_t src0_type, const void *src0, int64_t ne00, int64_t ne01, int64_t ne02, int64_t nb01, int64_t nb02,
                        const float *src1, int64_t ne11, int64_t ne12, int64_t nb11, int64_t nb12, float *dst, int64_t nbd1, int64_t nbd2, int32_t causal_past);
/* quantize_row_q8_K (LC/k_quants.c:1133-1183) of B rows of K floats -> B * K/256 block_q8_K {f32 d; i8 qs[256]; i16 bsums[16]} (292 bytes each), bit-exact */
int  b200_op_quantize_q8_K(const float *x, int64_t K, int64_t B, void *blocks_out);
/* LoraAdapter::patch of one adapter on host buffers: w (N rows of K, F32 or Q4_0/Q4_1/Q5_0/Q5_1/Q8_0 GGML blocks) += scaling * ba, ba[n][k] = dot(a row k,
 * b row n), a: K rows of r (a_type 0 F32 / 1 F16), b: N rows of r f32 -- bit-exact with the reference's ggml_mul_mat / ggml_scale / ggml_add on the CPU */
int  b200_op_lora_patch(int32_t wtype, void *w_ggml_inout, int64_t K, int64_t N, int32_t a_type, const void *a, const float *b, int64_t r, float scaling);
/* the scoring step of b200_session_perplexity on host rows: terms_out[r] = -ln(softmax(logits row r)[targets[r]]), `rows` rows of n_vocab f32 */
int  b200_op_nll_rows(const float *logits, int64_t rows, int64_t n_vocab, const int32_t *targets, float *terms_out);
/* the sampler of b200_session_infer_next_token on one host row of n_vocab logits, with the penalty window history[max(0, n_past - last_n), n_past)
 * (history may be NULL when n_past is 0).  id_out: the sampled id; n_kept_out: the candidates top-p kept; cand_ids_out / cand_probs_out
 * (nullable, min(top_k, n_vocab, 1024) entries): the top-k candidates in order and their top-p probabilities.  B200_ERR_SAMPLER_FAILURE on a NaN. */
int  b200_op_sample(const float *logits, int64_t n_vocab, const int32_t *history, int32_t n_past, const b200_sampler *sampler, int32_t *id_out,
                    int32_t *n_kept_out, int32_t *cand_ids_out, float *cand_probs_out);
enum { B200_MM_AUTO = 0, B200_MM_VEC = 1, B200_MM_SIMPLE = 2, B200_MM_TENSOR = 3, B200_MM_EXACT = 4, B200_MM_EXACT_STREAM = 5, B200_MM_EXACT_MMA = 6, B200_MM_EXACT_TC5 = 7, B200_MM_FAST_TC5 = 8 };   /* AUTO = the exact kernel the sessions pick for B rows (the streaming mat-vec at B == 1 where K allows it, EXACT below 16, EXACT_MMA below 96, EXACT_TC5 from 96; K-quants: EXACT); TC5 = the tensor-core prefill GEMMs (the name predates the sm_90a port): wgmma/TMA kernel (exact_tc5.cu); FAST_TC5 = order-free dequant->wgmma GEMM (mmq_tc5.cu, non-conformant) */

#ifdef __cplusplus
}
#endif
#endif
