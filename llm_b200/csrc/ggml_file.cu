// llm_b200/csrc/ggml_file.cu -- the GGML / GGMF / GGJT container (SURVEY.md §8f-2): parse, inspect, write, and load into a b200_model.
//
// Mirrors, event for event, what the reference's loader does with a file:
//   ggml::format::load           crates/ggml/src/format/loader.rs:160-208   magic (+version), hyperparameters, vocabulary, tensors
//   load_weights                 crates/ggml/src/format/loader.rs:214-281   per tensor: n_dims, name_len, element type, dims (ne0 first), name,
//                                                                            [GGJT/GGLA: seek to the next multiple of 32], data;
//                                                                            n_dims <= 2, Q4_0/Q4_1 rows need ne0 % 64 == 0
//   ContainerType::read          crates/ggml/src/lib.rs:58-86               'ggml' unversioned; 'ggmf' 1; 'ggjt' 1..3; 'ggla' 1
//   llama Hyperparameters        crates/models/llama/src/lib.rs:425-447     7 x i32: n_vocab n_embd n_mult n_head n_layer n_rot file_type
//   gpt2 Hyperparameters         crates/models/gpt2/src/lib.rs:394-416      6 x i32: n_vocab n_ctx n_embd n_head n_layer file_type, then n_vocab AGAIN (must match)
//   gptneox Hyperparameters      crates/models/gptneox/src/lib.rs:431-442   8 x i32: n_vocab n_ctx n_embd n_head n_layer n_rot use_parallel_residual(0|1) file_type
//   mpt Hyperparameters          crates/models/mpt/src/lib.rs:317-330       n_embd max_seq_len n_head n_layer n_vocab (i32), alibi_bias_max clip_kqv (f32), file_type
//   bloom Hyperparameters        crates/models/bloom/src/lib.rs             6 x i32: n_vocab n_embd n_mult n_head n_layer file_type
//   lora LoraParameters          crates/llm-base/src/lora.rs:27-35          2 x i32: r alpha, no vocabulary (r <= 0: InvariantBroken, a deliberate deviation)
//   FileType                     crates/llm-base/src/loader.rs:32-50        file_type = quantization_version * 1000 + llama_ftype
//   quantization version rule    crates/llm-base/src/loader.rs:459-484      0 is read as 1 (GGJT v2) / 2 (GGJT v3); quantized tensors require 2
//   ggml::format::save           crates/ggml/src/format/saver.rs:86-160     the writer (GGJT v3)
// The parser is plain host code (mmap, no CUDA): the CPU test-suite exercises it without a GPU.  b200_llama_load_file() then feeds every tensor
// to b200_model_load_tensor straight from the mapping (TensorLoader::load + transfer_to(Backend::Gpu)).
#include <fcntl.h>
#include <stdio.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <string>
#include <vector>

#include "../../include/llm_b200.h"
#include "common.cuh"
#include "host.h"

namespace {

constexpr uint32_t MAGIC_GGML = 0x67676d6c, MAGIC_GGMF = 0x67676d66, MAGIC_GGJT = 0x67676a74, MAGIC_GGLA = 0x67676c61;

struct TensorInfo { std::string name; int32_t type; int32_t n_dims; int64_t ne[2]; uint64_t offset, nbytes; };

// bytes of `n` elements of a ggml element type (crates/ggml/src/format/loader.rs:121-123); 0 = unknown type
uint64_t data_size(int32_t type, uint64_t n) {
    switch (type) {
        case b200::T_F32: return n * 4;
        case b200::T_F16: return n * 2;
        case b200::T_Q4_0: case b200::T_Q4_1: case b200::T_Q5_0: case b200::T_Q5_1: case b200::T_Q8_0: case b200::T_Q8_1:
            return n / b200::QK * (uint64_t)b200::ggml_block_bytes(type);
        // K-quants (LC/k_quants.h, QK_K = 256): parsed and sized like the reference's loader does; the native sessions stream the five 32-element formats only (kquants.cu serves Q2_K..Q6_K per operator), so
        // b200_llama_load_file reports the tensor by name instead of failing the whole parse (GGJT v3 "Q4_0" files of the vendored llama.cpp
        // quantizer carry output.weight as Q6_K, LC/llama.cpp:2938-2944)
        case 10: return n / 256 * 84;  case 11: return n / 256 * 110; case 12: return n / 256 * 144; case 13: return n / 256 * 176; case 14: return n / 256 * 210;
        case b200::T_I8: return n; case b200::T_I32: return n * 4;
        default: return 0;
    }
}
// every ElementType the reference's Type::try_from accepts (crates/ggml/src/lib.rs:156-230)
bool known_type(int32_t t) { return t == b200::T_F32 || t == b200::T_F16 || b200::is_quant(t) || t == b200::T_Q8_1 || (t >= 10 && t <= 14) || t == b200::T_I8 || t == b200::T_I32; }
const char *type_name(int32_t t) {
    switch (t) { case 0: return "F32"; case 1: return "F16"; case 2: return "Q4_0"; case 3: return "Q4_1"; case 6: return "Q5_0"; case 7: return "Q5_1"; case 8: return "Q8_0";
                 case 9: return "Q8_1"; case 10: return "Q2_K"; case 11: return "Q3_K"; case 12: return "Q4_K"; case 13: return "Q5_K"; case 14: return "Q6_K"; case 16: return "I8"; case 18: return "I32"; }
    return "?";
}

}  // namespace

struct b200_ggml_file {
    int fd = -1;
    const uint8_t *map = nullptr;
    uint64_t size = 0;
    uint32_t magic = 0, version = 0;
    int32_t arch = 0, n_hp = 7;
    int32_t hp[8] = {0, 0, 0, 0, 0, 0, 0, 0};       // the architecture's hyperparameter words, file order (llama: n_vocab n_embd n_mult n_head n_layer n_rot file_type)
    std::vector<std::pair<uint64_t, uint32_t>> tokens;   // (offset of the bytes, length)
    std::vector<float> scores;
    std::vector<TensorInfo> tensors;
};

// ---- the LoRA hook's view of an adapter file (host.h) ----
int64_t b200::ggml_find_tensor(const b200_ggml_file *f, const char *name) {
    for (size_t i = 0; i < f->tensors.size(); i++) if (f->tensors[i].name == name) return (int64_t)i;
    return -1;
}
bool b200::lora_in_patch_set(const b200_ggml_file *f, const char *name) {     // rsplit_once('.') of some tensor name gives `name`
    const size_t n = strlen(name);
    for (const TensorInfo &t : f->tensors)
        if (t.name.size() > n && t.name.compare(0, n, name) == 0 && t.name[n] == '.' && t.name.find('.', n + 1) == std::string::npos) return true;
    return false;
}
float b200::lora_scaling(const b200_ggml_file *f) { return (float)f->hp[1] / (float)f->hp[0]; }    // LoraParameters::calculate_scaling

// ---- the writers' view (host.h) ----
const char *b200::ggml_tensor_name(const b200_ggml_file *f, int64_t i, size_t *len) {
    const std::string &n = f->tensors[(size_t)i].name;
    *len = n.size();
    return n.data();
}
// one tensor record of ggml::format::save (saver.rs:136-153): n_dims, name length, element type, ne[0..n_dims), the name, and with `align`
// (GGJT) zeros up to the next multiple of 32 bytes of the file; the caller writes the data
bool b200::ggml_write_record(FILE *fp, const char *name, size_t name_len, int32_t n_dims, int32_t type, const int64_t *ne, bool align) {
    bool ok = true;
    auto w32 = [&](uint32_t v) { ok &= fwrite(&v, 4, 1, fp) == 1; };
    w32((uint32_t)n_dims); w32((uint32_t)name_len); w32((uint32_t)type);
    for (int d = 0; d < n_dims; d++) w32((uint32_t)ne[d]);
    ok &= fwrite(name, 1, name_len, fp) == name_len;
    if (align) {
        const long pos = ftell(fp);
        static const uint8_t zeros[32] = {0};
        const size_t pad = (size_t)(((pos + 31) & ~31L) - pos);
        if (pad) ok &= fwrite(zeros, 1, pad, fp) == pad;
    }
    return ok;
}

extern "C" {

void b200_ggml_close(b200_ggml_file *f) {
    if (!f) return;
    if (f->map) munmap((void *)f->map, f->size);
    if (f->fd >= 0) close(f->fd);
    delete f;
}

static b200_ggml_file *open_arch_impl(const char *path, int32_t arch, int *err) {
    int dummy; if (!err) err = &dummy;
    if (arch < 0 || arch > B200_ARCH_LORA) { *err = B200_ERR_BAD_ARG; return nullptr; }
    *err = B200_OK;
    b200_ggml_file *f = new b200_ggml_file();
    f->arch = arch; f->n_hp = arch == B200_ARCH_LLAMA ? 7 : arch == B200_ARCH_GPT2 ? 7 : arch == B200_ARCH_BLOOM ? 6 : arch == B200_ARCH_LORA ? 2 : 8;
    auto fail = [&](int code) -> b200_ggml_file * { *err = code; b200_ggml_close(f); return nullptr; };
    f->fd = open(path, O_RDONLY);
    struct stat sb;
    if (f->fd < 0 || fstat(f->fd, &sb) != 0) return fail(B200_ERR_IO);
    f->size = (uint64_t)sb.st_size;
    if (f->size < 4) return fail(B200_ERR_IO);
    void *m = mmap(nullptr, f->size, PROT_READ, MAP_PRIVATE, f->fd, 0);
    if (m == MAP_FAILED) return fail(B200_ERR_IO);
    f->map = (const uint8_t *)m;

    uint64_t pos = 0;
    bool eof = false;
    auto rd32 = [&]() -> uint32_t { if (pos + 4 > f->size) { eof = true; return 0; } uint32_t v; memcpy(&v, f->map + pos, 4); pos += 4; return v; };

    f->magic = rd32();
    if (f->magic == MAGIC_GGML) f->version = 0;
    else if (f->magic == MAGIC_GGMF || f->magic == MAGIC_GGJT || f->magic == MAGIC_GGLA) f->version = rd32();
    else return fail(B200_ERR_INVALID_MAGIC);
    const bool ok_version = f->magic == MAGIC_GGML || (f->magic == MAGIC_GGMF && f->version == 1) || (f->magic == MAGIC_GGJT && f->version >= 1 && f->version <= 3) ||
                            (f->magic == MAGIC_GGLA && f->version == 1);
    if (eof || !ok_version) return fail(eof ? B200_ERR_IO : B200_ERR_INVALID_FORMAT_VERSION);

    for (int i = 0; i < f->n_hp; i++) f->hp[i] = (int32_t)rd32();
    if (eof) return fail(B200_ERR_IO);
    for (int i = 0; i < f->n_hp; i++)                                                                 // usize::try_from in the reference; MPT's words 5 and 6
        if (f->hp[i] < 0 && !(arch == B200_ARCH_MPT && (i == 5 || i == 6)) && arch != B200_ARCH_LORA) return fail(B200_ERR_INVARIANT_BROKEN);   // are f32 (read_f32 takes any value)
    if (arch == B200_ARCH_LORA && f->hp[0] <= 0) return fail(B200_ERR_INVARIANT_BROKEN);             // r and alpha are i32; the scaling alpha / r needs r > 0
    if (arch == B200_ARCH_GPT2 && f->hp[6] != f->hp[0]) return fail(B200_ERR_INVARIANT_BROKEN);     // "GPT2 model expected n_vocab {} found {}"
    if (arch == B200_ARCH_GPTJ && f->hp[7] != f->hp[0]) return fail(B200_ERR_INVARIANT_BROKEN);     // "GPTJ model expected n_vocab {} found {}" (gptj lib.rs:377-386)
    if (arch == B200_ARCH_GPTNEOX && f->hp[6] > 1) return fail(B200_ERR_IO);                        // read_bool: InvalidData

    const bool scored = f->magic == MAGIC_GGMF || f->magic == MAGIC_GGJT;
    const int32_t n_vocab = arch == B200_ARCH_LORA ? 0 : f->hp[arch == B200_ARCH_MPT ? 4 : 0];   // MPT: n_embd max_seq_len n_head n_layer n_vocab ...; LoRA: none
    if ((uint64_t)n_vocab > (f->size - pos) / 4) return fail(B200_ERR_IO);       // every token record takes at least 4 bytes: a corrupt count cannot ask for gigabytes
    f->tokens.reserve((size_t)n_vocab);
    for (int32_t i = 0; i < n_vocab; i++) {
        const uint32_t len = rd32();
        if (eof || pos + len > f->size) return fail(B200_ERR_IO);
        f->tokens.emplace_back(pos, len);
        pos += len;
        float sc = 0.f;
        if (scored) { const uint32_t b = rd32(); memcpy(&sc, &b, 4); }
        if (eof) return fail(B200_ERR_IO);
        f->scores.push_back(sc);
    }

    const bool align = f->magic == MAGIC_GGJT || f->magic == MAGIC_GGLA;
    while (pos < f->size) {                                                     // has_data_left
        TensorInfo t;
        const int32_t n_dims = (int32_t)rd32(), name_len = (int32_t)rd32();
        const uint32_t ftype = rd32();
        if (eof) return fail(B200_ERR_IO);
        if (n_dims < 0 || name_len < 0) return fail(B200_ERR_INVARIANT_BROKEN);
        if (n_dims > 2) return fail(B200_ERR_INVARIANT_BROKEN);
        t.n_dims = n_dims; t.ne[0] = t.ne[1] = 1;
        uint64_t n_elements = 1;
        for (int i = 0; i < n_dims; i++) { const int32_t d = (int32_t)rd32(); if (d < 0) return fail(B200_ERR_INVARIANT_BROKEN); t.ne[i] = d; n_elements *= (uint64_t)d; }
        if (eof || pos + (uint64_t)name_len > f->size) return fail(B200_ERR_IO);
        t.name.assign((const char *)f->map + pos, (size_t)name_len);
        pos += (uint64_t)name_len;
        t.type = (int32_t)ftype;
        if (!known_type(t.type)) return fail(B200_ERR_UNSUPPORTED_ELEMENT_TYPE);
        if ((t.type == b200::T_Q4_0 || t.type == b200::T_Q4_1) && t.ne[0] % 64 != 0) return fail(B200_ERR_INVARIANT_BROKEN);
        t.offset = align ? (pos + 31) & ~(uint64_t)31 : pos;
        t.nbytes = data_size(t.type, n_elements);
        if (t.offset + t.nbytes > f->size) return fail(B200_ERR_IO);
        pos = t.offset + t.nbytes;
        f->tensors.push_back(t);
    }
    return f;
}

// no C++ exception (e.g. std::bad_alloc on a hostile header) may cross the C ABI: it becomes LoadError::Io
b200_ggml_file *b200_ggml_open_arch(const char *path, int32_t arch, int *err) {
    try { return open_arch_impl(path, arch, err); }
    catch (...) { if (err) *err = B200_ERR_IO; return nullptr; }
}

b200_ggml_file *b200_ggml_open(const char *path, int *err) { return b200_ggml_open_arch(path, B200_ARCH_LLAMA, err); }

int b200_ggml_hparams(const b200_ggml_file *f, int32_t *arch, int32_t *words8, int32_t *n_words) {
    if (!f) return B200_ERR_BAD_ARG;
    if (arch) *arch = f->arch;
    if (words8) memcpy(words8, f->hp, sizeof(f->hp));
    if (n_words) *n_words = f->n_hp;
    return B200_OK;
}

int b200_ggml_container(const b200_ggml_file *f, uint32_t *magic, uint32_t *version) {
    if (!f) return B200_ERR_BAD_ARG;
    if (magic) *magic = f->magic;
    if (version) *version = f->version;
    return B200_OK;
}

int64_t b200_ggml_n_tensors(const b200_ggml_file *f) { return f ? (int64_t)f->tensors.size() : -1; }
int64_t b200_ggml_n_vocab(const b200_ggml_file *f) { return f ? (int64_t)f->tokens.size() : -1; }

int b200_ggml_tensor(const b200_ggml_file *f, int64_t i, b200_ggml_tensor_info *out) {
    if (!f || !out || i < 0 || i >= (int64_t)f->tensors.size()) return B200_ERR_BAD_ARG;
    const TensorInfo &t = f->tensors[(size_t)i];
    memset(out, 0, sizeof(*out));
    snprintf(out->name, sizeof(out->name), "%s", t.name.c_str());
    out->type = t.type; out->n_dims = t.n_dims; out->ne[0] = t.ne[0]; out->ne[1] = t.ne[1]; out->offset = t.offset; out->nbytes = t.nbytes;
    return B200_OK;
}

int b200_ggml_token(const b200_ggml_file *f, int64_t i, const uint8_t **bytes, uint32_t *len, float *score) {
    if (!f || i < 0 || i >= (int64_t)f->tokens.size()) return B200_ERR_BAD_ARG;
    if (bytes) *bytes = f->map + f->tokens[(size_t)i].first;
    if (len) *len = f->tokens[(size_t)i].second;
    if (score) *score = f->scores[(size_t)i];
    return B200_OK;
}

const void *b200_ggml_tensor_data(const b200_ggml_file *f, int64_t i) {
    if (!f || i < 0 || i >= (int64_t)f->tensors.size()) return nullptr;
    return f->map + f->tensors[(size_t)i].offset;
}

// LLaMA view of the header: hyperparameters + what the tensors add (n_ff = rows of feed_forward.w1, weight type = type of attention.wq),
// and the quantization-version rule of crates/llm-base/src/loader.rs:459-484.
int b200_ggml_llama_hparams(const b200_ggml_file *f, b200_llama_hparams *out, int32_t *n_mult, int32_t *llama_ftype, int32_t *quantization_version) {
    if (!f || !out || f->arch != B200_ARCH_LLAMA) return B200_ERR_BAD_ARG;
    memset(out, 0, sizeof(*out));
    out->n_vocab = f->hp[0]; out->n_embd = f->hp[1]; out->n_head = f->hp[3]; out->n_head_kv = f->hp[3]; out->n_layer = f->hp[4]; out->n_rot = f->hp[5];
    out->context_size = 2048; out->rope_freq_base = 10000.0f; out->rope_freq_scale = 1.0f;
    int32_t qv = (int32_t)((uint32_t)f->hp[6] / 1000u);
    if (qv == 0 && f->magic == MAGIC_GGJT) qv = f->version == 2 ? 1 : f->version == 3 ? 2 : 0;
    if (n_mult) *n_mult = f->hp[2];
    if (llama_ftype) *llama_ftype = (int32_t)((uint32_t)f->hp[6] % 1000u);
    if (quantization_version) *quantization_version = qv;
    bool any_quant = false;
    out->wtype = -1;                                                             // "not found" (F32 = 0 is a valid element type)
    for (const TensorInfo &t : f->tensors) {
        any_quant |= b200::is_quant(t.type);
        if (t.name == "layers.0.feed_forward.w1.weight") out->n_ff = (int32_t)t.ne[1];
        if (t.name == "layers.0.attention.wq.weight") out->wtype = t.type;
    }
    if (any_quant && qv != 2) return B200_ERR_QUANTIZATION_VERSION;
    if (out->n_ff == 0 || out->wtype < 0) return B200_ERR_UNKNOWN_TENSOR;
    return B200_OK;
}

// ggml::format::save: GGJT v3, the architecture's hyperparameter words verbatim, tensor data 32-byte aligned.  tensors = n_tensors x {name, type, n_dims, ne,
// nbytes} with data[i] the GGML-layout bytes; tokens/scores may be NULL (every token is then written empty with score 0).
int b200_ggml_write(const char *path, const int32_t *hparam_words, int32_t n_words, int32_t n_vocab, const uint8_t *const *token_bytes, const uint32_t *token_len,
                    const float *token_score, const b200_ggml_tensor_info *tensors, const void *const *data, int64_t n_tensors) {
    if (!path || !hparam_words || n_words < 1 || n_words > 8 || (n_tensors > 0 && (!tensors || !data))) return B200_ERR_BAD_ARG;
    FILE *fp = fopen(path, "wb");
    if (!fp) return B200_ERR_IO;
    bool ok = true;
    auto w32 = [&](uint32_t v) { ok &= fwrite(&v, 4, 1, fp) == 1; };
    w32(MAGIC_GGJT); w32(3);
    for (int i = 0; i < n_words; i++) w32((uint32_t)hparam_words[i]);
    for (int32_t i = 0; i < n_vocab; i++) {
        const uint32_t len = token_len ? token_len[i] : 0;
        w32(len);
        if (len) ok &= fwrite(token_bytes[i], 1, len, fp) == len;
        float sc = token_score ? token_score[i] : 0.f; uint32_t b; memcpy(&b, &sc, 4); w32(b);
    }
    for (int64_t i = 0; i < n_tensors && ok; i++) {
        const b200_ggml_tensor_info &t = tensors[i];
        ok &= b200::ggml_write_record(fp, t.name, strnlen(t.name, sizeof(t.name)), t.n_dims, t.type, t.ne, true);
        if (t.nbytes) ok &= fwrite(data[i], 1, (size_t)t.nbytes, fp) == (size_t)t.nbytes;
    }
    ok &= fclose(fp) == 0;
    return ok ? B200_OK : B200_ERR_IO;
}

int b200_ggml_write_llama(const char *path, const b200_llama_hparams *hp, int32_t n_mult, int32_t file_type, const uint8_t *const *token_bytes, const uint32_t *token_len,
                          const float *token_score, const b200_ggml_tensor_info *tensors, const void *const *data, int64_t n_tensors) {
    if (!hp) return B200_ERR_BAD_ARG;
    const int32_t h[7] = {hp->n_vocab, hp->n_embd, n_mult, hp->n_head, hp->n_layer, hp->n_rot, file_type};
    return b200_ggml_write(path, h, 7, hp->n_vocab, token_bytes, token_len, token_score, tensors, data, n_tensors);
}

// llm::load::<Llama>(path, params): parse, build the model for the file's geometry, upload every tensor from the mapping.
// n_gqa > 1: ModelParameters::n_gqa (grouped-query attention, e.g. 8 for LLaMA-2 70B): n_head_kv = n_head / n_gqa (llama lib.rs:403-447).
// With adapters, each tensor goes through b200_model_load_tensor_lora (MmapCompatibleLoader::load, crates/llm-base/src/loader.rs:661-669).
static b200_model *load_file_impl(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int32_t n_gqa,
                                  const b200_ggml_file *const *adapters, int32_t n_adapters, int *err) {
    b200_ggml_file *f = b200_ggml_open(path, err);
    if (!f) return nullptr;
    b200_llama_hparams hp;
    *err = b200_ggml_llama_hparams(f, &hp, nullptr, nullptr, nullptr);
    if (*err != B200_OK) { b200_ggml_close(f); return nullptr; }
    if (!b200::is_qweight_type(hp.wtype)) {     // F32 / K-quant files parse, but this backend streams F16 and the five 32-element block formats only
        fprintf(stderr, "llm_b200: %s: layers.0.attention.wq.weight is %s; this backend loads F16/Q4_0/Q4_1/Q5_0/Q5_1/Q8_0 weights\n", path, type_name(hp.wtype));
        *err = B200_ERR_UNSUPPORTED_ELEMENT_TYPE; b200_ggml_close(f); return nullptr;
    }
    if (context_size > 0) hp.context_size = context_size;
    if (rope_freq_base > 0.f) hp.rope_freq_base = rope_freq_base;
    if (rope_freq_scale > 0.f) hp.rope_freq_scale = rope_freq_scale;
    if (n_gqa > 1) { if (hp.n_head % n_gqa) { *err = B200_ERR_BAD_ARG; b200_ggml_close(f); return nullptr; } hp.n_head_kv = hp.n_head / n_gqa; }
    b200_model *m = b200_llama_new(&hp);
    if (!m) { *err = B200_ERR_BAD_ARG; b200_ggml_close(f); return nullptr; }
    for (size_t i = 0; i < f->tensors.size(); i++) {
        const TensorInfo &t = f->tensors[i];
        const bool is_norm = t.n_dims == 1;
        if (!is_norm && t.type != hp.wtype) {     // one weight type per model (QWeight planes are per matrix, the decode graph is instantiated per type)
            fprintf(stderr, "llm_b200: %s: tensor %s is %s, the model's weight type is %s: mixed-type files are not supported by this backend\n", path, t.name.c_str(),
                    type_name(t.type), type_name(hp.wtype));
            *err = B200_ERR_UNSUPPORTED_ELEMENT_TYPE; b200_model_free(m); b200_ggml_close(f); return nullptr;
        }
        const int rc = b200_model_load_tensor_lora(m, t.name.c_str(), t.type, t.n_dims, t.ne[0], t.ne[1], f->map + t.offset, (size_t)t.nbytes, adapters, n_adapters);
        if (rc != B200_OK) { *err = rc; b200_model_free(m); b200_ggml_close(f); return nullptr; }
    }
    if (!b200_model_is_loaded(m)) { *err = B200_ERR_NOT_LOADED; b200_model_free(m); b200_ggml_close(f); return nullptr; }
    b200_ggml_close(f);
    *err = B200_OK;
    return m;
}
b200_model *b200_llama_load_file_gqa(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int32_t n_gqa, int *err) {
    int dummy; if (!err) err = &dummy;
    return load_file_impl(path, context_size, rope_freq_base, rope_freq_scale, n_gqa, nullptr, 0, err);
}

// ModelParameters::lora_adapters: every adapter is opened (ggml::format::load with LoraParameters) and stays open while the model's tensors load
b200_model *b200_llama_load_file_lora(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int32_t n_gqa,
                                      const char *const *lora_paths, int32_t n_lora, int *err) {
    int dummy; if (!err) err = &dummy;
    if (n_lora < 0 || (n_lora > 0 && !lora_paths)) { *err = B200_ERR_BAD_ARG; return nullptr; }
    std::vector<b200_ggml_file *> ad;
    auto close_all = [&]() { for (b200_ggml_file *a : ad) b200_ggml_close(a); };
    for (int32_t i = 0; i < n_lora; i++) {
        b200_ggml_file *a = b200_ggml_open_arch(lora_paths[i], B200_ARCH_LORA, err);
        if (!a) { close_all(); return nullptr; }
        ad.push_back(a);
    }
    b200_model *m = load_file_impl(path, context_size, rope_freq_base, rope_freq_scale, n_gqa, ad.data(), n_lora, err);
    close_all();
    return m;
}
b200_model *b200_llama_load_file(const char *path, int32_t context_size, float rope_freq_base, float rope_freq_scale, int *err) {
    return b200_llama_load_file_gqa(path, context_size, rope_freq_base, rope_freq_scale, 1, err);
}

}  // extern "C"
