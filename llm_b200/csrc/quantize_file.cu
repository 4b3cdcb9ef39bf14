// llm_b200/csrc/quantize_file.cu -- model quantization: F16 / F32 model files to Q4_0 / Q4_1 / Q5_0 / Q5_1 / Q8_0, byte-identical with the reference's
// `quantize` (llm_base::quantize, crates/llm-base/src/quantize.rs:139-414, + ggml::format::save, crates/ggml/src/format/saver.rs:86-160).
//
// The reference widens each selected tensor to f32 and calls ggml_quantize_q* (LC/ggml.c:18083-18208): quantize_row_*_reference per row, then a
// 16-bin histogram of the quants.  Here one kernel does both in one pass over the source rows (quantize_blocks_kernel), and the host streams every
// selected tensor through a ring of pinned and device buffers, so the device memory in use is bounded by the ring, never by the model.
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#include <regex>
#include <string>
#include <vector>

#include "../../include/llm_b200.h"
#include "host.h"
#include "kernels.cuh"
#include "quant_rules.cuh"
#include "runtime.h"

namespace b200 {

namespace {

template <typename SRC> __device__ __forceinline__ float widen(SRC x);
template <> __device__ __forceinline__ float widen<float>(float x) { return x; }
template <> __device__ __forceinline__ float widen<__half>(__half x) { return __half2float(x); }     // exact, as half::f16::to_f32

// ggml_quantize_q* on a contiguous run of nblk 32-element blocks: one warp per block (lane j <-> element j, quantize_block_ref), 8 consecutive
// blocks per CTA assembled in shared memory in GGML's file layout (2-byte aligned d [m] [qh] qs) and stored with 16-byte stores: 8 blocks are
// 144 / 160 / 176 / 192 / 272 bytes, so every CTA but the tail one starts and ends on a 16-byte boundary of a 16-byte aligned dst.
// hist (nullable): the blocks' histogram of LC/ggml.c:18092-18202 added to 16 counters -- Q4_x the stored nibble, Q5_x (nibble | fifth bit) / 2
// with the fifth bits the reference's x86 build pairs with each nibble (below), Q8_0 q / 16 + 8 (C's truncating division: bin 8 takes -15..15,
// bin 0 stays empty); counted per CTA in shared memory, one atomic per bin.
template <typename SRC>
__global__ void __launch_bounds__(256) quantize_blocks_kernel(int type, const SRC *__restrict__ src, int64_t nblk, uint8_t *__restrict__ dst,
                                                              unsigned long long *__restrict__ hist) {
    __shared__ __align__(16) uint8_t sbuf[8 * 34];
    __shared__ unsigned int sh[16];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t blk0 = (int64_t)blockIdx.x * 8;
    const int nb = (int)min((int64_t)8, nblk - blk0);
    const int bb = ggml_block_bytes(type);
    if (threadIdx.x < 16) sh[threadIdx.x] = 0;
    __syncthreads();
    if (warp < nb) {
        float d, mn;
        const int q = quantize_block_ref<true>(type, widen<SRC>(src[(blk0 + warp) * 32 + lane]), d, mn);
        uint8_t *o = sbuf + warp * bb;
        int bin;
        if (type == T_Q8_0) {
            o[2 + lane] = (uint8_t)(int8_t)q;
            bin = (int8_t)q / 16 + 8;
        } else {
            const int hdr = 2 + (has_min(type) ? 2 : 0);                  // qh (Q5_x) follows d [m]; qs follows qh
            const int hi = __shfl_down_sync(0xffffffffu, q, 16);
            if (lane < 16) o[hdr + (has_qh(type) ? 4 : 0) + lane] = (uint8_t)((q & 0xF) | ((hi & 0xF) << 4));
            if (has_qh(type)) {
                const unsigned qh = __ballot_sync(0xffffffffu, (q & 0x10) != 0);
                if (lane == 0) { ((uint16_t *)(o + hdr))[0] = (uint16_t)qh; ((uint16_t *)(o + hdr))[1] = (uint16_t)(qh >> 16); }
                // the reference's loop (j = 0, 2, .., 30) pairs qs[j / 2] with fifth bits j and j + 16, and its shifts past bit 31 take their
                // count mod 32 on x86: (qh & 1 << (j + 16)) >> (j + 12) is bit j + 16 for j <= 14, 0 for j = 16, 18 and bit j - 16 for j >= 20
                const int j = 2 * (lane & 15);
                const unsigned vh = lane < 16 ? ((qh & (1u << j)) >> j) << 4 : (uint8_t)((qh & (1u << ((j + 16) & 31))) >> ((j + 12) & 31));
                bin = ((q & 0xF) | vh) >> 1;
            } else {
                bin = q & 0xF;
            }
        }
        if (lane == 0) {
            ((__half *)o)[0] = __float2half_rn(d);
            if (has_min(type)) ((__half *)o)[1] = __float2half_rn(mn);
        }
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (lane == __ffs(peers) - 1) atomicAdd(&sh[bin], (unsigned)__popc(peers));
    }
    __syncthreads();
    const int bytes = nb * bb, n16 = bytes / 16;
    uint8_t *out = dst + blk0 * bb;
    if (threadIdx.x < n16) ((int4 *)out)[threadIdx.x] = ((const int4 *)sbuf)[threadIdx.x];
    if (threadIdx.x < bytes - n16 * 16) out[n16 * 16 + threadIdx.x] = sbuf[n16 * 16 + threadIdx.x];
    if (hist && threadIdx.x < 16 && sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}

}  // namespace

void quantize_blocks(int type, int src_type, const void *src, int64_t nblk, void *dst, unsigned long long *hist, cudaStream_t st) {
    B200_ASSERT(is_quant(type) && (src_type == T_F32 || src_type == T_F16) && ((uintptr_t)dst & 15) == 0);
    if (nblk <= 0) return;
    const unsigned grid = (unsigned)((nblk + 7) / 8);
    if (src_type == T_F32) quantize_blocks_kernel<float><<<grid, 256, 0, st>>>(type, (const float *)src, nblk, (uint8_t *)dst, hist);
    else quantize_blocks_kernel<__half><<<grid, 256, 0, st>>>(type, (const __half *)src, nblk, (uint8_t *)dst, hist);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200

using namespace b200;

namespace {

constexpr int RING = 4;                        // chunks in flight: chunk i+1's read and H2D overlap chunk i's kernel, D2H and write
constexpr int64_t CHUNK_BLOCKS = 1 << 16;      // 2 Mi elements per chunk: 4 / 8 MiB of F16 / F32 source (a multiple of 8 blocks)

// KnownModel::quantize_tensors() of each architecture (llama / gptneox / mpt / bloom / gptj lib.rs: ".*weight"; gpt2 lib.rs:357-369), matched
// unanchored like Regex::is_match; skip_quantize_tensors() is empty for all six
bool selected_for_quantization(int32_t arch, const std::string &name) {
    static const std::vector<std::regex> weight = {std::regex(".*weight")};
    static const std::vector<std::regex> gpt2 = {std::regex("model/wte"), std::regex("model/lm_head"), std::regex("model/h.*/attn/c_attn/w"),
                                                 std::regex("model/h.*/attn/c_proj/w"), std::regex("model/h.*/mlp/c_fc/w"),
                                                 std::regex("model/h.*/mlp/c_proj/w")};
    for (const std::regex &re : arch == B200_ARCH_GPT2 ? gpt2 : weight)
        if (std::regex_search(name, re)) return true;
    return false;
}

// index of the file-type word in each architecture's header (file_type_mut + write_ggml of each model)
int file_type_word(int32_t arch) {
    switch (arch) { case B200_ARCH_LLAMA: return 6; case B200_ARCH_GPT2: return 5; case B200_ARCH_GPTNEOX: return 7; case B200_ARCH_MPT: return 7;
                    case B200_ARCH_BLOOM: return 5; case B200_ARCH_GPTJ: return 6; }
    return -1;
}

// FileTypeFormat::MostlyQ* of the target (crates/llm-base/src/loader.rs:32-50), -1 for anything but the five QuantizationTargets
int llama_ftype(int32_t target) {
    switch (target) { case T_Q4_0: return 2; case T_Q4_1: return 3; case T_Q5_0: return 8; case T_Q5_1: return 9; case T_Q8_0: return 7; }
    return -1;
}

struct Plan { b200_ggml_tensor_info info; bool quantize; int64_t out_bytes; };

int quantize_file_impl(const char *src_path, const char *dst_path, int32_t arch, int32_t target, int32_t container, b200_quantize_callback cb,
                       void *user, int64_t *original_size_out, int64_t *reduced_size_out, int64_t *hist_out, bool &created) {
    if (llama_ftype(target) < 0) return B200_ERR_INVALID_QUANTIZATION_TARGET;
    if (!src_path || !dst_path || arch < 0 || arch >= B200_ARCH_LORA || (container != 0 && container != 1)) return B200_ERR_BAD_ARG;
    struct stat ss, ds;
    if (stat(dst_path, &ds) == 0 && stat(src_path, &ss) == 0 && ss.st_dev == ds.st_dev && ss.st_ino == ds.st_ino) return B200_ERR_BAD_ARG;
    int err = B200_OK;
    b200_ggml_file *f = b200_ggml_open_arch(src_path, arch, &err);
    if (!f) return err;
    struct Closer { b200_ggml_file *f; ~Closer() { b200_ggml_close(f); } } closer{f};

    // every check before the output exists
    std::vector<Plan> plan((size_t)b200_ggml_n_tensors(f));
    bool any_quantized = false;
    for (size_t i = 0; i < plan.size(); i++) {
        Plan &p = plan[i];
        b200_ggml_tensor(f, (int64_t)i, &p.info);
        size_t name_len;
        const char *name = ggml_tensor_name(f, (int64_t)i, &name_len);
        p.quantize = p.info.n_dims == 2 && selected_for_quantization(arch, std::string(name, name_len));
        p.out_bytes = (int64_t)p.info.nbytes;
        if (!p.quantize) continue;
        if (p.info.type != T_F32 && p.info.type != T_F16) return B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
        if (p.info.ne[0] % QK) return B200_ERR_INVARIANT_BROKEN;                                                   // ggml_quantize_*'s assert
        if ((target == T_Q4_0 || target == T_Q4_1) && p.info.ne[0] % 64) return B200_ERR_INVARIANT_BROKEN;         // saver.rs:124-131
        p.out_bytes = p.info.ne[0] * p.info.ne[1] / QK * ggml_block_bytes(target);
        any_quantized = true;
    }
    const int64_t n_vocab = b200_ggml_n_vocab(f);
    if (container == 1)
        for (int64_t i = 0; i < n_vocab; i++) {
            float score;
            b200_ggml_token(f, i, nullptr, nullptr, &score);
            if (score != 0.f) return B200_ERR_VOCABULARY_SCORING_NOT_SUPPORTED;                                  // saver.rs:96-100
        }
    int32_t words[8], n_words = 0;
    b200_ggml_hparams(f, nullptr, words, &n_words);
    words[file_type_word(arch)] = 2 * 1000 + llama_ftype(target);           // quantization_version ggml::QNT_VERSION, format MostlyQ*

    // each slot's buffers: the source chunk (IN bytes), then its blocks; d_hist: 16 counters per slot for the current tensor
    constexpr size_t IN = CHUNK_BLOCKS * QK * 4, OUT = CHUNK_BLOCKS * 34;
    unsigned long long *d_hist = nullptr;
    struct Release { unsigned long long *&d_hist; ~Release() { if (d_hist) cudaFree(d_hist); } } release{d_hist};
    std::unique_ptr<StreamRing> ring;             // destroyed first: its streams are idle before d_hist goes
    if (any_quantized) {
        ring.reset(new StreamRing(RING, IN + OUT, IN + OUT));
        B200_CHECK(cudaMalloc(&d_hist, RING * 16 * sizeof(unsigned long long)));
    }

    FILE *fp = fopen(dst_path, "wb");
    if (!fp) return B200_ERR_IO;
    created = true;
    bool ok = true;
    auto w32 = [&](uint32_t v) { ok &= fwrite(&v, 4, 1, fp) == 1; };
    w32(container == 0 ? 0x67676a74u : 0x67676d6cu);                        // ContainerType::write: 'ggjt' 3, or 'ggml' alone
    if (container == 0) w32(3);
    for (int i = 0; i < n_words; i++) w32((uint32_t)words[i]);
    for (int64_t i = 0; i < n_vocab && ok; i++) {
        const uint8_t *bytes; uint32_t len; float score;
        b200_ggml_token(f, i, &bytes, &len, &score);
        w32(len);
        if (len) ok &= fwrite(bytes, 1, len, fp) == len;
        if (container == 0) { uint32_t b; memcpy(&b, &score, 4); w32(b); }
    }

    int64_t total_in = 0, total_out = 0, hist_all[16] = {0};
    auto retire = [&](StreamRing::Slot &sl) {
        StreamRing::wait(sl);
        ok &= fwrite(sl.h + IN, 1, sl.bytes, fp) == sl.bytes;
    };
    for (size_t i = 0; i < plan.size() && ok; i++) {
        const Plan &p = plan[i];
        size_t name_len;
        const char *name = ggml_tensor_name(f, (int64_t)i, &name_len);
        const int32_t type = p.quantize ? target : p.info.type;
        ok &= ggml_write_record(fp, name, name_len, p.info.n_dims, type, p.info.ne, container == 0);
        const uint8_t *data = (const uint8_t *)b200_ggml_tensor_data(f, (int64_t)i);
        b200_quantize_report r;
        memset(&r, 0, sizeof(r));
        if (!p.quantize) {
            if (p.info.nbytes) ok &= fwrite(data, 1, (size_t)p.info.nbytes, fp) == (size_t)p.info.nbytes;
        } else {
            const int64_t nblk = p.info.ne[0] * p.info.ne[1] / QK, es = p.info.type == T_F16 ? 2 : 4;
            for (int k = 0; k < RING; k++) B200_CHECK(cudaMemsetAsync(d_hist + k * 16, 0, 16 * sizeof(unsigned long long), ring->at(k).st));
            int64_t c = 0;
            for (int64_t b0 = 0; b0 < nblk && ok; b0 += CHUNK_BLOCKS, c++) {
                StreamRing::Slot &sl = ring->at(c);
                if (sl.busy) retire(sl);                                   // chunk c - RING, the oldest in flight: writes stay in file order
                const int64_t nb = std::min(CHUNK_BLOCKS, nblk - b0);
                memcpy(sl.h, data + b0 * QK * es, (size_t)(nb * QK * es));
                B200_CHECK(cudaMemcpyAsync(sl.d, sl.h, (size_t)(nb * QK * es), cudaMemcpyHostToDevice, sl.st));
                quantize_blocks(target, p.info.type, sl.d, nb, sl.d + IN, d_hist + (c % RING) * 16, sl.st);
                sl.bytes = (size_t)(nb * ggml_block_bytes(target));
                B200_CHECK(cudaMemcpyAsync(sl.h + IN, sl.d + IN, sl.bytes, cudaMemcpyDeviceToHost, sl.st));
                B200_CHECK(cudaEventRecord(sl.done, sl.st));
                sl.busy = true;
            }
            for (int k = 0; k < RING; k++) {
                StreamRing::Slot &sl = ring->at(c + k);
                if (sl.busy) retire(sl);
            }
            unsigned long long h[RING * 16];
            B200_CHECK(cudaMemcpy(h, d_hist, sizeof(h), cudaMemcpyDeviceToHost));
            for (int s = 0; s < RING; s++)
                for (int b = 0; b < 16; b++) r.hist[b] += (int64_t)h[s * 16 + b];
        }
        if (!ok) break;
        snprintf(r.name, sizeof(r.name), "%.*s", (int)name_len, name);
        r.n_dims = p.info.n_dims; r.src_type = p.info.type; r.dst_type = type;
        r.ne[0] = p.info.ne[0]; r.ne[1] = p.info.ne[1]; r.n_elements = p.info.ne[0] * p.info.ne[1];
        r.original_size = (int64_t)p.info.nbytes; r.reduced_size = p.out_bytes;
        total_in += r.original_size; total_out += r.reduced_size;
        for (int b = 0; b < 16; b++) hist_all[b] += r.hist[b];
        if (cb) cb(user, &r);
    }
    ok &= fclose(fp) == 0;
    if (!ok) return B200_ERR_IO;
    if (original_size_out) *original_size_out = total_in;
    if (reduced_size_out) *reduced_size_out = total_out;
    if (hist_out) memcpy(hist_out, hist_all, sizeof(hist_all));
    return B200_OK;
}

}  // namespace

extern "C" int b200_quantize_file(const char *src_path, const char *dst_path, int32_t arch, int32_t target_type, int32_t container,
                                  b200_quantize_callback cb, void *user, int64_t *original_size_out, int64_t *reduced_size_out, int64_t *hist_out) {
    bool created = false;
    int rc;
    try { rc = quantize_file_impl(src_path, dst_path, arch, target_type, container, cb, user, original_size_out, reduced_size_out, hist_out, created); }
    catch (...) { rc = B200_ERR_IO; }                                         // no C++ exception crosses the C ABI
    if (rc != B200_OK && created) unlink(dst_path);                          // no partial output
    return rc;
}
