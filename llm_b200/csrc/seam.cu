// llm_b200/csrc/seam.cu -- the ggml_cuda_* C ABI (include/ggml_b200.h) served by the project's CUDA kernels.
//
// This is the per-node, drop-in front end: the reference's graph executor (LC/ggml.c:14584-14591) calls
// ggml_cuda_compute_forward for every node and the Rust side (crates/ggml/src/tensor.rs, accelerator/mod.rs) manages
// buffers through transform_tensor / assign_buffers*.  Semantics follow LC/ggml-cuda.cu:3807-4135 (what the callers rely
// on), the mechanism is ours: weights are re-laid out into 16-byte planes at upload, mat-muls run the bit-exact
// kernels mul_mat.cu picks (B200_FAST=1: those of mmvq.cu / mmq.cu), row ops run rowops.cu.  Single device per process (GGML_BACKEND_GPU_SPLIT is rejected: the
// reference's Rust API can never produce it, crates/llm-base/src/model/mod.rs:244-250).
#include <string.h>

#include <mutex>
#include <vector>

#include "../../include/ggml_b200.h"
#include "kernels.cuh"
#include "runtime.h"

using namespace b200;

namespace b200 {

// ---- process-wide runtime (device, stream, arenas) -----------------------------------------------------------------------
Runtime &rt() {
    static Runtime R;
    return R;
}

void Runtime::ensure_init() {
    if (inited) return;
    std::lock_guard<std::mutex> lock(mu);
    if (inited) return;
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        fprintf(stderr, "llm_b200: no CUDA device available (%s). This backend has no CPU fallback.\n", cudaGetErrorString(e));
        exit(1);
    }
    device_count = n;
    if (device < 0 || device >= n) device = 0;
    B200_CHECK(cudaSetDevice(device));
    B200_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    cudaDeviceProp prop;
    B200_CHECK(cudaGetDeviceProperties(&prop, device));
    sm_count = prop.multiProcessorCount;
    { const char *f = getenv("B200_FAST"); fast = f && f[0] == '1'; }
    luts();
    inited = true;
}

void *Arena::get(size_t bytes, cudaStream_t st) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (off + bytes > cap) {
        // grow: everything enqueued so far may still be using the old block
        B200_CHECK(cudaStreamSynchronize(st));
        size_t ncap = cap ? cap : (size_t)64 << 20;
        while (ncap < off + bytes) ncap *= 2;
        void *nb;
        B200_CHECK(cudaMalloc(&nb, ncap));
        if (base) { retired.push_back(base); }
        base = (char *)nb; cap = ncap; off = 0;   // callers never hold arena pointers across get() of a NEW op
    }
    void *p = base + off;
    off += bytes;
    return p;
}
void Arena::reset() { off = 0; for (void *p : retired) cudaFree(p); retired.clear(); }
void Arena::release() { reset(); if (base) cudaFree(base); base = nullptr; cap = 0; }

}  // namespace b200

namespace {

struct Extra {              // what tensor->extra points at
    void *data = nullptr;   // device pointer of element (0,0,0,0)
    QWeight qw;             // valid when the tensor is an uploaded quantized matrix
    bool is_q = false;
    bool owned = false;
};

// ---- small restatements of the ggml.h helpers the seam needs (LC/ggml.c:4070-4215) ----------------------------------------
inline int64_t nelements(const ggml_tensor *t) { return t->ne[0] * t->ne[1] * t->ne[2] * t->ne[3]; }
inline int64_t nrows(const ggml_tensor *t) { return t->ne[1] * t->ne[2] * t->ne[3]; }
inline size_t nbytes(const ggml_tensor *t) {
    const size_t a = (size_t)t->ne[3] * t->nb[3];
    const size_t b = (size_t)nelements(t) * ggml_type_size(t->type) / ggml_blck_size(t->type);
    return a > b ? a : b;
}
inline bool is_contiguous(const ggml_tensor *t) {
    return t->nb[0] == ggml_type_size(t->type) && t->nb[1] == t->nb[0] * t->ne[0] / ggml_blck_size(t->type) &&
           t->nb[2] == t->nb[1] * t->ne[1] && t->nb[3] == t->nb[2] * t->ne[2];
}
inline bool on_device(const ggml_tensor *t) { return t->backend == B200_BACKEND_GPU || t->backend == B200_BACKEND_GPU_SPLIT; }

struct Scratch { size_t size = 0, offset = 0; char *buffer = nullptr; } g_scratch;   // LC/ggml-cuda.cu:2598-2604
std::vector<Extra> g_temp_extras;                                                   // ring of 4096, :3895-3909
size_t g_temp_extra_index = 0;

Extra *alloc_temp_extra() {
    if (g_temp_extras.empty()) g_temp_extras.resize(4096);                            // GGML_MAX_NODES
    Extra *e = &g_temp_extras[g_temp_extra_index];
    g_temp_extra_index = (g_temp_extra_index + 1) % g_temp_extras.size();
    *e = Extra();
    return e;
}

// device view of a source operand; host-resident operands are staged through the op arena (LC/ggml-cuda.cu:3476-3504)
const void *src_dev(const ggml_tensor *t) {
    Runtime &R = rt();
    if (on_device(t)) { B200_ASSERT(t->extra); return ((Extra *)t->extra)->data; }
    B200_ASSERT(is_contiguous(t));
    const size_t n = nbytes(t);
    void *d = R.op_arena.get(n, R.stream);
    B200_CHECK(cudaMemcpyAsync(d, t->data, n, cudaMemcpyHostToDevice, R.stream));
    return d;
}
void *dst_dev(ggml_tensor *t) {
    Runtime &R = rt();
    if (on_device(t)) { B200_ASSERT(t->extra); return ((Extra *)t->extra)->data; }
    B200_ASSERT(is_contiguous(t));
    return R.op_arena.get(nbytes(t), R.stream);
}
// results that live on the host are copied back and the stream drained (LC/ggml-cuda.cu:3516-3543, 3585-3588)
void dst_finish(ggml_tensor *t, void *d) {
    Runtime &R = rt();
    if (on_device(t)) return;
    B200_CHECK(cudaMemcpyAsync(t->data, d, nbytes(t), cudaMemcpyDeviceToHost, R.stream));
    B200_CHECK(cudaStreamSynchronize(R.stream));
}

StridedDesc desc_of(const ggml_tensor *t) {
    StridedDesc d;
    for (int i = 0; i < 4; i++) { d.ne[i] = t->ne[i]; d.nb[i] = (int64_t)t->nb[i]; }
    return d;
}

// ---- ops ------------------------------------------------------------------------------------------------------------------
void op_mul_mat(const ggml_tensor *src0, const ggml_tensor *src1, ggml_tensor *dst) {
    Runtime &R = rt();
    cudaStream_t st = R.stream;
    B200_ASSERT(src1->type == B200_TYPE_F32 && dst->type == B200_TYPE_F32);
    B200_ASSERT(src0->backend != B200_BACKEND_GPU_SPLIT);
    if (is_quant(src0->type)) {
        // W[type; K, N] x X[f32; K, B] -> dst[N, B]   (contract asserts of LC/ggml.c:10419-10431)
        B200_ASSERT(src0->ne[2] == 1 && src0->ne[3] == 1 && is_contiguous(src0));
        B200_ASSERT(src1->nb[0] == 4 && src1->ne[2] * src1->ne[3] == 1 || is_contiguous(src1));
        B200_ASSERT(is_contiguous(dst));
        const int64_t K = src0->ne[0], N = src0->ne[1], B = nrows(src1);
        QWeight w;
        if (on_device(src0)) {
            Extra *e = (Extra *)src0->extra;
            B200_ASSERT(e && e->is_q);
            w = e->qw;
        } else {   // host-resident weights (ggml_cuda_can_mul_mat path): upload + re-layout for this call
            const size_t raw_bytes = (size_t)N * (K / QK) * ggml_block_bytes(src0->type);
            void *raw = R.op_arena.get(raw_bytes, st);
            B200_CHECK(cudaMemcpyAsync(raw, src0->data, raw_bytes, cudaMemcpyHostToDevice, st));
            const size_t pb = qweight_layout(w, src0->type, K, N, nullptr);
            qweight_layout(w, src0->type, K, N, R.op_arena.get(pb, st));
            repack_weights(w, raw, st);
        }
        const float *x = (const float *)src_dev(src1);
        float *d = (float *)dst_dev(dst);
        const int64_t ldx = is_contiguous(src1) ? K : (int64_t)(src1->nb[1] / 4);
        int8_t *xq = (int8_t *)R.op_arena.get((size_t)B * K, st);
        float2 *xds = (float2 *)R.op_arena.get((size_t)B * (K / QK) * sizeof(float2), st);
        if (!R.fast) {
            int4 *xpack = (int4 *)R.op_arena.get((size_t)(K / QK) * 64, st);
            __half *xh = (__half *)R.op_arena.get(xh_bytes(K, B), st);
            mul_mat_exact_auto(w, x, ldx, B, d, N, nullptr, 0, {xq, xds, xpack, xh}, st);
        } else {
            quantize_act(vec_dot_type(src0->type), x, ldx, xq, xds, K, B, st);
            if (B == 1)      mul_mat_vec_q(w, xq, xds, d, nullptr, st);
            else if (B < 16) mul_mat_q_simple(w, xq, xds, d, N, B, nullptr, 0, st);
            else             mul_mat_q(w, xq, xds, d, N, B, nullptr, 0, st);
        }
        dst_finish(dst, d);
        return;
    }
    if (is_kquant(src0->type)) {
        // Q2_K .. Q6_K: the super-blocks stay in GGML's own layout (transform_tensor uploaded them as they are); quantize_row_q8_K + vec_dot order of the AVX2 build
        B200_ASSERT(src0->ne[2] == 1 && src0->ne[3] == 1 && is_contiguous(src0) && is_contiguous(dst));
        B200_ASSERT(src1->nb[0] == 4 && src1->ne[2] * src1->ne[3] == 1 || is_contiguous(src1));
        const int64_t K = src0->ne[0], N = src0->ne[1], B = nrows(src1);
        B200_ASSERT(K % 256 == 0);
        const void *wraw;
        if (on_device(src0)) { Extra *e = (Extra *)src0->extra; B200_ASSERT(e && e->data); wraw = e->data; }
        else {
            const size_t raw_bytes = (size_t)N * (K / 256) * kquant_block_bytes(src0->type);
            void *raw = R.op_arena.get(raw_bytes, st);
            B200_CHECK(cudaMemcpyAsync(raw, src0->data, raw_bytes, cudaMemcpyHostToDevice, st));
            wraw = raw;
        }
        const float *x = (const float *)src_dev(src1);
        float *d = (float *)dst_dev(dst);
        const int64_t ldx = is_contiguous(src1) ? K : (int64_t)(src1->nb[1] / 4);
        void *xq = R.op_arena.get(q8k_bytes(K, B), st);
        quantize_act_q8k(x, ldx, xq, K, B, st);
        mul_mat_kq_exact(src0->type, wraw, xq, d, N, K, N, B, nullptr, 0, st);
        dst_finish(dst, d);
        return;
    }
    if (src0->type == B200_TYPE_F16) {
        B200_ASSERT(src0->nb[0] == 2 && src1->nb[0] == 4 && dst->nb[0] == 4);
        B200_ASSERT(src0->ne[3] == 1 && src1->ne[3] == 1);
        B200_ASSERT(on_device(src0));
        const __half *a = (const __half *)((Extra *)src0->extra)->data;
        const float *b;
        if (on_device(src1)) b = (const float *)((Extra *)src1->extra)->data; else b = (const float *)src_dev(src1);
        float *d = (float *)dst_dev(dst);
        if (R.fast) mul_mat_f16(a, src0->ne[0], src0->ne[1], src0->ne[2], src0->nb[1], src0->nb[2],
                                b, src1->ne[1], src1->ne[2], src1->nb[1], src1->nb[2], d, dst->nb[1], dst->nb[2], st);
        else mul_mat_f16_exact(a, src0->ne[0], src0->ne[1], src0->ne[2], src0->nb[1], src0->nb[2],
                               b, src1->ne[1], src1->ne[2], src1->nb[1], src1->nb[2], d, dst->nb[1], dst->nb[2], -1, st);
        dst_finish(dst, d);
        return;
    }
    fprintf(stderr, "llm_b200: ggml_cuda_mul_mat: unsupported src0 type %d\n", src0->type);
    abort();
}

void op_binary(int which, const ggml_tensor *src0, const ggml_tensor *src1, ggml_tensor *dst) {
    B200_ASSERT(src0->type == B200_TYPE_F32 && src1->type == B200_TYPE_F32 && dst->type == B200_TYPE_F32);
    B200_ASSERT(is_contiguous(src0) && is_contiguous(src1) && is_contiguous(dst));
    B200_ASSERT(src1->ne[0] == src0->ne[0] && nelements(src0) % nelements(src1) == 0);
    const float *a = (const float *)src_dev(src0), *b = (const float *)src_dev(src1);
    float *d = (float *)dst_dev(dst);
    if (which == 0) add_f32(a, b, d, nelements(src0), nelements(src1), rt().stream);
    else            mul_f32(a, b, d, nelements(src0), nelements(src1), rt().stream);
    dst_finish(dst, d);
}

void op_rows(const ggml_tensor *src0, ggml_tensor *dst) {   // NORM, RMS_NORM, SOFT_MAX, DIAG_MASK_INF, SCALE, UNARY
    Runtime &R = rt();
    B200_ASSERT(src0->type == B200_TYPE_F32 && is_contiguous(src0) && is_contiguous(dst));
    const float *x = (const float *)src_dev(src0);
    float *y = (float *)dst_dev(dst);
    const int64_t n = src0->ne[0], rows = nrows(src0);
    switch (dst->op) {
        case B200_OP_RMS_NORM: { float eps; memcpy(&eps, dst->op_params, 4); rms_norm(x, y, nullptr, n, rows, eps, R.stream); } break;
        case B200_OP_NORM: layer_norm(x, y, nullptr, nullptr, n, rows, R.stream); break;
        case B200_OP_SOFT_MAX: soft_max(x, y, n, rows, src0->ne[1], 1.f, false, 0, false, true, R.stream); break;
        case B200_OP_DIAG_MASK_INF: soft_max(x, y, n, rows, src0->ne[1], 1.f, false, dst->op_params[0], true, false, R.stream); break;
        case B200_OP_SCALE: {
            // src1 is a 1-element HOST tensor even when flagged GPU (ggml_new_f32 writes tensor->data; LC/ggml-cuda.cu:3259, 3328-3329)
            const float s = *(const float *)dst->src[1]->data;
            scale_f32(x, s, y, nelements(src0), R.stream);
        } break;
        case B200_OP_UNARY:
            unary_lut(dst->op_params[0] == B200_UNARY_GELU ? UNARY_GELU : UNARY_SILU, x, y, nelements(src0), R.stream);
            break;
        default: B200_ASSERT(!"op_rows");
    }
    dst_finish(dst, y);
}

void op_rope(const ggml_tensor *src0, ggml_tensor *dst) {
    Runtime &R = rt();
    B200_ASSERT(src0->type == B200_TYPE_F32 && src0->nb[0] == 4 && dst->nb[0] == 4 && src0->ne[3] == 1);
    const int n_past = dst->op_params[0], n_dims = dst->op_params[1], mode = dst->op_params[2];
    float freq_base, freq_scale;
    memcpy(&freq_base, dst->op_params + 4, 4);
    memcpy(&freq_scale, dst->op_params + 5, 4);
    B200_ASSERT((mode & 1) == 0 && (mode & 4) == 0);        // modes 0 and 2 (LLaMA, NeoX); GLM is out of scope
    const float *x = (const float *)src_dev(src0);
    float *y = (float *)dst_dev(dst);
    const RopeTable &tab = rope_table(n_dims, mode, freq_base, freq_scale, (int)src0->ne[0], n_past + (int)src0->ne[2]);
    rope_f32(x, y, src0->ne[0], src0->ne[1], src0->ne[2], src0->nb[1] / 4, src0->nb[2] / 4, dst->nb[1] / 4, dst->nb[2] / 4, n_past, tab, R.stream);
    dst_finish(dst, y);
}

void op_cpy(const ggml_tensor *src0, ggml_tensor *dst) {    // CPY, DUP, CONT: dst already carries the target layout
    const void *s = src_dev(src0);
    void *d = dst_dev(dst);
    cpy_strided(s, src0->type, desc_of(src0), d, dst->type, desc_of(dst), rt().stream);
    dst_finish(dst, d);
}

bool op_supported(const ggml_tensor *t) {
    switch (t->op) {
        case B200_OP_DUP: case B200_OP_ADD: case B200_OP_MUL: case B200_OP_NORM: case B200_OP_RMS_NORM: case B200_OP_MUL_MAT:
        case B200_OP_SCALE: case B200_OP_CPY: case B200_OP_CONT: case B200_OP_RESHAPE: case B200_OP_VIEW: case B200_OP_PERMUTE:
        case B200_OP_TRANSPOSE: case B200_OP_DIAG_MASK_INF: case B200_OP_SOFT_MAX: case B200_OP_ROPE:
            return true;
        case B200_OP_UNARY: return t->op_params[0] == B200_UNARY_GELU || t->op_params[0] == B200_UNARY_SILU;
        default: return false;
    }
}

void assign_buffers_impl(ggml_tensor *tensor, bool scratch, bool force_inplace) {   // LC/ggml-cuda.cu:3911-3977
    Runtime &R = rt();
    if (scratch && g_scratch.size == 0) return;
    R.ensure_init();
    if (tensor->src[0] != nullptr && tensor->src[0]->backend == B200_BACKEND_CPU) {
        const int op0 = tensor->src[0]->op;
        if (op0 == B200_OP_RESHAPE || op0 == B200_OP_TRANSPOSE || op0 == B200_OP_VIEW || op0 == B200_OP_PERMUTE)
            assign_buffers_impl(tensor->src[0], scratch, force_inplace);
    }
    if (tensor->op == B200_OP_CPY && tensor->src[1]->backend == B200_BACKEND_CPU) assign_buffers_impl(tensor->src[1], scratch, force_inplace);

    tensor->backend = B200_BACKEND_GPU;
    Extra *extra;
    const bool inplace = (tensor->src[0] != nullptr && tensor->src[0]->data == tensor->data) || tensor->op == B200_OP_VIEW || force_inplace;
    const size_t size = nbytes(tensor);
    if (inplace && tensor->src[0] != nullptr && on_device(tensor->src[0])) {
        Extra *e0 = (Extra *)tensor->src[0]->extra;
        size_t offset = 0;
        if (tensor->op == B200_OP_VIEW) memcpy(&offset, tensor->op_params, sizeof(size_t));
        extra = alloc_temp_extra();
        extra->data = (char *)e0->data + offset;
    } else if (tensor->op == B200_OP_CPY) {
        Extra *e1 = (Extra *)tensor->src[1]->extra;
        extra = alloc_temp_extra();
        extra->data = e1->data;
    } else if (scratch) {
        B200_ASSERT(size <= g_scratch.size);
        const size_t asz = (size + 255) & ~(size_t)255;        // keep every activation 256-byte aligned (vector loads, TMA)
        if (g_scratch.offset + asz > g_scratch.size) g_scratch.offset = 0;
        if (g_scratch.buffer == nullptr) B200_CHECK(cudaMalloc(&g_scratch.buffer, g_scratch.size + 256));
        extra = alloc_temp_extra();
        extra->data = g_scratch.buffer + g_scratch.offset;
        g_scratch.offset += asz;
    } else {
        void *data;
        B200_CHECK(cudaMalloc(&data, size));
        B200_CHECK(cudaMemset(data, 0, size));
        B200_CHECK(cudaDeviceSynchronize());   // legacy-stream copy/memset: not ordered with our non-blocking stream, and a pageable H2D cudaMemcpy may return before its DMA lands
        extra = new Extra();
        extra->data = data;
        extra->owned = true;
    }
    tensor->extra = extra;
}

}  // namespace

// ==== exported C ABI ==========================================================================================================
extern "C" {

void ggml_init_cublas(void) { rt().ensure_init(); }

void ggml_cuda_set_main_device(int main_device) {
    Runtime &R = rt();
    if (R.inited) {
        if (main_device != R.device)
            fprintf(stderr, "llm_b200: warning: main device already fixed to %d; ignoring request for %d\n", R.device, main_device);
        return;
    }
    R.device = main_device;
}

void ggml_cuda_set_tensor_split(const float *tensor_split) {
    // One process drives one GPU (DESIGN.md §multi-GPU); the only value the Rust side ever passes is a single 1.0f
    // (crates/ggml/src/accelerator/mod.rs:68-77), so exactly one float is read here -- never g_device_count of them.
    (void)tensor_split;
}

void ggml_cuda_set_scratch_size(size_t scratch_size) { g_scratch.size = scratch_size; }

void ggml_cuda_free_scratch(void) {
    if (!g_scratch.buffer) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    B200_CHECK(cudaFree(g_scratch.buffer));
    g_scratch.buffer = nullptr;
    g_scratch.offset = 0;
}

void ggml_cuda_transform_tensor(void *data, struct ggml_tensor *tensor) {     // LC/ggml-cuda.cu:3807-3871
    Runtime &R = rt();
    R.ensure_init();
    B200_ASSERT(tensor->backend == B200_BACKEND_GPU);    // GPU_SPLIT unreachable from the Rust API
    Extra *e = new Extra();
    e->owned = true;
    if (is_quant(tensor->type)) {
        B200_ASSERT(tensor->ne[2] == 1 && tensor->ne[3] == 1 && is_contiguous(tensor));
        const int64_t K = tensor->ne[0], N = tensor->ne[1];
        const size_t pb = qweight_layout(e->qw, tensor->type, K, N, nullptr);
        void *base;
        B200_CHECK(cudaMalloc(&base, pb));
        qweight_layout(e->qw, tensor->type, K, N, base);
        const size_t raw_bytes = nbytes(tensor);
        R.op_arena.reset();
        void *raw = R.op_arena.get(raw_bytes, R.stream);
        B200_CHECK(cudaMemcpyAsync(raw, data, raw_bytes, cudaMemcpyHostToDevice, R.stream));
        repack_weights(e->qw, raw, R.stream);
        B200_CHECK(cudaStreamSynchronize(R.stream));
        e->is_q = true;
        e->data = base;
    } else {
        const size_t n = nbytes(tensor);
        B200_CHECK(cudaMalloc(&e->data, n));
        B200_CHECK(cudaMemcpy(e->data, data, n, cudaMemcpyHostToDevice));
        B200_CHECK(cudaDeviceSynchronize());   // legacy-stream copy/memset: not ordered with our non-blocking stream, and a pageable H2D cudaMemcpy may return before its DMA lands
    }
    tensor->extra = e;
}

void ggml_cuda_free_data(struct ggml_tensor *tensor) {                        // LC/ggml-cuda.cu:3873-3893
    if (!tensor || !on_device(tensor) || !tensor->extra) return;
    Extra *e = (Extra *)tensor->extra;
    if (!e->owned) return;
    B200_CHECK(cudaStreamSynchronize(rt().stream));
    if (e->data) B200_CHECK(cudaFree(e->data));
    delete e;
    tensor->extra = nullptr;
}

void ggml_cuda_assign_buffers(struct ggml_tensor *tensor) { assign_buffers_impl(tensor, true, false); }
void ggml_cuda_assign_buffers_no_scratch(struct ggml_tensor *tensor) { assign_buffers_impl(tensor, false, false); }
void ggml_cuda_assign_buffers_force_inplace(struct ggml_tensor *tensor) { assign_buffers_impl(tensor, false, true); }

bool ggml_cuda_can_mul_mat(const struct ggml_tensor *src0, const struct ggml_tensor *src1, struct ggml_tensor *dst) {   // :3627-3642
    const int64_t ne10 = src1->ne[0], ne0 = dst->ne[0], ne1 = dst->ne[1];
    // F32/F16 host-resident weights are not on this backend's path (only the five block formats are): let the CPU keep them.
    if (is_kquant(src0->type))
        return src1->type == B200_TYPE_F32 && dst->type == B200_TYPE_F32 && ne0 >= 32 && ne1 >= 32 && ne10 >= 32 && src0->ne[0] % 256 == 0 && src0->ne[2] == 1 && src0->ne[3] == 1;
    return is_quant(src0->type) && src1->type == B200_TYPE_F32 && dst->type == B200_TYPE_F32 && ne0 >= 32 && ne1 >= 32 && ne10 >= 32 &&
           src0->ne[0] % 64 == 0 && src0->ne[2] == 1 && src0->ne[3] == 1;
}

bool ggml_cuda_compute_forward(struct ggml_compute_params *params, struct ggml_tensor *tensor) {   // LC/ggml-cuda.cu:4018-4135
    const bool any_on_device = tensor->backend == B200_BACKEND_GPU ||
        (tensor->src[0] != nullptr && on_device(tensor->src[0])) ||
        (tensor->src[1] != nullptr && tensor->src[1]->backend == B200_BACKEND_GPU);
    if (!op_supported(tensor)) {
        if (any_on_device && tensor->op != B200_OP_NONE && tensor->op != B200_OP_GET_ROWS) {
            fprintf(stderr, "llm_b200: op %d has device-resident operands but is not served by this backend (no CPU fallback)\n", tensor->op);
            abort();
        }
        return false;
    }
    if (tensor->op == B200_OP_MUL_MAT) {
        if (!any_on_device && !ggml_cuda_can_mul_mat(tensor->src[0], tensor->src[1], tensor)) return false;
    } else if (!any_on_device) {
        return false;
    }
    if (params->ith != 0) return true;
    if (params->type == B200_TASK_INIT || params->type == B200_TASK_FINALIZE) return true;

    Runtime &R = rt();
    R.ensure_init();
    R.op_arena.reset();
    const ggml_tensor *s0 = tensor->src[0], *s1 = tensor->src[1];
    switch (tensor->op) {
        case B200_OP_MUL_MAT: op_mul_mat(s0, s1, tensor); break;
        case B200_OP_ADD: op_binary(0, s0, s1, tensor); break;
        case B200_OP_MUL: op_binary(1, s0, s1, tensor); break;
        case B200_OP_NORM: case B200_OP_RMS_NORM: case B200_OP_SOFT_MAX: case B200_OP_DIAG_MASK_INF: case B200_OP_SCALE: case B200_OP_UNARY:
            op_rows(s0, tensor); break;
        case B200_OP_ROPE: op_rope(s0, tensor); break;
        case B200_OP_CPY: case B200_OP_DUP: case B200_OP_CONT: op_cpy(s0, tensor); break;
        case B200_OP_RESHAPE: case B200_OP_VIEW: case B200_OP_PERMUTE: case B200_OP_TRANSPOSE: break;   // ggml_cuda_nop
        default: B200_ASSERT(!"unreachable");
    }
    return true;
}

void ggml_cuda_mul(const struct ggml_tensor *src0, const struct ggml_tensor *src1, struct ggml_tensor *dst) {
    rt().ensure_init();
    rt().op_arena.reset();
    op_binary(1, src0, src1, dst);
}
size_t ggml_cuda_mul_mat_get_wsize(const struct ggml_tensor *, const struct ggml_tensor *, struct ggml_tensor *) { return 0; }
void ggml_cuda_mul_mat(const struct ggml_tensor *src0, const struct ggml_tensor *src1, struct ggml_tensor *dst, void *, size_t) {
    rt().ensure_init();
    rt().op_arena.reset();
    op_mul_mat(src0, src1, dst);
}
void *ggml_cuda_host_malloc(size_t size) {       // LC/ggml-cuda.cu:2754-2771: NULL (caller falls back to malloc) on failure
    rt().ensure_init();
    void *p = nullptr;
    if (cudaMallocHost(&p, size) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void ggml_cuda_host_free(void *ptr) { if (ptr) B200_CHECK(cudaFreeHost(ptr)); }
void ggml_cuda_set_mul_mat_q(bool) {}

}  // extern "C"
