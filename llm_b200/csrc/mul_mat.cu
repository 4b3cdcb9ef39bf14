// llm_b200/csrc/mul_mat.cu -- ggml_mul_mat(w, x) on the conformant path: which bit-exact kernel serves a quantized weight at a batch size.
// The one place that choice is made for the LLaMA session (session.cu), the GPT-NeoX / GPT-2 session (neox.cu) and the ggml_cuda_* seam (seam.cu).
#include <stdlib.h>
#include <string.h>

#include "kernels.cuh"

namespace b200 {

// B200_PREFILL_GEMM=mma selects the round-1 mma.sync kernel for every batch size (default: wgmma for batches >= 96 tokens)
bool prefill_gemm_tc5() {
    static int v = -1;
    if (v < 0) { const char *e = getenv("B200_PREFILL_GEMM"); v = (e && !strcmp(e, "mma")) ? 0 : 1; }
    return v != 0;
}

int mul_mat_exact_auto(const QWeight &w, const float *x, int64_t ldx, int64_t B, float *dst, int64_t ldd, const float *addend, int64_t lda,
                       const ExactActs &a, cudaStream_t st) {
    if (w.type == T_F16) {                                   // ggml_fp32_to_fp16_row, then ggml_vec_dot_f16 per output (exact_f16.cu)
        cvt_act_f16(x, ldx, a.xh, w.K, B, st);
        if (B == 1 && mmv_f16_supported(w)) mul_mat_vec_f16(w, a.xh, dst, addend, st);
        else mul_mat_f16_gemm(w, a.xh, dst, ldd, B, addend, lda, st);
        return 2;
    }
    if (is_kquant(w.type)) {                                 // quantize_row_q8_K, then ggml_vec_dot_q*_K_q8_K per output (kquants.cu)
        quantize_act_q8k(x, ldx, a.xq8k, w.K, B, st);
        mul_mat_kq_exact(w.type, w.qs, a.xq8k, dst, ldd, w.K, w.N, B, addend, lda, st);
        return 2;
    }
    const int vdt = vec_dot_type(w.type);
    if (B == 1 && mmv_exact_stream_supported(w)) {          // decode: TMA bulk-copy ring at HBM speed (exact_stream.cu)
        quantize_act_pack(w.type, x, a.xpack, w.K, st);
        mul_mat_vec_q_exact_stream(w, a.xpack, dst, addend, st);
    } else if (B >= 96 && prefill_gemm_tc5()) {              // wgmma / TMA kernel: 128-token tiles (exact_tc5.cu)
        quantize_act_f16_rm(vdt, x, ldx, a.xh, a.xds, w.K, B, st);
        mul_mat_q_exact_tc5(w, a.xh, a.xds, dst, ldd, B, addend, lda, st);
    } else if (B >= 16) {                                    // mma.sync kernel: 64-token tiles, better for short batches (exact_mma.cu)
        quantize_act_f16(vdt, x, ldx, a.xh, a.xds, w.K, B, st);
        mul_mat_q_exact_mma(w, a.xh, a.xds, dst, ldd, B, addend, lda, st);
    } else {
        quantize_act(vdt, x, ldx, a.xq, a.xds, w.K, B, st);
        mul_mat_q_exact(w, a.xq, a.xds, dst, ldd, B, addend, lda, st);
    }
    return 2;
}

}  // namespace b200
