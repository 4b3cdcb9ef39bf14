// llm_b200/csrc/lora.cu -- LoRA adapters patched into a weight as it is loaded (LoraAdapter::patch, crates/llm-base/src/lora.rs:71-140), bit-exact
// with the reference's CPU graph for one adapter on a target W [ne0 = K, ne1 = N]:
//   ba = ggml_mul_mat(A [r, K], B [r, NB])     ba[n][k] = vec_dot(A row k, B row n): ggml_vec_dot_f32 (A F32) or ggml_vec_dot_f16 on B rounded to fp16 (A F16)
//   ba = ggml_scale(ba, alpha / r)            only when the scaling is not 1
//   W  = ggml_add(W, ba)                      block types: ggml_compute_forward_add_q_f32 (LC/ggml.c:8273-8345), dequantize_row -> + ba -> from_float,
//                                             where from_float is quantize_row_*_reference for Q4_0..Q5_1 and the AVX2 quantize_row_q8_0 for Q8_0;
//                                             F32: add_f32, the rows of ba repeated over W's (NB divides N)
// One fused kernel: no K x N intermediate leaves the CTA.  CTA = 16 rows of W x one 32-element block column; warp w owns rows 2w, 2w + 1 and lane j
// element j of the block, so the warp ends holding exactly one block per row and dequantizes, adds and requantizes it in place with the shared rules
// of quant_rules.cuh.  The dots run on CUDA cores in the reference's order (tensor cores cannot reproduce it): each thread keeps the 32 chains of
// the AVX code (element i of a 32-element step -> chain i % 32) for its two outputs, fed from 32-element slices of A and B staged in shared memory.
#include "../../include/llm_b200.h"
#include "f32dot.cuh"
#include "kernels.cuh"
#include "quant_rules.cuh"

namespace b200 {

constexpr int LP_ROWS = 16, LP_THREADS = 256, LP_RPW = LP_ROWS / (LP_THREADS / 32), LP_STRIDE = 36;   // stride 36: the float4 reads of a quarter-warp hit disjoint banks

// the 32 chains of one output end in f32x8_reduce (f32dot.cuh), the GGML_F32x8_REDUCE that ggml_vec_dot_f32 and ggml_vec_dot_f16 share

// w: N rows of the target in GGML layout (WT = T_F32: N rows of K floats).  a: K rows of r (f32, or f16 when A16); b: NB rows of r floats.
template <int WT, bool A16>
__global__ void __launch_bounds__(LP_THREADS) lora_patch_kernel(uint8_t *__restrict__ w, int64_t K, int64_t N, const void *__restrict__ a,
                                                                 const float *__restrict__ b, int64_t r, int64_t nb_rows, float scaling) {
    __shared__ __align__(16) float sa[32][LP_STRIDE];
    __shared__ __align__(16) float sb[LP_ROWS][LP_STRIDE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t n0 = (int64_t)blockIdx.x * LP_ROWS, kb = blockIdx.y;

    // slice [c0, c0 + 32) of A's rows kb*32.. and of B's rows for n0.., zero past r, K or N; B rounded to fp16 for the f16 dot (from_float of F16)
    auto stage = [&](int64_t c0) {
#pragma unroll
        for (int i = 0; i < 32 * 32 / LP_THREADS; i++) {
            const int idx = tid + i * LP_THREADS, row = idx >> 5, col = idx & 31;
            const int64_t k = kb * 32 + row, c = c0 + col;
            float v = 0.f;
            if (k < K && c < r) v = A16 ? __half2float(((const __half *)a)[k * r + c]) : ((const float *)a)[k * r + c];
            sa[row][col] = v;
        }
#pragma unroll
        for (int i = 0; i < LP_ROWS * 32 / LP_THREADS; i++) {
            const int idx = tid + i * LP_THREADS, row = idx >> 5, col = idx & 31;
            const int64_t n = n0 + row, c = c0 + col;
            float v = 0.f;
            if (n < N && c < r) {
                v = b[(n % nb_rows) * r + c];
                if (A16) v = __half2float(__float2half_rn(v));
            }
            sb[row][col] = v;
        }
    };

    float acc[LP_RPW][32];
#pragma unroll
    for (int j = 0; j < LP_RPW; j++)
#pragma unroll
        for (int l = 0; l < 32; l++) acc[j][l] = 0.f;
    const int64_t np = r & ~(int64_t)31;
    for (int64_t c0 = 0; c0 < np; c0 += 32) {                       // GGML_F32_STEP / GGML_F16_STEP = 32: one fma per chain and step
        __syncthreads();
        stage(c0);
        __syncthreads();
#pragma unroll
        for (int l = 0; l < 32; l += 4) {
            const float4 x = *(const float4 *)&sa[lane][l];
#pragma unroll
            for (int j = 0; j < LP_RPW; j++) {
                const float4 y = *(const float4 *)&sb[warp * LP_RPW + j][l];
                acc[j][l] = __fmaf_rn(x.x, y.x, acc[j][l]);     acc[j][l + 1] = __fmaf_rn(x.y, y.y, acc[j][l + 1]);
                acc[j][l + 2] = __fmaf_rn(x.z, y.z, acc[j][l + 2]); acc[j][l + 3] = __fmaf_rn(x.w, y.w, acc[j][l + 3]);
            }
        }
    }
    float s[LP_RPW];
#pragma unroll
    for (int j = 0; j < LP_RPW; j++) s[j] = f32x8_reduce(acc[j]);
    if (np < r) {                                                     // leftovers, one by one in order
        __syncthreads();
        stage(np);
        __syncthreads();
        const int left = (int)(r - np);
#pragma unroll
        for (int j = 0; j < LP_RPW; j++) {
            const float *y = sb[warp * LP_RPW + j];
            if (A16) {                                                // ggml_vec_dot_f16: sumf is a double, += (double)(f32 product)
                double sd = (double)s[j];
                for (int i = 0; i < left; i++) sd += (double)__fmul_rn(sa[lane][i], y[i]);
                s[j] = (float)sd;
            } else {                                                  // ggml_vec_dot_f32 as compiled (f32dot.cuh)
                s[j] = f32_leftovers(s[j], left, [&](int i) { return sa[lane][i]; }, [&](int i) { return y[i]; });
            }
        }
    }

#pragma unroll
    for (int j = 0; j < LP_RPW; j++) {
        const int64_t n = n0 + warp * LP_RPW + j;                     // warp-uniform
        if (n >= N) break;
        const float v = scaling != 1.0f ? __fmul_rn(s[j], scaling) : s[j];
        if (WT == T_F32) {
            const int64_t k = kb * 32 + lane;
            if (k < K) { float *p = (float *)w + n * K + k; *p = __fadd_rn(*p, v); }
            continue;
        }
        if (WT == T_F16) {                                            // add_f16_f32 (LC/ggml.c:8165-8215): fp16(f32(w) + ba)
            const int64_t k = kb * 32 + lane;
            if (k < K) { __half *p = (__half *)w + n * K + k; *p = __float2half_rn(__fadd_rn(__half2float(*p), v)); }
            continue;
        }
        uint8_t *blk = w + (n * (K / QK) + kb) * ggml_block_bytes(WT);
        float d, m, lo, hi;
        uint32_t qh;
        const uint8_t *qs = raw_block_header(WT, blk, d, m, qh);
        dequant_block(WT, qs, qh, d, m, lane & 15, lo, hi);
        const float x = __fadd_rn(lane < 16 ? lo : hi, v);           // dequantize_row_q -> ggml_vec_acc_f32
        __syncwarp();                                                 // every lane has read the block before it is overwritten
        uint16_t *h16 = (uint16_t *)blk;
        if (WT == T_Q8_0) {
            float dq;
            const int q = quantize_q8_avx2(x, dq);
            ((int8_t *)blk)[2 + lane] = (int8_t)q;
            if (lane == 0) h16[0] = f32_to_f16_bits(dq);
            continue;
        }
        float dq, mn;
        const int q = quantize_block_ref(WT, x, dq, mn);
        const int qhi = __shfl_down_sync(0xffffffffu, q, 16);
        const unsigned bits5 = __ballot_sync(0xffffffffu, (q & 0x10) != 0);
        uint8_t *qs_out = (uint8_t *)qs;
        if (lane < 16) qs_out[lane] = (uint8_t)((q & 0xF) | ((qhi & 0xF) << 4));
        if (lane == 0) {
            int o = 0;
            h16[o++] = f32_to_f16_bits(dq);
            if (has_min(WT)) h16[o++] = f32_to_f16_bits(mn);
            if (has_qh(WT)) { h16[o] = (uint16_t)(bits5 & 0xffffu); h16[o + 1] = (uint16_t)(bits5 >> 16); }
        }
    }
}

template <int WT>
static void launch_lora(uint8_t *w, int64_t K, int64_t N, int a_type, const void *a, const float *b, int64_t r, int64_t nb_rows, float scaling, cudaStream_t st) {
    const dim3 grid((unsigned)((N + LP_ROWS - 1) / LP_ROWS), (unsigned)((K + 31) / 32));
    if (a_type == T_F16) lora_patch_kernel<WT, true><<<grid, LP_THREADS, 0, st>>>(w, K, N, a, b, r, nb_rows, scaling);
    else                 lora_patch_kernel<WT, false><<<grid, LP_THREADS, 0, st>>>(w, K, N, a, b, r, nb_rows, scaling);
    B200_CHECK(cudaGetLastError());
}

int lora_check(int wtype, int64_t K, int64_t N, int a_type, int64_t a_ne0, int64_t a_ne1, int b_type, int64_t b_ne0, int64_t b_ne1) {
    if ((a_type != T_F32 && a_type != T_F16) || b_type != T_F32) return B200_ERR_UNSUPPORTED_ELEMENT_TYPE;   // nb10 == sizeof(float), LC/ggml.c:10424-10427
    if (wtype != T_F32 && wtype != T_F16 && !is_quant(wtype)) return B200_ERR_UNSUPPORTED_ELEMENT_TYPE;
    if (a_ne0 != b_ne0 || a_ne1 != K || b_ne1 < 1) return B200_ERR_TENSOR_SHAPE;                         // ggml_can_mul_mat; ba has K rows
    if (wtype == T_F32 ? N % b_ne1 != 0 : b_ne1 != N) return B200_ERR_TENSOR_SHAPE;                      // ggml_can_repeat_rows / add_q_f32's same shape
    if (is_quant(wtype) && K % QK) return B200_ERR_TENSOR_SHAPE;
    if ((K + 31) / 32 > 65535 || (N + LP_ROWS - 1) / LP_ROWS > 0x7fffffff) return B200_ERR_TENSOR_SHAPE;   // grid limits
    return B200_OK;
}

void lora_patch(int wtype, void *w, int64_t K, int64_t N, int a_type, const void *a, const float *b, int64_t r, int64_t nb_rows, float scaling, cudaStream_t st) {
    if (K == 0 || N == 0) return;
    uint8_t *p = (uint8_t *)w;
    switch (wtype) {
        case T_F32:  launch_lora<T_F32>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        case T_F16:  launch_lora<T_F16>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        case T_Q4_0: launch_lora<T_Q4_0>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        case T_Q4_1: launch_lora<T_Q4_1>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        case T_Q5_0: launch_lora<T_Q5_0>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        case T_Q5_1: launch_lora<T_Q5_1>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        case T_Q8_0: launch_lora<T_Q8_0>(p, K, N, a_type, a, b, r, nb_rows, scaling, st); break;
        default: B200_ASSERT(!"lora_patch: unsupported target type");
    }
}

}  // namespace b200
