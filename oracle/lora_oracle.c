/*
 * oracle/lora_oracle.c -- TEST INFRASTRUCTURE (parity oracle): the LoRA patch of LoraAdapter::patch (crates/llm-base/src/lora.rs:71-140) restated in
 * plain C on the rules of ggml_oracle.c.  Built with ggml_oracle.c into liboracle_lora.so (oracle/lora.mk) and pinned bit for bit to the reference's
 * own ggml.c driven by ref_lora.c (tests/test_lora_file.py).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "ggml_oracle.h"

/* ggml_vec_dot_f32, AVX body (LC/ggml.c:2288-2323, GGML_F32_STEP 32, GGML_F32_EPR 8): element i of each 32-element step goes to lane i % 32, fused
 * multiply-add in order; GGML_F32x8_REDUCE (:1897-1915) adds lanes l and l + 16, then l and l + 8, then the 128-bit halves (l and l + 4), then two hadds.
 * The leftovers (n % 32) are added one by one, in order, but the reference build (gcc -O3 -mavx2 -mfma, GNU C) vectorizes their products: groups of
 * eight, then one of four, are multiplied as vectors (each product rounded to f32, then added), and only the last (n % 32) % 4 are contracted
 * into scalar FMAs (the compiled ggml_vec_dot_f32 of oracle/_ref; tests/test_lora_file.py pins r = 3, 7, 8, 31, 35 and 40). */
float or_vec_dot_f32(int64_t n, const float *x, const float *y) {
    const int64_t np = n & ~(int64_t)31;
    float acc[32] = {0};
    for (int64_t i = 0; i < np; i += 32)
        for (int l = 0; l < 32; l++) acc[l] = fmaf(x[i + l], y[i + l], acc[l]);
    for (int l = 0; l < 16; l++) acc[l] = acc[l] + acc[l + 16];
    for (int l = 0; l < 8; l++) acc[l] = acc[l] + acc[l + 8];
    for (int l = 0; l < 4; l++) acc[l] = acc[l] + acc[l + 4];
    float sumf = (acc[0] + acc[1]) + (acc[2] + acc[3]);
    const int64_t nv = np + ((n - np) & ~(int64_t)3);
    for (int64_t i = np; i < nv; i++) sumf += x[i] * y[i];
    for (int64_t i = nv; i < n; i++) sumf = fmaf(x[i], y[i], sumf);
    return sumf;
}

/* One adapter on one target W [K, N] in GGML layout (type wtype: F32 or one of the five block types), in place:
 *   ba[n][k] = vec_dot(A row k, B row n % nb_rows)     A: K rows of r (F32, or F16 with B's rows rounded to fp16 first, LC/ggml.c:10504-10520)
 *   ba *= scaling if scaling != 1                     ggml_vec_scale_f32
 *   W row n = from_float(to_float(W row n) + ba row)  ggml_compute_forward_add_q_f32 (:8273-8345): from_float is quantize_row_*_reference for
 *                                                     Q4_0..Q5_1 and the AVX2 quantize_row_q8_0 (round half to even) for Q8_0; F32: add_f32 */
void or_lora_patch(int wtype, void *w, int64_t K, int64_t N, int a_type, const void *a, const float *b, int64_t r, int64_t nb_rows, float scaling) {
    float *row = malloc((size_t)K * 4), *ba = malloc((size_t)K * 4);
    uint16_t *b16 = malloc((size_t)r * 2);
    const size_t rb = or_row_bytes(wtype, K);
    for (int64_t n = 0; n < N; n++) {
        const float *bn = b + (n % nb_rows) * r;
        if (a_type == OR_F16)
            for (int64_t i = 0; i < r; i++) b16[i] = or_fp32_to_fp16(bn[i]);
        for (int64_t k = 0; k < K; k++) {
            const float v = a_type == OR_F16 ? or_vec_dot_f16(r, (const uint16_t *)a + k * r, b16) : or_vec_dot_f32(r, (const float *)a + k * r, bn);
            ba[k] = scaling != 1.0f ? v * scaling : v;
        }
        char *wn = (char *)w + n * rb;
        if (wtype == OR_F32) {
            for (int64_t k = 0; k < K; k++) ((float *)wn)[k] += ba[k];
            continue;
        }
        or_dequantize_row(wtype, wn, row, K);
        for (int64_t k = 0; k < K; k++) row[k] += ba[k];
        if (wtype == OR_Q8_0) or_quantize_row_q8_0(row, wn, K);
        else or_quantize_weights(wtype, row, wn, 1, K);
    }
    free(row); free(ba); free(b16);
}
