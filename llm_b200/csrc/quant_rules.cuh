// llm_b200/csrc/quant_rules.cuh -- the reference's per-block quantization arithmetic as device functions, one 32-element block per warp
// (lane j <-> element j) or per 16 threads (dequant_block).  Shared by the weight upload and get_rows (quant.cu), the synthetic weights (synth.cu)
// and the LoRA patch (lora.cu), so that each rule is written once.
#pragma once
#include "common.cuh"

namespace b200 {

// One GGML block in file layout (2-byte aligned): d [m] [qh] qs.  Reads the header, returns the qs pointer.
__device__ __forceinline__ const uint8_t *raw_block_header(int type, const uint8_t *p, float &d, float &m, uint32_t &qh) {
    const uint16_t *p16 = (const uint16_t *)p;
    int o = 0;
    d = f16_bits_to_f32(p16[o++]);
    m = 0.f;
    if (has_min(type)) m = f16_bits_to_f32(p16[o++]);
    qh = 0;
    if (has_qh(type)) { qh = (uint32_t)p16[o] | ((uint32_t)p16[o + 1] << 16); o += 2; }
    return p + 2 * o;
}

// dequantize_row_* (LC/ggml.c:1525-1635).  `x*d + m` is a fused multiply-add in the reference build.
__device__ __forceinline__ void dequant_block(int type, const uint8_t *qs, uint32_t qh, float d, float m, int lane16, float &lo, float &hi) {
    // element lane16 (lo half) and lane16 + 16 (hi half) of the block
    if (type == T_Q8_0) { lo = (float)((const int8_t *)qs)[lane16] * d; hi = (float)((const int8_t *)qs)[lane16 + 16] * d; return; }
    const int q = qs[lane16];
    int q0 = q & 0xF, q1 = q >> 4;
    if (has_qh(type)) { q0 |= ((qh >> lane16) & 1) << 4; q1 |= ((qh >> (lane16 + 16)) & 1) << 4; }
    switch (type) {
        case T_Q4_0: lo = (float)(q0 - 8) * d;  hi = (float)(q1 - 8) * d; break;
        case T_Q5_0: lo = (float)(q0 - 16) * d; hi = (float)(q1 - 16) * d; break;
        default:     lo = __fmaf_rn((float)q0, d, m); hi = __fmaf_rn((float)q1, d, m); break;   // Q4_1, Q5_1
    }
}

// quantize_row_q{4_0,4_1,5_0,5_1,8_0}_reference (LC/ggml.c:943-1145), what ggml_quantize_* calls: the lane's quant q (the 5-bit value for Q5_x),
// and the block's d and min (Q4_1 / Q5_1), in f32 before the fp16 store.  All 32 lanes take part.
// FMA: `x0 = x*id; (int8_t)(x0 + 8.5f)` (16.5f, and `(x - min)*id + 0.5f` for Q4_1 / Q5_1) is one fused multiply-add, as the reference's release
// build executes it (gcc -O3 -mfma contracts across the two statements; oracle/_ref/libggml_ref.so has vfmadd there): the file quantizer.  Without
// it each step is rounded, as oracle/ggml_oracle.c restates the rule: the synthetic weights and the LoRA patch.  The two differ only where the
// sum lands within an ulp of an integer (about one block in 400 of F16 values).  Signed zeros follow the reference's scans in both forms.
template <bool FMA = false>
__device__ __forceinline__ int quantize_block_ref(int type, float v, float &d, float &mn) {
    int q = 0;
    d = 0.f; mn = 0.f;
    if (type == T_Q4_0 || type == T_Q5_0) {
        const float amax = warp_max(fabsf(v));
        const unsigned who = __ballot_sync(0xffffffffu, fabsf(v) == amax);
        // the first element attaining amax (strict `<` scan from max = 0.0f: an all-zero block keeps +0, whatever the signs of its zeros)
        const float mx = amax == 0.f ? 0.f : __shfl_sync(0xffffffffu, v, __ffs(who) - 1);
        const float div = type == T_Q4_0 ? -8.f : -16.f;
        d = __fdiv_rn(mx, div);
        const float id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.f;
        const float off = type == T_Q4_0 ? 8.5f : 16.5f;
        q = min(type == T_Q4_0 ? 15 : 31, (int)(int8_t)__float2int_rz(FMA ? __fmaf_rn(v, id, off) : __fadd_rn(__fmul_rn(v, id), off)));
    } else if (type == T_Q4_1 || type == T_Q5_1) {
        // the first element equal to the minimum / maximum (strict `<` / `>` scans): the sign of a zero extreme is that element's
        const float lo = -warp_max(-v), hi = warp_max(v);
        mn = __shfl_sync(0xffffffffu, v, __ffs(__ballot_sync(0xffffffffu, v == lo)) - 1);
        const float mx = __shfl_sync(0xffffffffu, v, __ffs(__ballot_sync(0xffffffffu, v == hi)) - 1);
        const int levels = type == T_Q4_1 ? 15 : 31;
        d = __fdiv_rn(__fsub_rn(mx, mn), (float)levels);
        const float id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.f;
        q = __float2int_rz(FMA ? __fmaf_rn(__fsub_rn(v, mn), id, 0.5f) : __fadd_rn(__fmul_rn(__fsub_rn(v, mn), id), 0.5f));
        if (type == T_Q4_1) q = min(15, q);
        q &= 0xff;
    } else {   // Q8_0
        const float amax = warp_max(fabsf(v));
        d = __fdiv_rn(amax, 127.f);
        const float id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.f;
        q = (int)roundf(__fmul_rn(v, id));
    }
    return q;
}

// The AVX2 bodies of quantize_row_q8_0 / q8_1 (LC/ggml.c:1239-1254 / 1449-1474):
//   d = amax / 127 ; id = amax != 0 ? 127 / amax : 0 ; q = round-half-even(x * id)      (NOT 1/d, NOT roundf)
// IEEE division and a separately rounded multiply are forced with __fdiv_rn / __fmul_rn.  All 32 lanes take part; d is f32 (q8_0 stores fp16(d)).
__device__ __forceinline__ int quantize_q8_avx2(float v, float &d) {
    const float amax = warp_max(fabsf(v));
    d = __fdiv_rn(amax, 127.f);
    const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
    return __float2int_rn(__fmul_rn(v, id));
}

}  // namespace b200
