// llm_b200/csrc/stream_core.cuh -- building blocks of the bit-exact streaming mat-vec, shared by the stand-alone kernel
// (exact_stream.cu) and the fused mat-vecs of the decode schedules (decode_ops.cu).  See exact_stream.cu for the design notes.
#pragma once
#include "kernels.cuh"

#ifndef B200_PROF_SLOTS
#define B200_PROF_SLOTS 1024
#endif

namespace b200 {
namespace stream {

constexpr int SR = 32;        // rows per tile
constexpr int SCB = 16;       // quant blocks per ring stage
constexpr int SST = 4;        // ring stages of the stand-alone mat-vec kernel (the decode kernel uses a deeper ring: Ring::nst)
constexpr int SCOMPUTE = 128; // 4 compute warps (4 threads per row)
constexpr int STHREADS = SCOMPUTE + 32;   // + 1 producer warp

template <int TYPE, int ROWS = SR, int CB = SCB> struct St {
    static constexpr int QS = (TYPE == T_Q8_0) ? 32 : 16;
    static constexpr int DM = (TYPE == T_Q4_1 || TYPE == T_Q5_1) ? 4 : 2;
    static constexpr bool QH = (TYPE == T_Q5_0 || TYPE == T_Q5_1);
    static constexpr bool MIN = (TYPE == T_Q4_1 || TYPE == T_Q5_1);
    static constexpr int QS_STRIDE = CB * QS + 16;     // +16 B: the 8 rows of a warp land in different banks
    static constexpr int DM_STRIDE = CB * DM + 16;
    static constexpr int QH_STRIDE = CB * 4 + 16;
    static constexpr int QS_BYTES = ROWS * QS_STRIDE, DM_BYTES = ROWS * DM_STRIDE, QH_BYTES = QH ? ROWS * QH_STRIDE : 0;
    static constexpr int STAGE_BYTES = QS_BYTES + DM_BYTES + QH_BYTES;
    static constexpr int RING_BYTES = SST * STAGE_BYTES;
    __host__ __device__ static constexpr int ring_bytes(int nst) { return nst * STAGE_BYTES; }
};

// int -> float without the conversion unit: the block dots start from the accumulator seed 0x4B400000 (the bits of 12582912.0f = 1.5 * 2^23), so the
// integer result, read as a float, is exactly 12582912 + s for |s| < 2^22 (here |s| <= 4 * 128 * 127 + seeds), and one FADD on the FMA pipe returns
// exactly (float)s.  The I2F of the straightforward form runs on the quarter-rate XU pipe, which would otherwise be the busiest pipe of the
// mat-vec steady state while the FMA pipe idles.
constexpr int I2F_MAGIC = 0x4B400000;
__device__ __forceinline__ float i2f_magic(int biased) { return __fadd_rn(__int_as_float(biased), -12582912.0f); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) { asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void cp16(uint32_t dst, const void *src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
// arrive on `bar` once all cp.async issued so far by this thread have landed (counts against the barrier's expected arrivals)
__device__ __forceinline__ void cp_async_arrive(uint64_t *bar) { asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void compute_sync() { asm volatile("bar.sync 1, %0;" ::"n"(SCOMPUTE) : "memory"); }   // the 4 compute warps only

constexpr int SST_MAX = 12;    // barrier arrays: full[12] | empty[12] in the first 192 bytes of the CTA's shared memory
struct Ring {                 // per-CTA streaming state (lives in registers; the storage is shared memory)
    uint64_t *full, *empty;   // [nst] each
    uint8_t *base;
    uint32_t g;               // running stage counter: producer and consumers enumerate stages in the same order
    uint32_t nst;             // ring depth (<= SST_MAX)
    uint32_t slot, phase;     // g % nst and (g / nst) & 1, kept incrementally (nst is a run-time value: no division per stage)
    __device__ __forceinline__ void advance() { g++; if (++slot == nst) { slot = 0; phase ^= 1u; } }
};

__device__ __forceinline__ void ring_init(uint64_t *full, uint64_t *empty, int nst) {   // one thread, before a CTA-wide barrier
    for (int s = 0; s < nst; s++) { mbar_init(&full[s], 32); mbar_init(&empty[s], SCOMPUTE / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// One plane of a stage: SR rows x (COLS x 16 B), global row pitch src_pitch bytes, shared row pitch dst_pitch.  No divisions:
// COLS is a power of two, a warp instruction covers 32/COLS rows (COLS <= 32) or half a row (COLS == 64).
template <int COLS, int ROWS = SR>
__device__ __forceinline__ void stream_plane(uint32_t dst, int dst_pitch, const uint8_t *src, int64_t src_pitch, int cols_valid, int rows_valid, int lane) {
    if (COLS >= 32) {
#pragma unroll 8
        for (int rr = 0; rr < ROWS; rr++) {
            const uint8_t *srow = src + (int64_t)(rr < rows_valid ? rr : rows_valid - 1) * src_pitch;      // tail tile: re-read a valid row
#pragma unroll
            for (int k = 0; k < COLS / 32; k++) { const int cc = lane + 32 * k; if (cc < cols_valid) cp16(dst + rr * dst_pitch + cc * 16, srow + cc * 16); }
        }
    } else {
        constexpr int RPI = COLS >= 32 ? 1 : 32 / COLS;               // (this branch is dead for COLS >= 32)
        const int r0 = lane / COLS, cc = lane % COLS;
#pragma unroll
        for (int it = 0; it < ROWS / RPI; it++) {
            const int rr = it * RPI + r0;
            const uint8_t *srow = src + (int64_t)(rr < rows_valid ? rr : rows_valid - 1) * src_pitch;
            if (cc < cols_valid) cp16(dst + rr * dst_pitch + cc * 16, srow + cc * 16);
        }
    }
}

// Producer warp: stream every row tile (tile0, tile0 + tstride, ...) of W through the ring.
// Tiles are handed out in groups of G consecutive tiles (G = 2 lets an epilogue see 64 consecutive rows, e.g. 32 rows of w1 and the
// matching 32 rows of w3): group g = tile0, tile0 + tstride, ... covers tiles [g*G, g*G + G).
template <int TYPE, int ROWS = SR, int CB = SCB>
__device__ __forceinline__ void produce_matvec(const QWeight &w, Ring &R, int tile0, int tstride, int lane, int G = 1) {
    using T = St<TYPE, ROWS, CB>;
    const int nb = (int)w.nb, nchunks = (nb + CB - 1) / CB, ntiles = (int)((w.N + ROWS - 1) / ROWS);
    const uint32_t ring_u32 = smem_u32(R.base);
    for (int grp = tile0; grp * G < ntiles; grp += tstride)
    for (int tile = grp * G; tile < grp * G + G && tile < ntiles; tile++) {
        const int64_t row_base = (int64_t)tile * ROWS;
        const int rows_valid = (int)(w.N - row_base < ROWS ? w.N - row_base : ROWS);
        for (int c = 0; c < nchunks; c++, R.advance()) {
            const int s = R.slot;
            const int b0 = c * CB, cb = nb - b0 < CB ? nb - b0 : CB;
            mbar_wait(&R.empty[s], R.phase ^ 1u);
            const uint32_t st = ring_u32 + s * T::STAGE_BYTES;
            stream_plane<CB * T::QS / 16, ROWS>(st, T::QS_STRIDE, w.qs + (row_base * nb + b0) * T::QS, (int64_t)nb * T::QS, cb * T::QS / 16, rows_valid, lane);
            stream_plane<CB * T::DM / 16, ROWS>(st + T::QS_BYTES, T::DM_STRIDE, (const uint8_t *)w.dm + (row_base * nb + b0) * T::DM, (int64_t)nb * T::DM,
                                           cb * T::DM / 16, rows_valid, lane);
            if (T::QH)
                stream_plane<CB * 4 / 16, ROWS>(st + T::QS_BYTES + T::DM_BYTES, T::QH_STRIDE, (const uint8_t *)(w.qh + row_base * nb + b0), (int64_t)nb * 4,
                                           cb * 4 / 16, rows_valid, lane);
            cp_async_arrive(&R.full[s]);
        }
    }
}

// Compute warps: walk the AVX2 lane chains of the tiles this CTA owns.  epi(row, value) is called by ALL 128 threads once per tile
// (value = the finished dot product of `row`, identical in the 4 threads of a quad; row may be >= w.N on the tail tile).
template <int TYPE, class Epi>
__device__ __forceinline__ void consume_matvec(const QWeight &w, const int4 *sx, Ring &R, int tile0, int tstride, int tid, Epi epi, int G = 1,
                                               unsigned long long *prof = nullptr) {
    using T = St<TYPE>;
    const int nb = (int)w.nb, nchunks = (nb + SCB - 1) / SCB, ntiles = (int)((w.N + SR - 1) / SR);
    const int r = tid >> 2, wd = tid & 3, lane = tid & 31;
    for (int grp = tile0; grp * G < ntiles; grp += tstride)
    for (int tile = grp * G; tile < grp * G + G && tile < ntiles; tile++) {
        float a_lo = 0.f, a_hi = 0.f, summs = 0.f;
        for (int c = 0; c < nchunks; c++, R.advance()) {
            const int s = R.slot;
            const int b0 = c * SCB, cb = nb - b0 < SCB ? nb - b0 : SCB;
            mbar_wait(&R.full[s], R.phase);
            if (prof && tid == 0) {                                        // tuning aid (b200_session_decode_timeline): first / latest stage arrival
                unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                if (R.g == 0) { atomicMin(prof + 5 * B200_PROF_SLOTS, t); atomicMax(prof + 6 * B200_PROF_SLOTS, t); }
                atomicMax(prof + 7 * B200_PROF_SLOTS, t);
            }
            const uint8_t *st = R.base + s * T::STAGE_BYTES;
            const uint8_t *qrow = st + r * T::QS_STRIDE, *drow = st + T::QS_BYTES + r * T::DM_STRIDE, *hrow = st + T::QS_BYTES + T::DM_BYTES + r * T::QH_STRIDE;
#pragma unroll 8
            for (int b = 0; b < cb; b++) {
                const int4 xp = sx[(b0 + b) * 4 + wd];
                float dw, mw = 0.f;
                if (T::MIN) { const __half2 dm = *(const __half2 *)(drow + b * T::DM); dw = __low2float(dm); mw = __high2float(dm); }
                else dw = __half2float(*(const __half *)(drow + b * T::DM));
                int s_lo, s_hi;
                if (TYPE == T_Q8_0) {
                    s_lo = __dp4a(*(const int *)(qrow + b * T::QS + 4 * wd), xp.x, I2F_MAGIC);
                    s_hi = __dp4a(*(const int *)(qrow + b * T::QS + 16 + 4 * wd), xp.y, I2F_MAGIC);
                } else if (TYPE == T_Q4_0) {
                    // (q - 8) as a 4-bit two's complement value is q ^ 8; parked in the HIGH nibble of each byte it reads as 16*(q-8):
                    // the dp4a result is exactly 16 * sum (q-8) x, and the 1/16 rides (exactly, a power of two) in the packed d_x.
                    const uint32_t q = *(const uint32_t *)(qrow + b * T::QS + 4 * wd);
                    s_lo = __dp4a((int)(((q << 4) ^ 0x80808080u) & 0xF0F0F0F0u), xp.x, I2F_MAGIC);
                    s_hi = __dp4a((int)((q ^ 0x88888888u) & 0xF0F0F0F0u), xp.y, I2F_MAGIC);
                } else {
                    const uint32_t q = *(const uint32_t *)(qrow + b * T::QS + 4 * wd);
                    uint32_t l = q & 0x0F0F0F0Fu, h = (q >> 4) & 0x0F0F0F0Fu;
                    if (T::QH) {
                        const uint32_t qh = *(const uint32_t *)(hrow + b * 4);
                        l |= spread4_to_bit4(qh >> (4 * wd));
                        h |= spread4_to_bit4(qh >> (16 + 4 * wd));
                    }
                    // Q5_0: the -16 offset of every value is pre-multiplied into the accumulator seeds (exact integers); Q4_1/Q5_1: no offset
                    const int seed_lo = TYPE == T_Q5_0 ? (int)(short)(xp.z & 0xffff) + I2F_MAGIC : I2F_MAGIC;
                    const int seed_hi = TYPE == T_Q5_0 ? (xp.z >> 16) + I2F_MAGIC : I2F_MAGIC;
                    s_lo = __dp4a((int)l, xp.x, seed_lo);
                    s_hi = __dp4a((int)h, xp.y, seed_hi);
                }
                const float d = __fmul_rn(dw, __int_as_float(xp.w));
                a_lo = __fmaf_rn(d, i2f_magic(s_lo), a_lo);
                a_hi = __fmaf_rn(d, i2f_magic(s_hi), a_hi);
                if (T::MIN) summs = __fmaf_rn(mw, __int_as_float(xp.z), summs);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&R.empty[s]);
        }
        float v = __fadd_rn(a_hi, a_lo);                                   // hsum_float_8 (see exact.cu)
        v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 2));
        v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 1));
        if (T::MIN) v = __fadd_rn(v, summs);
        epi((int64_t)tile * SR + r, v);
    }
}

// Quantize one 32-element block held one value per lane (reference AVX2 arithmetic, see quant.cu) and emit its 4 packed records.
// record (block, word w) = { x bytes 4w..4w+3, x bytes 16+4w..16+4w+3, z, d_x }:
//   Q8_0 activations: z = 2 x int16 { -off * sum(bytes of word w), -off * sum(bytes of word w+4) } (off = 16 for Q5_0 weights, else 0),
//                     d_x = f32(fp16(amax/127)), pre-divided by 16 for Q4_0 weights (exact; the consumer computes 16 x the block dot)
//   Q8_1 activations: z = bits of s = d * sum(q), d_x = amax/127
__device__ __forceinline__ void pack_block(float v, int4 *rec4, int lane, int q81, int off, int scale16) {
    const float amax = warp_max(fabsf(v));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
    const int q = __float2int_rn(__fmul_rn(v, id));
    const int isum = warp_sum(q);
    uint32_t word = (uint32_t)(q & 0xff) << (8 * (lane & 3));
    word |= __shfl_xor_sync(0xffffffffu, word, 1);
    word |= __shfl_xor_sync(0xffffffffu, word, 2);
    int s4 = q + __shfl_xor_sync(0xffffffffu, q, 1);
    s4 += __shfl_xor_sync(0xffffffffu, s4, 2);
    const uint32_t word_hi = __shfl_down_sync(0xffffffffu, word, 16);
    const int s4_hi = __shfl_down_sync(0xffffffffu, s4, 16);
    if (lane < 16 && (lane & 3) == 0) {
        int4 rec;
        rec.x = (int)word; rec.y = (int)word_hi;
        if (q81) { rec.z = __float_as_int(__fmul_rn(d, (float)isum)); rec.w = __float_as_int(d); }
        else {
            rec.z = (int)(((uint32_t)(-off * s4) & 0xffffu) | ((uint32_t)(-off * s4_hi) << 16));
            const float dx = __half2float(__float2half_rn(d));
            rec.w = __float_as_int(scale16 ? dx * 0.0625f : dx);
        }
        rec4[lane >> 2] = rec;
    }
}

// Same arithmetic, 4 blocks per warp pass: lane l owns word (l & 7) = elements 4*(l&7) .. +3 of block (l >> 3).  The block maximum and
// the quant sum need 3 xor-shuffles each inside the 8-lane group, the packed word and its byte sum are lane-local, and the record's
// second word comes from 4 lanes up: 8 shuffles per 4 blocks instead of 16 per block.  `active` = this lane's block exists.
// returns true in the lanes that hold a record (word lane & 7 < 4 of an existing block); the caller stores it at [block * 4 + (lane & 7)]
__device__ __forceinline__ bool pack_quad_rec(float4 v, int lane, bool active, int q81, int off, int scale16, int4 &rec) {
    float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
    const int q0 = __float2int_rn(__fmul_rn(v.x, id)), q1 = __float2int_rn(__fmul_rn(v.y, id));
    const int q2 = __float2int_rn(__fmul_rn(v.z, id)), q3 = __float2int_rn(__fmul_rn(v.w, id));
    const uint32_t word = (uint32_t)(q0 & 0xff) | ((uint32_t)(q1 & 0xff) << 8) | ((uint32_t)(q2 & 0xff) << 16) | ((uint32_t)(q3 & 0xff) << 24);
    const int s4 = q0 + q1 + q2 + q3;
    int isum = s4 + __shfl_xor_sync(0xffffffffu, s4, 1);
    isum += __shfl_xor_sync(0xffffffffu, isum, 2);
    isum += __shfl_xor_sync(0xffffffffu, isum, 4);
    const uint32_t word_hi = __shfl_down_sync(0xffffffffu, word, 4);
    const int s4_hi = __shfl_down_sync(0xffffffffu, s4, 4);
    rec.x = (int)word; rec.y = (int)word_hi;
    if (q81) { rec.z = __float_as_int(__fmul_rn(d, (float)isum)); rec.w = __float_as_int(d); }
    else {
        rec.z = (int)(((uint32_t)(-off * s4) & 0xffffu) | ((uint32_t)(-off * s4_hi) << 16));
        const float dx = __half2float(__float2half_rn(d));
        rec.w = __float_as_int(scale16 ? dx * 0.0625f : dx);
    }
    return active && (lane & 7) < 4;
}
__device__ __forceinline__ void pack_quad(float4 v, int4 *rec4_of_my_block, int lane, bool active, int q81, int off, int scale16) {
    int4 rec;
    if (pack_quad_rec(v, lane, active, q81, off, scale16, rec)) rec4_of_my_block[lane & 7] = rec;
}

}  // namespace stream
}  // namespace b200
