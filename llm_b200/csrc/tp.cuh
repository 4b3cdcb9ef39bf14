// llm_b200/csrc/tp.cuh -- tensor-parallel decode: the exchange of activation slices between the GPUs of one NVSwitch box.
//
// Scheme (DESIGN.md section 5): every weight matrix is split by OUTPUT ROWS (heads for wq|wk|wv, n_ff/G rows of w1|w3, n_embd/G rows of wo / w2,
// n_vocab/G rows of the lm_head), so every dst element is still one complete ggml_vec_dot over the full K (LC/ggml.c:10570-10572) and the result is
// bit-identical to the single-GPU / CPU result by construction.  What travels between GPUs are the OUTPUT slices a following operator needs whole:
//   attention rows (as Q8 records)  -> wo's input        buffer XD
//   wo x + inpSA  (f32)             -> ffn rms_norm      buffer FF
//   silu(w1 x) * (w3 x) (records)   -> w2's input        buffer XF
//   w2 h + inpFF  (f32)             -> next rms_norm     buffer X
//   logits (f32)                    -> the caller        buffer LOGITS
// There is no collective call and no fence on the data path.  Every 32-bit word travels as an 8-byte unit {payload, tag} written with ONE 64-bit store
// straight into EVERY rank's buffer through peer-mapped pointers (NVLink / NVSwitch P2P stores, CUDA IPC mappings of one "exchange slab" per rank); an
// aligned 8-byte store is single-copy atomic, so a consumer that polls a unit until its tag equals the expected one has the payload -- the low-latency
// protocol NCCL calls LL.  tag = epoch * (n_layer + 1) + layer stamp + 1, epoch = tokens decoded so far: monotonic, nothing is ever reset, and a unit is
// only rewritten after every rank consumed its previous content (the next write of a buffer needs results that depend on all ranks having read it).
// The alternative -- plain stores + __threadfence_system() + a per-kernel flag -- puts a system-scope fence and a flag round trip into every exchanging kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

constexpr int TP_MAX = 8;
enum { TPB_X = 0, TPB_FF = 1, TPB_XD = 2, TPB_XF = 3, TPB_LOGITS = 4, TPB_COUNT = 5 };

struct TpCtx {                 // kernel argument (POD); world == 1: single GPU, the kernels use their plain local buffers
    int world = 1, rank = 0;
    char *peer[TP_MAX] = {};   // base of rank p's exchange slab as mapped in THIS process (peer[rank] is the local slab)
    unsigned *epoch = nullptr;     // local: [0] tokens decoded so far, [1] number of polls that timed out (a peer died)
    uint32_t off[TPB_COUNT] = {};  // byte offsets of the buffers (arrays of 8-byte units) inside a slab
    unsigned vmul = 1;             // n_layer + 1
    int nowait = 0;                // measurement aid (b200_session_tp_set_nowait): 1 = accept whatever a unit holds -- results are garbage, the time is compute + stores;
                                   // 2 = additionally store to the local slab only: the time is compute alone
    int relax = 0;                 // bit 0: the norm kernels, bit 1: the mat-vecs fed by exchanged records -- kernels whose every dependence on their predecessor
                                   // travels through tagged units may skip griddepcontrol.wait (which also waits for the predecessor's peer stores to be
                                   // acknowledged across NVLink).  Compute alone gets faster that way,
                                   // but the early-resident pollers take issue slots and L2 bandwidth from the producers and the token need not get faster:
                                   // default 0 = every kernel waits for its predecessor grid.  B200_TP_RELAX overrides.
};

// what one kernel instance reads / writes (baked into the CUDA graph; the epoch is read from device memory)
struct TpSync {
    int in_buf = -1; unsigned in_v = 0;       // input vector / records come from this exchange buffer with layer stamp in_v (-1: local plain buffer)
    int add_buf = -1; unsigned add_v = 0;     // residual addend (this rank's own slice of it)
    int out_buf = -1; unsigned out_v = 0;     // results go to this buffer of every rank
};

__device__ __forceinline__ unsigned tp_tag(const TpCtx &T, unsigned v) { return *(volatile unsigned *)T.epoch * T.vmul + v + 1u; }   // never 0 (the slab starts zeroed)

__device__ __forceinline__ void tp_put(const TpCtx &T, int buf, int64_t unit, uint32_t payload, unsigned tag) {
#pragma unroll 1
    for (int p = 0; p < T.world; p++) {
        if (T.nowait == 2 && p != T.rank) continue;
        uint2 *dst = (uint2 *)(T.peer[p] + T.off[buf]) + unit;
        asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(dst), "r"(payload), "r"(tag) : "memory");
    }
}
__device__ __forceinline__ void tp_put_f32(const TpCtx &T, int buf, int64_t unit, float v, unsigned tag) { tp_put(T, buf, unit, __float_as_uint(v), tag); }
__device__ __forceinline__ void tp_put_rec(const TpCtx &T, int buf, int64_t rec, int4 r, unsigned tag) {    // a 16-byte record = 4 units
    tp_put(T, buf, rec * 4 + 0, (uint32_t)r.x, tag); tp_put(T, buf, rec * 4 + 1, (uint32_t)r.y, tag);
    tp_put(T, buf, rec * 4 + 2, (uint32_t)r.z, tag); tp_put(T, buf, rec * 4 + 3, (uint32_t)r.w, tag);
}

// poll the LOCAL copy of a unit until its tag is the expected one
__device__ __forceinline__ uint32_t tp_get(const TpCtx &T, int buf, int64_t unit, unsigned tag) {
    const uint2 *src = (const uint2 *)(T.peer[T.rank] + T.off[buf]) + unit;
    uint32_t v, t;
    asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v), "=r"(t) : "l"(src) : "memory");
    if (t == tag || T.nowait || *(volatile unsigned *)(T.epoch + 1)) return v;      // after the first timeout nothing waits any more: the session is dead, the host reports it
    const long long t0 = clock64();
    unsigned ns = 32;
    do {
        __nanosleep(ns); if (ns < 512) ns *= 2;                  // back off: thousands of spinning threads would otherwise flood L2 while the producers still stream weights
        asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v), "=r"(t) : "l"(src) : "memory");
        if (clock64() - t0 > 6000000000LL) { atomicAdd(T.epoch + 1, 1u); break; }        // a peer is gone: do not hang the GPU, count it (b200_session_tp_timeouts)
    } while (t != tag);
    return v;
}
// One warp waits for a spread sample of a buffer (32 units, one per lane) before the CTA gathers it: a consumer that was launched ahead of its data
// (TpCtx::relax) then polls 32 words per CTA with back-off instead of re-reading the whole buffer from L2 until it is complete.
__device__ __forceinline__ void tp_wait_sample(const TpCtx &T, int buf, int64_t nunits, unsigned tag, int lane) {
    const int64_t unit = nunits <= 32 ? (lane < nunits ? lane : nunits - 1) : (int64_t)lane * (nunits - 1) / 31;
    (void)tp_get(T, buf, unit, tag);
}
// Two units per 16-byte load, for consumers that read many units: issue ALL the loads first (tp_ld2), then check the tags (tp_fix2) -- the polling branch
// of tp_get serialises a thread's loads at one L2 round trip each.
__device__ __forceinline__ uint4 tp_ld2(const TpCtx &T, int buf, int64_t pair) {
    const uint4 *src = (const uint4 *)(T.peer[T.rank] + T.off[buf]) + pair;
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src) : "memory");
    return v;
}
__device__ __forceinline__ void tp_fix2(const TpCtx &T, int buf, int64_t pair, unsigned tag, uint4 &v) {     // payloads end up in v.x and v.z
    if (T.nowait) return;
    if (v.y != tag) v.x = tp_get(T, buf, 2 * pair, tag);
    if (v.w != tag) v.z = tp_get(T, buf, 2 * pair + 1, tag);
}
__device__ __forceinline__ float tp_get_f32(const TpCtx &T, int buf, int64_t unit, unsigned tag) { return __uint_as_float(tp_get(T, buf, unit, tag)); }

}  // namespace b200
