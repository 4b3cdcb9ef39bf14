// llm_b200/csrc/tc5.cuh -- thin inline-PTX wrappers of the Hopper (sm_90a) machinery used by the wgmma GEMMs:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma.mma_async with shared-memory descriptors, setmaxnreg.
// Descriptor bit layout: PTX ISA "Matrix Descriptor Format" for wgmma (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {
namespace tc5 {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Spin with a watchdog: a protocol bug must not hang the GPU.  After ~1 s without progress the thread records
// (bar, parity, block, thread) in g_timeout, turns "dead" (all its later waits return at once) and the kernel runs to completion with
// garbage results; the host reads g_timeout (check_timeout) in the op-level entry points and the tests.
static __device__ unsigned int g_timeout[8];   // one copy per translation unit (each kernel file has its own *_check_timeout)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, bool &dead) {
    if (dead || mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 2000000000LL) {
            dead = true;
            if (atomicAdd(&g_timeout[0], 1u) == 0u) { g_timeout[1] = bar; g_timeout[2] = parity; g_timeout[3] = blockIdx.x; g_timeout[4] = blockIdx.y; g_timeout[5] = threadIdx.x; }
            return;
        }
    }
}
// generic-proxy writes to shared memory -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- TMA ----------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *m) { asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory"); }
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *m, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(m), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// ---- wgmma ----------------------------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (K-major operands).  Canonical layouts in 16-byte units (cute/atom/mma_traits_sm90_gmma.hpp):
//   no swizzle : ((8,n),2):((1,SBO),LBO)   -- 8 rows x 16 B core matrices; LBO = stride between the two K halves, SBO = between 8-row groups
//   128B swizzle: ((8,n),2):((8,SBO),1)    -- rows of 128 B, 16-byte chunk c of row r at chunk (c ^ (r & 7)); SBO = 1024 B; LBO unused
constexpr uint64_t LAYOUT_NONE = 0, LAYOUT_SW128 = 1;
__host__ __device__ inline uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (layout << 62);
}
// wgmma issue protocol of a warpgroup: fence (orders earlier register / shared-memory accesses before the async reads), the MMAs,
// commit them as one group, wait until at most N groups are pending
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads of wgmma accumulators above the wait that makes them valid
template <int R> __device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, f16 inputs from shared memory (K-major descriptors), f32 accumulators in registers.
// Thread `lane` of warp w of the warpgroup holds rows 16w + lane/4 (d[4i], d[4i+1]) and 16w + lane/4 + 8 (d[4i+2], d[4i+3]), columns 8i + 2(lane%4) + {0, 1}.
// Operand lists: SM90_OPS(t) names %t0 .. %t9, SM90_ACC8(i) binds d[i .. i+7] read-write.
#define SM90_OPS(t) "%" #t "0, %" #t "1, %" #t "2, %" #t "3, %" #t "4, %" #t "5, %" #t "6, %" #t "7, %" #t "8, %" #t "9"
#define SM90_OPS0 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9"
#define SM90_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define SM90_ACC32(i) SM90_ACC8(i), SM90_ACC8(i + 8), SM90_ACC8(i + 16), SM90_ACC8(i + 24)
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
                 SM90_OPS0 ", " SM90_OPS(1) ", " SM90_OPS(2) ", %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : SM90_ACC32(0) : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
// the same with N = 128 (64 accumulators per thread, i < 16)
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
                 SM90_OPS0 ", " SM90_OPS(1) ", " SM90_OPS(2) ", " SM90_OPS(3) ", " SM90_OPS(4) ", " SM90_OPS(5) ", %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : SM90_ACC32(0), SM90_ACC32(32) : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

template <int N> __device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// cuTensorMapEncodeTiled through the runtime's driver entry point (the library links cudart statically and not libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// returns 0 if no mbarrier wait of this translation unit's kernels ever timed out; prints the first record otherwise
inline int check_timeout(const char *what) {
    unsigned int h[8] = {0};
    if (cudaMemcpyFromSymbol(h, g_timeout, sizeof(h)) != cudaSuccess) return -1;
    if (h[0] == 0) return 0;
    fprintf(stderr, "llm_b200: %s: %u mbarrier waits timed out; first: bar +%u parity %u block (%u,%u) thread %u\n", what, h[0], h[1], h[2], h[3], h[4], h[5]);
    return 1;
}
inline EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) {
            fprintf(stderr, "llm_b200: cuTensorMapEncodeTiled is not available\n");
            exit(1);
        }
        fn = (EncodeTiledFn)p;
    }
    return fn;
}
// 2-D f16/bf16 row-major [rows][cols] tensor, box [box_rows][64 columns = 128 B], 128-byte swizzle, out-of-bounds rows read as zero
inline CUtensorMap make_tmap_2d_f16_sw128(const void *base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes, uint32_t box_rows, bool bf16 = false) {
    CUtensorMap m;
    cuuint64_t dims[2] = {cols, rows}, strides[1] = {row_stride_bytes};
    cuuint32_t box[2] = {64, box_rows}, estr[2] = {1, 1};
    CUresult r = encode_tiled_fn()(&m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)base, dims, strides, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { fprintf(stderr, "llm_b200: cuTensorMapEncodeTiled failed (%d)\n", (int)r); exit(1); }
    return m;
}

}  // namespace tc5
}  // namespace b200
