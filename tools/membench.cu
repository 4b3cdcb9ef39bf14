// tools/membench.cu -- micro-benchmark behind the weight layout decision: how fast can a ring of shared-memory
// stages be filled from HBM when a stage is (A) 32 row segments of 256 B at the row pitch of a [N][K/32][16 B] plane (16-byte cp.async
// by one producer warp) versus (B) one contiguous 9 KB region fetched by a single bulk (TMA) copy.  No arithmetic: consumers only
// wait for the stage and hand it back.   nvcc -arch=sm_90a -O3 -o membench tools/membench.cu && ./membench
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t su32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, uint32_t c) { asm volatile("mbarrier.init.shared.b64 [%0], %1;" ::"r"(su32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *b) { asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(su32(b)) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t *b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.release.cta.shared::cta.b64 _, [%0], %1;" ::"r"(su32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *b, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(su32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void cp16(uint32_t dst, const void *src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_arrive(uint64_t *b) { asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(su32(b)) : "memory"); }
__device__ __forceinline__ void bulk(uint32_t dst, const void *src, uint32_t bytes, uint64_t *b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(su32(b)) : "memory");
}

constexpr int STAGE = 9216, STAGE_A = 10240, ROWS = 32, SEG = 256;   // Q4_0 stage: 32 rows x 16 blocks x 16 B (+ 1 KB of scales, fetched as 32 x 32 B in mode A)

// mode 0: strided 16-byte cp.async (qs 256 B + dm 32 B per row, row pitches pitch and pitch/8), mode 1: one bulk copy per stage
template <int MODE>
__global__ void __launch_bounds__(160) fill_kernel(const uint8_t *base, size_t pitch, int chunks_per_tile, int ntiles, int nst, unsigned long long *sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *full = (uint64_t *)smem, *empty = full + 16;
    uint8_t *ring = smem + 256;
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < nst; s++) { mbar_init(&full[s], MODE == 0 ? 32 : 1); mbar_init(&empty[s], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t slot = 0, phase = 0;
    if (tid >= 128) {
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
            for (int c = 0; c < chunks_per_tile; c++) {
                mbar_wait(&empty[slot], phase ^ 1u);
                const uint32_t dst = su32(ring + (size_t)slot * (MODE == 0 ? STAGE_A : STAGE));
                if (MODE == 0) {
                    const uint8_t *q = base + (size_t)tile * ROWS * pitch + (size_t)c * SEG;
#pragma unroll
                    for (int it = 0; it < 16; it++) { const int rr = it * 2 + (lane >> 4), cc = lane & 15; cp16(dst + rr * 272 + cc * 16, q + rr * pitch + cc * 16); }
                    const uint8_t *d = base + (size_t)ntiles * ROWS * pitch + (size_t)tile * ROWS * (pitch / 8) + (size_t)c * 32;
#pragma unroll
                    for (int it = 0; it < 2; it++) { const int rr = it * 16 + (lane >> 1), cc = lane & 1; cp16(dst + 8704 + rr * 48 + cc * 16, d + rr * (pitch / 8) + cc * 16); }
                    cp_arrive(&full[slot]);
                } else if (lane == 0) {
                    mbar_expect(&full[slot], STAGE);
                    bulk(dst, base + ((size_t)tile * chunks_per_tile + c) * STAGE, STAGE, &full[slot]);
                }
                if (++slot == (uint32_t)nst) { slot = 0; phase ^= 1u; }
            }
        return;
    }
    unsigned long long acc = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int c = 0; c < chunks_per_tile; c++) {
            mbar_wait(&full[slot], phase);
            acc += *(const uint32_t *)(ring + (size_t)slot * (MODE == 0 ? STAGE_A : STAGE) + tid * 4);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[slot]);
            if (++slot == (uint32_t)nst) { slot = 0; phase ^= 1u; }
        }
    if (acc == 0x123456789ull) *sink = acc;
}

// mode 2: plain grid-stride 16-byte loads, 8 in flight per thread (no shared memory, no barriers): the floor for "read this matrix once"
__global__ void __launch_bounds__(256) read_kernel(const int4 *base, size_t n16, unsigned long long *sink) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned acc = 0;
    for (; i + 7 * stride < n16; i += 8 * stride) {
        int4 v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = __ldcs(base + i + k * stride);
#pragma unroll
        for (int k = 0; k < 8; k++) acc += v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
    }
    for (; i < n16; i += stride) { const int4 v = __ldcs(base + i); acc += v.x ^ v.y ^ v.z ^ v.w; }
    if (acc == 0x12345u) *sink = acc;
}

int main() {
    int sms; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const size_t total = (size_t)3 << 30;
    const size_t alloc = total / 8 * 9 + ((size_t)256 << 20);
    uint8_t *buf; CK(cudaMalloc(&buf, alloc)); CK(cudaMemset(buf, 1, alloc));
    unsigned long long *sink; CK(cudaMalloc(&sink, 8));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    struct Shape { const char *name; int N, nb; } shapes[] = {{"wo   4096x4096", 4096, 128}, {"w2   4096x11008", 4096, 344}, {"qkv 12288x4096", 12288, 128}, {"w13 22016x4096", 22016, 128}};
    for (auto &sh : shapes) {
        const int ntiles = sh.N / 32, chunks = (sh.nb + 15) / 16;
        const size_t pitch = (size_t)sh.nb * 16, bytes = (size_t)ntiles * chunks * STAGE;
        const int reps = (int)(total / bytes) < 64 ? (int)(total / bytes) : 64;        // distinct matrices back to back (nothing stays in L2)
        cudaStream_t st; CK(cudaStreamCreate(&st));
        for (int mode = 0; mode < 3; mode++)
            for (int nst : {4, 8}) {
                if (mode == 2 && nst == 8) continue;
                const int smem = 256 + nst * (mode == 0 ? STAGE_A : STAGE);
                int occ = 0;
                if (mode == 0) { CK(cudaFuncSetAttribute(fill_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fill_kernel<0>, 160, smem)); }
                else if (mode == 1) { CK(cudaFuncSetAttribute(fill_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fill_kernel<1>, 160, smem)); }
                if (occ > 4) occ = 4;
                const int grid = mode == 2 ? sms * 8 : (ntiles < sms * occ ? ntiles : sms * occ);
                auto enqueue = [&]() {
                    for (int r = 0; r < reps; r++) {
                        const uint8_t *b = buf + (size_t)r * bytes * 9 / 8 / 256 * 256;
                        if (mode == 0) fill_kernel<0><<<grid, 160, smem, st>>>(b, pitch, chunks, ntiles, nst, sink);
                        else if (mode == 1) fill_kernel<1><<<grid, 160, smem, st>>>(b, pitch, chunks, ntiles, nst, sink);
                        else read_kernel<<<grid, 256, 0, st>>>((const int4 *)b, bytes / 16, sink);
                    }
                };
                float best = 1e9f, bestg = 1e9f;
                for (int trial = 0; trial < 3; trial++) {
                    CK(cudaEventRecord(e0, st)); enqueue(); CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1));
                    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
                }
                cudaGraph_t g; cudaGraphExec_t ge;
                CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal)); enqueue(); CK(cudaStreamEndCapture(st, &g));
                CK(cudaGraphInstantiate(&ge, g, 0));
                for (int trial = 0; trial < 4; trial++) {
                    CK(cudaEventRecord(e0, st)); CK(cudaGraphLaunch(ge, st)); CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1));
                    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (trial && ms < bestg) bestg = ms;
                }
                CK(cudaGraphExecDestroy(ge)); CK(cudaGraphDestroy(g));
                printf("%-16s %-12s ring %d grid %4d: stream %6.2f us/launch %5.0f GB/s | graph %6.2f us/launch %5.0f GB/s\n", sh.name,
                       mode == 0 ? "16B-strided" : mode == 1 ? "bulk-9KB" : "plain-LDG", nst, grid, best * 1e3f / reps, (double)bytes * reps / (best * 1e-3) / 1e9,
                       bestg * 1e3f / reps, (double)bytes * reps / (bestg * 1e-3) / 1e9);
            }
        CK(cudaStreamDestroy(st));
    }
    CK(cudaGetLastError());
    return 0;
}
