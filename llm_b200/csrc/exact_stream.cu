// llm_b200/csrc/exact_stream.cu -- the decode mat-vec at HBM speed WITH the reference's bit-exact operation order.
//
// Arithmetic = exact.cu (AVX2 lane chains of ggml_vec_dot_q*_q8_*).  Data movement is what changes (stream_core.cuh):
//   * a dedicated producer warp streams the weight rows of a 32-row tile stage by stage (16 quant blocks = 256 B of nibbles per
//     row) into a 4-stage shared-memory ring with 16-byte cp.async and signals each stage through an mbarrier
//     (cp.async.mbarrier.arrive): the compute warps never touch global memory for weights.  The kernel is persistent: a CTA walks
//     several row tiles and the ring keeps streaming across them.  (v1 used one cp.async.bulk per row and per plane: 64 TMA requests
//     of 64..512 B per stage made the request rate, not the bytes, the limit of an SM.)
//   * 4 compute warps (4 threads per row: thread w owns AVX lanes w and w+4 == packed word w of every block) walk the blocks
//     IN ORDER out of shared memory: 3 LDS + 3 unpack + 2 dp4a + 2 i2f + 1 cvt + 1 fmul + 2 fma per block;
//   * the quantized activation row is re-packed once per mat-vec (quantize_act_pack) into 16-byte records per (block, word).
// Algorithmic bytes per row of K weights: K/32 * {18, 20, 22, 24, 34}; each is read exactly once.
#include "stream_core.cuh"

namespace b200 {

using namespace stream;

namespace {

template <int TYPE>
__global__ void __launch_bounds__(STHREADS) mmv_exact_stream_kernel(const QWeight w, const int4 *__restrict__ xpack, float *__restrict__ dst,
                                                                    const float *__restrict__ addend) {
    using T = St<TYPE>;
    extern __shared__ __align__(128) uint8_t smem[];
    Ring R{(uint64_t *)smem, (uint64_t *)smem + SST_MAX, smem + 256, 0u, SST};
    int4 *sx = (int4 *)(R.base + T::RING_BYTES);          // [nb][4] activation records
    const int tid = threadIdx.x;
    if (tid == 0) ring_init(R.full, R.empty, SST);
    __syncthreads();
    if (tid >= SCOMPUTE) { produce_matvec<TYPE>(w, R, blockIdx.x, gridDim.x, tid & 31); return; }
    for (int i = tid; i < (int)w.nb * 4; i += SCOMPUTE) cp16(smem_u32(sx + i), xpack + i);     // all 16-byte copies in flight at once
    asm volatile("cp.async.wait_all;" ::: "memory");
    compute_sync();
    consume_matvec<TYPE>(w, sx, R, blockIdx.x, gridDim.x, tid, [&](int64_t row, float v) {
        if ((tid & 3) == 0 && row < w.N) dst[row] = addend ? __fadd_rn(v, addend[row]) : v;
    });
}

__global__ void __launch_bounds__(256) quantize_act_pack_kernel(const float *__restrict__ x, int4 *__restrict__ pack, int nbk, int q81, int off, int scale16) {
    const int blk = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (blk >= nbk) return;
    const int lane = threadIdx.x & 31;
    pack_block(x[blk * QK + lane], pack + blk * 4, lane, q81, off, scale16);
}

template <int TYPE>
void launch_stream(const QWeight &w, const int4 *xpack, float *dst, const float *addend, cudaStream_t st) {
    using T = St<TYPE>;
    const int smem = 256 + T::RING_BYTES + (int)w.nb * 64;
    static int smem_set = 0;
    if (smem > smem_set) {
        B200_ASSERT(smem <= 227 * 1024);
        B200_CHECK(cudaFuncSetAttribute(mmv_exact_stream_kernel<TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        smem_set = smem;
    }
    static int ctas_per_sm = 0, sms = 0, occ_smem = -1;
    if (!sms) { int dev; B200_CHECK(cudaGetDevice(&dev)); B200_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)); }
    if (occ_smem != smem) { B200_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, mmv_exact_stream_kernel<TYPE>, STHREADS, smem)); occ_smem = smem; }
    const int64_t tiles = (w.N + SR - 1) / SR;
    const int64_t slots = (int64_t)sms * (ctas_per_sm > 0 ? ctas_per_sm : 1);
    // persistent: never more CTAs than can be resident; when there are more tiles than slots every CTA walks ceil(tiles/slots) tiles
    const unsigned grid = (unsigned)(tiles < slots ? tiles : slots);
    mmv_exact_stream_kernel<TYPE><<<grid, STHREADS, smem, st>>>(w, xpack, dst, addend);
    B200_CHECK(cudaGetLastError());
}

}  // namespace

bool mmv_exact_stream_supported(const QWeight &w) { return w.nb % 8 == 0 && w.nb * 64 + 256 + St<T_Q8_0>::RING_BYTES <= 227 * 1024; }

void quantize_act_pack(int wtype, const float *x, int4 *pack, int64_t K, cudaStream_t st) {
    const int nbk = (int)(K / QK);
    quantize_act_pack_kernel<<<(nbk + 7) / 8, 256, 0, st>>>(x, pack, nbk, has_min(wtype) ? 1 : 0, wtype == T_Q5_0 ? 16 : 0, wtype == T_Q4_0 ? 1 : 0);
    B200_CHECK(cudaGetLastError());
}

void mul_mat_vec_q_exact_stream(const QWeight &w, const int4 *xpack, float *dst, const float *addend, cudaStream_t st) {
    if (w.N == 0) return;
    B200_ASSERT(mmv_exact_stream_supported(w));
    switch (w.type) {
        case T_Q4_0: launch_stream<T_Q4_0>(w, xpack, dst, addend, st); break;
        case T_Q4_1: launch_stream<T_Q4_1>(w, xpack, dst, addend, st); break;
        case T_Q5_0: launch_stream<T_Q5_0>(w, xpack, dst, addend, st); break;
        case T_Q5_1: launch_stream<T_Q5_1>(w, xpack, dst, addend, st); break;
        case T_Q8_0: launch_stream<T_Q8_0>(w, xpack, dst, addend, st); break;
        default: B200_ASSERT(!"mul_mat_vec_q_exact_stream: unsupported weight type");
    }
}

}  // namespace b200
