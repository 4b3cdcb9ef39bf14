// llm_b200/csrc/quant.cu -- weight re-layout at upload, the bit-faithful activation quantizer, get_rows.
#include "kernels.cuh"
#include "quant_rules.cuh"

namespace b200 {

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

size_t qweight_layout(QWeight &w, int type, int64_t K, int64_t N, void *base) {
    B200_ASSERT((is_qweight_type(type) && K % QK == 0) || (is_kquant(type) && K % 256 == 0));
    w.type = type; w.K = K; w.N = N; w.nb = K / (is_kquant(type) ? 256 : QK);
    if (type == T_F16 || is_kquant(type)) {              // one plane: the file's [N][K] halves, or its [N][K/256] super-blocks
        w.bytes = align_up((size_t)N * w.nb * qweight_block_bytes(type), 256);
        if (base) { w.base = base; w.qs = (const uint8_t *)base; w.qh = nullptr; w.dm = nullptr; }
        return w.bytes;
    }
    const size_t nblk = (size_t)N * (size_t)w.nb;
    size_t off = 0;
    const size_t qs_off = off; off = align_up(off + nblk * qs_bytes(type), 256);
    const size_t qh_off = off; if (has_qh(type)) off = align_up(off + nblk * 4, 256);
    const size_t dm_off = off; off = align_up(off + nblk * (has_min(type) ? 4 : 2), 256);
    w.bytes = off;
    if (base) {
        w.base = base;
        w.qs = (const uint8_t *)base + qs_off;
        w.qh = has_qh(type) ? (const uint32_t *)((const uint8_t *)base + qh_off) : nullptr;
        w.dm = (const uint8_t *)base + dm_off;
    }
    return off;
}

// One thread per quant block. GGML blocks are only 2-byte aligned (18/20/22/24/34 B), so the raw side moves as u16.
template <bool TO_PLANES>
__global__ void repack_kernel(int type, int64_t nblk, uint8_t *raw, uint8_t *qs, uint32_t *qh, uint8_t *dm) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nblk) return;
    const int bb = ggml_block_bytes(type);
    uint16_t *r = (uint16_t *)(raw + i * bb);
    int o = 0;  // offset in u16 units inside the GGML block: d [m] [qh] qs
    uint16_t *pd = (uint16_t *)(dm + i * (has_min(type) ? 4 : 2));
    if (TO_PLANES) pd[0] = r[o]; else r[o] = pd[0];
    o++;
    if (has_min(type)) { if (TO_PLANES) pd[1] = r[o]; else r[o] = pd[1]; o++; }
    if (has_qh(type)) {
        if (TO_PLANES) qh[i] = (uint32_t)r[o] | ((uint32_t)r[o + 1] << 16);
        else { r[o] = (uint16_t)(qh[i] & 0xffffu); r[o + 1] = (uint16_t)(qh[i] >> 16); }
        o += 2;
    }
    const int nq = qs_bytes(type) / 2;
    uint16_t *pq = (uint16_t *)(qs + i * qs_bytes(type));
    for (int j = 0; j < nq; j++) { if (TO_PLANES) pq[j] = r[o + j]; else r[o + j] = pq[j]; }
}

void repack_weights(const QWeight &w, const void *raw, cudaStream_t st) {
    const int64_t nblk = w.N * w.nb;
    if (nblk == 0) return;
    if (w.type == T_F16 || is_kquant(w.type)) { B200_CHECK(cudaMemcpyAsync((void *)w.qs, raw, (size_t)nblk * qweight_block_bytes(w.type), cudaMemcpyDeviceToDevice, st)); return; }
    repack_kernel<true><<<(unsigned)((nblk + 255) / 256), 256, 0, st>>>(w.type, nblk, (uint8_t *)raw, (uint8_t *)w.qs, (uint32_t *)w.qh, (uint8_t *)w.dm);
    B200_CHECK(cudaGetLastError());
}
void unpack_weights(const QWeight &w, void *raw, cudaStream_t st) {
    const int64_t nblk = w.N * w.nb;
    if (nblk == 0) return;
    if (w.type == T_F16 || is_kquant(w.type)) { B200_CHECK(cudaMemcpyAsync(raw, w.qs, (size_t)nblk * qweight_block_bytes(w.type), cudaMemcpyDeviceToDevice, st)); return; }
    repack_kernel<false><<<(unsigned)((nblk + 255) / 256), 256, 0, st>>>(w.type, nblk, (uint8_t *)raw, (uint8_t *)w.qs, (uint32_t *)w.qh, (uint8_t *)w.dm);
    B200_CHECK(cudaGetLastError());
}

// ---- activation quantizer ----------------------------------------------------------------------------------------
// One warp per 32-element block, lane j <-> element j: the AVX2 rule of quantize_q8_avx2 (quant_rules.cuh).
template <bool Q81>
__global__ void __launch_bounds__(256) quantize_act_kernel(const float *__restrict__ x, int64_t ldx, int8_t *__restrict__ qs,
                                                           float2 *__restrict__ ds, int64_t nbk, int64_t total_blocks) {
    const int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (blk >= total_blocks) return;
    const int lane = threadIdx.x & 31;
    const int64_t row = blk / nbk, b = blk - row * nbk;
    const float v = x[row * ldx + b * QK + lane];
    float d;
    const int q = quantize_q8_avx2(v, d);
    const int isum = warp_sum(q);
    qs[blk * QK + lane] = (int8_t)q;
    if (lane == 0) {
        if (Q81) ds[blk] = make_float2(d, __fmul_rn(d, (float)isum));
        else     ds[blk] = make_float2(__half2float(__float2half_rn(d)), (float)isum);
    }
}

void quantize_act(int vdt, const float *x, int64_t ldx, int8_t *qs, float2 *ds, int64_t K, int64_t B, cudaStream_t st) {
    B200_ASSERT(K % QK == 0);
    const int64_t nbk = K / QK, total = nbk * B;
    if (total == 0) return;
    const unsigned grid = (unsigned)((total + 7) / 8);
    if (vdt == T_Q8_1) quantize_act_kernel<true><<<grid, 256, 0, st>>>(x, ldx, qs, ds, nbk, total);
    else               quantize_act_kernel<false><<<grid, 256, 0, st>>>(x, ldx, qs, ds, nbk, total);
    B200_CHECK(cudaGetLastError());
}

// ---- get_rows: dequantize_row_* (dequant_block, quant_rules.cuh) -----------------------------------------------------
// 16 threads per block; planes layout
__global__ void get_rows_q_kernel(QWeight w, const int32_t *__restrict__ ids, float *__restrict__ dst, int64_t n) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t blk = t >> 4; const int j = (int)(t & 15);
    if (blk >= n * w.nb) return;
    const int64_t i = blk / w.nb, b = blk - i * w.nb;
    const int64_t src = (int64_t)ids[i] * w.nb + b;
    float d, m = 0.f;
    if (has_min(w.type)) { const __half2 dm = ((const __half2 *)w.dm)[src]; d = __low2float(dm); m = __high2float(dm); }
    else d = __half2float(((const __half *)w.dm)[src]);
    const uint32_t qh = has_qh(w.type) ? w.qh[src] : 0u;
    float lo, hi;
    dequant_block(w.type, w.qs + src * qs_bytes(w.type), qh, d, m, j, lo, hi);
    dst[i * w.K + b * QK + j] = lo;
    dst[i * w.K + b * QK + j + 16] = hi;
}

void get_rows_q(const QWeight &w, const int32_t *ids, float *dst, int64_t n, cudaStream_t st) {
    if (w.type == T_F16) { get_rows_f16(w, ids, dst, n, st); return; }
    if (is_kquant(w.type)) { get_rows_kq(w.type, w.qs, w.K, ids, dst, n, st); return; }
    const int64_t threads = n * w.nb * 16;
    if (threads == 0) return;
    get_rows_q_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(w, ids, dst, n);
    B200_CHECK(cudaGetLastError());
}

// GGML array-of-blocks source
__global__ void get_rows_raw_kernel(int type, const uint8_t *__restrict__ raw, int64_t nb, const int32_t *__restrict__ ids,
                                    float *__restrict__ dst, int64_t n) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t blk = t >> 4; const int j = (int)(t & 15);
    if (blk >= n * nb) return;
    const int64_t i = blk / nb, b = blk - i * nb;
    float d, m, lo, hi;
    uint32_t qh;
    const uint8_t *qs = raw_block_header(type, raw + ((int64_t)ids[i] * nb + b) * ggml_block_bytes(type), d, m, qh);
    dequant_block(type, qs, qh, d, m, j, lo, hi);
    const int64_t K = nb * QK;
    dst[i * K + b * QK + j] = lo;
    dst[i * K + b * QK + j + 16] = hi;
}

void get_rows_raw(int type, const void *raw, int64_t K, const int32_t *ids, float *dst, int64_t n, cudaStream_t st) {
    const int64_t nb = K / QK, threads = n * nb * 16;
    if (threads == 0) return;
    get_rows_raw_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(type, (const uint8_t *)raw, nb, ids, dst, n);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
