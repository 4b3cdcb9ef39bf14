// llm_b200/csrc/sample.cu -- the default sampler chain of the reference (crates/llm-base/src/samplers.rs:97-211) on a logits row in HBM:
// repetition penalty -> top-k -> top-p -> temperature -> one draw from the kept distribution.
//
// Arithmetic (oracle/sampler_oracle.c states the same chain in plain C; every operation below is its f32 operation, in its order):
//   repetition   each DISTINCT id of tokens[max(0, n_past - last_n), n_past): l <= 0 ? l * penalty : l / penalty; then every value + 0.0f
//                (-0 becomes +0, so that equal values are equal keys; no result of the chain depends on the sign of a zero)
//   top-k        value descending, ties by ascending id; k capped at min(k, n_vocab, 1024); a NaN anywhere in the row is a sampler failure
//   top-p        p_i = expf(l_i - l_0) / S, S the f32 sum over the k candidates in order; keep the shortest prefix whose running f32 sum of
//                p_i is >= p (at least one)
//   temperature  t_i = l_i / T
//   draw         w_i = expf(t_i - t_0), x = u * (f32 sum of w_i in order), the first i whose running sum is > x (none: the last kept);
//                u = (z >> 40) * 2^-24, z = the draw-th SplitMix64 output of seed
// expf is glibc's (libm_f32.h).
//
// Shape: the row is read once.  Each CTA of sample_select_kernel turns a 4096-id slice into 64-bit keys (orderable value bits << 32 | ~id, so
// that descending key order is the chain's order and every key is distinct), bitonic-sorts them in shared memory and writes its top k.
// sample_merge_kernel does the same to the candidates until at most 4096 are left (k <= 1024, so each level shrinks them 4x or more); then
// sample_tail_kernel, one CTA, sorts them and runs top-p, temperature and the draw: the exps in parallel, each ordered sum in one thread.
#include "kernels.cuh"
#include "libm_f32.h"

namespace b200 {

namespace {

constexpr int TILE = 4096;            // keys sorted per CTA (32 KB of shared memory)
constexpr int THREADS = 1024;

__device__ __forceinline__ uint32_t ord_bits(float v) { const uint32_t b = __float_as_uint(v); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
__device__ __forceinline__ float ord_value(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }
__device__ __forceinline__ uint64_t make_key(float v, int id) { return ((uint64_t)ord_bits(v) << 32) | (uint32_t)(0xffffffffu - (uint32_t)id); }
__device__ __forceinline__ int key_id(uint64_t k) { return (int)(0xffffffffu - (uint32_t)k); }
__device__ __forceinline__ float key_value(uint64_t k) { return ord_value((uint32_t)(k >> 32)); }
// key 0 sorts below every real key (the least real one, -inf at the last id, has high word 0x007fffff): it pads a tile

// descending bitonic sort of s[0, n), n a power of two <= TILE, all threads of the CTA
__device__ __forceinline__ void sort_desc(uint64_t *s, int n = TILE) {
    for (int k = 2; k <= n; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < n / 2; t += THREADS) {
                const int i = 2 * t - (t & (j - 1)), l = i + j;     // the pair (i, i + j), bit j of i clear
                const uint64_t a = s[i], b = s[l];
                if ((i & k) == 0 ? a < b : a > b) { s[i] = b; s[l] = a; }
            }
            __syncthreads();
        }
}

// the kernels' bodies take their CTA's index `blk`: the single-row kernels pass blockIdx.x, the many-row ones (sample_rows) blockIdx.x of the
// row blockIdx.y
__device__ __forceinline__ void sample_select(const float *__restrict__ row, int n_vocab, const int32_t *__restrict__ hist, int lo, int hi,
                                              float penalty, int kk, uint64_t *__restrict__ out, int *fail, unsigned blk) {
    __shared__ uint64_t s[TILE];
    __shared__ uint32_t mark[TILE / 32];          // ids of this slice in the penalty window
    const int base = blk * TILE, tid = threadIdx.x;
    for (int t = tid; t < TILE / 32; t += THREADS) mark[t] = 0;
    __syncthreads();
    for (int j = lo + tid; j < hi; j += THREADS) {
        const int id = hist[j] - base;
        if (id >= 0 && id < TILE) atomicOr(&mark[id >> 5], 1u << (id & 31));
    }
    __syncthreads();
    int nan = 0;
    for (int t = tid; t < TILE; t += THREADS) {
        const int i = base + t;
        uint64_t key = 0;
        if (i < n_vocab) {
            float v = row[i];
            nan |= v != v;
            if ((mark[t >> 5] >> (t & 31)) & 1u) v = v <= 0.0f ? __fmul_rn(v, penalty) : __fdiv_rn(v, penalty);
            key = make_key(__fadd_rn(v, 0.0f), i);
        }
        s[t] = key;
    }
    if (__syncthreads_or(nan) && tid == 0) atomicOr(fail, 1);
    sort_desc(s);
    for (int t = tid; t < kk; t += THREADS) out[(size_t)blk * kk + t] = s[t];
}
__global__ void __launch_bounds__(THREADS) sample_select_kernel(const float *__restrict__ row, int n_vocab, const int32_t *__restrict__ hist, int lo, int hi,
                                                                float penalty, int kk, uint64_t *__restrict__ out, int *fail) {
    sample_select(row, n_vocab, hist, lo, hi, penalty, kk, out, fail, blockIdx.x);
}

__device__ __forceinline__ void sample_merge(const uint64_t *__restrict__ in, int n, int kk, uint64_t *__restrict__ out, unsigned blk) {
    __shared__ uint64_t s[TILE];
    const int base = blk * TILE;
    for (int t = threadIdx.x; t < TILE; t += THREADS) s[t] = base + t < n ? in[base + t] : 0;
    __syncthreads();
    sort_desc(s);
    for (int t = threadIdx.x; t < kk; t += THREADS) out[(size_t)blk * kk + t] = s[t];
}
__global__ void __launch_bounds__(THREADS) sample_merge_kernel(const uint64_t *__restrict__ in, int n, int kk, uint64_t *__restrict__ out) {
    sample_merge(in, n, kk, out, blockIdx.x);
}

struct TailArgs {
    int n_vocab, kk;
    float top_p, temperature;
    uint64_t seed, draw;
};

__device__ __forceinline__ void sample_tail(const uint64_t *__restrict__ in, int n, const TailArgs &a, const float *__restrict__ row, int *fail,
                                            SampleResult *res, int32_t *tok_dst, int32_t *hist_dst, int32_t *cand_ids, float *cand_vals,
                                            float *cand_probs, float *backup) {
    __shared__ uint64_t s[TILE];
    __shared__ int failed, n_kept;
    __shared__ float S;
    const int tid = threadIdx.x, kk = a.kk;
    int np2 = 2;                                                 // the candidates fill a power of two, padded with key 0
    while (np2 < n) np2 <<= 1;
    for (int t = tid; t < np2; t += THREADS) s[t] = t < n ? in[t] : 0;
    if (tid == 0) { failed = *fail; *fail = 0; }                 // the flag is re-armed for the next call
    __syncthreads();
    if (failed) {                                                // Logits::try_from_iter refuses the row; keep a copy of it for the host to restore
        if (backup) for (int i = tid; i < a.n_vocab; i += THREADS) backup[i] = row[i];
        if (tid == 0 && res) {
            volatile SampleResult *r = res;
            r->id = -1; r->n_cand = 0; r->n_kept = 0; r->status = 1;
            __threadfence_system();
        }
        return;
    }
    sort_desc(s, np2);
    const uint64_t key = tid < kk ? s[tid] : 0;
    const float v = key_value(key), v0 = key_value(s[0]);
    const int id = key_id(key);
    __syncthreads();                                             // s is reused below
    float *e = (float *)s, *pr = e + THREADS, *w = e + 2 * THREADS;
    int *ids = (int *)(e + 3 * THREADS);
    if (tid < kk) { e[tid] = lm_expf(__fsub_rn(v, v0)); ids[tid] = id; }
    __syncthreads();
    if (tid == 0) { float sum = 0.0f; for (int i = 0; i < kk; i++) sum = __fadd_rn(sum, e[i]); S = sum; }
    __syncthreads();
    if (tid < kk) pr[tid] = __fdiv_rn(e[tid], S);
    __syncthreads();
    if (tid == 0) {
        float cum = 0.0f; int m = kk;
        for (int i = 0; i < kk; i++) { cum = __fadd_rn(cum, pr[i]); if (cum >= a.top_p) { m = i + 1; break; } }
        n_kept = m;
    }
    __syncthreads();
    const int nk = n_kept;
    if (tid < nk) w[tid] = lm_expf(__fsub_rn(__fdiv_rn(v, a.temperature), __fdiv_rn(v0, a.temperature)));
    if (tid < kk) {
        if (cand_ids) cand_ids[tid] = id;
        if (cand_vals) cand_vals[tid] = row[id];
        if (cand_probs) cand_probs[tid] = pr[tid];
    }
    __syncthreads();
    if (tid == 0) {
        float sum = 0.0f;
        for (int i = 0; i < nk; i++) sum = __fadd_rn(sum, w[i]);
        const float u = __fmul_rn((float)(uint32_t)(splitmix64(a.seed, a.draw) >> 40), 0x1p-24f);
        const float x = __fmul_rn(u, sum);
        float run = 0.0f; int pick = nk - 1;
        for (int i = 0; i < nk; i++) { run = __fadd_rn(run, w[i]); if (run > x) { pick = i; break; } }
        const int tok = ids[pick];
        if (tok_dst) *tok_dst = tok;
        if (hist_dst) *hist_dst = tok;
        if (res) {
            volatile SampleResult *r = res;
            r->id = tok; r->n_cand = kk; r->n_kept = nk; r->status = 0;
            __threadfence_system();
        }
    }
}
__global__ void __launch_bounds__(THREADS) sample_tail_kernel(const uint64_t *__restrict__ in, int n, TailArgs a, const float *__restrict__ row, int *fail,
                                                              SampleResult *res, int32_t *tok_dst, int32_t *hist_dst, int32_t *cand_ids, float *cand_vals,
                                                              float *cand_probs, float *backup) {
    sample_tail(in, n, a, row, fail, res, tok_dst, hist_dst, cand_ids, cand_vals, cand_probs, backup);
}

// ---- many rows (sample_rows): job blockIdx.y, or blockIdx.x for the tail -----------------------------------------------------------
// A job's chain: select over ceil(n_vocab / TILE) CTAs into keys[0], then merge levels while more than TILE candidates are left, each from
// keys[l & 1] into keys[(l + 1) & 1], then the tail on keys[levels & 1] -- sample_row's launches, in the same buffers.
__device__ __forceinline__ int job_lo(const SampleJob &j) {
    return j.a.penalty == 1.0f || j.a.last_n <= 0 ? j.n_past : (j.n_past > j.a.last_n ? j.n_past - j.a.last_n : 0);
}
__global__ void __launch_bounds__(THREADS) sample_select_rows_kernel(const SampleJob *__restrict__ jobs) {
    const SampleJob &j = jobs[blockIdx.y];
    if ((int)blockIdx.x * TILE >= j.n_vocab) return;
    sample_select(j.row, j.n_vocab, j.hist, job_lo(j), j.n_past, j.a.penalty, sample_kk(j.a.top_k, j.n_vocab), j.b.keys[0], j.b.fail, blockIdx.x);
}
// merge level `level` (0-based) of every job that has one
__global__ void __launch_bounds__(THREADS) sample_merge_rows_kernel(const SampleJob *__restrict__ jobs, int level) {
    const SampleJob &j = jobs[blockIdx.y];
    const int kk = sample_kk(j.a.top_k, j.n_vocab);
    int n = (j.n_vocab + TILE - 1) / TILE * kk;
    for (int l = 0; l < level && n > TILE; l++) n = (n + TILE - 1) / TILE * kk;
    if (n <= TILE || (int)blockIdx.x * TILE >= n) return;
    sample_merge(j.b.keys[level & 1], n, kk, j.b.keys[(level + 1) & 1], blockIdx.x);
}
__global__ void __launch_bounds__(THREADS) sample_tail_rows_kernel(const SampleJob *__restrict__ jobs) {
    const SampleJob &j = jobs[blockIdx.x];
    const int kk = sample_kk(j.a.top_k, j.n_vocab);
    int n = (j.n_vocab + TILE - 1) / TILE * kk, cur = 0;
    while (n > TILE) { n = (n + TILE - 1) / TILE * kk; cur ^= 1; }
    const TailArgs t{j.n_vocab, kk, j.a.top_p, j.a.temperature, j.a.seed, j.a.draw};
    sample_tail(j.b.keys[cur], n, t, j.row, j.b.fail, j.res, j.tok_dst, j.hist_dst, nullptr, nullptr, nullptr, j.b.backup);
}

}  // namespace

size_t sample_key_bytes(int n_vocab) { return (size_t)((n_vocab + TILE - 1) / TILE) * 1024 * sizeof(uint64_t); }

int sample_rows(const SampleJob *jobs, int n, int max_n_vocab, int max_kk, cudaStream_t st) {
    B200_ASSERT(n >= 1 && n <= 65535 && max_kk >= 1 && max_n_vocab >= 1);
    int grid = (max_n_vocab + TILE - 1) / TILE, launches = 2;
    sample_select_rows_kernel<<<dim3((unsigned)grid, (unsigned)n), THREADS, 0, st>>>(jobs);
    B200_CHECK(cudaGetLastError());
    // the most candidates any job has at each level: the widest row with the most candidates per CTA
    for (int64_t m = (int64_t)grid * max_kk, level = 0; m > TILE; level++) {
        grid = (int)((m + TILE - 1) / TILE);
        sample_merge_rows_kernel<<<dim3((unsigned)grid, (unsigned)n), THREADS, 0, st>>>(jobs, (int)level);
        B200_CHECK(cudaGetLastError());
        m = (int64_t)grid * max_kk;
        launches++;
    }
    sample_tail_rows_kernel<<<(unsigned)n, THREADS, 0, st>>>(jobs);
    B200_CHECK(cudaGetLastError());
    return launches;
}

void sample_row(const float *row, int n_vocab, const int32_t *hist, int n_past, const SampleArgs &a, const SampleBufs &b, int32_t *tok_dst, int32_t *hist_dst,
                SampleResult *res, int32_t *cand_ids, float *cand_vals, float *cand_probs, cudaStream_t st) {
    const int kk = a.top_k < n_vocab ? (a.top_k < 1024 ? a.top_k : 1024) : (n_vocab < 1024 ? n_vocab : 1024);
    B200_ASSERT(kk >= 1 && n_vocab >= 1);
    const int lo = a.penalty == 1.0f || a.last_n <= 0 ? n_past : (n_past > a.last_n ? n_past - a.last_n : 0);   // penalty off: an empty window
    int grid = (n_vocab + TILE - 1) / TILE;
    sample_select_kernel<<<grid, THREADS, 0, st>>>(row, n_vocab, hist, lo, n_past, a.penalty, kk, b.keys[0], b.fail);
    B200_CHECK(cudaGetLastError());
    int n = grid * kk, cur = 0;
    while (n > TILE) {
        grid = (n + TILE - 1) / TILE;
        sample_merge_kernel<<<grid, THREADS, 0, st>>>(b.keys[cur], n, kk, b.keys[cur ^ 1]);
        B200_CHECK(cudaGetLastError());
        n = grid * kk; cur ^= 1;
    }
    const TailArgs t{n_vocab, kk, a.top_p, a.temperature, a.seed, a.draw};
    sample_tail_kernel<<<1, THREADS, 0, st>>>(b.keys[cur], n, t, row, b.fail, res, tok_dst, hist_dst, cand_ids, cand_vals, cand_probs, b.backup);
    B200_CHECK(cudaGetLastError());
}

}  // namespace b200
