/* oracle/sampler_oracle.c -- TEST INFRASTRUCTURE: the default sampler chain of llm_b200 (include/llm_b200.h, b200_sampler) in plain C, one
 * function per stage, on the host libm (expf is a call into libm: -fno-builtin; -ffp-contract=off: no fused operations the source does not write).
 *
 *   or_repetition   each distinct id of history[max(0, n_past - last_n), n_past): l <= 0 ? l * penalty : l / penalty; then every value + 0.0f
 *   or_top_k        value descending, ties by ascending id; min(k, n_vocab, 1024) candidates; a NaN in the row fails the chain
 *   or_top_p        p_i = expf(l_i - l_0) / S (S: f32 sum over the candidates in order); shortest prefix with running sum >= p, at least 1
 *   or_temperature  l_i / T
 *   or_draw         w_i = expf(l_i - l_0); x = u * (sum of w_i in order); the first i whose running sum is > x, else the last
 *   or_uniform      u = (z >> 40) * 2^-24, z = or_splitmix64(seed, draw) */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

uint64_t or_splitmix64(uint64_t seed, uint64_t draw) {
    uint64_t z = seed + (draw + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

float or_uniform(uint64_t seed, uint64_t draw) { return (float)(uint32_t)(or_splitmix64(seed, draw) >> 40) * 0x1p-24f; }

/* out = the row with the penalty applied (row itself untouched); 0, or -1 if the row holds a NaN */
int or_repetition(const float *row, int64_t n_vocab, const int32_t *history, int32_t n_past, int32_t last_n, float penalty, float *out) {
    int nan = 0;
    for (int64_t i = 0; i < n_vocab; i++) { out[i] = row[i]; nan |= row[i] != row[i]; }
    if (penalty != 1.0f && last_n > 0) {
        unsigned char *seen = calloc((size_t)n_vocab, 1);
        for (int32_t j = n_past > last_n ? n_past - last_n : 0; j < n_past; j++) {
            const int32_t id = history[j];
            if (seen[id]) continue;
            seen[id] = 1;
            out[id] = out[id] <= 0.0f ? out[id] * penalty : out[id] / penalty;
        }
        free(seen);
    }
    for (int64_t i = 0; i < n_vocab; i++) out[i] = out[i] + 0.0f;
    return nan ? -1 : 0;
}

static const float *g_vals;
static int cmp_desc(const void *a, const void *b) {
    const int32_t i = *(const int32_t *)a, j = *(const int32_t *)b;
    if (g_vals[i] > g_vals[j]) return -1;
    if (g_vals[i] < g_vals[j]) return 1;
    return i < j ? -1 : i > j;
}

/* the candidates, in order: ids_out / vals_out of min(k, n_vocab, 1024) entries; returns that count */
int32_t or_top_k(const float *vals, int64_t n_vocab, int32_t k, int32_t *ids_out, float *vals_out) {
    int32_t *idx = malloc((size_t)n_vocab * sizeof(int32_t));
    for (int64_t i = 0; i < n_vocab; i++) idx[i] = (int32_t)i;
    g_vals = vals;
    qsort(idx, (size_t)n_vocab, sizeof(int32_t), cmp_desc);
    int32_t kk = k < n_vocab ? k : (int32_t)n_vocab;
    if (kk > 1024) kk = 1024;
    for (int32_t i = 0; i < kk; i++) { ids_out[i] = idx[i]; vals_out[i] = vals[idx[i]]; }
    free(idx);
    return kk;
}

/* probs_out[i] = p_i for the n candidates; returns how many are kept */
int32_t or_top_p(const float *vals, int32_t n, float p, float *probs_out) {
    float sum = 0.0f;
    for (int32_t i = 0; i < n; i++) { probs_out[i] = expf(vals[i] - vals[0]); sum += probs_out[i]; }
    for (int32_t i = 0; i < n; i++) probs_out[i] = probs_out[i] / sum;
    float cum = 0.0f;
    for (int32_t i = 0; i < n; i++) { cum += probs_out[i]; if (cum >= p) return i + 1; }
    return n;
}

void or_temperature(float *vals, int32_t n, float t) {
    for (int32_t i = 0; i < n; i++) vals[i] = vals[i] / t;
}

int32_t or_draw(const float *vals, int32_t n, float u) {
    float *w = malloc((size_t)n * sizeof(float)), sum = 0.0f;
    for (int32_t i = 0; i < n; i++) { w[i] = expf(vals[i] - vals[0]); sum += w[i]; }
    const float x = u * sum;
    float run = 0.0f;
    int32_t pick = n - 1;
    for (int32_t i = 0; i < n; i++) { run += w[i]; if (run > x) { pick = i; break; } }
    free(w);
    return pick;
}

/* the whole chain: 0 and *id_out, *n_kept_out, cand_ids_out / cand_probs_out (min(k, n_vocab, 1024) entries each); -1 on a NaN */
int or_sample(const float *row, int64_t n_vocab, const int32_t *history, int32_t n_past, float penalty, int32_t last_n, int32_t k, float p, float t,
              uint64_t seed, uint64_t draw, int32_t *id_out, int32_t *n_kept_out, int32_t *cand_ids_out, float *cand_probs_out) {
    float *pen = malloc((size_t)n_vocab * sizeof(float)), vals[1024];
    if (or_repetition(row, n_vocab, history, n_past, last_n, penalty, pen) != 0) { free(pen); return -1; }
    const int32_t kk = or_top_k(pen, n_vocab, k, cand_ids_out, vals);
    free(pen);
    const int32_t n = or_top_p(vals, kk, p, cand_probs_out);
    or_temperature(vals, n, t);
    *id_out = cand_ids_out[or_draw(vals, n, or_uniform(seed, draw))];
    *n_kept_out = n;
    return 0;
}
