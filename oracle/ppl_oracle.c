/* oracle/ppl_oracle.c -- TEST INFRASTRUCTURE: the reference's perplexity arithmetic in plain C (InferenceSession::perplexity,
 * crates/llm-base/src/inference_session.rs:514-589, with util::softmax, crates/llm-base/src/util.rs:143-151), on logits the caller computed.
 *
 * Built with -ffp-contract=off and linked to the host libm: exp and ln are libm's expf / logf, which is what Rust's f32::exp / f32::ln call on
 * x86_64-linux-gnu.  Every sum is the reference's left-to-right f32 fold. */
#include <math.h>
#include <stdint.h>

/* -ln(softmax(row)[target]) of `rows` rows of n_vocab logits: max = fold(-inf, f32::max), sum = in-order f32 sum of expf(v - max) from 0,
 * p = expf(l[target] - max) / sum */
void or_nll_rows(const float *logits, int64_t rows, int64_t n_vocab, const int32_t *targets, float *terms) {
    for (int64_t r = 0; r < rows; r++) {
        const float *l = logits + r * n_vocab;
        float mx = -INFINITY;
        for (int64_t j = 0; j < n_vocab; j++) mx = fmaxf(mx, l[j]);
        float sum = 0.0f;
        for (int64_t j = 0; j < n_vocab; j++) sum += expf(l[j] - mx);
        const float p = expf(l[targets[r]] - mx) / sum;
        terms[r] = -logf(p);
    }
}

/* One chunk of the loop: `logits` holds the C rows the chunk's evaluation produced ([C][n_vocab]), `tokens` the chunk's C + 1 tokens
 * t[iC .. iC + C] (the last one is only read when it exists: rows j in [min(512, C/2), C - 1) are scored against t[iC + j + 1]).  nll and count
 * carry over between chunks, as in the reference.  terms_out (nullable) receives the chunk's scored terms in row order; returns the chunk's
 * perplexity expf(nll / count). */
float or_perplexity_chunk(const float *logits, int64_t C, int64_t n_vocab, const int32_t *tokens, float *nll, int64_t *count, float *terms_out) {
    const int64_t first = C / 2 < 512 ? C / 2 : 512;
    for (int64_t j = first; j < C - 1; j++) {
        float term;
        or_nll_rows(logits + j * n_vocab, 1, n_vocab, tokens + j + 1, &term);
        if (terms_out) terms_out[j - first] = term;
        *nll += term;
        *count += 1;
    }
    return expf(*nll / (float)*count);
}

/* the scalar libm functions themselves, for the restatement check */
float or_expf(float x) { return expf(x); }
float or_logf(float x) { return logf(x); }
