/* oracle/libm_f32_check.c -- TEST INFRASTRUCTURE: compares the product's restatement of glibc's expf / logf (llm_b200/csrc/libm_f32.h, the
 * source the perplexity kernel compiles) with the host libm, bit for bit, over a range of float bit patterns.  Built by gcc with
 * -ffp-contract=off, so the header's operations are the ones written. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../llm_b200/csrc/libm_f32.h"

static uint32_t bits(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }

/* Walks the bit patterns [lo, hi] (inclusive; as unsigned 32-bit words, so a range of negative floats runs from -0 towards -inf).
 * which = 0: expf, 1: logf.  Returns the number of inputs whose result differs; *first_bad gets the first such pattern (untouched if none). */
int64_t lm_check_range(int which, uint32_t lo, uint32_t hi, uint32_t *first_bad) {
    int64_t bad = 0;
    for (uint64_t u = lo; u <= hi; u++) {
        float x;
        const uint32_t w = (uint32_t)u;
        memcpy(&x, &w, 4);
        const float want = which ? logf(x) : expf(x);
        const float got = which ? lm_logf(x) : lm_expf(x);
        const uint32_t a = bits(want), b = bits(got);
        /* a nan matches any nan (the payload is not part of the contract) */
        if (a != b && !(isnan(want) && isnan(got))) {
            if (!bad && first_bad) *first_bad = w;
            bad++;
        }
    }
    return bad;
}

float lm_check_expf(float x) { return lm_expf(x); }
float lm_check_logf(float x) { return lm_logf(x); }
