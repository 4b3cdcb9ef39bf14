# oracle/ppl.mk -- TEST INFRASTRUCTURE build recipe for the perplexity checkers (make -C oracle -f ppl.mk).  Plain C, no reference sources.
#
#   liboracle_ppl.so       ppl_oracle.c: the reference's softmax / log-likelihood loop on given logits, calling the host libm's expf / logf
#   liblibm_f32_check.so   libm_f32_check.c: the product's restated expf / logf (llm_b200/csrc/libm_f32.h) against the host libm, per input
#
# -ffp-contract=off: the C source's operations are the ones executed (no fused multiply-adds the source does not write), and -fno-builtin keeps
# every expf / logf a call into libm.

CC     = /usr/bin/gcc
PFLAGS = -O2 -std=c11 -fPIC -Wall -Wextra -ffp-contract=off -fno-builtin -fno-fast-math

ppl: liboracle_ppl.so liblibm_f32_check.so

liboracle_ppl.so: ppl_oracle.c
	$(CC) $(PFLAGS) -shared -o $@ ppl_oracle.c -lm

liblibm_f32_check.so: libm_f32_check.c ../llm_b200/csrc/libm_f32.h
	$(CC) $(PFLAGS) -shared -o $@ libm_f32_check.c -lm

.PHONY: ppl
