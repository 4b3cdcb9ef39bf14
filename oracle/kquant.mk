# oracle/kquant.mk -- TEST INFRASTRUCTURE build recipe for the reference's LLaMA graph on a model whose 2-D weights each have their own element type
# (make -C oracle -f kquant.mk): the mixed-type files the reference's quantizer writes (Q6_K output.weight, the Q4_K_M / Q5_K_M / Q3_K_M mixes).
#
#   _ref/libggml_ref_kq.so   the reference's OWN LC/ggml.c + LC/k_quants.c (oracle/Makefile's objects and flags) + a copy of ref_harness.c
#
# ref_harness.c stays as it is: the copy made under _ref/ differs from it in these lines only, and the recipe checks them:
#   * kquant_types.inc after the ggml include (rk_set_types: the table the next rh_llama_new reads);
#   * the nine 2-D weights of rh_llama_new take rk_type(wt) instead of wt, and the model context is sized by rk_ctx_bytes.
# A harness that no longer matches these patterns fails the build.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)

ifneq ($(wildcard $(REF)/ggml.c),)
kq: _ref/libggml_ref_kq.so
else
kq:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/libggml_ref_kq.so (if any)"
endif

_ref/ref_harness_kq.c: ref_harness.c kquant_types.inc
	mkdir -p _ref
	sed -e '/^#include "ggml.h"/r kquant_types.inc' \
	    -e 's/ggml_new_tensor_2d(c, wt, /ggml_new_tensor_2d(c, rk_type(wt), /' \
	    -e 's/struct ggml_init_params ip = { wbytes, NULL, false };/struct ggml_init_params ip = { rk_ctx_bytes(wbytes, p), NULL, false };/' $< > $@
	test "$$(grep -c '^void rk_set_types' $@)" = 1
	test "$$(grep -c 'ggml_new_tensor_2d(c, rk_type(wt), ' $@)" = 9
	test "$$(grep -c 'ip = { rk_ctx_bytes(wbytes, p), NULL' $@)" = 1

_ref/ref_harness_kq.o: _ref/ref_harness_kq.c
	$(CC) $(RFLAGS) -I. -c $< -o $@

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/libggml_ref_kq.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_harness_kq.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: kq
.SECONDARY:
