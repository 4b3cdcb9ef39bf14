# oracle/neox_kquant.mk -- TEST INFRASTRUCTURE build recipe for the reference's GPT-NeoX, GPT-2, MPT, BLOOM and GPT-J graphs on models whose 2-D
# weights each have their own element type, and with ModelParameters::rope_overrides (make -C oracle -f neox_kquant.mk).
#
#   _ref/libggml_ref_nxkq.so     GPT-2, GPT-NeoX  (ref_harness.c as oracle/Makefile compiles it + a copy of ref_gpt2.c; the RefLib API of bindings.py)
#   _ref/libggml_alibi_kq.so     MPT, BLOOM       (a copy of ref_alibi.c)
#   _ref/libggml_gptj_kq.so      GPT-J            (a copy of ref_gptj.c)
#
# The reference's OWN LC/ggml.c + LC/k_quants.c (oracle/Makefile's objects and flags).  The committed harnesses stay as they are: each copy made
# under _ref/ differs from its harness in these lines only, and the recipe counts every substitution:
#   * kquant_types.inc after the ggml include (rk_set_types: the table the next model allocation reads), and in ref_gpt2.c / ref_gptj.c
#     rope_custom.inc (rk_set_rope);
#   * every 2-D weight allocated with the harness's weight type takes rk_type(wt) instead (ref_gpt2.c 6, ref_alibi.c 6, ref_gptj.c 8);
#   * the weight context is sized for F16 weights (8 x the one-type bytes) while a table is armed;
#   * the RoPE nodes call rk_rope instead of ggml_rope_inplace (2 in ref_gpt2.c's GPT-NeoX graph, 2 in ref_gptj.c).
# A harness that no longer matches these patterns fails the build.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)
SUBST  = -e '/^\#include "ggml.h"/r kquant_types.inc' \
         -e 's/ggml_new_tensor_2d(c, wt, /ggml_new_tensor_2d(c, rk_type(wt), /g' \
         -e 's/struct ggml_init_params ip = { wbytes, NULL, false };/struct ggml_init_params ip = { rk_n ? 8 * wbytes : wbytes, NULL, false };/'
ROPE   = -e '/^\#include "ggml.h"/r rope_custom.inc' -e 's/ggml_rope_inplace(ctx0, /rk_rope(ctx0, /g'

ifneq ($(wildcard $(REF)/ggml.c),)
nxkq: _ref/libggml_ref_nxkq.so _ref/libggml_alibi_kq.so _ref/libggml_gptj_kq.so
else
nxkq:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/*_kq.so (if any)"
endif

_ref/ref_gpt2_kq.c: ref_gpt2.c kquant_types.inc rope_custom.inc
	mkdir -p _ref
	sed $(SUBST) $(ROPE) $< > $@
	test "$$(grep -o '^void rk_set_types' $@ | wc -l)" = 1
	test "$$(grep -o '^void rk_set_rope' $@ | wc -l)" = 1
	test "$$(grep -o 'ggml_new_tensor_2d(c, rk_type(wt), ' $@ | wc -l)" = 6
	test "$$(grep -o 'ip = { rk_n ? 8 \* wbytes : wbytes' $@ | wc -l)" = 1
	test "$$(grep -o 'rk_rope(ctx0, ' $@ | wc -l)" = 2

_ref/ref_gptj_kq.c: ref_gptj.c kquant_types.inc rope_custom.inc
	mkdir -p _ref
	sed $(SUBST) $(ROPE) $< > $@
	test "$$(grep -o '^void rk_set_types' $@ | wc -l)" = 1
	test "$$(grep -o '^void rk_set_rope' $@ | wc -l)" = 1
	test "$$(grep -o 'ggml_new_tensor_2d(c, rk_type(wt), ' $@ | wc -l)" = 8
	test "$$(grep -o 'ip = { rk_n ? 8 \* wbytes : wbytes' $@ | wc -l)" = 1
	test "$$(grep -o 'rk_rope(ctx0, ' $@ | wc -l)" = 2

_ref/ref_alibi_kq.c: ref_alibi.c kquant_types.inc
	mkdir -p _ref
	sed $(SUBST) $< > $@
	test "$$(grep -o '^void rk_set_types' $@ | wc -l)" = 1
	test "$$(grep -o 'ggml_new_tensor_2d(c, rk_type(wt), ' $@ | wc -l)" = 6
	test "$$(grep -o 'ip = { rk_n ? 8 \* wbytes : wbytes' $@ | wc -l)" = 1

_ref/%_kq.o: _ref/%_kq.c
	$(CC) $(RFLAGS) -I. -c $< -o $@

_ref/harness_cpu.o: ref_harness.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c ref_harness.c -o $@

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/libggml_ref_nxkq.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/harness_cpu.o _ref/ref_gpt2_kq.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_alibi_kq.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_alibi_kq.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_gptj_kq.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_gptj_kq.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: nxkq
.SECONDARY:
