# oracle/embd.mk -- TEST INFRASTRUCTURE build recipe for the reference graphs with their embeddings exposed (make -C oracle -f embd.mk):
# OutputRequest::embeddings (crates/llm-base/src/model/common.rs:40-59), the final norm's output, and the residual stream that norm reads.
#
#   _ref/libggml_ref_embd.so          LLaMA, GPT-2, GPT-NeoX   (ref_harness.c + a copy of ref_gpt2.c)
#   _ref/libggml_alibi_embd.so        MPT, BLOOM               (a copy of ref_alibi.c)
#   _ref/libggml_gptj_embd.so         GPT-J                    (a copy of ref_gptj.c)
#   _ref/libggml_*_kv32_embd.so       the same on an F32 KV cache: copies of oracle/kv32.mk's F32-cache copies
#
# The reference's OWN LC/ggml.c + LC/k_quants.c, compiled unmodified with the flags of oracle/Makefile (RFLAGS).  The committed harnesses and
# their libraries stay as they are: each library here links a copy made under _ref/ that differs from its source in these lines only, and the
# recipe checks them:
#   * embd_capture.inc after the ggml include (rx_set_outputs: where the next evals write their rows);
#   * the residual named before the final norm, the norm's output named after its last node (gain, or the bias add), both copied out right
#     after the logits -- once per eval function of the harness (ref_gpt2.c: 2, the others: 1).
# A harness that no longer matches these patterns fails the build instead of silently giving no rows.
# The ggml objects are the ones oracle/Makefile makes (same names, same flags): whichever recipe runs first compiles them.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)

LIBS = _ref/libggml_ref_embd.so _ref/libggml_alibi_embd.so _ref/libggml_gptj_embd.so \
       _ref/libggml_ref_kv32_embd.so _ref/libggml_alibi_kv32_embd.so _ref/libggml_gptj_kv32_embd.so

ifneq ($(wildcard $(REF)/ggml.c),)
embd: $(LIBS)
else
embd:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/*_embd.so (if any)"
endif

# eval functions per harness: each must gain exactly one capture
N_ref_gpt2 = 2
N_ref_gpt2_kv32 = 2
N_ref_alibi = 1
N_ref_alibi_kv32 = 1
N_ref_gptj = 1
N_ref_gptj_kv32 = 1

define embd_copy
	mkdir -p _ref
	sed -e '/^#include "ggml.h"/r embd_capture.inc' \
	    -e 's/^\(    \)\(inpL = G(m, ggml_norm(ctx0, inpL));\)/\1struct ggml_tensor *rx_resid = inpL; \2/' \
	    -e 's/^\(    inpL = G(m, ggml_add(ctx0, G(m, ggml_mul(ctx0, inpL, m->ln_f_g)), m->ln_f_b));\)/\1 struct ggml_tensor *rx_embd = inpL;/' \
	    -e 's/^\(    \)\(inpL = ra_ln(ctx0, inpL, m->out_g, m->out_b);\)/\1struct ggml_tensor *rx_resid = inpL; \2 struct ggml_tensor *rx_embd = inpL;/' \
	    -e 's/^\(    \)\(inpL = ggml_add(ctx0, ggml_mul(ctx0, ggml_norm(ctx0, inpL), m->ln_f_g), m->ln_f_b);\)/\1struct ggml_tensor *rx_resid = inpL; \2 struct ggml_tensor *rx_embd = inpL;/' \
	    -e 's/^\(    if (logits_out) memcpy(logits_out, inpL->data, .*\)$$/\1 rx_capture(rx_embd, rx_resid);/' $< > $@
	test "$$(grep -c '^static void rx_capture' $@)" = 1
	test "$$(grep -c 'struct ggml_tensor \*rx_resid = inpL; ' $@)" = $(N_$*)
	test "$$(grep -c 'struct ggml_tensor \*rx_embd = inpL;' $@)" = $(N_$*)
	test "$$(grep -c ' rx_capture(rx_embd, rx_resid);$$' $@)" = $(N_$*)
endef

_ref/%_embd.c: %.c embd_capture.inc
	$(embd_copy)

_ref/%_kv32_embd.c: _ref/%_kv32.c embd_capture.inc
	$(embd_copy)

# kv32.mk's F32-cache copies (and its checks)
_ref/%_kv32.c: %.c
	$(MAKE) -f kv32.mk $@

_ref/%_embd.o: _ref/%_embd.c
	$(CC) $(RFLAGS) -I. -c $< -o $@

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/harness_cpu.o: ref_harness.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c ref_harness.c -o $@

_ref/ref_harness_kv32.o: _ref/ref_harness_kv32.c
	$(CC) $(RFLAGS) -I. -c $< -o $@

_ref/libggml_ref_embd.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/harness_cpu.o _ref/ref_gpt2_embd.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_ref_kv32_embd.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_harness_kv32.o _ref/ref_gpt2_kv32_embd.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_%_embd.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_%_embd.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: embd
.SECONDARY:
