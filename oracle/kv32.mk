# oracle/kv32.mk -- TEST INFRASTRUCTURE build recipe for the reference graphs on an F32 KV cache (make -C oracle -f kv32.mk):
# InferenceSessionConfig::memory_k_type = memory_v_type = ModelKVMemoryType::Float32, the reference CLI's --no-float16.
#
#   _ref/libggml_ref_kv32.so     LLaMA, GPT-2, GPT-NeoX  (ref_harness.c + ref_gpt2.c, the RefLib API of oracle/bindings.py)
#   _ref/libggml_alibi_kv32.so   MPT, BLOOM               (ref_alibi.c)
#   _ref/libggml_gptj_kv32.so    GPT-J                    (ref_gptj.c)
#
# The reference's OWN LC/ggml.c + LC/k_quants.c, compiled unmodified with the flags of oracle/Makefile (RFLAGS), with a copy of each harness made
# here under _ref/ (the committed harnesses and their libraries stay as they are).  The copy differs in the harness's f16 cache choices and in
# nothing else, and the recipe checks each of them:
#   * memory_k and memory_v are allocated as GGML_TYPE_F32 instead of GGML_TYPE_F16 (both lines, in every harness);
#   * the context that holds them is sized for 4-byte elements (n_elements * 4 * 2 instead of n_elements * 2 * 2);
#   * the graph builders' cache views take a 4-byte element size where the harness writes the f16 constant (ref_gptj.c asks
#     ggml_element_size and needs no change there).
# A harness that no longer matches these patterns fails the build instead of silently giving an f16 cache.
# The ggml objects are the ones oracle/Makefile makes (same names, same flags): whichever recipe runs first compiles them.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)

ifneq ($(wildcard $(REF)/ggml.c),)
kv32: _ref/libggml_ref_kv32.so _ref/libggml_alibi_kv32.so _ref/libggml_gptj_kv32.so
else
kv32:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/*_kv32.so (if any)"
endif

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/%_kv32.c: %.c
	mkdir -p _ref
	sed -e 's/\(m->memory_[kv] = ggml_new_tensor_1d(m->session_ctx, \)GGML_TYPE_F16, n_elements)/\1GGML_TYPE_F32, n_elements)/' \
	    -e 's/{ n_elements \* 2 \* 2 + /{ n_elements * 4 * 2 + /' \
	    -e 's/const size_t ksz = 2, vsz = 2/const size_t ksz = 4, vsz = 4/' $< > $@
	test "$$(grep -c 'm->memory_[kv] = ggml_new_tensor_1d(m->session_ctx, GGML_TYPE_F32, n_elements)' $@)" = 2
	test "$$(grep -c '{ n_elements \* 4 \* 2 + ' $@)" = 1
	! grep -n 'GGML_TYPE_F16\|ksz = 2\|vsz = 2' $@

_ref/%_kv32.o: _ref/%_kv32.c
	$(CC) $(RFLAGS) -I. -c $< -o $@

_ref/libggml_ref_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_harness_kv32.o _ref/ref_gpt2_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_alibi_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_alibi_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_gptj_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_gptj_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: kv32
