# oracle/kquant_kv32.mk -- TEST INFRASTRUCTURE build recipe for the reference graphs on models whose 2-D weights each have their own element type,
# with an F32 KV cache (make -C oracle -f kquant_kv32.mk): the typed harness copies of kquant.mk / neox_kquant.mk with kv32.mk's cache substitutions.
#
#   _ref/libggml_ref_kq_kv32.so     LLaMA            (the typed copy of ref_harness.c; RefKq(kv32=True) in oracle/kquant.py)
#   _ref/libggml_ref_nxkq_kv32.so   GPT-2, GPT-NeoX  (kv32.mk's ref_harness copy + the typed copy of ref_gpt2.c; the RefLib API of bindings.py)
#   _ref/libggml_alibi_kq_kv32.so   MPT, BLOOM       (the typed copy of ref_alibi.c)
#   _ref/libggml_gptj_kq_kv32.so    GPT-J            (the typed copy of ref_gptj.c)
#
# The reference's OWN LC/ggml.c + LC/k_quants.c (oracle/Makefile's objects and flags).  The typed copies _ref/*_kq.c are the ones kquant.mk and
# neox_kquant.mk make (and check); this recipe asks those recipes for them and makes a second copy of each, _ref/*_kq_kv32.c, that differs from
# it in kv32.mk's three substitutions only, each counted as kv32.mk counts it on the same harness:
#   * memory_k and memory_v are allocated as GGML_TYPE_F32 instead of GGML_TYPE_F16 (both lines, in every harness);
#   * the context that holds them is sized for 4-byte elements (one line, in every harness);
#   * the graph builders' cache views take a 4-byte element size (ref_harness.c 1 line, ref_gpt2.c 2, ref_alibi.c 1; ref_gptj.c asks
#     ggml_element_size and has none).
# No GGML_TYPE_F16 may remain in a copy.  A harness that no longer matches these patterns fails the build instead of silently giving an f16 cache.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)
KSZ_ref_harness = 1
KSZ_ref_gpt2    = 2
KSZ_ref_alibi   = 1
KSZ_ref_gptj    = 0

ifneq ($(wildcard $(REF)/ggml.c),)
kqkv32: _ref/libggml_ref_kq_kv32.so _ref/libggml_ref_nxkq_kv32.so _ref/libggml_alibi_kq_kv32.so _ref/libggml_gptj_kq_kv32.so
else
kqkv32:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/*_kq_kv32.so (if any)"
endif

# the typed copies and the F32-cache harness object, from the recipes that own them (with their own checks)
_ref/ref_harness_kq.c: ref_harness.c kquant_types.inc
	$(MAKE) -f kquant.mk $@
_ref/ref_gpt2_kq.c: ref_gpt2.c kquant_types.inc rope_custom.inc
	$(MAKE) -f neox_kquant.mk $@
_ref/ref_gptj_kq.c: ref_gptj.c kquant_types.inc rope_custom.inc
	$(MAKE) -f neox_kquant.mk $@
_ref/ref_alibi_kq.c: ref_alibi.c kquant_types.inc
	$(MAKE) -f neox_kquant.mk $@
_ref/ref_harness_kv32.o: ref_harness.c
	$(MAKE) -f kv32.mk $@

_ref/%_kq_kv32.c: _ref/%_kq.c
	sed -e 's/\(m->memory_[kv] = ggml_new_tensor_1d(m->session_ctx, \)GGML_TYPE_F16, n_elements)/\1GGML_TYPE_F32, n_elements)/' \
	    -e 's/{ n_elements \* 2 \* 2 + /{ n_elements * 4 * 2 + /' \
	    -e 's/const size_t ksz = 2, vsz = 2/const size_t ksz = 4, vsz = 4/' $< > $@
	test "$$(grep -c 'm->memory_[kv] = ggml_new_tensor_1d(m->session_ctx, GGML_TYPE_F32, n_elements)' $@)" = 2
	test "$$(grep -c '{ n_elements \* 4 \* 2 + ' $@)" = 1
	test "$$(grep -c 'const size_t ksz = 4, vsz = 4' $@)" = $(KSZ_$*)
	! grep -n 'GGML_TYPE_F16\|ksz = 2\|vsz = 2' $@

_ref/%_kq_kv32.o: _ref/%_kq_kv32.c
	$(CC) $(RFLAGS) -I. -c $< -o $@

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/libggml_ref_kq_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_harness_kq_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_ref_nxkq_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_harness_kv32.o _ref/ref_gpt2_kq_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_alibi_kq_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_alibi_kq_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

_ref/libggml_gptj_kq_kv32.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/ref_gptj_kq_kv32.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: kqkv32
.SECONDARY:
