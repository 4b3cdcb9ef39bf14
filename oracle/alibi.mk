# oracle/alibi.mk -- TEST INFRASTRUCTURE build recipe for the MPT / BLOOM reference graphs (make -C oracle -f alibi.mk).
#
#   _ref/libggml_alibi.so   the reference's OWN LC/ggml.c + LC/k_quants.c, compiled unmodified from where they lie with the flags of
#                           oracle/Makefile (RFLAGS), plus ref_alibi.c (the MPT and BLOOM graph builders restated on the C API).
#
# A library of its own beside _ref/libggml_ref.so, so that the LLaMA / GPT-2 / GPT-NeoX harness library is built exactly as before.
# The object files are the ones oracle/Makefile makes (same names, same flags): whichever recipe runs first compiles them.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)

ifneq ($(wildcard $(REF)/ggml.c),)
alibi: _ref/libggml_alibi.so
else
alibi:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/libggml_alibi.so (if any)"
endif

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/alibi_cpu.o: ref_alibi.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c ref_alibi.c -o $@

_ref/libggml_alibi.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/alibi_cpu.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: alibi
