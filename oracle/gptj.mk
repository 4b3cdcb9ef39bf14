# oracle/gptj.mk -- TEST INFRASTRUCTURE build recipe for the GPT-J reference graph (make -C oracle -f gptj.mk).
#
#   _ref/libggml_gptj.so   the reference's OWN LC/ggml.c + LC/k_quants.c, compiled unmodified from where they lie with the flags of
#                           oracle/Makefile (RFLAGS), plus ref_gptj.c (the GPT-J graph builder restated on the C API).
#
# A library of its own beside _ref/libggml_ref.so, so that the other reference libraries are built exactly as before.
# The object files are the ones oracle/Makefile makes (same names, same flags): whichever recipe runs first compiles them.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)

ifneq ($(wildcard $(REF)/ggml.c),)
gptj: _ref/libggml_gptj.so
else
gptj:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/libggml_gptj.so (if any)"
endif

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/gptj_cpu.o: ref_gptj.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c ref_gptj.c -o $@

_ref/libggml_gptj.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/gptj_cpu.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: gptj
