# oracle/lora.mk -- TEST INFRASTRUCTURE build recipe for the LoRA patch checkers (make -C oracle -f lora.mk).
#
#   liboracle_lora.so      plain-C restatement (lora_oracle.c on ggml_oracle.c); builds anywhere, no reference sources needed.
#   _ref/libggml_lora.so   the reference's OWN LC/ggml.c + LC/k_quants.c, compiled unmodified from where they lie with the flags of
#                          oracle/Makefile (RFLAGS), plus ref_lora.c (LoraAdapter::patch restated on the C API).
#
# The object files are the ones oracle/Makefile makes (same names, same flags): whichever recipe runs first compiles them.

REF   ?= /root/reference/crates/ggml/sys/llama-cpp
CC     = /usr/bin/gcc
RFLAGS = -O3 -DNDEBUG -DGGML_USE_K_QUANTS -pthread -mavx -mavx2 -mfma -mf16c -msse3 -fPIC -w -I$(REF)
OFLAGS = -O3 -std=c11 -fPIC -Wall -Wextra -Wno-unused-parameter -mavx2 -mfma -mf16c -fopenmp -ffp-contract=off

ifneq ($(wildcard $(REF)/ggml.c),)
lora: liboracle_lora.so _ref/libggml_lora.so
else
lora: liboracle_lora.so
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/libggml_lora.so (if any)"
endif

liboracle_lora.so: lora_oracle.c ggml_oracle.c ggml_oracle.h
	$(CC) $(OFLAGS) -shared -o $@ lora_oracle.c ggml_oracle.c -lm

_ref/ggml_cpu.o: $(REF)/ggml.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/ggml.c -o $@

_ref/k_quants.o: $(REF)/k_quants.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c $(REF)/k_quants.c -o $@

_ref/lora_cpu.o: ref_lora.c
	mkdir -p _ref
	$(CC) $(RFLAGS) -c ref_lora.c -o $@

_ref/libggml_lora.so: _ref/ggml_cpu.o _ref/k_quants.o _ref/lora_cpu.o
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm -pthread

.PHONY: lora
