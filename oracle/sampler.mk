# oracle/sampler.mk -- TEST INFRASTRUCTURE build recipe for the sampler checker (make -C oracle -f sampler.mk).  Plain C, no reference sources.
#
#   liboracle_sampler.so   sampler_oracle.c: the default sampler chain of b200_sampler, stage by stage, calling the host libm's expf
#
# -ffp-contract=off: the C source's operations are the ones executed (no fused multiply-adds the source does not write), and -fno-builtin keeps
# every expf a call into libm.

CC     = /usr/bin/gcc
PFLAGS = -O2 -std=c11 -fPIC -Wall -Wextra -ffp-contract=off -fno-builtin -fno-fast-math

sampler: liboracle_sampler.so

liboracle_sampler.so: sampler_oracle.c
	$(CC) $(PFLAGS) -shared -o $@ sampler_oracle.c -lm

.PHONY: sampler
