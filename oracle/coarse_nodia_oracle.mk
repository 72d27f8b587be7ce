# Builds the nodia CPU oracle (oracle/coarse_nodia_oracle.c, test infrastructure only) into oracle/_build/, with the flags of
# oracle/Makefile: fp32 without FMA contraction, like the __f*_rn intrinsics of the kernels it checks.
CC ?= gcc
CFLAGS := -O2 -fPIC -shared -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function
all: _build/libcoarse_nodia_oracle.so
_build/libcoarse_nodia_oracle.so: coarse_nodia_oracle.c
	@mkdir -p _build
	$(CC) $(CFLAGS) -o $@ $< -lm
