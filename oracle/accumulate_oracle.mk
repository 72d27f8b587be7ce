# Builds the n13 CPU oracle (oracle/accumulate_oracle.c, test infrastructure only) into oracle/_build/, with the flags of
# oracle/Makefile: fp32 without FMA contraction, like the __f*_rn intrinsics of the kernels it checks.
CC ?= gcc
CFLAGS := -O2 -fPIC -shared -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function
all: _build/libaccumulate_oracle.so
_build/libaccumulate_oracle.so: accumulate_oracle.c
	@mkdir -p _build
	$(CC) $(CFLAGS) -o $@ $< -lm
