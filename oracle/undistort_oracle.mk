# Builds the n11 CPU oracle (oracle/undistort_oracle.c, which includes front_oracle.c's pyramid; test infrastructure only) into
# oracle/_build/, with the flags of oracle/Makefile: fp32 without FMA contraction, like the __f*_rn intrinsics of the kernels
# it checks.
CC ?= gcc
CFLAGS := -O2 -fPIC -shared -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function
all: _build/libundistort_oracle.so
_build/libundistort_oracle.so: undistort_oracle.c front_oracle.c
	@mkdir -p _build
	$(CC) $(CFLAGS) -o $@ $< -lm
