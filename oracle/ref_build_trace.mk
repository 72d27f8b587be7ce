# Pin of n8: DSO's immature-point constructor and traceOn (ImmaturePoint.cpp:32-61, 75-414), the three interpolation helpers
# they call (globalFuncs.h) and the point pattern (settings.cpp), cut out of the files where they lie into _ref/gen_trace/
# (build output, git-ignored - nothing is copied into the repo) and compiled, unmodified, against the stand-in Eigen of
# ref_shim/trace_eigen and the harness ref_wrap_trace.cpp, with NDEBUG as in the reference's release build (traceOn's
# assert(dist>0) is then not evaluated; a zero maxPixSearch reaches the non-finite dx/dy return behind it).  CPU only; only
# oracle/gen_reference_pins_trace.py uses the results.
#   make -C oracle -f ref_build_trace.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
SRC := $(REFERENCE)/tandem/src
GEN := _ref/gen_trace
CXX ?= g++
all: _ref/libtrace_ref.so
$(GEN)/ctor.inc: $(SRC)/FullSystem/ImmaturePoint.cpp
	@mkdir -p $(GEN)
	sed -n '32,61p' $< > $@
$(GEN)/trace_on.inc: $(SRC)/FullSystem/ImmaturePoint.cpp
	@mkdir -p $(GEN)
	sed -n '75,414p' $< > $@
$(GEN)/interp33.inc: $(SRC)/util/globalFuncs.h
	@mkdir -p $(GEN)
	sed -n '75,89p' $< > $@
$(GEN)/interp31.inc: $(SRC)/util/globalFuncs.h
	@mkdir -p $(GEN)
	sed -n '126,140p' $< > $@
$(GEN)/interp33bilin.inc: $(SRC)/util/globalFuncs.h
	@mkdir -p $(GEN)
	sed -n '166,188p' $< > $@
$(GEN)/pattern.inc: $(SRC)/util/settings.cpp
	@mkdir -p $(GEN)
	sed -n '216,266p' $< > $@
_ref/libtrace_ref.so: ref_wrap_trace.cpp $(GEN)/ctor.inc $(GEN)/trace_on.inc $(GEN)/interp33.inc $(GEN)/interp31.inc $(GEN)/interp33bilin.inc $(GEN)/pattern.inc ref_shim/trace_eigen/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -DNDEBUG -w -I. -Iref_shim/trace_eigen -o $@ ref_wrap_trace.cpp
