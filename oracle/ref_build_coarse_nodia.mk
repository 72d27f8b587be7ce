# Pin of the undilated level-0 cloud and MVSNet's depth-range quantile: the body of CoarseTracker::makeCoarseDepthL0
# (CoarseTracker.cpp:148-374) and get_idepth_quantile (tandem_backend.cpp:354-361), cut out of the files where they lie into
# _ref/gen_nodia/ (build output, git-ignored - nothing is copied into the repo) and compiled, unmodified, against the stand-in
# Eigen of tests/cpp/eigen_stub and the harness ref_wrap_coarse_nodia.cpp.  CPU only; only
# oracle/gen_reference_pins_coarse_nodia.py uses the results.
#   make -C oracle -f ref_build_coarse_nodia.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
FS := $(REFERENCE)/tandem/src/FullSystem
TB := $(REFERENCE)/tandem/src/tandem
OUT := _ref
CXX ?= g++
all: $(OUT)/libcoarse_nodia_ref.so
$(OUT)/gen_nodia/make_coarse_depth.inc: $(FS)/CoarseTracker.cpp
	@mkdir -p $(OUT)/gen_nodia
	sed -n '148,374p' $< > $@
$(OUT)/gen_nodia/idepth_quantile.inc: $(TB)/tandem_backend.cpp
	@mkdir -p $(OUT)/gen_nodia
	sed -n '354,361p' $< > $@
$(OUT)/libcoarse_nodia_ref.so: ref_wrap_coarse_nodia.cpp $(OUT)/gen_nodia/make_coarse_depth.inc $(OUT)/gen_nodia/idepth_quantile.inc ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub -o $@ ref_wrap_coarse_nodia.cpp
