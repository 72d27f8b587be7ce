# n7 pin (SURVEY.md 8f): the body of CoarseTracker::makeCoarseDepthL0 (CoarseTracker.cpp:148-374), cut out of the file where
# it lies into _ref/gen/ (build output, git-ignored - nothing is copied into the repo) and compiled, unmodified, against the
# stand-in Eigen of tests/cpp/eigen_stub and the harness ref_wrap_coarse_ref.cpp.  CPU only.  The dense block it is chained with
# is ref_build.mk's libfront_ref.so; only oracle/gen_reference_pins_coarse_ref.py uses the results.
#   make -C oracle -f ref_build.mk REFERENCE=<dir>
#   make -C oracle -f ref_build_coarse_ref.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
FS := $(REFERENCE)/tandem/src/FullSystem
OUT := _ref
CXX ?= g++
all: $(OUT)/libcoarse_ref_ref.so
$(OUT)/gen/make_coarse_depth.inc: $(FS)/CoarseTracker.cpp
	@mkdir -p $(OUT)/gen
	sed -n '148,374p' $< > $@
$(OUT)/libcoarse_ref_ref.so: ref_wrap_coarse_ref.cpp $(OUT)/gen/make_coarse_depth.inc ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub -o $@ ref_wrap_coarse_ref.cpp
