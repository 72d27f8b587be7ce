# n5 pin (SURVEY.md 8f): the whole coarse-to-fine body of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-936), cut
# out of the file where it lies into _ref/gen/ (build output, git-ignored - nothing is copied into the repo) and compiled,
# unmodified, against the stand-in Eigen of tests/cpp/eigen_stub and the harness ref_wrap_pyramid.cpp.  CPU only.  Same
# recipe style as ref_build.mk; only oracle/gen_reference_pins_pyramid.py uses the result.
#   make -C oracle -f ref_build_pyramid.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
FS := $(REFERENCE)/tandem/src/FullSystem
OUT := _ref
CXX ?= g++
all: $(OUT)/libpyramid_ref.so
$(OUT)/gen/track_pyramid.inc: $(FS)/CoarseTracker.cpp
	@mkdir -p $(OUT)/gen
	sed -n '750,936p' $< > $@
$(OUT)/libpyramid_ref.so: ref_wrap_pyramid.cpp $(OUT)/gen/track_pyramid.inc ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub -o $@ ref_wrap_pyramid.cpp
