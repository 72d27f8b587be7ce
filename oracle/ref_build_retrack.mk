# n6 pin (SURVEY.md 8f): the motion-hypothesis loop of FullSystem::trackNewCoarse (FullSystem.cpp:538-617), cut out of the file
# where it lies into _ref/gen/ (build output, git-ignored - nothing is copied into the repo) and compiled, unmodified, in the
# harness ref_wrap_retrack.cpp.  Its trackNewestCoarse is the reference's own body (CoarseTracker.cpp:750-936) through
# ref_wrap_pyramid.cpp, linked into the same library.  CPU only; only oracle/gen_reference_pins_retrack.py uses the result.
#   make -C oracle -f ref_build_retrack.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
FS := $(REFERENCE)/tandem/src/FullSystem
OUT := _ref
CXX ?= g++
CXXFLAGS := -O2 -std=c++14 -fPIC -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub
all: $(OUT)/libretrack_ref.so
$(OUT)/gen/track_pyramid.inc: $(FS)/CoarseTracker.cpp
	@mkdir -p $(OUT)/gen
	sed -n '750,936p' $< > $@
$(OUT)/gen/retrack.inc: $(FS)/FullSystem.cpp
	@mkdir -p $(OUT)/gen
	sed -n '538,617p' $< > $@
$(OUT)/libretrack_ref.so: ref_wrap_retrack.cpp ref_wrap_pyramid.cpp $(OUT)/gen/retrack.inc $(OUT)/gen/track_pyramid.inc ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_wrap_retrack.cpp ref_wrap_pyramid.cpp
