# Compiles the REFERENCE's own sources, unmodified and from where they lie in a checkout of the reference
# (make -f ref_build.mk REFERENCE=<dir>), into oracle/_ref/ (git-ignored).  Nothing is copied into the repo.  Only
# oracle/gen_reference_pins.py uses the result.  The reference's CMake build is not used (it needs OpenCV/Eigen/Boost).
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
REF := $(REFERENCE)/tandem/libdr
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
OUT := _ref
FUS := $(REF)/dr_fusion/src
FUS_SRCS := $(FUS)/tsdfvh/heap.cu $(FUS)/tsdfvh/hash_table.cu $(FUS)/tsdfvh/tsdf_volume.cu $(FUS)/marching_cubes/mesh.cu \
            $(FUS)/marching_cubes/mesh_extractor.cu $(FUS)/utils/rgbd_image.cu
TRK := $(REF)/cuda_coarse_tracker

all: $(OUT)/libdr_fusion_ref.so $(OUT)/libtracker_ref.so

# DR_FUSION_DEBUG_SYNC_LAUNCH is a PUBLIC compile definition of the reference target (dr_fusion/CMakeLists.txt:40-41)
$(OUT)/libdr_fusion_ref.so: ref_wrap_fusion.cpp
	@mkdir -p $(OUT)
	$(NVCC) -O2 -std=c++17 $(ARCH) -rdc=true -DDR_FUSION_DEBUG_SYNC_LAUNCH -Xcompiler -fPIC -w -I$(FUS) -shared -cudart static \
	    -o $@ $(FUS_SRCS) -x cu $(FUS)/dr_fusion/dr_fusion.cpp -x cu ref_wrap_fusion.cpp

$(OUT)/libtracker_ref.so: ref_wrap_tracker.cu
	@mkdir -p $(OUT)
	$(NVCC) -O2 -std=c++17 $(ARCH) -Xcompiler -fPIC -w -Iref_shim -I$(TRK)/include/private -shared -cudart static \
	    -o $@ $(TRK)/src/cuda_coarse_tracker_private.cu ref_wrap_tracker.cu

# n1 / n2 pins (SURVEY.md 8f): two function bodies of tandem/src/FullSystem, cut out of the files where they lie (line ranges
# as cited in oracle/front_oracle.c) into _ref/gen/ (build output, git-ignored - nothing is copied into the repo) and
# compiled, unmodified, against the stand-in Eigen of tests/cpp/eigen_stub and the harness ref_wrap_front.cpp.  CPU only.
FS := $(REFERENCE)/tandem/src/FullSystem
CXX ?= g++
all: $(OUT)/libfront_ref.so
$(OUT)/gen/make_images.inc: $(FS)/HessianBlocks.cpp
	@mkdir -p $(OUT)/gen
	sed -n '128,191p' $< > $@
$(OUT)/gen/dense_ref.inc: $(FS)/CoarseTracker.cpp
	@mkdir -p $(OUT)/gen
	sed -n '655,725p' $< > $@
$(OUT)/libfront_ref.so: ref_wrap_front.cpp $(OUT)/gen/make_images.inc $(OUT)/gen/dense_ref.inc ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub -o $@ ref_wrap_front.cpp

# n3 pin: the LM level loop of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-916), same recipe style.
all: $(OUT)/liblm_ref.so
$(OUT)/gen/lm_loop.inc: $(FS)/CoarseTracker.cpp
	@mkdir -p $(OUT)/gen
	sed -n '750,916p' $< > $@
$(OUT)/liblm_ref.so: ref_wrap_lm.cpp $(OUT)/gen/lm_loop.inc ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub -o $@ ref_wrap_lm.cpp
