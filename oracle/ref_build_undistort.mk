# Pin of n11: DSO's per-frame input, cut out of the files where they lie into _ref/gen_undistort/ (build output, git-ignored -
# nothing is copied into the repo) and compiled, unmodified, with -ffp-contract=off -fno-fast-math against the stand-ins of the
# harness ref_wrap_undistort.cpp and the stand-in Eigen of tests/cpp/eigen_stub:
#   PhotometricUndistorter and Undistort (declarations)   tandem/src/util/Undistort.h:40-64, :67-109
#   PhotometricUndistorter's constructor and destructor   tandem/src/util/Undistort.cpp:50-185
#   PhotometricUndistorter::processFrame                  tandem/src/util/Undistort.cpp:213-252
#   Undistort::undistort                                  tandem/src/util/Undistort.cpp:393-490
#   getImageBGR_8UC3_undistort_internal                   tandem/src/util/DatasetReader.h:354-400
#   FullSystem::setGammaFunction                          tandem/src/FullSystem/FullSystem.cpp:232-253
#   CalibHessian::getBGradOnly                            tandem/src/FullSystem/HessianBlocks.h:446-452
#   FrameHessian::makeImages                              tandem/src/FullSystem/HessianBlocks.cpp:128-191
# The constructor reads the response with iostreams inside the Python process that loads the library, so build it with the
# C++ compiler whose libstdc++ that process resolves (the system g++: CXX=g++).  CPU only; only
# oracle/gen_reference_pins_undistort.py uses the result.
#   make -C oracle -f ref_build_undistort.mk REFERENCE=<dir> CXX=g++
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
SRC := $(REFERENCE)/tandem/src
UGEN := _ref/gen_undistort
CXX ?= g++
INCS := $(UGEN)/photometric_class.inc $(UGEN)/undistort_class.inc $(UGEN)/photometric_ctor.inc $(UGEN)/process_frame.inc \
        $(UGEN)/undistort.inc $(UGEN)/bgr.inc $(UGEN)/set_gamma.inc $(UGEN)/bgrad.inc $(UGEN)/make_images.inc
all: _ref/libundistort_ref.so
$(UGEN)/photometric_class.inc: $(SRC)/util/Undistort.h
	@mkdir -p $(UGEN)
	sed -n '40,64p' $< > $@
$(UGEN)/undistort_class.inc: $(SRC)/util/Undistort.h
	@mkdir -p $(UGEN)
	sed -n '67,109p' $< > $@
$(UGEN)/photometric_ctor.inc: $(SRC)/util/Undistort.cpp
	@mkdir -p $(UGEN)
	sed -n '50,185p' $< > $@
$(UGEN)/process_frame.inc: $(SRC)/util/Undistort.cpp
	@mkdir -p $(UGEN)
	sed -n '213,252p' $< > $@
$(UGEN)/undistort.inc: $(SRC)/util/Undistort.cpp
	@mkdir -p $(UGEN)
	sed -n '393,490p' $< > $@
$(UGEN)/bgr.inc: $(SRC)/util/DatasetReader.h
	@mkdir -p $(UGEN)
	sed -n '354,400p' $< > $@
$(UGEN)/set_gamma.inc: $(SRC)/FullSystem/FullSystem.cpp
	@mkdir -p $(UGEN)
	sed -n '232,253p' $< > $@
$(UGEN)/bgrad.inc: $(SRC)/FullSystem/HessianBlocks.h
	@mkdir -p $(UGEN)
	sed -n '446,452p' $< > $@
$(UGEN)/make_images.inc: $(SRC)/FullSystem/HessianBlocks.cpp
	@mkdir -p $(UGEN)
	sed -n '128,191p' $< > $@
_ref/libundistort_ref.so: ref_wrap_undistort.cpp $(INCS) ../tests/cpp/eigen_stub/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -w -I. -I../tests/cpp/eigen_stub -o $@ ref_wrap_undistort.cpp
