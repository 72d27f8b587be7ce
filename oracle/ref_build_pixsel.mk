# Pin of n10: DSO's PixelSelector (PixelSelector2.cpp:41-438: the constructor with its srand / rand pattern, makeHists,
# makeMaps and select) and its class declaration (PixelSelector2.h:32-66), cut out of the files where they lie into
# _ref/gen_pixsel/ (build output, git-ignored - nothing is copied into the repo) and compiled, unmodified, against a stand-in
# Eigen of its own (ref_shim/pixsel_eigen) and the harness ref_wrap_pixsel.cpp, with NDEBUG as in the reference's release build.
# The harness uses the real srand / rand of the C library.  CPU only; only oracle/gen_reference_pins_pixsel.py uses the results.
#   make -C oracle -f ref_build_pixsel.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
SRC := $(REFERENCE)/tandem/src
PGEN := _ref/gen_pixsel
CXX ?= g++
all: _ref/libpixsel_ref.so
$(PGEN)/class.inc: $(SRC)/FullSystem/PixelSelector2.h
	@mkdir -p $(PGEN)
	sed -n '32,66p' $< > $@
$(PGEN)/selector.inc: $(SRC)/FullSystem/PixelSelector2.cpp
	@mkdir -p $(PGEN)
	sed -n '41,438p' $< > $@
_ref/libpixsel_ref.so: ref_wrap_pixsel.cpp $(PGEN)/class.inc $(PGEN)/selector.inc ref_shim/pixsel_eigen/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -DNDEBUG -w -I. -Iref_shim/pixsel_eigen -o $@ ref_wrap_pixsel.cpp
