# Pin of n12: DSO's PointFrameResidual::linearize and applyRes (Residuals.cpp:78-274, 306-328), FullSystem's
# linearizeAll_Reductor, applyRes_Reductor, setNewFrameEnergyTH and linearizeAll (FullSystemOptimize.cpp:52-210), cut out of
# the files where they lie into _ref/gen_linearize/ (build output, git-ignored - nothing is copied into the repo) and compiled,
# unmodified, with n9's cut of both projectPoint forms (ResidualProjections.h:36-87) and n8's cut of the interpolation helpers
# and the pattern (ref_build_activate.mk, ref_build_trace.mk), against the stand-ins of ref_wrap_linearize.cpp, the stand-in
# Eigen of ref_shim/linearize_eigen and the boost::bind stand-in of ref_shim/boost.  NDEBUG as in the reference's release
# build.  CPU only; only oracle/gen_reference_pins_linearize.py uses the results.
#   make -C oracle -f ref_build_linearize.mk REFERENCE=<dir>
linearize: _ref/liblinearize_ref.so
include ref_build_activate.mk
LGEN := _ref/gen_linearize
$(LGEN)/linearize.inc: $(SRC)/FullSystem/Residuals.cpp
	@mkdir -p $(LGEN)
	sed -n '78,274p' $< > $@
$(LGEN)/apply_res.inc: $(SRC)/FullSystem/Residuals.cpp
	@mkdir -p $(LGEN)
	sed -n '306,328p' $< > $@
$(LGEN)/linearize_all.inc: $(SRC)/FullSystem/FullSystemOptimize.cpp
	@mkdir -p $(LGEN)
	sed -n '52,210p' $< > $@
_ref/liblinearize_ref.so: ref_wrap_linearize.cpp $(LGEN)/linearize.inc $(LGEN)/apply_res.inc $(LGEN)/linearize_all.inc $(AGEN)/projections.inc $(GEN)/interp33.inc $(GEN)/pattern.inc ref_shim/linearize_eigen/Eigen/Dense ref_shim/boost/bind.hpp
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -DNDEBUG -w -I. -Iref_shim/linearize_eigen -Iref_shim -o $@ ref_wrap_linearize.cpp
