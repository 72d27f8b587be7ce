# Pin of n9: DSO's optimizeImmaturePoint (FullSystemOptPoint.cpp:51-205), ImmaturePoint::linearizeResidual
# (ImmaturePoint.cpp:476-543) and derive_idepth / both projectPoint (ResidualProjections.h:36-87), cut out of the files where
# they lie into _ref/gen_activate/ (build output, git-ignored - nothing is copied into the repo) and compiled, unmodified,
# together with n8's cut of the constructor, traceOn, the interpolation helpers and the pattern (ref_build_trace.mk), so the
# pinned inputs are points the reference itself traced.  Stand-ins for the DSO types they touch are in ref_wrap_activate.cpp;
# Eigen is n8's stand-in (ref_shim/trace_eigen), unchanged.  NDEBUG as in the reference's release build.  CPU only; only
# oracle/gen_reference_pins_activate.py uses the results.
#   make -C oracle -f ref_build_activate.mk REFERENCE=<dir>
activate: _ref/libactivate_ref.so
include ref_build_trace.mk
AGEN := _ref/gen_activate
$(AGEN)/opt_point.inc: $(SRC)/FullSystem/FullSystemOptPoint.cpp
	@mkdir -p $(AGEN)
	sed -n '51,205p' $< > $@
$(AGEN)/linearize.inc: $(SRC)/FullSystem/ImmaturePoint.cpp
	@mkdir -p $(AGEN)
	sed -n '476,543p' $< > $@
$(AGEN)/projections.inc: $(SRC)/FullSystem/ResidualProjections.h
	@mkdir -p $(AGEN)
	sed -n '36,87p' $< > $@
_ref/libactivate_ref.so: ref_wrap_activate.cpp $(AGEN)/opt_point.inc $(AGEN)/linearize.inc $(AGEN)/projections.inc $(GEN)/ctor.inc $(GEN)/trace_on.inc $(GEN)/interp33.inc $(GEN)/interp31.inc $(GEN)/interp33bilin.inc $(GEN)/pattern.inc ref_shim/trace_eigen/Eigen/Dense
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -DNDEBUG -w -I. -Iref_shim/trace_eigen -o $@ ref_wrap_activate.cpp
