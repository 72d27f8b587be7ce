# Pin of n13: DSO's EFResidual::takeDataF (EnergyFunctionalStructs.cpp:39-50), the accumulators AccumulatorXX, AccumulatorX
# and AccumulatorApprox (MatrixAccumulators.h:36-89, 177-237, 595-972), AccumulatedTopHessianSSE (the class body of
# AccumulatedTopHessian.h:44-166, addPoint<0/1/2> and stitchDoubleInternal of AccumulatedTopHessian.cpp:36-162, 241-303),
# AccumulatedSCHessianSSE (AccumulatedSCHessian.h:42-156, AccumulatedSCHessian.cpp:34-157) and EnergyFunctional's
# accumulateAF_MT, accumulateLF_MT, accumulateSCF_MT, resubstituteF_MT and resubstituteFPt (EnergyFunctional.cpp:196-318),
# cut out of the files where they lie into _ref/gen_accumulate/ (build output, git-ignored - nothing is copied into the repo)
# and compiled, unmodified, against the stand-ins of ref_wrap_accumulate.cpp, the stand-in Eigen of ref_shim/accumulate_eigen
# and the boost::bind stand-in of ref_shim/boost.  SSE intrinsics compile as they are on x86.  NDEBUG as in the reference's
# release build.  CPU only; only oracle/gen_reference_pins_accumulate.py uses the results.
#   make -C oracle -f ref_build_accumulate.mk REFERENCE=<dir>
ifndef REFERENCE
$(error set REFERENCE to the root of a checkout of the reference)
endif
OB := $(REFERENCE)/tandem/src/OptimizationBackend
CG := _ref/gen_accumulate
accumulate: _ref/libaccumulate_ref.so
$(CG)/acc_xx.inc: $(OB)/MatrixAccumulators.h
	@mkdir -p $(CG)
	sed -n '36,89p' $< > $@
$(CG)/acc_x.inc: $(OB)/MatrixAccumulators.h
	@mkdir -p $(CG)
	sed -n '177,237p' $< > $@
$(CG)/acc_approx.inc: $(OB)/MatrixAccumulators.h
	@mkdir -p $(CG)
	sed -n '595,972p' $< > $@
$(CG)/top_class.inc: $(OB)/AccumulatedTopHessian.h
	@mkdir -p $(CG)
	sed -n '44,166p' $< > $@
$(CG)/sc_class.inc: $(OB)/AccumulatedSCHessian.h
	@mkdir -p $(CG)
	sed -n '42,156p' $< > $@
$(CG)/take_data.inc: $(OB)/EnergyFunctionalStructs.cpp
	@mkdir -p $(CG)
	sed -n '39,50p' $< > $@
$(CG)/top_add.inc: $(OB)/AccumulatedTopHessian.cpp
	@mkdir -p $(CG)
	sed -n '36,162p' $< > $@
$(CG)/top_stitch.inc: $(OB)/AccumulatedTopHessian.cpp
	@mkdir -p $(CG)
	sed -n '241,303p' $< > $@
$(CG)/sc.inc: $(OB)/AccumulatedSCHessian.cpp
	@mkdir -p $(CG)
	sed -n '34,157p' $< > $@
$(CG)/ef.inc: $(OB)/EnergyFunctional.cpp
	@mkdir -p $(CG)
	sed -n '196,318p' $< > $@
INCS := $(addprefix $(CG)/,acc_xx.inc acc_x.inc acc_approx.inc top_class.inc sc_class.inc take_data.inc top_add.inc top_stitch.inc sc.inc ef.inc)
_ref/libaccumulate_ref.so: ref_wrap_accumulate.cpp $(INCS) ref_shim/accumulate_eigen/Eigen/Dense ref_shim/boost/bind.hpp
	$(CXX) -O2 -std=c++14 -fPIC -shared -ffp-contract=off -fno-fast-math -DNDEBUG -w -I. -Iref_shim/accumulate_eigen -Iref_shim -o $@ ref_wrap_accumulate.cpp
