// Drop-in replacement header for tandem/libdr/dr_mvsnet/src/dr_mvsnet/dr_mvsnet.h (class surface :36-66,
// DrMvsnetOutput :12-34, test_dr_mvsnet :68) implemented over the tandem_b200 C ABI (include/tandem_b200.h).
// tandem/src (FullSystem.cpp:284-285, tandem_backend.cpp:147,264,268,286,347) compiles against it unchanged.
#ifndef DR_MVSNET_H
#define DR_MVSNET_H

#include <cstdlib>
#include <memory>
#include <utility>
#include <vector>

class DrMvsnetImpl;  // opaque: owns a tdm_mvsnet handle (shims/dr_mvsnet.cpp)
struct tdm_mvsnet;   // include/tandem_b200.h

class DrMvsnetOutput {
public:
  DrMvsnetOutput(int height, int width) : height(height), width(width) {
    depth = (float *) malloc(sizeof(float) * width * height);
    confidence = (float *) malloc(sizeof(float) * width * height);
    depth_dense = (float *) malloc(sizeof(float) * width * height);
    confidence_dense = (float *) malloc(sizeof(float) * width * height);
  }

  ~DrMvsnetOutput() {
    free(depth);
    free(confidence);
    free(depth_dense);
    free(confidence_dense);
  }

  float *depth;
  float *confidence;
  float *depth_dense;
  float *confidence_dense;
  const int height;
  const int width;
};

class DrMvsnet {
public:
  // filename: ".../model.pt" as passed by FullSystem::initDr; the weights are read from ".../model.tdmw" beside it.
  explicit DrMvsnet(char const *filename);

  ~DrMvsnet();

  // Blocking for last input. Non-blocking for this input.
  void CallAsync(int height, int width, int view_num, int ref_index, unsigned char **bgrs, float const *intrinsic_matrix,
                 float **cam_to_worlds, float depth_min, float depth_max, float discard_percentage,
                 bool debug_print = false);

  // Extension: the same call with the feature cache (tdm_mvsnet_call_async_ids).  view_ids[i] names view i (TANDEM:
  // frameHessians[i]->shell->id); FeatureNet runs only for the ids the previous such call did not hold.  bgrs[i] may be
  // NULL for a held id and is ignored for one.
  void CallAsync(int height, int width, int view_num, int ref_index, std::vector<long long> const &view_ids,
                 unsigned char **bgrs, float const *intrinsic_matrix, float **cam_to_worlds, float depth_min,
                 float depth_max, float discard_percentage, bool debug_print = false);

  // Blocking. Ownership of the result passes to the caller (delete it).
  DrMvsnetOutput *GetResult();

  // Blocking
  void Wait();

  // Non-blocking
  bool Ready();

  // Extension: the C-ABI handle, so that DrFusion::IntegrateScanAsync(DrMvsnet const&) can read the result on the device.
  tdm_mvsnet* handle() const;

private:
  DrMvsnetImpl *impl;
};

// Known-answer test of the reference (dr_mvsnet.cpp:376-556). filename_inputs: the converted golden container
// "sample_inputs.bin" written by tools/convert_sample_inputs.py next to the reference's sample_inputs.pt
// (a TorchScript zip cannot be read without libtorch).
bool test_dr_mvsnet(DrMvsnet &model, char const *filename_inputs, bool print = false, int repetitions = 1,
                    char const *out_folder = NULL);

#endif  // DR_MVSNET_H
