// class DrFusion over the tandem_b200 C ABI (replaces tandem/libdr/dr_fusion/src/dr_fusion/dr_fusion.cpp).
// Error convention of the reference: print + exit(EXIT_FAILURE) (tsdf_volume.cu:520-524).
#include "dr_fusion/dr_fusion.h"
#include "dr_mvsnet/dr_mvsnet.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>

#include "tandem_b200.h"

static void die(const char* where) {
  std::cerr << "ERROR: " << where << ": " << tdm_last_error() << std::endl;
  exit(EXIT_FAILURE);
}

DrFusion::DrFusion(struct DrFusionOptions const& o) {
  static_assert(sizeof(DrFusionOptions) == sizeof(tdm_fusion_options), "DrFusionOptions must match tdm_fusion_options");
  tdm_fusion_options t;
  std::memcpy(&t, &o, sizeof(t));
  if (tdm_fusion_create(&t, getenv("TDM_DEVICE") ? atoi(getenv("TDM_DEVICE")) : 0, &handle_)   /* TDM_DEVICE: CUDA ordinal, default 0 */ != TDM_OK) die("DrFusion::DrFusion");
  dr_mesh_vert = (float*)malloc(sizeof(float) * dr_mesh_num_max * 3);  // dr_fusion.cpp:36-37
  dr_mesh_cols = (float*)malloc(sizeof(float) * dr_mesh_num_max * 3);
}

DrFusion::~DrFusion() {
  tdm_fusion_destroy(handle_);
  free(dr_mesh_vert);
  free(dr_mesh_cols);
}

void DrFusion::IntegrateScanAsync(unsigned char* bgr, float* depth, float const* pose) {
  if (tdm_fusion_integrate_async(handle_, bgr, depth, pose) != TDM_OK) die("DrFusion::IntegrateScanAsync");
}

void DrFusion::IntegrateScanAsync(DrMvsnet const& mvsnet, float const* pose) {
  if (tdm_fusion_integrate_mvsnet(handle_, mvsnet.handle(), pose) != TDM_OK) die("DrFusion::IntegrateScanAsync(DrMvsnet)");
}

void DrFusion::RenderAsync(std::vector<float const*> camera_poses) {
  if (tdm_fusion_render_async(handle_, camera_poses.data(), (int)camera_poses.size()) != TDM_OK) die("DrFusion::RenderAsync");
  n_render_ = (int)camera_poses.size();
}

void DrFusion::GetRenderResult(std::vector<unsigned char*>& bgr, std::vector<float*>& depth) {
  if (!bgr.empty() || !depth.empty()) {  // tsdf_volume.cu:710-713
    std::cerr << "GetRenderResult: output vectors must be empty on entry" << std::endl;
    exit(EXIT_FAILURE);
  }
  bgr.resize(n_render_);
  depth.resize(n_render_);
  if (tdm_fusion_get_render_result(handle_, bgr.data(), depth.data(), n_render_) != TDM_OK) die("DrFusion::GetRenderResult");
}

void DrFusion::ExtractMeshAsync(float lower_corner[3], float upper_corner[3]) {   // dr_fusion.cpp:151-153
  if (tdm_fusion_extract_mesh_async(handle_, lower_corner, upper_corner) != TDM_OK) die("DrFusion::ExtractMeshAsync");
}

void DrFusion::GetMeshSync() {   // dr_fusion.cpp:155-157: fills dr_mesh_num / dr_mesh_vert / dr_mesh_cols
  long long n = tdm_fusion_get_mesh(handle_, dr_mesh_vert, dr_mesh_cols, dr_mesh_num_max);
  if (n < 0) die("DrFusion::GetMeshSync");
  dr_mesh_num = (size_t)n;
}

struct DrMesh DrFusion::GetMesh(float lower_corner[3], float upper_corner[3]) {   // dr_fusion.cpp:95-149 (caller frees)
  DrMesh m;
  long long n = tdm_fusion_extract_mesh(handle_, lower_corner, upper_corner, nullptr, nullptr, 0);   // count, mesh stays on the device
  if (n < 0) die("DrFusion::GetMesh");
  m.num = (size_t)n;
  m.vert = (float*)malloc((m.num + 1) * 3 * sizeof(float));
  m.cols = (float*)malloc((m.num + 1) * 3 * sizeof(float));
  if (tdm_fusion_extract_mesh(handle_, lower_corner, upper_corner, m.vert, m.cols, m.num) < 0) die("DrFusion::GetMesh");
  return m;
}

void DrFusion::SaveMeshToFile(std::string const& filename, float lower_corner[3], float upper_corner[3]) {
  DrMesh m = GetMesh(lower_corner, upper_corner);  // .obj, one "v x y z r g b" line per vertex then the faces: Mesh::SaveToFile(bgr=true), mesh.cu:26-66
  std::ofstream f(filename);
  for (size_t i = 0; i < m.num; ++i)
    f << "v " << m.vert[3 * i] << " " << m.vert[3 * i + 1] << " " << m.vert[3 * i + 2] << " " << m.cols[3 * i] << " "
      << m.cols[3 * i + 1] << " " << m.cols[3 * i + 2] << "\n";
  for (size_t i = 0; i + 2 < m.num; i += 3) f << "f " << i + 1 << " " << i + 2 << " " << i + 3 << "\n";
  free(m.vert);
  free(m.cols);
}

void DrFusion::Synchronize() {
  if (tdm_fusion_synchronize(handle_) != TDM_OK) die("DrFusion::Synchronize");
}
