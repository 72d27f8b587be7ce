// Drop-in replacement header for tandem/libdr/dr_fusion/src/dr_fusion/dr_fusion.h (:18-73) implemented over the
// tandem_b200 C ABI.  Callers: FullSystem.cpp:259-281, tandem_backend.cpp:166-200, main_tandem_pangolin.cpp:296-300.
#ifndef DR_FUSION_DR_FUSION_H
#define DR_FUSION_DR_FUSION_H

#include <cstddef>
#include <memory>
#include <string>
#include <vector>

struct tdm_fusion;  // include/tandem_b200.h
class DrMvsnet;     // include/dr_mvsnet/dr_mvsnet.h

struct DrFusionOptions {
    float voxel_size;
    int num_buckets;
    int bucket_size;
    int num_blocks;
    int block_size;
    int max_sdf_weight;
    float truncation_distance;
    float max_sensor_depth;
    float min_sensor_depth;
    int num_render_streams;

    float fx;
    float fy;
    float cx;
    float cy;
    int height;
    int width;
};

struct DrMesh {
    size_t num = 0;
    float* vert = nullptr;
    float* cols = nullptr;
};

class DrFusion {
public:
    DrFusion(struct DrFusionOptions const &options);

    ~DrFusion();

    void IntegrateScanAsync(unsigned char *bgr, float *depth, float const *pose);

    // Extension: integrates the result mvsnet.GetResult() last returned where it sits on the device - its depth, the
    // window's reference BGR image and (pose == nullptr) reference cam_to_world, i.e. what tandem_backend.cpp:166 passes -
    // with no host round trip.  Legal until the next GetResult, also after the next CallAsync (tdm_fusion_integrate_mvsnet).
    void IntegrateScanAsync(DrMvsnet const &mvsnet, float const *pose = nullptr);

    void RenderAsync(std::vector<float const *> camera_poses);

    void GetRenderResult(std::vector<unsigned char *> &bgr, std::vector<float *> &depth);

    void SaveMeshToFile(std::string const& filename,  float lower_corner[3], float upper_corner[3]);

    struct DrMesh GetMesh(float lower_corner[3], float upper_corner[3]);

    void ExtractMeshAsync(float lower_corner[3], float upper_corner[3]);
    void GetMeshSync();

    void Synchronize();

    // Extension: the C-ABI handle, so that CudaCoarseTracker::setReferenceDense can read the rendered depth on the device.
    tdm_fusion* handle() const { return handle_; }

    size_t dr_mesh_num = 0;
    const size_t dr_mesh_num_max = 60000000;
    float* dr_mesh_vert;
    float* dr_mesh_cols;

private:
    tdm_fusion* handle_;
    int n_render_ = 0;
};

#endif  // DR_FUSION_DR_FUSION_H
