// vp_kernels.cuh — device layout of the J-Linkage VP clustering (see vp_kernels.cu).
#pragma once
#include "lm_math.cuh"

namespace lm {

struct VPParams {
  const float4 *pts;        // [sum n] valid segments (x1,y1,x2,y2) as float
  const int64_t *valid_off; // [n_images+1]
  const int64_t *image_index; // [n_images] index seeding the hypotheses of each image, or NULL (= position in the call)
  int32_t *labels;          // [sum n] out: raw cluster id of every valid segment
  int32_t *n_clusters;      // [n_images] out
  uint32_t *ps_slab;        // [grid][max_n][W] preference bit matrices
  uint32_t *mat_slab;       // [grid][max_n][max_n] cached (intersection << 16 | union)
  int n_images, n_models, max_n, min_lines;
  float inlier_threshold;
  uint64_t seed;
};

// Dynamic shared memory of one launch. The kernel's static shared memory (vp_static_smem_bytes) comes on top, and the
// two together must fit the per-block opt-in limit, and above 48 KB together the launch needs the opt-in attribute.
size_t vp_smem_bytes(int n_models, int max_n);
cudaError_t vp_static_smem_bytes(size_t *out);
cudaError_t launch_jlinkage(const VPParams &p, int grid, size_t static_smem, cudaStream_t s);

} // namespace lm
