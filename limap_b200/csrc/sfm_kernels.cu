// sfm_kernels.cu — see sfm_kernels.cuh. Integer/sort-bound: the only arithmetic is one triangulation angle per
// (point, image pair); everything else is keys for CUB radix sorts and run-length encoding (plumbing).
#include "sfm_kernels.cuh"

namespace lm {

__global__ void sfm_pair_keys_kernel(const double *__restrict__ centres, const double *__restrict__ xyz,
                                     const int64_t *__restrict__ track_off, const int32_t *__restrict__ track_img,
                                     const int64_t *__restrict__ rec_off, int64_t n_points, int64_t n_rec,
                                     unsigned long long *__restrict__ keys, unsigned int *__restrict__ num_points) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rec; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = last_le(rec_off, n_points, r);
    const int64_t k = r - rec_off[p]; // pair index in the track: (a, b), a > b, k = a (a - 1) / 2 + b
    int64_t a = (int64_t)((1.0 + sqrt(1.0 + 8.0 * (double)k)) * 0.5);
    while (a * (a - 1) / 2 > k) --a;
    while ((a + 1) * a / 2 <= k) ++a;
    const int64_t b = k - a * (a - 1) / 2;
    const int i = track_img[track_off[p] + a], j = track_img[track_off[p] + b];
    unsigned long long key = ~0ull; // same image twice in one track: no pair (sorted to the end, ignored)
    if (i != j) {
      const double *X = xyz + 3 * p, *c1 = centres + 3 * (int64_t)i, *c2 = centres + 3 * (int64_t)j;
      double bl2 = 0, r1 = 0, r2 = 0;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        bl2 += (c1[q] - c2[q]) * (c1[q] - c2[q]);
        r1 += (X[q] - c1[q]) * (X[q] - c1[q]);
        r2 += (X[q] - c2[q]) * (X[q] - c2[q]);
      }
      const double denom = 2.0 * sqrt(r1 * r2);
      double angle = 0.0;
      if (denom != 0.0) {
        angle = fabs(acos((r1 + r2 - bl2) / denom));
        angle = fmin(angle, 3.14159265358979323846 - angle);
      }
      const float af = (float)angle; // COLMAP keeps the angles as float
      const unsigned int lo_img = (unsigned int)min(i, j), hi_img = (unsigned int)max(i, j);
      key = ((unsigned long long)((lo_img << 16) | hi_img) << 32) | (unsigned long long)__float_as_uint(af);
    }
    keys[r] = key;
  }
  // points per image (SfmModel::ComputeNumPoints): one thread per track entry
  const int64_t n_ent = track_off[n_points];
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n_ent; e += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(&num_points[track_img[e]], 1u);
}

__global__ void sfm_pair_ids_kernel(const unsigned long long *__restrict__ keys, int64_t n_rec, unsigned int *__restrict__ ids) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r < n_rec) ids[r] = (unsigned int)(keys[r] >> 32);
}

__global__ void sfm_scores_kernel(const unsigned long long *__restrict__ keys, const unsigned int *__restrict__ run_pair,
                                  const unsigned int *__restrict__ run_len, const unsigned int *__restrict__ run_start,
                                  int n_runs, const unsigned int *__restrict__ num_points, float min_angle_rad, int mode,
                                  unsigned int *__restrict__ dir_val, unsigned long long *__restrict__ dir_key,
                                  unsigned int *__restrict__ n_dir) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_runs) return;
  const unsigned int pair = run_pair[r];
  if (pair == 0xffffffffu) return; // the ignored records
  const unsigned int n = run_len[r], st = run_start[r];
  // Percentile(angles, 75): element round(0.75 (n - 1)) of the sorted angles (the records are sorted by angle)
  const unsigned int idx = (unsigned int)llround(75.0 / 100.0 * (double)(n - 1));
  const float perc = __uint_as_float((unsigned int)(keys[st + idx] & 0xffffffffull));
  if (!(perc >= min_angle_rad)) return;
  const unsigned int i = pair >> 16, j = pair & 0xffffu;
  const int inter = (int)n, uni = (int)num_points[i] + (int)num_points[j] - inter;
  double score;
  if (mode == 0) score = (double)inter / (double)uni;                    // IoU (sfm_model.cc:130-133)
  else if (mode == 1) score = (double)(2 * inter) / (double)(uni + inter); // Dice (:196-198)
  else score = (double)inter;                                             // shared points (COLMAP GetMaxOverlappingImages)
  // descending score = ascending key; scores are positive doubles, so their bit patterns order like the values
  const unsigned long long k = ~(unsigned long long)__double_as_longlong(score);
  const unsigned int o = atomicAdd(n_dir, 2u);
  dir_val[o] = (i << 16) | j; dir_key[o] = k;
  dir_val[o + 1] = (j << 16) | i; dir_key[o + 1] = k;
}

__global__ void sfm_take_kernel(const unsigned int *__restrict__ dir_val, int64_t n_dir, int n_images, int num_images,
                                int32_t *__restrict__ out_neighbors, int32_t *__restrict__ out_count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_images) return;
  int64_t lo = 0, hi = n_dir; // first record of source image i
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((dir_val[mid] >> 16) < (unsigned int)i) lo = mid + 1; else hi = mid;
  }
  int n = 0;
  for (int64_t r = lo; r < n_dir && n < num_images && (dir_val[r] >> 16) == (unsigned int)i; ++r)
    out_neighbors[(int64_t)i * num_images + n++] = (int32_t)(dir_val[r] & 0xffffu);
  out_count[i] = n;
  for (int k = n; k < num_images; ++k) out_neighbors[(int64_t)i * num_images + k] = -1;
}

void launch_sfm_pair_keys(const double *centres, const double *xyz, const int64_t *track_off, const int32_t *track_img,
                          const int64_t *rec_off, int64_t n_points, int64_t n_rec, unsigned long long *keys,
                          unsigned int *num_points, cudaStream_t s) {
  sfm_pair_keys_kernel<<<current_device_sms() * 8, 256, 0, s>>>(centres, xyz, track_off, track_img, rec_off, n_points, n_rec, keys, num_points);
}
void launch_sfm_pair_ids(const unsigned long long *keys, int64_t n_rec, unsigned int *pair_ids, cudaStream_t s) {
  if (n_rec <= 0) return;
  sfm_pair_ids_kernel<<<(int)((n_rec + 255) / 256), 256, 0, s>>>(keys, n_rec, pair_ids);
}
void launch_sfm_scores(const unsigned long long *keys, const unsigned int *run_pair, const unsigned int *run_len,
                       const unsigned int *run_start, int n_runs, const unsigned int *num_points, float min_angle_rad,
                       int mode, unsigned int *dir_val, unsigned long long *dir_key, unsigned int *n_dir, cudaStream_t s) {
  if (n_runs <= 0) return;
  sfm_scores_kernel<<<(n_runs + 255) / 256, 256, 0, s>>>(keys, run_pair, run_len, run_start, n_runs, num_points,
                                                          min_angle_rad, mode, dir_val, dir_key, n_dir);
}
void launch_sfm_take(const unsigned int *dir_val, int64_t n_dir, int n_images, int num_images, int32_t *out_neighbors,
                     int32_t *out_count, cudaStream_t s) {
  sfm_take_kernel<<<(n_images + 127) / 128, 128, 0, s>>>(dir_val, n_dir, n_images, num_images, out_neighbors, out_count);
}

} // namespace lm
