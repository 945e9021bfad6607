// engine_sfm.cu — visual-neighbour ranking and robust ranges from a sparse point model (SURVEY.md 8 f4)
#include "engine.cuh"
#include "sfm_kernels.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>

extern "C" {

int lm_sfm_rank_neighbors(lm_ctx *c, int32_t n_images, const double *centres, int64_t n_points, const double *xyz,
                          const int64_t *track_off, const int32_t *track_img, int32_t num_images,
                          double min_triangulation_angle_deg, int32_t mode, int32_t *out_neighbors, int32_t *out_count) {
  if (!c || !centres || !track_off || !out_neighbors || !out_count) return fail(LM_ERR_INVALID, "NULL argument");
  if (n_images <= 0 || n_images > 65535 || n_points < 0 || num_images <= 0 || mode < 0 || mode > 2)
    return fail(LM_ERR_INVALID, "bad sizes");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const int64_t n_ent = track_off[n_points];
  for (int64_t e = 0; e < n_ent; ++e)
    if (track_img[e] < 0 || track_img[e] >= n_images) return fail(LM_ERR_INVALID, "track image index out of range");
  // records per point: pairs of its track entries
  std::vector<int64_t> rec_off(n_points + 1, 0);
  for (int64_t p = 0; p < n_points; ++p) {
    const int64_t t = track_off[p + 1] - track_off[p];
    rec_off[p + 1] = rec_off[p] + t * (t - 1) / 2;
  }
  const int64_t n_rec = rec_off[n_points];
  if (n_rec >= ((int64_t)1 << 31) - 64) return fail(LM_ERR_INVALID, "more than 2^31 (point, image pair) records");
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  const size_t o_c = take(24 * (size_t)n_images), o_x = take(24 * (size_t)std::max<int64_t>(n_points, 1)),
               o_to = take(8 * (size_t)(n_points + 1)), o_ti = take(4 * (size_t)std::max<int64_t>(n_ent, 1)),
               o_ro = take(8 * (size_t)(n_points + 1)), o_np = take(4 * (size_t)n_images), o_sc = take(64),
               o_out = take(4 * (size_t)n_images * num_images), o_cnt = take(4 * (size_t)n_images);
  CU(c->d_sfm_in.ensure(off + 256));
  char *in = c->d_sfm_in.as<char>();
  CU(cudaMemcpyAsync(in + o_c, centres, 24 * (size_t)n_images, cudaMemcpyHostToDevice, s));
  if (n_points) CU(cudaMemcpyAsync(in + o_x, xyz, 24 * (size_t)n_points, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_to, track_off, 8 * (size_t)(n_points + 1), cudaMemcpyHostToDevice, s));
  if (n_ent) CU(cudaMemcpyAsync(in + o_ti, track_img, 4 * (size_t)n_ent, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_ro, rec_off.data(), 8 * (size_t)(n_points + 1), cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(in + o_np, 0, 4 * (size_t)n_images, s));
  CU(cudaMemsetAsync(in + o_sc, 0, 64, s));
  unsigned int *d_np = reinterpret_cast<unsigned int *>(in + o_np);
  unsigned int *d_ndir = reinterpret_cast<unsigned int *>(in + o_sc);
  int *d_nruns = reinterpret_cast<int *>(in + o_sc + 16);
  int64_t n_dir = 0;
  if (n_rec > 0) {
    // (a pair seen once yields two directed records: the scratch is sized for 2 n_rec)
    CU(c->d_sfm_keys.ensure(16 * (size_t)n_rec));
    CU(c->d_sfm_keys2.ensure(16 * (size_t)n_rec));
    lm::launch_sfm_pair_keys(reinterpret_cast<const double *>(in + o_c), reinterpret_cast<const double *>(in + o_x),
                             reinterpret_cast<const int64_t *>(in + o_to), reinterpret_cast<const int32_t *>(in + o_ti),
                             reinterpret_cast<const int64_t *>(in + o_ro), n_points, n_rec,
                             c->d_sfm_keys.as<unsigned long long>(), d_np, s);
    cub::DoubleBuffer<unsigned long long> dk(c->d_sfm_keys.as<unsigned long long>(), c->d_sfm_keys2.as<unsigned long long>());
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortKeys(t, b, dk, (int)n_rec, 0, 64, s); }));
    const unsigned long long *sorted = dk.Current();
    // runs of equal image pairs: ids -> run-length encode -> starts
    CU(c->d_sfm_a.ensure(8 * (size_t)n_rec));       // pair ids, later the directed records
    CU(c->d_sfm_b.ensure(8 * (size_t)n_rec + 16));  // unique pairs, later the sort's alternate buffer
    CU(c->d_sfm_c.ensure(4 * (size_t)n_rec + 16));  // run lengths
    CU(c->d_sfm_d.ensure(4 * (size_t)n_rec + 16));  // run starts
    lm::launch_sfm_pair_ids(sorted, n_rec, c->d_sfm_a.as<unsigned int>(), s);
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) {
      return cub::DeviceRunLengthEncode::Encode(t, b, c->d_sfm_a.as<unsigned int>(), c->d_sfm_b.as<unsigned int>(),
                                                c->d_sfm_c.as<unsigned int>(), d_nruns, (int)n_rec, s);
    }));
    int n_runs = 0;
    CU(cudaMemcpyAsync(&n_runs, d_nruns, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) {
      return cub::DeviceScan::ExclusiveSum(t, b, c->d_sfm_c.as<unsigned int>(), c->d_sfm_d.as<unsigned int>(), n_runs, s);
    }));
    // directed (source, destination) records of the pairs that pass the angle test; the sorted keys are dead afterwards,
    // so their buffers carry the records: values in d_sfm_a (reused), keys in the alternate key buffer
    unsigned int *dir_val = c->d_sfm_a.as<unsigned int>();
    unsigned long long *dir_key = dk.Alternate();
    const float min_angle = (float)(min_triangulation_angle_deg * 3.14159265358979323846 / 180.0);
    lm::launch_sfm_scores(sorted, c->d_sfm_b.as<unsigned int>(), c->d_sfm_c.as<unsigned int>(), c->d_sfm_d.as<unsigned int>(),
                          n_runs, d_np, min_angle, mode, dir_val, dir_key, d_ndir, s);
    unsigned int h_ndir = 0;
    CU(cudaMemcpyAsync(&h_ndir, d_ndir, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    n_dir = h_ndir;
    if (n_dir > 0) {
      // order: source ascending, score descending, destination ascending = three stable radix sorts, least significant first
      unsigned int *val2 = c->d_sfm_b.as<unsigned int>();
      unsigned long long *key2 = const_cast<unsigned long long *>(sorted); // the sorted pair keys are dead now
      {
        cub::DoubleBuffer<unsigned int> k(dir_val, val2);
        cub::DoubleBuffer<unsigned long long> v(dir_key, key2);
        // by (source, destination)
        CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, k, v, (int)n_dir, 0, 32, s); }));
        cub::DoubleBuffer<unsigned long long> k2(v.Current(), v.Alternate());
        cub::DoubleBuffer<unsigned int> v2(k.Current(), k.Alternate());
        // by score, descending
        CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, k2, v2, (int)n_dir, 0, 64, s); }));
        cub::DoubleBuffer<unsigned int> k3(v2.Current(), v2.Alternate());
        // by source (stable)
        CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortKeys(t, b, k3, (int)n_dir, 16, 32, s); }));
        dir_val = k3.Current();
      }
    }
    lm::launch_sfm_take(dir_val, n_dir, n_images, num_images, reinterpret_cast<int32_t *>(in + o_out),
                        reinterpret_cast<int32_t *>(in + o_cnt), s);
  } else {
    lm::launch_sfm_take(nullptr, 0, n_images, num_images, reinterpret_cast<int32_t *>(in + o_out),
                        reinterpret_cast<int32_t *>(in + o_cnt), s);
  }
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out_neighbors, in + o_out, 4 * (size_t)n_images * num_images, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(out_count, in + o_cnt, 4 * (size_t)n_images, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  c->stats.n_kernel_launches += 12;
  return LM_OK;
}

int lm_sfm_robust_ranges(lm_ctx *c, int64_t n_points, const double *xyz, double q_lo, double q_hi, double kstretch,
                         double out[6]) {
  if (!c || !xyz || !out) return fail(LM_ERR_INVALID, "NULL argument");
  if (n_points <= 0 || n_points >= ((int64_t)1 << 31) - 64) return fail(LM_ERR_INVALID, "bad point count");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  // SfmModel::ComputeRanges keeps the coordinates as float (sfm_model.cc:245-252): one float column per axis, sorted
  std::vector<float> col((size_t)n_points);
  CU(c->d_sfm_a.ensure(4 * (size_t)n_points));
  CU(c->d_sfm_b.ensure(4 * (size_t)n_points));
  for (int ax = 0; ax < 3; ++ax) {
    for (int64_t p = 0; p < n_points; ++p) col[p] = (float)xyz[3 * p + ax];
    CU(cudaMemcpyAsync(c->d_sfm_a.p, col.data(), 4 * (size_t)n_points, cudaMemcpyHostToDevice, s));
    cub::DoubleBuffer<float> dk(c->d_sfm_a.as<float>(), c->d_sfm_b.as<float>());
    CU(cub_call(c->d_sort_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortKeys(t, b, dk, (int)n_points, 0, 32, s); }));
    const float kmin = (float)q_lo, kmax = (float)q_hi;
    const size_t i_lo = (size_t)((float)n_points * kmin), i_hi = (size_t)((float)n_points * kmax); // data[data.size() * k]
    float lo = 0, hi = 0;
    CU(cudaMemcpyAsync(&lo, dk.Current() + std::min<size_t>(i_lo, n_points - 1), 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&hi, dk.Current() + std::min<size_t>(i_hi, n_points - 1), 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    const float ks = (float)kstretch, diff = hi - lo;
    lo -= ks * diff;
    hi += ks * diff;
    out[ax] = lo;
    out[3 + ax] = hi;
  }
  c->stats.n_kernel_launches += 12;
  return LM_OK;
}

} // extern "C"
