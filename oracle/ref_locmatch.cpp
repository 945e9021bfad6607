// oracle/ref_locmatch.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
// The reference's compiled compute_epipolar_IoU (oracle/_ref/liblimap_ref.so, ref_api.cpp) in a plain C loop over the
// (query line, target line) pairs of many items, parallel over items on all host cores: the CPU rate of the epipolar
// matcher as the reference computes it, without the Python loop around it. Built by oracle/locmatch.py.
#include <cstdint>

extern "C" double ref_compute_epipolar_IoU(const double *l1, const double *cam1, const double *l2, const double *cam2);

extern "C" void ref_locmatch_count(int64_t n_items, const int64_t *item_cams /*[n][2] rows of cams*/,
                                   const double *cams /*[][12]*/, const int64_t *line_off, const double *lines,
                                   const int64_t *item_lines /*[n][2] images of the query / target lines*/, double th,
                                   int64_t *out_counts) {
#pragma omp parallel for schedule(dynamic, 1)
  for (int64_t k = 0; k < n_items; ++k) {
    const double *c1 = cams + 12 * item_cams[2 * k], *c2 = cams + 12 * item_cams[2 * k + 1];
    const int64_t a = item_lines[2 * k], b = item_lines[2 * k + 1];
    int64_t n = 0;
    for (int64_t i = line_off[a]; i < line_off[a + 1]; ++i)
      for (int64_t j = line_off[b]; j < line_off[b + 1]; ++j)
        n += ref_compute_epipolar_IoU(lines + 4 * i, c1, lines + 4 * j, c2) > th;
    out_counts[k] = n;
  }
}
