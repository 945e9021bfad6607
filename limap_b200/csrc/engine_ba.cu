// engine_ba.cu — line refinement: the per-track bundle adjustment of the 3D lines (lm_kernels.cu) and the segments cut
// from its results.
#include "engine.cuh"
#include "lm_kernels.cuh"
#include <algorithm>

namespace {

struct V3h { double x, y, z; };
inline V3h v3(double x, double y, double z) { return V3h{x, y, z}; }
inline V3h crossh(V3h a, V3h b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// MinimalInfiniteLine3d::GetInfiniteLine (:220-231) + GetLineSegmentFromInfiniteLine3d (:265-287)
void segment_from_minimal(const double x[6], const double *l3d, int64_t n, int num_outliers, double out[6]) {
  M3h Q = quat_to_R(x);
  const V3h d = v3(Q.m[0], Q.m[3], Q.m[6]);
  const double f = std::fabs(x[5]) / std::fabs(x[4]);
  const V3h m = v3(Q.m[1] * f, Q.m[4] * f, Q.m[7] * f);
  auto point_projection = [&](V3h q) { // InfiniteLine3d::point_projection (:73-78)
    V3h dq = crossh(d, q);
    V3h mq = v3(m.x + dq.x, m.y + dq.y, m.z + dq.z);
    V3h c = crossh(d, mq);
    return v3(q.x + c.x, q.y + c.y, q.z + c.z);
  };
  const V3h pref = point_projection(v3(l3d[0], l3d[1], l3d[2]));
  std::vector<double> vals;
  vals.reserve(2 * n);
  for (int64_t k = 0; k < n; ++k)
    for (int e = 0; e < 2; ++e) {
      const double *p = l3d + 6 * k + 3 * e;
      vals.push_back((p[0] - pref.x) * d.x + (p[1] - pref.y) * d.y + (p[2] - pref.z) * d.z);
    }
  std::sort(vals.begin(), vals.end());
  const double a = vals[num_outliers], b = vals[2 * n - 1 - num_outliers];
  out[0] = pref.x + d.x * a; out[1] = pref.y + d.y * a; out[2] = pref.z + d.z * a;
  out[3] = pref.x + d.x * b; out[4] = pref.y + d.y * b; out[5] = pref.z + d.z * b;
}

} // namespace

extern "C" {

int lm_ba_solve(lm_ctx *c, int32_t n_views, const double *kvec, const double *qvec, const double *tvec, int64_t T,
                const int64_t *sup_off, const int32_t *sup_view, const double *segs, const double *line3d,
                const double *line_init, const double *sup_vp, const lm_ba_config *cfg, double *out_line,
                double *out_minimal, int32_t *out_iters, double *out_cost) {
  if (!c || !cfg || !sup_off) return fail(LM_ERR_INVALID, "NULL argument");
  if (T < 0 || n_views <= 0) return fail(LM_ERR_INVALID, "bad sizes");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const int64_t n = sup_off[T];
  for (int64_t k = 0; k < n; ++k)
    if (sup_view[k] < 0 || sup_view[k] >= n_views) return fail(LM_ERR_INVALID, "support view index out of range");
  // device input arena: [kvec | qvec | tvec | segs | x0 | sup_off | sup_view | active]
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  const size_t o_k = take(32 * n_views), o_q = take(32 * n_views), o_t = take(24 * n_views), o_s = take(32 * n),
               o_x = take(48 * T), o_so = take(8 * (T + 1)), o_sv = take(4 * n), o_a = take(T),
               o_vp = take(sup_vp ? 24 * n : 0), o_l3 = take((line3d && out_line) ? 48 * n : 0), o_li = take(48 * T),
               o_err = take(32);
  CU(c->d_ba_in.ensure(off + 256));
  char *in = c->d_ba_in.as<char>();
  CU(cudaMemcpyAsync(in + o_k, kvec, 32 * n_views, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_q, qvec, 32 * n_views, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_t, tvec, 24 * n_views, cudaMemcpyHostToDevice, s));
  if (n) CU(cudaMemcpyAsync(in + o_s, segs, 32 * n, cudaMemcpyHostToDevice, s));
  if (T) CU(cudaMemcpyAsync(in + o_li, line_init, 48 * T, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(in + o_so, sup_off, 8 * (T + 1), cudaMemcpyHostToDevice, s));
  if (n) CU(cudaMemcpyAsync(in + o_sv, sup_view, 4 * n, cudaMemcpyHostToDevice, s));
  if (sup_vp && n) CU(cudaMemcpyAsync(in + o_vp, sup_vp, 24 * n, cudaMemcpyHostToDevice, s));
  const bool dev_seg = line3d && out_line && n;
  if (dev_seg) CU(cudaMemcpyAsync(in + o_l3, line3d, 48 * n, cudaMemcpyHostToDevice, s));
  CU(c->d_ba_blocks.ensure(sizeof(lm::LMBlockDev) * std::max<int64_t>(n, 1)));
  size_t oo = 0;
  auto take_o = [&](size_t bytes) { size_t o = oo; oo += (bytes + 255) / 256 * 256; return o; };
  const size_t oo_x = take_o(48 * T), oo_i = take_o(8 * T), oo_c = take_o(16 * T), oo_t = take_o(4 * T),
               oo_s = take_o(48 * T);
  CU(c->d_ba_out.ensure(oo + 256));
  char *out = c->d_ba_out.as<char>();
  CU(cudaEventRecord(c->ev0, s));
  // per-track prologue on the device: minimal parameterisation of the start lines, constant-track flags
  lm::launch_zero_words(in + o_err, 8, s);
  lm::launch_lm_prologue(reinterpret_cast<const double *>(in + o_li), reinterpret_cast<const int64_t *>(in + o_so),
                         reinterpret_cast<const int32_t *>(in + o_sv), T, cfg->min_num_images,
                         reinterpret_cast<double *>(in + o_x), reinterpret_cast<uint8_t *>(in + o_a),
                         reinterpret_cast<int *>(in + o_err), s);
  lm::launch_lm_prepare(reinterpret_cast<const double *>(in + o_s), reinterpret_cast<const int32_t *>(in + o_sv),
                        reinterpret_cast<const double *>(in + o_k), reinterpret_cast<const double *>(in + o_q),
                        reinterpret_cast<const double *>(in + o_t),
                        (sup_vp && n) ? reinterpret_cast<const double *>(in + o_vp) : nullptr, cfg->vp_multiplier, n,
                        c->d_ba_blocks.as<lm::LMBlockDev>(), s);
  CU(cudaEventRecord(c->evk0, s));
  lm::LMParams p;
  p.blocks = c->d_ba_blocks.as<lm::LMBlockDev>();
  p.sup_off = reinterpret_cast<const int64_t *>(in + o_so);
  p.x0 = reinterpret_cast<const double *>(in + o_x);
  p.active = reinterpret_cast<const uint8_t *>(in + o_a);
  p.x_out = reinterpret_cast<double *>(out + oo_x);
  p.iters = reinterpret_cast<int32_t *>(out + oo_i);
  p.cost = reinterpret_cast<double *>(out + oo_c);
  p.term = reinterpret_cast<int32_t *>(out + oo_t);
  p.line3d = dev_seg ? reinterpret_cast<const double *>(in + o_l3) : nullptr;
  p.seg_out = dev_seg ? reinterpret_cast<double *>(out + oo_s) : nullptr;
  p.next_track = reinterpret_cast<unsigned long long *>(in + o_err + 16);
  p.num_outliers = cfg->num_outliers;
  p.T = T;
  p.geometric_alpha = cfg->geometric_alpha;
  p.cauchy_scale = cfg->cauchy_scale;
  p.max_num_iterations = cfg->max_num_iterations;
  p.max_invalid = cfg->max_num_consecutive_invalid_steps;
  lm::launch_lm_refine(p, s);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->evk1, s));
  // results land in a pinned staging area of the context (a pageable destination would serialise the copies)
  const size_t T1 = (size_t)std::max<int64_t>(T, 1);
  const size_t need_pin = T1 * (48 + 16 + 8 + 48) + 64;
  if (need_pin > c->h_ba_pin_cap) {
    if (c->h_ba_pin) cudaFreeHost(c->h_ba_pin);
    c->h_ba_pin = nullptr;
    c->h_ba_pin_cap = 0;
    CU(cudaHostAlloc(&c->h_ba_pin, need_pin + need_pin / 4, cudaHostAllocDefault));
    c->h_ba_pin_cap = need_pin + need_pin / 4;
  }
  double *xf = reinterpret_cast<double *>(c->h_ba_pin);
  double *cost = xf + 6 * T1;
  double *segd = cost + 2 * T1;
  int32_t *iters = reinterpret_cast<int32_t *>(segd + 6 * T1);
  int *h_err = reinterpret_cast<int *>(iters + 2 * T1);
  *h_err = 0;
  if (T) {
    if (dev_seg) CU(cudaMemcpyAsync(segd, out + oo_s, 48 * T, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(xf, out + oo_x, 48 * T, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(iters, out + oo_i, 8 * T, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(cost, out + oo_c, 16 * T, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(h_err, in + o_err, 4, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  if (*h_err) return fail(LM_ERR_INVALID, "track with a zero-length 3D line (CHECK_GT(line.length(), 0))");
  float ms0 = 0, ms1 = 0;
  CU(cudaEventElapsedTime(&ms0, c->ev0, c->evk0));
  CU(cudaEventElapsedTime(&ms1, c->evk0, c->evk1));
  c->stats.n_kernel_launches += 4;
  c->ba_stats.n_tracks = T;
  c->ba_stats.n_blocks = n;
  c->ba_stats.prepare_ms = ms0;
  c->ba_stats.solve_ms = ms1;
  c->ba_stats.total_iterations = c->ba_stats.total_successful = 0;
  for (int64_t t = 0; t < T; ++t) {
    c->ba_stats.total_iterations += iters[2 * t];
    c->ba_stats.total_successful += iters[2 * t + 1];
    if (out_minimal) memcpy(out_minimal + 6 * t, &xf[6 * t], 48);
    if (out_iters) { out_iters[2 * t] = iters[2 * t]; out_iters[2 * t + 1] = iters[2 * t + 1]; }
    if (out_cost) { out_cost[2 * t] = cost[2 * t]; out_cost[2 * t + 1] = cost[2 * t + 1]; }
    if (out_line && dev_seg && !std::isnan(segd[6 * t])) {
      memcpy(out_line + 6 * t, &segd[6 * t], 48); // cut on the device
    } else if (out_line) {
      const int64_t a = sup_off[t], b = sup_off[t + 1];
      if (b > a && 2 * (b - a) - 1 - cfg->num_outliers >= 0 && cfg->num_outliers < 2 * (b - a))
        segment_from_minimal(&xf[6 * t], line3d + 6 * a, b - a, cfg->num_outliers, out_line + 6 * t);
      else
        memcpy(out_line + 6 * t, line_init + 6 * t, 48);
    }
  }
  return LM_OK;
}

int lm_ba_get_stats(lm_ctx *c, lm_ba_stats *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  *out = c->ba_stats;
  return LM_OK;
}

} // extern "C"
