// engine_vp.cu — vanishing points: J-Linkage clustering on the device (vp_kernels.cu), cluster filtering and the VP fit
// of every cluster on the host.
#include "engine.cuh"
#include "vp_kernels.cuh"
#include <algorithm>
#include <array>

namespace {

struct L2h { double x1, y1, x2, y2; };
inline double len_h(const L2h &l) { return std::sqrt((l.x1 - l.x2) * (l.x1 - l.x2) + (l.y1 - l.y2) * (l.y1 - l.y2)); }
// Line2d::coords (base/linebase.cc:35-39)
inline void coords_h(const L2h &l, double c[3]) {
  c[0] = l.y1 - l.y2; c[1] = l.x2 - l.x1; c[2] = l.x1 * l.y2 - l.x2 * l.y1;
  const double n2 = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
  if (n2 > 0) { const double n = std::sqrt(n2); c[0] /= n; c[1] /= n; c[2] /= n; }
}
// BaseVPDetector::count_valid_supports_2d (vplib/base_vp_detector.cc:41-73)
int count_valid_supports_2d_h(const std::vector<L2h> &lines, double th_perp) {
  const size_t n = lines.size();
  std::vector<int> parent(n, -1);
  auto root = [&](size_t i) { while (parent[i] != -1) i = parent[i]; return i; };
  auto dist = [&](const L2h &l, double qx, double qy) {
    double c[3];
    coords_h(l, c);
    return std::fabs(c[0] * qx + c[1] * qy + c[2]) / std::sqrt(c[0] * c[0] + c[1] * c[1]);
  };
  for (size_t i = 0; i + 1 < n; ++i) {
    const size_t ri = root(i);
    for (size_t j = i + 1; j < n; ++j) {
      const size_t rj = root(j);
      if (rj == ri) continue;
      size_t k1 = i, k2 = j;
      if (len_h(lines[i]) > len_h(lines[j])) { k1 = j; k2 = i; }
      const double ds = dist(lines[k2], lines[k1].x1, lines[k1].y1), de = dist(lines[k2], lines[k1].x2, lines[k1].y2);
      if (((ds < de) ? de : ds) > th_perp) continue;
      parent[rj] = (int)ri;
    }
  }
  int cnt = 0;
  for (size_t i = 0; i < n; ++i) cnt += parent[i] == -1;
  return cnt;
}
// JLinkage::fitVP (JLinkage.cc:86-100): right singular vector of the smallest singular value
void smallest_eigvec(const double A[3][3], double out[3]) {
  double V[3][3], ev[3];
  jacobi3(A, V, ev);
  int best = 0;
  if (ev[1] < ev[best]) best = 1;
  if (ev[2] < ev[best]) best = 2;
  double n = std::sqrt(V[0][best] * V[0][best] + V[1][best] * V[1][best] + V[2][best] * V[2][best]);
  for (int k = 0; k < 3; ++k) out[k] = V[k][best] / n;
}

} // namespace

extern "C" {

int64_t lm_vp_detect(lm_ctx *c, int32_t n_images, const int64_t *line_off, const double *segs, const lm_vp_config *cfg,
                     int32_t *labels, int64_t *vp_off, double *vps, int64_t vp_cap) {
  return lm_vp_detect_indexed(c, n_images, line_off, segs, cfg, nullptr, labels, vp_off, vps, vp_cap);
}
int lm_vp_get_stats(lm_ctx *c, lm_vp_stats *out) {
  if (!c || !out) return fail(LM_ERR_INVALID, "NULL argument");
  *out = c->vp_stats;
  return LM_OK;
}
int64_t lm_vp_detect_indexed(lm_ctx *c, int32_t n_images, const int64_t *line_off, const double *segs,
                             const lm_vp_config *cfg, const int64_t *image_index, int32_t *labels, int64_t *vp_off,
                             double *vps, int64_t vp_cap) {
  if (!c || !cfg || !line_off || !labels || !vp_off) return fail(LM_ERR_INVALID, "NULL argument");
  if (n_images < 0) return fail(LM_ERR_INVALID, "bad sizes");
  if (cfg->n_models <= 0 || cfg->n_models > 65535) return fail(LM_ERR_INVALID, "n_models must be in [1, 65535]");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  // ComputeVPLabels :17-36: segments of at least min_length px, cast to float
  std::vector<float> pts;
  std::vector<int64_t> valid_off(n_images + 1, 0);
  std::vector<int32_t> valid_ids;
  int max_n = 0;
  for (int im = 0; im < n_images; ++im) {
    for (int64_t l = line_off[im]; l < line_off[im + 1]; ++l) {
      const double *g = segs + 4 * l;
      const double len = std::sqrt((g[0] - g[2]) * (g[0] - g[2]) + (g[1] - g[3]) * (g[1] - g[3]));
      if (len < cfg->min_length) continue;
      valid_ids.push_back((int32_t)(l - line_off[im]));
      for (int k = 0; k < 4; ++k) pts.push_back((float)g[k]);
    }
    valid_off[im + 1] = (int64_t)valid_ids.size();
    max_n = std::max(max_n, (int)(valid_off[im + 1] - valid_off[im]));
  }
  if (max_n > 8192) return fail(LM_ERR_INVALID, "more than 8192 segments of min_length in one image");
  const int64_t nv = (int64_t)valid_ids.size();
  std::vector<int32_t> raw(std::max<int64_t>(nv, 1), -1), ncl(std::max(n_images, 1), 0);
  const int min_lines = 2 * std::max(cfg->min_num_supports, 10);
  bool vp_kernel_ran = false;
  if (nv > 0 && max_n >= min_lines) {
    const int W = (cfg->n_models + 31) / 32;
    int grid = std::min(n_images, c->sm_count * 2);
    CU(c->d_vp_pts.ensure(16 * nv));
    CU(c->d_vp_off.ensure(8 * (n_images + 1)));
    CU(c->d_vp_labels.ensure(4 * nv));
    CU(c->d_vp_nc.ensure(4 * n_images));
    CU(c->d_vp_ps.ensure((size_t)grid * max_n * W * 4));
    CU(c->d_vp_mat.ensure((size_t)grid * max_n * max_n * 4));
    CU(c->d_vp_idx.ensure(8 * std::max(n_images, 1)));
    CU(cudaMemcpyAsync(c->d_vp_pts.p, pts.data(), 16 * nv, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(c->d_vp_off.p, valid_off.data(), 8 * (n_images + 1), cudaMemcpyHostToDevice, s));
    if (image_index) CU(cudaMemcpyAsync(c->d_vp_idx.p, image_index, 8 * n_images, cudaMemcpyHostToDevice, s));
    lm::VPParams p;
    p.pts = c->d_vp_pts.as<float4>();
    p.valid_off = c->d_vp_off.as<int64_t>();
    p.image_index = image_index ? c->d_vp_idx.as<int64_t>() : nullptr;
    p.labels = c->d_vp_labels.as<int32_t>();
    p.n_clusters = c->d_vp_nc.as<int32_t>();
    p.ps_slab = c->d_vp_ps.as<uint32_t>();
    p.mat_slab = c->d_vp_mat.as<uint32_t>();
    p.n_images = n_images; p.n_models = cfg->n_models; p.max_n = max_n; p.min_lines = min_lines;
    p.inlier_threshold = (float)cfg->inlier_threshold;
    p.seed = cfg->seed;
    if (lm::vp_smem_bytes(p.n_models, p.max_n) > (size_t)c->max_smem_optin)
      return fail(LM_ERR_INVALID, "n_models too large for shared memory");
    CU(cudaEventRecord(c->evk0, s));
    lm::launch_jlinkage(p, grid, s);
    CU(cudaEventRecord(c->evk1, s));
    CU(cudaGetLastError());
    vp_kernel_ran = true;
    c->stats.n_kernel_launches += 1;
    CU(cudaMemcpyAsync(raw.data(), c->d_vp_labels.p, 4 * nv, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(ncl.data(), c->d_vp_nc.p, 4 * n_images, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
  }
  // JLinkage.cc:56-83 (cluster filtering) and AssociateVPs :102-127 (VP fitting), per image on the host
  int64_t n_vps = 0;
  for (int im = 0; im < n_images; ++im) {
    vp_off[im] = n_vps;
    const int64_t L = line_off[im + 1] - line_off[im];
    int32_t *lab = labels + line_off[im];
    for (int64_t l = 0; l < L; ++l) lab[l] = -1;
    const int64_t v0 = valid_off[im], v1 = valid_off[im + 1];
    const int nc = ncl[im];
    if (nc <= 0 || v1 - v0 < min_lines) continue;
    std::vector<std::vector<L2h>> sup(nc);
    for (int64_t k = v0; k < v1; ++k) {
      if (raw[k] < 0) continue;
      const double *g = segs + 4 * (line_off[im] + valid_ids[k]);
      sup[raw[k]].push_back(L2h{g[0], g[1], g[2], g[3]});
    }
    std::vector<int> vp_ids(nc, -1);
    int counter = 0;
    for (int q = 0; q < nc; ++q) {
      if ((int)sup[q].size() < cfg->min_num_supports) continue;
      if (count_valid_supports_2d_h(sup[q], cfg->th_perp_supports) < cfg->min_num_supports) continue;
      vp_ids[q] = counter++;
    }
    std::vector<std::array<double, 9>> S(counter, std::array<double, 9>{});
    for (int64_t k = v0; k < v1; ++k) {
      if (raw[k] < 0 || vp_ids[raw[k]] < 0) continue;
      const int v = vp_ids[raw[k]];
      lab[valid_ids[k]] = v;
      const double *g = segs + 4 * (line_off[im] + valid_ids[k]);
      double cc[3];
      coords_h(L2h{g[0], g[1], g[2], g[3]}, cc);
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) S[v][3 * a + b] += cc[a] * cc[b];
    }
    for (int v = 0; v < counter; ++v) {
      double A[3][3], e[3];
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) A[a][b] = S[v][3 * a + b];
      smallest_eigvec(A, e);
      if (vps && n_vps < vp_cap) { vps[3 * n_vps] = e[0]; vps[3 * n_vps + 1] = e[1]; vps[3 * n_vps + 2] = e[2]; }
      ++n_vps;
    }
  }
  vp_off[n_images] = n_vps;
  c->vp_stats.n_images = n_images;
  c->vp_stats.n_segments = nv;
  c->vp_stats.n_vps = n_vps;
  c->vp_stats.kernel_ms = 0;
  if (vp_kernel_ran) { float ms = 0; CU(cudaEventElapsedTime(&ms, c->evk0, c->evk1)); c->vp_stats.kernel_ms = ms; }
  return n_vps;
}

} // extern "C"
