// locmatch_kernels.cu — sm_90a kernels of the localization line matching (locmatch_kernels.cuh), fp64 throughout.
//
// Every output list is written in the reference's order by a count, an exclusive scan and a placement: the order of an
// entry never depends on the order in which threads finish.
#include "locmatch_kernels.cuh"
#include <math_constants.h>

namespace lm {

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kPlaceThreads = 256;

LM_D unsigned lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }

// CameraView::projection (base/camera_view.cc:61-65): dehomogeneous(K (R X + T)) with the EPS of util/types.h:40-42,
// every product and sum rounded on its own, in Eigen's order
LM_D vec2<double> project(const LocView &v, const double *X) {
  double pc[3];
  for (int i = 0; i < 3; ++i)
    pc[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(v.R[3 * i], X[0]), __dmul_rn(v.R[3 * i + 1], X[1])),
                                __dmul_rn(v.R[3 * i + 2], X[2])),
                      v.t[i]);
  const double hx = __dadd_rn(__dmul_rn(v.k[0], pc[0]), __dmul_rn(v.k[2], pc[2]));
  const double hy = __dadd_rn(__dmul_rn(v.k[1], pc[1]), __dmul_rn(v.k[3], pc[2]));
  const double d = __dadd_rn(pc[2], consts<double>::eps());
  return mk2(__ddiv_rn(hx, d), __ddiv_rn(hy, d));
}
// Line2d::length / direction (base/linebase.h:24-26): Eigen norm() and normalized()
LM_D double sq2(double x, double y) { return __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)); }
LM_D double seg_length(vec2<double> s, vec2<double> e) { return __dsqrt_rn(sq2(__dsub_rn(s.x, e.x), __dsub_rn(s.y, e.y))); }
LM_D vec2<double> seg_direction(vec2<double> s, vec2<double> e) {
  const double x = __dsub_rn(e.x, s.x), y = __dsub_rn(e.y, s.y);
  const double n2 = sq2(x, y);
  if (!(n2 > 0)) return mk2(x, y);
  const double n = __dsqrt_rn(n2);
  return mk2(__ddiv_rn(x, n), __ddiv_rn(y, n));
}
LM_D vec2<double> midpoint(vec2<double> s, vec2<double> e) {
  return mk2(__dmul_rn(0.5, __dadd_rn(s.x, e.x)), __dmul_rn(0.5, __dadd_rn(s.y, e.y)));
}
// np.cross of two 2-vectors
LM_D double cross2(vec2<double> a, vec2<double> b) { return __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x)); }

} // namespace

// ---- epipolar sweep ----------------------------------------------------------------------------------------------
struct RowCtx {
  int64_t item, ql, tbase;
  int nt;
  int2 it;
};
LM_D RowCtx row_ctx(const LocScene &s, const LocItems &it, int64_t r) {
  RowCtx c;
  c.item = last_le<true>(it.row_off, it.n_items, r);
  c.ql = r - __ldg(&it.row_off[c.item]);
  c.it = it.items[c.item];
  c.tbase = __ldg(&s.line_off[c.it.y]);
  c.nt = (int)(__ldg(&s.line_off[c.it.y + 1]) - c.tbase);
  return c;
}

__global__ void __launch_bounds__(32 * kWarpsPerBlock)
    sweep_count_kernel(const LocScene s, const LocItems it, const int64_t *__restrict__ word_off, double th,
                       int to_tracks, uint32_t *__restrict__ mask, int64_t *__restrict__ cnt,
                       unsigned long long *n_2to2) {
  const int lane = threadIdx.x & 31;
  const int64_t n_rows = it.row_off[it.n_items];
  const int64_t nw = (int64_t)gridDim.x * kWarpsPerBlock;
  for (int64_t r = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); r < n_rows; r += nw) {
    const RowCtx c = row_ctx(s, it, r);
    const LocView &vq = s.views[c.it.x];
    const LocView &vt = s.views[c.it.y];
    // the per-query-line terms: back-projected endpoints and the camera centres' baseline
    const double4 l1 = s.lines[__ldg(&s.line_off[c.it.x]) + c.ql];
    const vec3<double> w1s = mat3_mul_h(vq.M, l1.x, l1.y), w1e = mat3_mul_h(vq.M, l1.z, l1.w);
    const vec3<double> base = mk3(vq.C[0], vq.C[1], vq.C[2]) - mk3(vt.C[0], vt.C[1], vt.C[2]);
    const EpipolarLines ep(vt.M, base, w1s, w1e); // the endpoints' epipolar lines in the target view
    const int words = (c.nt + 31) >> 5;
    uint32_t *mrow = mask + __ldg(&word_off[c.item]) + c.ql * words;
    int64_t n_out = 0, n_pairs = 0;
    for (int w = 0; w < words; ++w) {
      const int j = (w << 5) + lane;
      bool hit = false, out = false;
      if (j < c.nt) {
        // accepted on IoU > th: NaN never matches, IoU == th does not match
        hit = epipolar_iou(ep, s.lines[c.tbase + j], th) > th;
        out = hit && (!to_tracks || __ldg(&s.line_track[c.tbase + j]) != -1);
      }
      const unsigned bo = __ballot_sync(0xffffffffu, out);
      n_pairs += __popc(__ballot_sync(0xffffffffu, hit));
      n_out += __popc(bo);
      if (lane == 0) mrow[w] = bo;
    }
    if (lane == 0) {
      cnt[r] = n_out;
      if (n_pairs) atomicAdd(n_2to2, (unsigned long long)n_pairs);
    }
  }
}
void launch_locmatch_sweep_count(const LocScene &s, const LocItems &it, const int64_t *word_off, double th,
                                 int to_tracks, uint32_t *mask, int64_t *cnt, unsigned long long *n_2to2,
                                 cudaStream_t st) {
  sweep_count_kernel<<<current_device_sms() * 8, 32 * kWarpsPerBlock, 0, st>>>(s, it, word_off, th, to_tracks, mask,
                                                                                cnt, n_2to2);
}

__global__ void __launch_bounds__(32 * kWarpsPerBlock)
    sweep_place_kernel(const LocScene s, const LocItems it, const int64_t *__restrict__ word_off,
                       const uint32_t *__restrict__ mask, const int64_t *__restrict__ off, int to_tracks,
                       int2 *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t n_rows = it.row_off[it.n_items];
  const int64_t nw = (int64_t)gridDim.x * kWarpsPerBlock;
  for (int64_t r = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); r < n_rows; r += nw) {
    int64_t pos = off[r];
    if (off[r + 1] == pos) continue;
    const RowCtx c = row_ctx(s, it, r);
    const int words = (c.nt + 31) >> 5;
    const uint32_t *mrow = mask + __ldg(&word_off[c.item]) + c.ql * words;
    for (int w = 0; w < words; ++w) {
      const uint32_t m = mrow[w];
      if ((m >> lane) & 1u) {
        const int j = (w << 5) + lane;
        out[pos + __popc(m & lanemask_lt())] = make_int2((int)c.ql, to_tracks ? s.line_track[c.tbase + j] : j);
      }
      pos += __popc(m);
    }
  }
}
void launch_locmatch_sweep_place(const LocScene &s, const LocItems &it, const int64_t *word_off, const uint32_t *mask,
                                 const int64_t *off, int to_tracks, int2 *out, cudaStream_t st) {
  sweep_place_kernel<<<current_device_sms() * 8, 32 * kWarpsPerBlock, 0, st>>>(s, it, word_off, mask, off, to_tracks,
                                                                                out);
}

// ---- given pairs -------------------------------------------------------------------------------------------------
__global__ void filter_flags_kernel(const LocScene s, const LocItems it, const int64_t *__restrict__ pair_off,
                                    const int2 *__restrict__ pairs, int64_t n_pairs, int use_iou, double th,
                                    int to_tracks, int64_t *__restrict__ flag, int *err, unsigned long long *n_2to2) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n_pairs) return;
  if (k == n_pairs) { flag[k] = 0; return; }
  const int64_t item = last_le<true>(pair_off, it.n_items, k);
  const int2 qt = it.items[item];
  const int2 p = pairs[k];
  const int64_t qb = s.line_off[qt.x], tb = s.line_off[qt.y];
  if (p.x < 0 || p.x >= s.line_off[qt.x + 1] - qb || p.y < 0 || p.y >= s.line_off[qt.y + 1] - tb) {
    *err = 1;
    flag[k] = 0;
    return;
  }
  bool keep = true;
  if (use_iou) {
    const LocView &vq = s.views[qt.x];
    const LocView &vt = s.views[qt.y];
    const double4 l1 = s.lines[qb + p.x];
    const vec3<double> w1s = mat3_mul_h(vq.M, l1.x, l1.y), w1e = mat3_mul_h(vq.M, l1.z, l1.w);
    const vec3<double> base = mk3(vq.C[0], vq.C[1], vq.C[2]) - mk3(vt.C[0], vt.C[1], vt.C[2]);
    keep = epipolar_iou(EpipolarFromRays{vt.M, base, w1s, w1e}, s.lines[tb + p.y], th) > th;
  }
  { // one atomic per group of converged lanes
    const unsigned act = __activemask(), b = __ballot_sync(act, keep);
    if ((threadIdx.x & 31) == __ffs(act) - 1 && b) atomicAdd(n_2to2, (unsigned long long)__popc(b));
  }
  if (to_tracks) keep = keep && s.line_track[tb + p.y] != -1;
  flag[k] = keep ? 1 : 0;
}
void launch_locmatch_filter_flags(const LocScene &s, const LocItems &it, const int64_t *pair_off, const int2 *pairs,
                                  int64_t n_pairs, int use_iou, double th, int to_tracks, int64_t *flag, int *err,
                                  unsigned long long *n_2to2, cudaStream_t st) {
  filter_flags_kernel<<<(unsigned)((n_pairs + 256) / 256), 256, 0, st>>>(s, it, pair_off, pairs, n_pairs, use_iou, th,
                                                                           to_tracks, flag, err, n_2to2);
}

__global__ void filter_place_kernel(const LocScene s, const LocItems it, const int64_t *__restrict__ pair_off,
                                    const int2 *__restrict__ pairs, int64_t n_pairs, const int64_t *__restrict__ pos,
                                    int to_tracks, int2 *__restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_pairs || pos[k + 1] == pos[k]) return;
  const int2 p = pairs[k];
  int y = p.y;
  if (to_tracks) {
    const int64_t item = last_le<true>(pair_off, it.n_items, k);
    y = s.line_track[s.line_off[it.items[item].y] + p.y];
  }
  out[pos[k]] = make_int2(p.x, y);
}
void launch_locmatch_filter_place(const LocScene &s, const LocItems &it, const int64_t *pair_off, const int2 *pairs,
                                  int64_t n_pairs, const int64_t *pos, int to_tracks, int2 *out, cudaStream_t st) {
  if (n_pairs <= 0) return;
  filter_place_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, st>>>(s, it, pair_off, pairs, n_pairs, pos,
                                                                           to_tracks, out);
}

__global__ void gather_offsets_kernel(const int64_t *__restrict__ off, const int64_t *__restrict__ first, int64_t n,
                                      int64_t *__restrict__ item_off) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k <= n) item_off[k] = off[first[k]];
}
void launch_gather_offsets(const int64_t *off, const int64_t *first, int64_t n, int64_t *item_off, cudaStream_t st) {
  gather_offsets_kernel<<<(unsigned)((n + 256) / 256), 256, 0, st>>>(off, first, n, item_off);
}

// ---- grouping ----------------------------------------------------------------------------------------------------
// (a) entries and first entry of every (item, line)
__global__ void group_count_kernel(const LocItems it, const LocGroup g) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g.n_e) return;
  const int64_t item = last_le<true>(g.item_off, it.n_items, e);
  const int64_t row = it.row_off[item] + g.E[e].x;
  atomicAdd(&g.cnt[row], 1u);
  atomicMin(&g.first[row], (unsigned long long)e);
}
void launch_group_count(const LocItems &it, const LocGroup &g, cudaStream_t st) {
  if (g.n_e > 0) group_count_kernel<<<(unsigned)((g.n_e + 255) / 256), 256, 0, st>>>(it, g);
}

LM_D bool query_row(const LocItems &it, const LocGroup &g, int64_t qr, int64_t &q, int64_t &l, int64_t &t0,
                    int64_t &t1) {
  q = last_le<true>(g.qrow_off, g.n_queries, qr);
  l = qr - g.qrow_off[q];
  t0 = g.q_item_off[q];
  t1 = g.q_item_off[q + 1];
  return t1 > t0;
}

// (b) per (query, line): entries of the earlier items (kept in key), total, and the first entry over the query's items
// (the items of a query are contiguous in E, so the smallest entry index is the first appearance)
__global__ void group_heads_kernel(const LocItems it, const LocGroup g) {
  const int64_t qr = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (qr >= g.qrow_off[g.n_queries]) return;
  int64_t q, l, t0, t1;
  g.qhead[qr] = -1;
  g.qtot[qr] = 0;
  if (!query_row(it, g, qr, q, l, t0, t1)) return;
  int64_t tot = 0;
  unsigned long long hd = ~0ull;
  for (int64_t t = t0; t < t1; ++t) {
    const int64_t row = it.row_off[t] + l;
    g.key[row] = tot;
    tot += g.cnt[row];
    hd = min(hd, g.first[row]);
  }
  if (tot == 0) return;
  g.head[hd] = tot;
  g.qhead[qr] = (int64_t)hd;
  g.qtot[qr] = tot;
}
void launch_group_heads(const LocItems &it, const LocGroup &g, int64_t n_qrows, cudaStream_t st) {
  if (n_qrows > 0) group_heads_kernel<<<(unsigned)((n_qrows + 255) / 256), 256, 0, st>>>(it, g);
}

// (c) after the exclusive scan of head: the key's first output position, per (item, line) and per (query, line)
__global__ void group_keys_kernel(const LocItems it, const LocGroup g) {
  const int64_t qr = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (qr >= g.qrow_off[g.n_queries] || g.qhead[qr] < 0) return;
  int64_t q, l, t0, t1;
  query_row(it, g, qr, q, l, t0, t1);
  const int64_t ks = g.head[g.qhead[qr]];
  for (int64_t t = t0; t < t1; ++t) g.key[it.row_off[t] + l] += ks;
  g.qhead[qr] = ks;
}
void launch_group_keys(const LocItems &it, const LocGroup &g, int64_t n_qrows, cudaStream_t st) {
  if (n_qrows > 0) group_keys_kernel<<<(unsigned)((n_qrows + 255) / 256), 256, 0, st>>>(it, g);
}

// (d) one CTA per item places the item's entries in order: a tile at a time, an entry's rank among the equal rows of
// its warp comes from __match_any_sync and the warps take turns, in entry order, to advance each row's running count
__global__ void __launch_bounds__(kPlaceThreads) group_place_kernel(const LocItems it, const LocGroup g,
                                                                     int2 *__restrict__ out) {
  __shared__ unsigned s_base[kPlaceThreads];
  const int64_t item = blockIdx.x;
  const int64_t e0 = g.item_off[item], e1 = g.item_off[item + 1];
  const int64_t rb = it.row_off[item];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t t0 = e0; t0 < e1; t0 += kPlaceThreads) {
    const int64_t e = t0 + threadIdx.x;
    const bool valid = e < e1;
    const int2 p = valid ? g.E[e] : make_int2(-1, 0);
    const int64_t row = rb + p.x;
    const unsigned same = __match_any_sync(0xffffffffu, valid ? (long long)row : -1ll);
    const int leader = __ffs(same) - 1;
    for (int w = 0; w < kPlaceThreads / 32; ++w) {
      if (w == warp && valid && lane == leader) {
        const unsigned k = g.run[row];
        g.run[row] = k + __popc(same);
        s_base[threadIdx.x] = k;
      }
      __syncthreads();
    }
    if (valid) {
      const unsigned k = s_base[(warp << 5) + leader] + __popc(same & lanemask_lt());
      out[g.key[row] + k] = p;
    }
    __syncthreads();
  }
}
void launch_group_place(const LocItems &it, const LocGroup &g, int2 *out, cudaStream_t st) {
  if (it.n_items > 0 && g.n_e > 0) group_place_kernel<<<(unsigned)it.n_items, kPlaceThreads, 0, st>>>(it, g, out);
}

// ---- reprojection filter -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * kWarpsPerBlock)
    reproj_filter_kernel(const LocScene s, const LocItems it, const LocGroup g, const int2 *__restrict__ G,
                         const ReprojParams rp, int64_t *__restrict__ flag, int32_t *__restrict__ sel) {
  const int lane = threadIdx.x & 31;
  const int64_t nqr = g.qrow_off[g.n_queries];
  const int64_t nw = (int64_t)gridDim.x * kWarpsPerBlock;
  for (int64_t qr = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); qr < nqr; qr += nw) {
    const int64_t ks = g.qhead[qr];
    if (ks < 0) continue;
    int64_t q, l, t0, t1;
    query_row(it, g, qr, q, l, t0, t1);
    const int qimg = it.items[t0].x;
    const LocView &v = s.views[qimg];
    const double4 L = s.lines[s.line_off[qimg] + l];
    const vec2<double> rs = mk2(L.x, L.y), re = mk2(L.z, L.w);
    const vec2<double> dir_ref = seg_direction(rs, re);
    const vec2<double> mref = midpoint(rs, re);
    const double len_ref = seg_length(rs, re);
    // the lexicographically smallest (loss, track) over the candidates whose loss is < inf: the reference's strict `<`
    // over ascending unique track ids from min_loss = inf (NaN never wins, ties go to the lowest track id)
    double best = 0.0;
    int bid = -1;
    const int64_t n = g.qtot[qr];
    for (int64_t k = lane; k < n; k += 32) {
      const int id = G[ks + k].y;
      const double *X = s.track_lines + 6 * (int64_t)id;
      const vec2<double> ps = project(v, X), pe = project(v, X + 3);
      const vec2<double> tdir = seg_direction(ps, pe);
      double dist;
      if (rp.dist_func == 1) { // midpoint_dist
        const vec2<double> mt = midpoint(ps, pe);
        dist = __dsqrt_rn(sq2(__dsub_rn(mref.x, mt.x), __dsub_rn(mref.y, mt.y)));
      } else if (rp.dist_func == 0) { // perpendicular_dist
        const double a = fabs(cross2(tdir, mk2(__dsub_rn(ps.x, rs.x), __dsub_rn(ps.y, rs.y))));
        const double b = fabs(cross2(tdir, mk2(__dsub_rn(ps.x, re.x), __dsub_rn(ps.y, re.y))));
        dist = __dmul_rn(0.5, __dadd_rn(a, b));
      } else { // midpoint_perpendicular_dist
        dist = __ddiv_rn(fabs(cross2(tdir, mk2(__dsub_rn(ps.x, mref.x), __dsub_rn(ps.y, mref.y)))), len_ref);
      }
      double loss = dist;
      bool skip = false;
      if (rp.dist_func == 1) {
        double c = __dadd_rn(__dmul_rn(dir_ref.x, tdir.x), __dmul_rn(dir_ref.y, tdir.y));
        c = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c); // np.clip keeps NaN
        const double sine = __dsqrt_rn(__dsub_rn(1.0, __dmul_rn(c, c)));
        loss = __dadd_rn(loss, __dmul_rn(__dmul_rn(rp.angle_scale, seg_length(ps, pe)), sine));
        skip = sine > rp.sine_thres;
      }
      skip = skip || dist > rp.dist_thres;
      if (!skip && loss < CUDART_INF && (bid < 0 || loss < best || (loss == best && id < bid))) {
        best = loss;
        bid = id;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_down_sync(0xffffffffu, best, o);
      const int oid = __shfl_down_sync(0xffffffffu, bid, o);
      if (oid >= 0 && (bid < 0 || ob < best || (ob == best && oid < bid))) {
        best = ob;
        bid = oid;
      }
    }
    if (lane == 0) {
      flag[ks] = bid >= 0 ? 1 : 0;
      sel[ks] = bid;
    }
  }
}
void launch_reproj_filter(const LocScene &s, const LocItems &it, const LocGroup &g, const int2 *G,
                          const ReprojParams &rp, int64_t *flag, int32_t *sel, cudaStream_t st) {
  reproj_filter_kernel<<<current_device_sms() * 8, 32 * kWarpsPerBlock, 0, st>>>(s, it, g, G, rp, flag, sel);
}

__global__ void reproj_place_kernel(int64_t n_e, const int2 *__restrict__ G, const int64_t *__restrict__ pos,
                                    const int32_t *__restrict__ sel, int2 *__restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n_e && pos[k + 1] != pos[k]) out[pos[k]] = make_int2(G[k].x, sel[k]);
}
void launch_reproj_place(const LocGroup &g, const int2 *G, const int64_t *pos, const int32_t *sel, int2 *out,
                         cudaStream_t st) {
  if (g.n_e > 0) reproj_place_kernel<<<(unsigned)((g.n_e + 255) / 256), 256, 0, st>>>(g.n_e, G, pos, sel, out);
}

} // namespace lm
