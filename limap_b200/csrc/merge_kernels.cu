// merge_kernels.cu — track filters + remerge pair test on sm_90a.
//
// support_flags_kernel: the three per-support predicates the runner applies between ComputeLineTracks and
//   the line BA (runners/line_triangulation.py:171-200): CheckReprojection (merging_utils.cc:27-48),
//   CheckSensitivity (:89-107) and the overlap test of FilterTracksByOverlap (:143-149). One thread per
//   supporting line, fp64, formulas in the reference's order; 32 B segment + 4 B view id in, 1 B out.
// remerge_pairs_kernel: RemergeLineTracks tests every pair of track lines with LineLinker3d::check_connection
//   (merging.cc:527-556, O(T^2)). Tiles of 256 x 256 pairs; the angle test is gated in fp32 on unit directions
//   (|cos| >= cos(th_angle) - 1e-5: a pair that fails the gate fails the fp64 angle test by > 1e3 ulp of fp32)
//   and, when the inner-segment test is on, on bounding balls grown by the largest passing distance,
//   survivors are queued per warp and checked densely in fp64 with the reference's formulas and argument
//   order. Output: unordered list of connected pairs (a < b); the union-find stays on the host (sequential).
#include "merge_kernels.cuh"
#include "graph_kernels.cuh"

namespace lm {

// LineLinker3d::check_connection (base/line_linker.cc:212-306) with uncertainty = min(l1, l2)
// (line_linker.cc:239-262), and LineLinker2d::check_connection (:120-137) with unc = 1 (th * 1.0 == th exactly).
// The scale-invariant test needs depths the 3D lines do not carry; every 3D caller runs under
// set_to_spatial_merging (line_linker.h:123-129), which switches it off, and the 2D linker has none.
template <typename V>
LM_D bool linker_check(const LinkerDev<double> &c, const seg<V> &l1, const seg<V> &l2, double unc) {
  double angle = 0.0, bio = 0.0;
  if (c.use_angle) {
    angle = compute_angle<double, V>(l1, l2);
    if (!(angle <= c.th_angle)) return false;
  }
  if (c.use_overlap) {
    bio = compute_bioverlap<double, V>(l1, l2);
    if (!(bio > c.th_overlap)) return false;
  }
  if (c.use_angle && c.use_overlap && c.use_smartangle) {
    double th_angle = c.th_angle;
    if (bio < c.th_smartoverlap) {
      double ratio = (c.th_smartoverlap - bio) / (c.th_smartoverlap - c.th_overlap);
      ratio = smin<double>(ratio, 1.0);
      th_angle = c.th_angle - ratio * (c.th_angle - c.th_smartangle);
    }
    if (!(thresh0(expscore(angle, th_angle * c.mult), c.score_th) >= c.score_th)) return false;
  }
  if (c.use_perp) {
    const double d = dist_endpoints_perpendicular<double, V>(l1, l2);
    if (!(thresh0(expscore(d, c.th_perp * unc * c.mult), c.score_th) >= c.score_th)) return false;
  }
  if (c.use_innerseg) {
    const double d = dist_innerseg<double, V>(l1, l2);
    if (!(thresh0(expscore(d, c.th_innerseg * unc * c.mult), c.score_th) >= c.score_th)) return false;
  }
  return true;
}

__global__ void __launch_bounds__(256) support_flags_kernel(const __grid_constant__ SupportParams p) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  // track of this support: last t with sup_off[t] <= s (its own loop: through last_le the kernel's SASS changes)
  int64_t lo = 0, hi = p.T;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(&p.sup_off[mid]) <= s) lo = mid; else hi = mid;
  }
  const double *tl = p.track_line + 6 * lo;
  seg<vec3<double>> L;
  L.s = mk3(tl[0], tl[1], tl[2]);
  L.e = mk3(tl[3], tl[4], tl[5]);
  const ViewD &v = p.views[p.sup_view[s]];
  const double2 a0 = __ldg(reinterpret_cast<const double2 *>(p.segs + s));
  const double2 a1 = __ldg(reinterpret_cast<const double2 *>(p.segs + s) + 1);
  seg<vec2<double>> l2d, proj;
  l2d.s = mk2(a0.x, a0.y);
  l2d.e = mk2(a1.x, a1.y);
  proj.s = dehom(proj_h(v.P, L.s)); // Line3d::projection (linebase.cc:93-98)
  proj.e = dehom(proj_h(v.P, L.e));
  uint8_t f = 0;
  {
    bool ok = true;
    const double angle = compute_angle<double, vec2<double>>(l2d, proj);
    if (angle > p.th_angular2d) ok = false;
    if (ok && dist_perp_oneway_max<double, vec2<double>>(l2d, proj) > p.th_perp2d) ok = false;
    if (ok) f |= 1;
  }
  { // Line3d::sensitivity (linebase.cc:100-107)
    const vec2<double> mid = (proj.s + proj.e) * 0.5;
    const vec3<double> dir3d = normalized(mat3_mul_h(v.M, mid.x, mid.y));
    const double cos_val = fabs(dot(direction(L), dir3d));
    const double sens = 90.0 - acos(cos_val) * consts<double>::rad2deg();
    if (!(sens > p.th_sv_angular3d)) f |= 2;
  }
  if (compute_overlap<double, vec2<double>>(proj, l2d) >= p.th_overlap) f |= 4;
  p.flags[s] = f;
}

void launch_support_flags(const SupportParams &p, cudaStream_t s) {
  if (p.S <= 0) return;
  support_flags_kernel<<<(unsigned)((p.S + 255) / 256), 256, 0, s>>>(p);
}

// fp32 gate records: unit direction, and a ball (midpoint relative to `origin`, radius) that contains the
// segment grown by the largest inner-segment distance that can still pass: score_innerseg >= score_th
// <=> dist <= th_innerseg * min(unc) (line_linker.cc:253-262 with multiplier() = 1/sqrt(-2 ln score_th)).
// Two segments whose inner-segment distance is d have points within d of each other, so their grown balls
// intersect; w carries the radius with the fp32 error budget (1e-3 relative + 1e-5 of the coordinates).
LM_D void gate_record(const double *l, double ox, double oy, double oz, double th_innerseg, float4 &dirf, float4 &ballf) {
  const vec3<double> v = mk3(l[3] - l[0], l[4] - l[1], l[5] - l[2]);
  const vec3<double> d = normalized(v);
  dirf = make_float4((float)d.x, (float)d.y, (float)d.z, 0.f);
  const double mx = 0.5 * (l[0] + l[3]) - ox, my = 0.5 * (l[1] + l[4]) - oy, mz = 0.5 * (l[2] + l[5]) - oz;
  double r = 0.5 * norm(v) + th_innerseg * fabs(l[6]);
  r = r * 1.001 + 1e-5 * (fabs(mx) + fabs(my) + fabs(mz)) + 1e-30;
  if (!(r == r) || !(mx == mx) || !(my == my) || !(mz == mz)) r = 3e38; // NaN input: never gate it away
  ballf = make_float4((float)mx, (float)my, (float)mz, (float)fmin(r, 1e18));
}
__global__ void remerge_dirs_kernel(const double *lines, int64_t T, double ox, double oy, double oz, double th_innerseg,
                                    float4 *dirf, float4 *ballf) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  gate_record(lines + 7 * t, ox, oy, oz, th_innerseg, dirf[t], ballf[t]);
}
void launch_remerge_dirs(const double *lines, int64_t T, const double origin[3], double th_innerseg, float4 *dirf,
                         float4 *ballf, cudaStream_t s) {
  if (T <= 0) return;
  remerge_dirs_kernel<<<(unsigned)((T + 255) / 256), 256, 0, s>>>(lines, T, origin[0], origin[1], origin[2],
                                                                 th_innerseg, dirf, ballf);
}

constexpr int kTile = 256;
constexpr int kQueue = 64; // per-warp survivor queue (drained at >= 32)

LM_D seg<vec3<double>> load_line(const double *lines, uint32_t t, double &unc) {
  const double *l = lines + 7 * (size_t)t;
  seg<vec3<double>> r;
  r.s = mk3(__ldg(l), __ldg(l + 1), __ldg(l + 2));
  r.e = mk3(__ldg(l + 3), __ldg(l + 4), __ldg(l + 5));
  unc = __ldg(l + 6);
  return r;
}

// The reference tests pair {a < b} as check(l_i, l_j) from the active side(s) (merging.cc:527-556):
//   all tracks active: from a when a + b is odd, from b when it is even (each pair once);
//   otherwise: from every active endpoint, the edge exists when any of the tests passes.
LM_D bool pair_connected(const RemergeParams &p, uint32_t a, uint32_t b) {
  double ua, ub;
  const seg<vec3<double>> la = load_line(p.lines, a, ua), lb = load_line(p.lines, b, ub);
  const double unc = smin<double>(ua, ub);
  const double unc_r = smin<double>(ub, ua);
  if (p.all_active) return ((a + b) & 1u) ? linker_check(p.lk, la, lb, unc) : linker_check(p.lk, lb, la, unc_r);
  bool ok = false;
  if (p.active[a]) ok = linker_check(p.lk, la, lb, unc);
  if (!ok && p.active[b]) ok = linker_check(p.lk, lb, la, unc_r);
  return ok;
}

__device__ __noinline__ void drain(const RemergeParams &p, const uint2 *q, int n, int lane) {
  if (lane < n) {
    const uint2 e = q[lane];
    if (pair_connected(p, e.x, e.y)) {
      const unsigned long long slot = atomicAdd(p.counter, 1ull);
      if (slot < p.capacity) { p.edges[2 * slot] = e.x; p.edges[2 * slot + 1] = e.y; }
    }
  }
}

__global__ void __launch_bounds__(kTile, 4) remerge_pairs_kernel(const __grid_constant__ RemergeParams p) {
  // upper-triangular tile grid: blockIdx.x enumerates (ta <= tb)
  const int64_t n_tiles = (p.T + kTile - 1) / kTile;
  int64_t ta = 0, rem = blockIdx.x;
  { // row ta holds n_tiles - ta tiles; solve by the closed form, fix up by one
    const double nt = (double)n_tiles;
    ta = (int64_t)floor(((2.0 * nt + 1.0) - sqrt((2.0 * nt + 1.0) * (2.0 * nt + 1.0) - 8.0 * (double)rem)) * 0.5);
    if (ta < 0) ta = 0;
    while (ta > 0 && ta * n_tiles - ta * (ta - 1) / 2 > rem) --ta;
    while ((ta + 1) * n_tiles - (ta + 1) * ta / 2 <= rem) ++ta;
    rem -= ta * n_tiles - ta * (ta - 1) / 2;
  }
  const int64_t tb = ta + rem;
  __shared__ float4 sb[kTile], sball[kTile];
  __shared__ uint8_t sact[kTile];
  __shared__ uint2 queue[kTile / 32][kQueue];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t a = ta * kTile + tid, b0 = tb * kTile;
  const int nb = (int)min((int64_t)kTile, p.T - b0);
  if (tid < nb) {
    sb[tid] = p.dirf[b0 + tid];
    sball[tid] = p.ballf[b0 + tid];
    sact[tid] = p.active[b0 + tid];
  } else {
    sb[tid] = make_float4(0.f, 0.f, 0.f, 0.f);
    sball[tid] = make_float4(1e30f, 1e30f, 1e30f, 0.f); // never inside a ball
    sact[tid] = 0;
  }
  __syncthreads();
  const bool a_ok = a < p.T;
  float4 da = make_float4(0.f, 0.f, 0.f, 0.f), ba = make_float4(0.f, 0.f, 0.f, 0.f);
  bool a_act = false;
  if (a_ok) { da = p.dirf[a]; ba = p.ballf[a]; a_act = p.active[a] != 0; }
  uint2 *q = queue[warp];
  int qn = 0; // warp-uniform
  unsigned long long gated = 0;
  const bool use_ball = p.use_ball != 0;
  const int jfirst = (ta == tb) ? (tid & ~31) : 0; // diagonal tile: b > a starts in this warp's own column block
  for (int j0 = jfirst & ~3; j0 < nb; j0 += 4) {
    bool ps[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4 bb = sball[j0 + u];
      const float dx = ba.x - bb.x, dy = ba.y - bb.y, dz = ba.z - bb.z, rs = ba.w + bb.w;
      ps[u] = !use_ball || !(dx * dx + dy * dy + dz * dz > rs * rs * 1.0001f); // NaN-safe: only a clear miss drops
    }
    if (!__any_sync(0xffffffffu, ps[0] | ps[1] | ps[2] | ps[3])) continue;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      const int64_t b = b0 + j;
      bool pass = ps[u] && a_ok && j < nb && b > a && (p.all_active || a_act || sact[j]);
      if (pass && p.use_gate) {
        const float4 db = sb[j];
        pass = fabsf(da.x * db.x + da.y * db.y + da.z * db.z) >= p.cos_gate;
      }
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (m) {
        if (pass) q[qn + __popc(m & ((1u << lane) - 1))] = make_uint2((uint32_t)a, (uint32_t)b);
        qn += __popc(m);
        gated += (lane == 0) ? __popc(m) : 0;
        __syncwarp();
        if (qn >= 32) {
          drain(p, q + (qn - 32), 32, lane);
          qn -= 32;
          __syncwarp();
        }
      }
    }
  }
  if (qn > 0) drain(p, q, qn, lane);
  if (lane == 0 && gated) atomicAdd(p.counter + 1, gated);
}

void launch_remerge_pairs(const RemergeParams &p, cudaStream_t s) {
  if (p.T <= 1) return;
  const int64_t n_tiles = (p.T + kTile - 1) / kTile;
  const int64_t grid = n_tiles * (n_tiles + 1) / 2;
  remerge_pairs_kernel<<<(unsigned)grid, kTile, 0, s>>>(p);
}

// ---- MergeToLineTracks (merging.cc:347-511) ---------------------------------------------------------------------------
// fit_prep_kernel: one thread per 3D fit. SetUncertaintySegs3d (merging_utils.cc:15-25), Line3d::length() (the compiled
// reference contracts its squared norm into two fused multiply-adds; sim = len1 + len2 is compared for ties, so the
// length is written operation for operation), the node flag `length != 0` (merging.cc:377) and the gate records.
LM_D double fit_depth(const FitView &w, const double *p) { // CameraPose::projdepth (camera.cc:276-279)
  return (w.R[6] * p[0] + w.R[7] * p[1] + w.R[8] * p[2]) + w.t[2];
}
__global__ void fit_prep_kernel(const __grid_constant__ FitPrepParams p) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n) return;
  const FitView &w = p.views[last_le<true>(p.line_off, p.V, g)]; // view of line g
  const double *l = p.lines3d + 6 * g;
  double *r = p.rec + 7 * g;
  for (int k = 0; k < 6; ++k) r[k] = l[k];
  r[6] = p.var2d * ((fit_depth(w, l) + fit_depth(w, l + 3)) / 2.0) / w.f; // computeUncertainty (linebase.cc:109-116)
  const double dx = __dsub_rn(l[0], l[3]), dy = __dsub_rn(l[1], l[4]), dz = __dsub_rn(l[2], l[5]);
  const double len = __dsqrt_rn(__fma_rn(dz, dz, __fma_rn(dy, dy, __dmul_rn(dx, dx))));
  p.len[g] = len;
  p.nonzero[g] = (len != 0.0) ? 1 : 0;
  gate_record(r, p.ox, p.oy, p.oz, p.th_innerseg, p.dirf[g], p.ballf[g]);
}
void launch_fit_prep(const FitPrepParams &p, cudaStream_t s) {
  if (p.n > 0) fit_prep_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, s>>>(p);
}

// Line3d::projection (linebase.cc:93-98) = dehomogeneous(K * (R * p + T)) (camera_view.cc:61-65); K's zero entries add
// exact zeros and are left out.
LM_D seg<vec2<double>> fit_project(const FitView &w, const seg<vec3<double>> &l) {
  seg<vec2<double>> o;
  const vec3<double> *pts[2] = {&l.s, &l.e};
  vec2<double> *out[2] = {&o.s, &o.e};
  for (int k = 0; k < 2; ++k) {
    const vec3<double> &p = *pts[k];
    const double X = (w.R[0] * p.x + w.R[1] * p.y + w.R[2] * p.z) + w.t[0];
    const double Y = (w.R[3] * p.x + w.R[4] * p.y + w.R[5] * p.z) + w.t[1];
    const double Z = (w.R[6] * p.x + w.R[7] * p.y + w.R[8] * p.z) + w.t[2];
    *out[k] = dehom(mk3(w.fx * X + w.cx * Z, w.fy * Y + w.cy * Z, Z));
  }
  return o;
}

// Exact test of one queued pair (a of view va, b of view vb, image-local indices) in the reference's argument order
// (merging.cc:405-412, :446-457); a passing pair is appended with its insertion key
//   va << 48 | cross << 47 | a << 31 | slot << 16 | b
// i.e. per source image: self pairs in (i, j) order, then cross pairs in (line, neighbour slot, neighbour line) order.
__device__ __noinline__ void fit_drain(const FitPairParams &p, const uint2 *q, int n, int lane, int va, int vb, int slot,
                                       int64_t ba, int64_t bb) {
  if (lane >= n) return;
  const uint2 e = q[lane];
  const int64_t ga = ba + e.x, gb = bb + e.y;
  double ua, ub;
  const seg<vec3<double>> la = load_line(p.rec, (uint32_t)ga, ua), lb = load_line(p.rec, (uint32_t)gb, ub);
  if (!linker_check(p.lk3, la, lb, smin<double>(ua, ub))) return;
  seg<vec2<double>> sa, sb;
  const double4 a4 = p.segs[ga], b4 = p.segs[gb];
  sa.s = mk2(a4.x, a4.y); sa.e = mk2(a4.z, a4.w);
  sb.s = mk2(b4.x, b4.y); sb.e = mk2(b4.z, b4.w);
  if (slot < 0) {
    if (!linker_check(p.lk2, sa, sb, 1.0)) return;
  } else {
    if (!linker_check(p.lk2, fit_project(p.views[vb], la), sb, 1.0)) return;
    if (!linker_check(p.lk2, fit_project(p.views[va], lb), sa, 1.0)) return;
  }
  const unsigned long long key = (unsigned long long)va << 48 | (slot < 0 ? 0ull : 1ull << 47) |
                                 (unsigned long long)e.x << 31 | (slot < 0 ? 0ull : (unsigned long long)slot << 16) |
                                 (unsigned long long)e.y;
  const unsigned long long k = atomicAdd(p.counter, 1ull);
  if (k < p.capacity) {
    p.keys[k] = key;
    p.pairs[k] = (unsigned long long)ga << 32 | (unsigned long long)gb;
  }
}

// One CTA per 256 x 256 tile of a (source image, self) or (source image, neighbour slot) block. Tested pairs are those
// the reference's loops hand to check_connection_3d: both lines non-zero, j > i in self blocks, and the parity rule of
// merging.cc:437-441 with its integer types in cross blocks. The fp32 ball and angle gates drop only pairs that fail the
// fp64 tests (DESIGN.md §3.5, §3.6); survivors go through the per-warp queues to fit_drain.
__global__ void __launch_bounds__(kTile, 4) fit_pairs_kernel(const __grid_constant__ FitPairParams p) {
  const FitTile tl = p.tiles[blockIdx.x];
  const int va = tl.va, vb = tl.vb, slot = tl.slot, ta = tl.tiles >> 16, tb = tl.tiles & 0xffff;
  const bool self = slot < 0;
  const int64_t ba = p.line_off[va], bb = p.line_off[vb];
  const int na = (int)(p.line_off[va + 1] - ba), nbt = (int)(p.line_off[vb + 1] - bb);
  __shared__ float4 sb[kTile], sball[kTile];
  __shared__ uint8_t snz[kTile];
  __shared__ uint2 queue[kTile / 32][kQueue];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int a = ta * kTile + tid, b0 = tb * kTile;
  const int nb = min(kTile, nbt - b0);
  if (tid < nb) {
    sb[tid] = p.dirf[bb + b0 + tid];
    sball[tid] = p.ballf[bb + b0 + tid];
    snz[tid] = p.nonzero[bb + b0 + tid];
  } else {
    sb[tid] = make_float4(0.f, 0.f, 0.f, 0.f);
    sball[tid] = make_float4(1e30f, 1e30f, 1e30f, 0.f);
    snz[tid] = 0;
  }
  __syncthreads();
  const bool a_ok = a < na && p.nonzero[ba + a];
  float4 da = make_float4(0.f, 0.f, 0.f, 0.f), qa = make_float4(0.f, 0.f, 0.f, 0.f);
  if (a_ok) { da = p.dirf[ba + a]; qa = p.ballf[ba + a]; }
  // merging.cc:437: `int key = image_id + line_id + ng_image_id + ng_line_id` summed as size_t, the images compared as size_t
  const unsigned long long ui = (unsigned long long)(long long)p.img_ids[va];
  const unsigned long long un = (unsigned long long)(long long)p.img_ids[vb];
  const unsigned long long kbase = ui + (unsigned long long)a + un + (unsigned long long)b0;
  uint2 *q = queue[warp];
  int qn = 0;
  unsigned long long gated = 0, tested = 0;
  const int jfirst = (self && ta == tb) ? (tid & ~31) : 0; // diagonal tile: j > i starts in this warp's own column block
  for (int j0 = jfirst & ~3; j0 < nb; j0 += 4) {
    bool ps[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      bool t = a_ok && snz[j]; // snz is 0 past nb
      if (self) {
        t = t && (b0 + j > a);
      } else {
        const int key = (int)(kbase + (unsigned long long)j);
        t = t && !((key % 2 == 0 && ui < un) || (key % 2 == 1 && ui > un));
      }
      tested += t ? 1 : 0;
      const float4 bq = sball[j];
      const float dx = qa.x - bq.x, dy = qa.y - bq.y, dz = qa.z - bq.z, rs = qa.w + bq.w;
      ps[u] = t && (!p.use_ball || !(dx * dx + dy * dy + dz * dz > rs * rs * 1.0001f));
    }
    if (!__any_sync(0xffffffffu, ps[0] | ps[1] | ps[2] | ps[3])) continue;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      bool pass = ps[u];
      if (pass && p.use_gate) {
        const float4 db = sb[j];
        pass = fabsf(da.x * db.x + da.y * db.y + da.z * db.z) >= p.cos_gate;
      }
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (m) {
        if (pass) q[qn + __popc(m & ((1u << lane) - 1))] = make_uint2((uint32_t)a, (uint32_t)(b0 + j));
        qn += __popc(m);
        gated += (lane == 0) ? __popc(m) : 0;
        __syncwarp();
        if (qn >= 32) {
          fit_drain(p, q + (qn - 32), 32, lane, va, vb, slot, ba, bb);
          qn -= 32;
          __syncwarp();
        }
      }
    }
  }
  if (qn > 0) fit_drain(p, q, qn, lane, va, vb, slot, ba, bb);
  for (int o = 16; o > 0; o >>= 1) tested += __shfl_xor_sync(0xffffffffu, tested, o);
  if (lane == 0) {
    if (gated) atomicAdd(p.counter + 1, gated);
    if (tested) atomicAdd(p.counter + 2, tested);
  }
}
void launch_fit_pairs(const FitPairParams &p, int64_t n_tiles, cudaStream_t s) {
  if (n_tiles > 0) fit_pairs_kernel<<<(unsigned)n_tiles, kTile, 0, s>>>(p);
}

__global__ void fit_order_keys_kernel(const unsigned long long *pairs, const double *len, int64_t n,
                                      unsigned long long *by_nodes, unsigned long long *by_score, double *sim) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const unsigned long long pr = pairs[e];
  const double w = __dadd_rn(len[pr >> 32], len[pr & 0xffffffffull]); // merging.cc:473-475
  sim[e] = w;
  by_nodes[e] = ~pr; // node ids are increasing in the line index: the line order is the node order
  by_score[e] = descending_double_key(w);
}
void launch_fit_order_keys(const unsigned long long *pairs, const double *len, int64_t n, unsigned long long *by_nodes,
                           unsigned long long *by_score, double *sim, cudaStream_t s) {
  if (n > 0) fit_order_keys_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(pairs, len, n, by_nodes, by_score, sim);
}

} // namespace lm
