// tri_kernels.cu — sm_90a kernels of the line-triangulation hot path.
//
//   tri_node_kernel : one CTA per 2D line ("node"). Fuses
//       BaseLineTriangulator::triangulateOneNode   (triangulation/base_line_triangulator.cc:161-337)
//       GlobalLineTriangulator::scoreOneNode       (triangulation/global_line_triangulator.cc:71-161)
//     so that the candidate set of a node lives only in shared memory: match rows are read once from
//     HBM, candidates are never written back unless debug_mode asks for them.
//   The plumbing kernels around it are in tri_plumbing.cu.
//
// Outputs and final decisions are fp64 (every gate of the reference is a hard threshold on a transcendental and
// the contract is bit-exact candidate indices); fp32 appears only in pruning gates with explicit margins
// (see DESIGN.md "Precision").
#include "tri_kernels.cuh"

namespace lm {

// CTAs per SM the registers of the headline instantiation tri_node_kernel<false, false, true> are sized for (5: 96
// registers, with the fast staging layout at cap 200 in 42.8 KB of shared memory); the slab, VP and generic
// instantiations stay at 4 (128 registers)
#ifndef LM_TRI_MIN_BLOCKS
#define LM_TRI_MIN_BLOCKS 5
#endif
static constexpr int kThreads = 128;
static constexpr int kWarps = kThreads / 32;
static constexpr int kFlush = 64; // generic phase B: a warp flushes its survivor list once it holds this many pairs
static constexpr int kListExtra = kFlush + 32;
static constexpr int kCandBytes = 17 * 8 + 48 + 8;

// FAST: reduced-form scorer and plane-pair triangulation only (the default configuration); the generic instantiation
// keeps the reference-structured scorer, the 2d margin gates and endpoint triangulation.
bool tri_fast(const TriParams &p) { return p.fast_forms && !p.use_endpoints_triangulation; }
// Capacities are multiples of 8 for the fast layout (gatef and the staged views of the VP instantiation stay 16-byte
// aligned; hypersim100's 200-row nodes fit at cap 200, five CTAs per SM) and of 32 for the generic one (its start-point
// prefilter pads a node's candidates to a multiple of 32).
int tri_cap_step(bool fast) { return fast ? 8 : 32; }

// Shared-memory staging per node. Generic layout: 17 doubles + 48-byte fp32 gate record + ng/row per candidate, two
// survivor lists and one prefilter list per warp. Fast layout (reduced-form scorer, plane-pair triangulation): 16 doubles
// (three reciprocals more, and not the matched 2D segment, which the scorer reloads through ng), a 32-byte gate record,
// ng/row, the depth-sorted order (float key + uint16 index) per candidate, and per warp one pair list (uint16) with its
// scores (double): 214 bytes per candidate slot, 42.8 KB at cap 200, which lets five CTAs share an SM.
size_t tri_smem_bytes(int cap, bool fast) {
  if (fast) return (size_t)cap * (16 * 8 + kWarps * 8 + 32 + 8 + 4 + 2 + kWarps * 2);
  return (size_t)cap * kCandBytes + (size_t)kWarps * 2 * (cap + kListExtra) * 4 + (size_t)kWarps * cap * 2;
}

// fp32 copy of a candidate for the pruning gates (three 16-byte loads, conflict-free at 48-byte stride):
// unit direction, endpoints relative to the source camera centre, squared scale-invariance limits of the
// candidate taken as l_i.
struct __align__(16) GateRec {
  float dx, dy, dz, lims2;
  float sx, sy, sz, lime2;
  float ex, ey, ez, pad;
};

// Fast-path gate record. Every candidate of a node starts on the ray of the source line's start point and ends on the
// ray of its end point (X = ray * lambda + C1 in both the plane-pair and the VP-constrained triangulation), so the
// scale-invariant endpoint test of LineLinker3d (line_linker.cc:269-277) is an interval test on lambda: 1-D, sortable.
struct __align__(16) GateRecF {
  float dx, dy, dz, lam_e; // unit direction; distance of the end point along the end ray
  float lam_s;             // distance of the start point along the start ray
  float lim_s, lim_e;      // largest |delta lambda| that can still pass, taken as l_i (widened, see phase A)
  int img;                 // neighbour view of the candidate
};

struct Slab {
  double *sx, *sy, *sz, *ex, *ey, *ez, *dx, *dy, *dz, *zs, *ze, *unc, *q0, *q1, *q2, *q3, *score;
  double *izs2, *ize2, *inb; // fast layout only: 1/(zs+EPS)^2, 1/(ze+EPS)^2, 1/|q|^2 (q0..q3: generic layout only)
  GateRec *gate;
  uint32_t *ng, *row;
  uint32_t *list;            // [kWarps][2][cap + kListExtra]: (row << 16 | j) survivor entries
  uint16_t *list0;           // [kWarps][cap]: j of the start-point prefilter
  // fast layout only
  GateRecF *gatef;
  float *slam;               // [cap] lam_s in ascending order
  uint16_t *sidx;            // [cap] candidate of each sorted position
  double *psc;               // [kWarps][cap] scores of a warp's pair list
  uint16_t *pent;            // [kWarps][cap] j of a warp's pair list (rows contiguous)
  LM_D void carve(char *base, int cap, bool fast) {
    if (fast) { carve_fast(base, cap); return; }
    gatef = nullptr; slam = nullptr; sidx = nullptr; psc = nullptr; pent = nullptr;
    double *d = reinterpret_cast<double *>(base);
    sx = d; sy = sx + cap; sz = sy + cap; ex = sz + cap; ey = ex + cap; ez = ey + cap;
    dx = ez + cap; dy = dx + cap; dz = dy + cap; zs = dz + cap; ze = zs + cap; unc = ze + cap;
    q0 = unc + cap; q1 = q0 + cap; q2 = q1 + cap; q3 = q2 + cap; score = q3 + cap;
    izs2 = ize2 = inb = nullptr;
    gate = reinterpret_cast<GateRec *>(score + cap);
    ng = reinterpret_cast<uint32_t *>(gate + cap);
    row = ng + cap;
    list = row + cap;
    list0 = reinterpret_cast<uint16_t *>(list + (size_t)kWarps * 2 * (cap + kListExtra));
  }
  // cap is a multiple of tri_cap_step(true) = 8: gatef and the staged views of the VP instantiation (psc + 4 cap) stay
  // 16-byte aligned
  LM_D void carve_fast(char *base, int cap) {
    double *d = reinterpret_cast<double *>(base);
    sx = d; sy = sx + cap; sz = sy + cap; ex = sz + cap; ey = ex + cap; ez = ey + cap;
    dx = ez + cap; dy = dx + cap; dz = dy + cap; zs = dz + cap; ze = zs + cap; unc = ze + cap;
    score = unc + cap; izs2 = score + cap; ize2 = izs2 + cap; inb = ize2 + cap;
    psc = inb + cap;                                              // byte 128 cap
    gatef = reinterpret_cast<GateRecF *>(psc + (size_t)kWarps * cap); // byte 160 cap
    ng = reinterpret_cast<uint32_t *>(gatef + cap);               // byte 192 cap
    row = ng + cap;
    slam = reinterpret_cast<float *>(row + cap);                  // byte 200 cap
    sidx = reinterpret_cast<uint16_t *>(slam + cap);              // byte 204 cap
    pent = sidx + cap;                                            // byte 206 cap, [kWarps][cap]
    q0 = q1 = q2 = q3 = nullptr; gate = nullptr; list = nullptr; list0 = nullptr;
  }
};

// ---- TMA bulk copies (cp.async.bulk + mbarrier): the neighbour views of a node are staged in shared memory ----------
LM_D uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
LM_D void mbar_init(unsigned long long *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
LM_D void mbar_arrive_expect_tx(unsigned long long *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
LM_D void bulk_copy_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
LM_D void mbar_wait(unsigned long long *bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(done)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
  }
}

struct Cand {
  vec3<double> s, e;
  double zs, ze, unc;
  double lam_s, lam_e; // s = ray1s * lam_s + C1, e = ray1e * lam_e + C1 (not set by endpoint triangulation)
};

LM_D double4 ld_seg(const double4 *p) {
  const double2 a = __ldg(reinterpret_cast<const double2 *>(p));
  const double2 b = __ldg(reinterpret_cast<const double2 *>(p) + 1);
  return make_double4(a.x, a.y, b.x, b.y);
}
LM_D double deg_from_cos_abs(double c) { return acos(fabs(c)) * consts<double>::rad2deg(); }
// depth of X in a view: row 2 of P times [X; 1] (CameraView::projdepth)
LM_D double projdepth(const ViewD &v, vec3<double> X) { return v.P[8] * X.x + v.P[9] * X.y + v.P[10] * X.z + v.P[11]; }

// triangulate_point (triangulation/functions.cc:100-117): mid-point method, 2x2 LDLT.
LM_D bool triangulate_point(const ViewD &v1, const ViewD &v2, vec3<double> n1e, vec3<double> n2e, vec3<double> C1,
                            vec3<double> C2, vec3<double> &out) {
  double a00 = dot(n1e, n1e), a01 = -dot(n1e, n2e), a10 = -dot(n2e, n1e), a11 = dot(n2e, n2e);
  double b0 = dot(n1e, C2 - C1), b1 = dot(n2e, C1 - C2);
  double r0, r1;
  if (a00 >= a11) {
    double l10 = a10 / a00, d1 = a11 - l10 * a01, y1 = b1 - l10 * b0;
    r1 = y1 / d1;
    r0 = (b0 - a01 * r1) / a00;
  } else {
    double l01 = a01 / a11, d0 = a00 - l01 * a10, y0 = b0 - l01 * b1;
    r0 = y0 / d0;
    r1 = (b1 - a10 * r0) / a11;
  }
  out = (n1e * r0 + C1 + n2e * r1 + C2) * 0.5;
  double z1 = projdepth(v1, out);
  double z2 = projdepth(v2, out);
  return !(z1 < consts<double>::eps() || z2 < consts<double>::eps());
}

// Per-node constants of the source line (computed by one thread into shared memory: ~60 flops).
struct Src {
  double4 l1;
  vec3<double> w1s, w1e;     // M1 [p;1] (unnormalised world rays)
  vec3<double> ray1s, ray1e; // normalised
  vec3<double> C1;
  vec3<double> n1;           // getNormalDirection(l1, view1) (only for VP proposals)
  bool ok;
};

// Margin comparison of squared quantities: returns +1 / -1 when lhs is above / below rhs by more than
// 1e-9 relative (far beyond fp64 rounding of these short expressions), 0 when too close to call -- the
// caller then evaluates the reference's transcendental form for that single test.
LM_D int cmp_margin(double lhs, double rhs) {
  const double REL = 1e-9;
  if (lhs > rhs * (1.0 + REL)) return 1;
  if (lhs < rhs * (1.0 - REL)) return -1;
  return 0;
}

// Line3d::sensitivity(view) > th  (base/linebase.cc:100-107), decided without acos when clear:
// 90 - acos|c| > th  <=>  |c| > sin(th).
LM_D bool sensitivity_exceeds(const TriParams &p, const ViewD &v, vec3<double> Xs, vec3<double> Xe, vec3<double> dir_raw) {
  const vec3<double> hs = proj_h(v.P, Xs), he = proj_h(v.P, Xe);
  const double is = 1.0 / (hs.z + consts<double>::eps()), ie = 1.0 / (he.z + consts<double>::eps());
  const vec2<double> mid = mk2((hs.x * is + he.x * ie) * 0.5, (hs.y * is + he.y * ie) * 0.5);
  const vec3<double> d3 = mat3_mul_h(v.M, mid.x, mid.y);
  const double t = dot(dir_raw, d3);
  const int cm = cmp_margin(t * t, p.sin2_sens * dot(dir_raw, dir_raw) * dot(d3, d3));
  if (cm != 0 && p.sens_poly_ok) return cm > 0;
  return 90.0 - deg_from_cos_abs(dot(normalized(dir_raw), normalized(d3))) > p.sensitivity_threshold;
}

// One match row -> candidate. Steps follow triangulateOneNode "Step 3" (base_line_triangulator.cc:290-326).
// Unit-vector normalisations that do not change a decision or an output beyond rounding are dropped; the
// angle / sensitivity gates use margin forms with the reference's acos form as the tie fallback.
// The gates of a match row that need no 3D point: segment length, ray-plane angles, epipolar IoU (:290-305).
LM_D bool cand_gates(const TriParams &p, const ViewD &v2, const Src &src, const double4 &l2) {
  const vec2<double> s2 = mk2(l2.x, l2.y), e2 = mk2(l2.z, l2.w);
  const vec2<double> v2d = e2 - s2;
  const double len2sq = dot(v2d, v2d);
  { // |l2| <= min_length_2d (:177), squared with an exact tie fallback
    const double m2 = p.min_length_2d * p.min_length_2d;
    if (p.min_length_2d >= 0.0) {
      if (len2sq <= m2 * (1.0 - 1e-12)) return false;
      if (len2sq < m2 * (1.0 + 1e-12) && sqrt(len2sq) <= p.min_length_2d) return false;
    }
  }
  if (p.disable_algebraic) return false;
  const vec3<double> c2s = mat3_mul_h(v2.M, l2.x, l2.y);
  const vec3<double> c2e = mat3_mul_h(v2.M, l2.z, l2.w);
  // getNormalDirection (functions.cc:28-35) + ray-plane angle tests (:292-302):
  // 90 - acos|n2.ray| < th  <=>  |n2.ray| < sin(th)
  {
    const vec3<double> n2 = cross(c2s, c2e);
    const double nn = dot(n2, n2);
    const double ts = dot(n2, src.ray1s), te = dot(n2, src.ray1e);
    int cs_ = cmp_margin(ts * ts, p.sin2_tri * nn), ce_ = cmp_margin(te * te, p.sin2_tri * nn);
    if (!p.tri_poly_ok) cs_ = ce_ = 0;
    if (cs_ < 0 || ce_ < 0) return false; // one endpoint ray clearly below the threshold
    if (cs_ == 0 || ce_ == 0) {           // too close to call: the reference's acos form decides
      const vec3<double> n2u = normalized(n2);
      if (cs_ == 0 && 90.0 - deg_from_cos_abs(dot(n2u, src.ray1s)) < p.line_tri_angle_threshold) return false;
      if (ce_ == 0 && 90.0 - deg_from_cos_abs(dot(n2u, src.ray1e)) < p.line_tri_angle_threshold) return false;
    }
  }
  const vec3<double> C2 = mk3(v2.C[0], v2.C[1], v2.C[2]);
  // compute_epipolar_IoU (functions.cc:76-98); rejects on IoU < th, so NaN and IoU == th pass
  if (epipolar_iou(EpipolarFromRays{v2.M, src.C1 - C2, src.w1s, src.w1e}, l2, s2, e2, v2d, len2sq, p.IoU_threshold) <
      p.IoU_threshold)
    return false;
  return true;
}

// Triangulation of a row that passed cand_gates, with the gates on the 3D points (:306-326).
template <bool ALLOW_ENDP>
LM_D bool cand_triangulate(const TriParams &p, const ViewD &v1, const ViewD &v2, const Src &src, const double4 &l2, Cand &c) {
  const vec3<double> c2s = mat3_mul_h(v2.M, l2.x, l2.y);
  const vec3<double> c2e = mat3_mul_h(v2.M, l2.z, l2.w);
  const vec3<double> C2 = mk3(v2.C[0], v2.C[1], v2.C[2]);
  vec3<double> Xs, Xe;
  const double EPS = consts<double>::eps();
  if (!ALLOW_ENDP || !p.use_endpoints_triangulation) {
    // line_triangulation (functions.cc:194-233): plane-pair intersection. Only lambda_0 is used, which
    // does not depend on the norms of the second and third column.
    const vec3<double> B = C2 - src.C1;
    const vec3<double> nb = mk3(-c2s.x, -c2s.y, -c2s.z), nc = mk3(-c2e.x, -c2e.y, -c2e.z);
    const vec3<double> ls = solve3_cols(src.ray1s, nb, nc, B);
    Xs = src.ray1s * ls.x + src.C1;
    const vec3<double> le = solve3_cols(src.ray1e, nb, nc, B);
    Xe = src.ray1e * le.x + src.C1;
    c.lam_s = ls.x;
    c.lam_e = le.x;
    c.zs = projdepth(v1, Xs);
    c.ze = projdepth(v1, Xe);
    if (c.zs < EPS || c.ze < EPS) return false;
    const double d21 = projdepth(v2, Xs);
    const double d22 = projdepth(v2, Xe);
    if (d21 < EPS || d22 < EPS) return false;
    if (isnan(Xs.x) || isnan(Xe.x)) return false;
  } else {
    // triangulate_line_by_endpoints (functions.cc:172-190)
    const vec3<double> r2s = normalized(c2s), r2e = normalized(c2e);
    if (!triangulate_point(v1, v2, src.ray1s, r2s, src.C1, C2, Xs)) return false;
    if (!triangulate_point(v1, v2, src.ray1e, r2e, src.C1, C2, Xe)) return false;
    c.zs = projdepth(v1, Xs);
    c.ze = projdepth(v1, Xe);
    c.lam_s = c.lam_e = 0.0;
  }
  // sensitivity in both views (:315-317)
  const vec3<double> dir_raw = Xe - Xs;
  if (sensitivity_exceeds(p, v1, Xs, Xe, dir_raw) && sensitivity_exceeds(p, v2, Xs, Xe, dir_raw)) return false;
  // uncertainty = min(u1, u2) (:319-321; linebase.cc:109-116; camera.cc:228-242)
  {
    const double d1 = (c.zs + c.ze) / 2.0;
    const double u1 = p.var2d * d1 / v1.fbar;
    const double z2s = projdepth(v2, Xs);
    const double z2e = projdepth(v2, Xe);
    const double u2 = p.var2d * ((z2s + z2e) / 2.0) / v2.fbar;
    c.unc = smin(u1, u2);
  }
  // test_line_inside_ranges (functions.cc:8-26), written out: through a helper it changes the hot kernel's SASS
  if (p.ranges_flag) {
    if (Xs.x < p.rlo[0] || Xs.x > p.rhi[0] || Xs.y < p.rlo[1] || Xs.y > p.rhi[1] || Xs.z < p.rlo[2] || Xs.z > p.rhi[2])
      return false;
    if (Xe.x < p.rlo[0] || Xe.x > p.rhi[0] || Xe.y < p.rlo[1] || Xe.y > p.rhi[1] || Xe.z < p.rlo[2] || Xe.z > p.rhi[2])
      return false;
  }
  c.s = Xs;
  c.e = Xe;
  return true;
}

template <bool ALLOW_ENDP>
LM_D bool gen_candidate(const TriParams &p, const ViewD &v1, const ViewD &v2, const Src &src, uint32_t ngv, uint32_t ngl,
                        Cand &c, double4 &l2out) {
  const double4 l2 = ld_seg(&p.segs[p.line_off[ngv] + ngl]);
  l2out = l2;
  return cand_gates(p, v2, src, l2) && cand_triangulate<ALLOW_ENDP>(p, v1, v2, src, l2, c);
}

// triangulate_line_with_direction (triangulation/functions.cc:389-446) for a VP proposal
// (base_line_triangulator.cc:258-288): fp64, formulas as in the reference (this path is off by default).
// `direction` is the unit world direction of the VP seen from view 1.
LM_D bool gen_vp_candidate(const TriParams &p, const ViewD &v1, const ViewD &v2, const Src &src, vec3<double> c2s,
                           vec3<double> c2e, vec3<double> direction, Cand &c) {
  const double EPS = consts<double>::eps();
  const vec3<double> n1 = src.n1;
  vec3<double> direc = direction - n1 * dot(n1, direction);
  if (norm(direc) < EPS) return false;
  direc = normalized(direc);
  const vec3<double> perp = cross(n1, direc);
  double a1s = dot(src.ray1s, perp), a1e = dot(src.ray1e, perp);
  if (a1s < 0) { a1s *= -1; a1e *= -1; }
  if (a1s < 0.001 || a1e < 0.001) return false; // MIN_VALUE
  const vec3<double> C2 = mk3(v2.C[0], v2.C[1], v2.C[2]);
  const vec3<double> n2 = normalized(cross(c2s, c2e));
  const double c1s = dot(n2, src.ray1s), c1e = dot(n2, src.ray1e), b = dot(n2, C2 - src.C1);
  const double c1 = c1s, c2 = c1e * a1s / a1e;
  const double d1s = (c1 + c2) * b / (c1 * c1 + c2 * c2);
  const double d1e = d1s * a1s / a1e;
  const vec3<double> Xs = src.ray1s * d1s + src.C1, Xe = src.ray1e * d1e + src.C1;
  c.lam_s = d1s;
  c.lam_e = d1e;
  c.zs = projdepth(v1, Xs);
  c.ze = projdepth(v1, Xe);
  if (c.zs < EPS || c.ze < EPS) return false;
  const double z2s = projdepth(v2, Xs);
  const double z2e = projdepth(v2, Xe);
  if (z2s < EPS || z2e < EPS) return false;
  if (isnan(Xs.x) || isnan(Xe.x)) return false;
  const double u1 = p.var2d * ((c.zs + c.ze) / 2.0) / v1.fbar;
  const double u2 = p.var2d * ((z2s + z2e) / 2.0) / v2.fbar;
  c.unc = smin(u1, u2);
  if (p.ranges_flag) { // test_line_inside_ranges, as in cand_triangulate
    if (Xs.x < p.rlo[0] || Xs.x > p.rhi[0] || Xs.y < p.rlo[1] || Xs.y > p.rhi[1] || Xs.z < p.rlo[2] || Xs.z > p.rhi[2])
      return false;
    if (Xe.x < p.rlo[0] || Xe.x > p.rhi[0] || Xe.y < p.rlo[1] || Xe.y > p.rhi[1] || Xe.z < p.rlo[2] || Xe.z > p.rhi[2])
      return false;
  }
  c.s = Xs;
  c.e = Xe;
  return true;
}

// Pair score of candidates (i, j) of one node (global_line_triangulator.cc:91-104):
// min(LineLinker3d::compute_score(l_i, l_j), LineLinker2d::compute_score(proj_{view j}(l_i), seg_j)),
// 0 when either is 0.
LM_D double pair_score(const TriParams &p, const seg<vec3<double>> &Li, vec3<double> di, double zsi, double zei,
                       const Slab &sl, int j, uint32_t vj) {
  // 3d: angle (line_linker.cc:185-192) then scale-invariant endpoint distance (:269-277)
  const LinkerDev<double> &c3 = p.l3d;
  double score3 = 1.0;
  {
    double cs = fabs(di.x * sl.dx[j] + di.y * sl.dy[j] + di.z * sl.dz[j]);
    double angle = acos(cs) * consts<double>::rad2deg();
    score3 = smin(score3, thresh0(expscore(angle, c3.th_angle * c3.mult), c3.score_th));
    if (score3 < c3.score_th) return 0.0;
    vec3<double> sj = mk3(sl.sx[j], sl.sy[j], sl.sz[j]), ej = mk3(sl.ex[j], sl.ey[j], sl.ez[j]);
    double ds = norm(Li.s - sj), de = norm(Li.e - ej);
    double dist = smax(ds / (zsi + consts<double>::eps()), de / (zei + consts<double>::eps()));
    score3 = smin(score3, thresh0(expscore(dist, c3.th_scaleinv * c3.mult), c3.score_th));
    if (score3 == 0.0) return 0.0;
  }
  // 2d: project l_i into the view of candidate j (linebase.cc:93-98) and score against its 2D segment
  const ViewD &v = p.views[vj];
  seg<vec2<double>> a, b;
  a.s = dehom(proj_h(v.P, Li.s));
  a.e = dehom(proj_h(v.P, Li.e));
  b.s = mk2(sl.q0[j], sl.q1[j]);
  b.e = mk2(sl.q2[j], sl.q3[j]);
  double score2 = linker_score<double, vec2<double>>(p.l2d, a, b, 1.0, false, 0.0, 0.0);
  if (score2 == 0.0) return 0.0;
  return smin(score3, score2);
}

// The same pair score in algebraically reduced form (used unless innerseg is enabled on the 2d linker):
// every sub-score of the two linkers is exp(-q_k/2) with q_k = (v_k/sigma_k)^2 zeroed below score_th, and
// their minimum is exp(-max_k q_k / 2) because exp is monotone -- one exp instead of up to six; distances
// enter as squares (no square roots: (d/sigma)^2 = d^2/sigma^2, max of the four perpendicular distances =
// sqrt of the max of their squares), directions are never normalised (|cos| = |a.b|/sqrt(|a|^2|b|^2)) and
// homogeneous divisions use one reciprocal. NaN angles are ignored exactly like std::min ignores a NaN
// sub-score (line_dists.h:62-66). Polynomial early-outs skip the transcendental part for clear failures.
// asin(sqrt(t))^2 / t for 0 <= t <= 1/16 (angles up to 14.4 deg): asin^2(x) = sum_n 2^(2n-1) x^(2n) / (n^2 C(2n,n));
// 14 terms leave a relative remainder below 3e-19.
LM_D double asin2_over_t(double t) {
  double r = 0.017069849551821746;
  r = fma(r, t, 0.019089950090498877);
  r = fma(r, t, 0.02154247840073658);
  r = fma(r, t, 0.02456910759753428);
  r = fma(r, t, 0.028377319275152094);
  r = fma(r, t, 0.03328204112517838);
  r = fma(r, t, 0.03978243978243978);
  r = fma(r, t, 0.04871319157033443);
  r = fma(r, t, 0.06156806156806157);
  r = fma(r, t, 0.08126984126984127);
  r = fma(r, t, 0.11428571428571428);
  r = fma(r, t, 0.17777777777777778);
  r = fma(r, t, 0.3333333333333333);
  r = fma(r, t, 1.0);
  return r;
}
// squared angle in degrees between two directions from sin^2 = t (t <= 1/16) or from |cos| otherwise
LM_D double angle2_deg(double t, double abs_cos) {
  const double k = consts<double>::rad2deg();
  if (t <= 0.0625) return t * asin2_over_t(t) * (k * k);
  const double a = acos(abs_cos) * k;
  return a * a;
}

// Reduced-form pair score: same value as pair_score() up to rounding. min over sub-scores of exp(-(v/sigma)^2/2)
// == exp(-max (v/sigma)^2 / 2), so the squared normalised deviations are maximised and one exponential is taken;
// angles come from sin^2 (cross products) through the asin^2 series, distances stay squared, and the divisors
// that depend on one candidate only (depths of l_i, |q_j|^2) are reciprocals prepared in phase A. The 2D segment q_j is
// read through ng_j from the segment table (L1/L2-resident) rather than staged per candidate.
LM_D double pair_score_fast(const TriParams &p, const Slab &sl, int i, int j, uint32_t ngj) {
  const uint32_t vj = ngj >> 16;
  const double EPS = consts<double>::eps();
  const LinkerDev<double> &c3 = p.l3d;
  const LinkerDev<double> &c2 = p.l2d;
  const vec3<double> si = mk3(sl.sx[i], sl.sy[i], sl.sz[i]), ei = mk3(sl.ex[i], sl.ey[i], sl.ez[i]);
  double Q = 0.0; // running maximum of the squared normalised deviations
  // ---- 3d: angle (line_linker.cc:185-192) + scale-invariant endpoint distance (:269-277)
  {
    const vec3<double> di = mk3(sl.dx[i], sl.dy[i], sl.dz[i]), dj = mk3(sl.dx[j], sl.dy[j], sl.dz[j]);
    // products rounded separately: cross(di, dj) == -cross(dj, di) bit for bit, so two candidates that support
    // only each other through the angle term tie exactly, as they do with the reference's symmetric acos(|di.dj|)
    const vec3<double> cr = mk3(__dmul_rn(di.y, dj.z) - __dmul_rn(di.z, dj.y), __dmul_rn(di.z, dj.x) - __dmul_rn(di.x, dj.z),
                                __dmul_rn(di.x, dj.y) - __dmul_rn(di.y, dj.x));
    double a2 = angle2_deg(dot(cr, cr), fabs(dot(di, dj)));
    if (!(dot(di, di) * dot(dj, dj) > 0.5)) a2 = 8100.0; // zero-length candidate: acos(0) = 90 deg
    if (a2 == a2) Q = a2 * (p.inv_sig_a3 * p.inv_sig_a3);
    const vec3<double> ds = si - mk3(sl.sx[j], sl.sy[j], sl.sz[j]), de = ei - mk3(sl.ex[j], sl.ey[j], sl.ez[j]);
    const double r2 = fmax(dot(ds, ds) * sl.izs2[i], dot(de, de) * sl.ize2[i]);
    Q = fmax(Q, r2 * p.inv_sig_s3 * p.inv_sig_s3);
    if (Q > p.q_cut3) return 0.0; // some 3d sub-score is clearly below score_th
  }
  // ---- 2d: projection of l_i into the view of candidate j (linebase.cc:93-98)
  const ViewD &v = p.views[vj];
  const vec3<double> hs = proj_h(v.P, si), he = proj_h(v.P, ei);
  const double ws = 1.0 / (hs.z + EPS), we = 1.0 / (he.z + EPS);
  const vec2<double> as = mk2(hs.x * ws, hs.y * ws), ae = mk2(he.x * we, he.y * we);
  const double4 q = ld_seg(&p.segs[p.line_off[vj] + (ngj & 0xffffu)]);
  const vec2<double> bs = mk2(q.x, q.y), be = mk2(q.z, q.w);
  const vec2<double> va = ae - as, vb = be - bs;
  const double na2 = dot(va, va), nb2 = dot(vb, vb);
  const double dab = dot(va, vb);
  const double ina = 1.0 / na2, inb = sl.inb[j];
  double Q2 = 0.0;
  double ang2 = 0.0; // squared 2d angle in degrees
  if (c2.use_angle) {
    if (dab * dab < p.cos2_th2d * na2 * nb2 * (1.0 - 1e-9)) return 0.0; // |cos| clearly below cos(th_angle)
    if (na2 > 0.0 && nb2 > 0.0) {
      const double cr = va.x * vb.y - va.y * vb.x;
      const double t = cr * cr * (ina * inb);
      ang2 = angle2_deg(t, (t <= 0.0625) ? 0.0 : fabs(dab) / sqrt(na2 * nb2));
    } else {
      ang2 = 8100.0; // acos(0) = 90 deg
    }
    if (ang2 == ang2) Q2 = ang2 * (p.inv_sig_a2 * p.inv_sig_a2);
  }
  double bio = 0.0;
  if (c2.use_overlap) { // compute_bioverlap (line_dists.h:190-208)
    double p1 = dot(as - bs, vb) * inb, p2 = dot(ae - bs, vb) * inb;
    if (p1 > p2) { const double t = p1; p1 = p2; p2 = t; }
    const double o1 = smin(p2, 1.0) - smax(p1, 0.0);
    double r1 = dot(bs - as, va) * ina, r2 = dot(be - as, va) * ina;
    if (r1 > r2) { const double t = r1; r1 = r2; r2 = t; }
    const double o2 = smin(r2, 1.0) - smax(r1, 0.0);
    bio = smax(o1, o2);
    if (!(bio > c2.th_overlap)) return 0.0;
  }
  if (c2.use_angle && c2.use_overlap && c2.use_smartangle && bio < c2.th_smartoverlap) { // line_linker.cc:49-65
    double ratio = (c2.th_smartoverlap - bio) * p.inv_smart_den2;
    ratio = smin(ratio, 1.0);
    const double sig = (c2.th_angle - ratio * (c2.th_angle - c2.th_smartangle)) * c2.mult;
    if (ang2 == ang2) Q2 = fmax(Q2, ang2 / (sig * sig));
  }
  if (c2.use_perp) { // max of the four endpoint-to-infinite-line distances, squared (line_dists.h:105-133)
    const vec2<double> d0 = as - bs, d1 = ae - bs, d2 = bs - as, d3 = be - as;
    const double t0 = dot(d0, vb), t1 = dot(d1, vb), t2 = dot(d2, va), t3 = dot(d3, va);
    double m = fmax(dot(d0, d0) - t0 * t0 * inb, 0.0);
    m = fmax(m, dot(d1, d1) - t1 * t1 * inb);
    m = fmax(m, dot(d2, d2) - t2 * t2 * ina);
    m = fmax(m, dot(d3, d3) - t3 * t3 * ina);
    Q2 = fmax(Q2, m * p.inv_sig_p2 * p.inv_sig_p2);
  }
  // each linker applies its own score_th: exp(-Q/2) >= th <=> Q <= -2 ln th. Clear of both cuts by 1e-9 relative,
  // one exponential of the larger deviation is the score; next to a cut the two exponentials decide.
  if (Q2 > p.q_cut2) return 0.0;
  if (Q < p.q_cut3_lo && Q2 < p.q_cut2_lo) return exp(-fmax(Q, Q2) * 0.5);
  const double e3 = exp(-Q * 0.5), e2 = exp(-Q2 * 0.5);
  if (e3 < c3.score_th || e2 < c2.score_th) return 0.0;
  return smin(e3, e2);
}

// ---- pruning gates -----------------------------------------------------------------------------------
// The reference decides every sub-test on exp(-(v/sigma)^2/2) >= score_th, i.e. v <= th. The gates below
// only discard pairs that fail a sub-test by a margin far above the arithmetic error of the gate (fp32
// for the 3d tests, fp64 polynomial forms for the 2d tests); every surviving pair is then scored by
// pair_score(), which evaluates the reference formulas in fp64 and takes all decisions itself. Pruned
// pairs would have scored exactly 0, so results do not depend on the gates.

// 3d gate, fp32: angle (line_linker.cc:185-192) and the end-point half of the scale-invariant endpoint distance
// (:269-277); the start-point half is the generic phase B's prefilter.
LM_D bool gate3d_rest(const GateRec &r, const GateRec *g, float cos_th) {
  const float4 a = *reinterpret_cast<const float4 *>(&g->dx);
  if (fabsf(r.dx * a.x + r.dy * a.y + r.dz * a.z) < cos_th) return false;
  const float4 c = *reinterpret_cast<const float4 *>(&g->ex);
  const float bx = r.ex - c.x, by = r.ey - c.y, bz = r.ez - c.z;
  return !(bx * bx + by * by + bz * bz > r.lime2);
}

// 2d gate, fp64 without transcendentals: angle, overlap and perpendicular tests of
// LineLinker2d::compute_score (line_linker.cc:139-160) in margin form.
LM_D bool gate2d(const TriParams &p, const seg<vec3<double>> &Li, const Slab &sl, int j, uint32_t vj) {
  const LinkerDev<double> &c = p.l2d;
  const ViewD &v = p.views[vj];
  const vec2<double> as = dehom(proj_h(v.P, Li.s)), ae = dehom(proj_h(v.P, Li.e));
  const vec2<double> bs = mk2(sl.q0[j], sl.q1[j]), be = mk2(sl.q2[j], sl.q3[j]);
  const vec2<double> va = ae - as, vb = be - bs;
  const double na2 = dot(va, va), nb2 = dot(vb, vb);
  const double REL = 1e-9;
  if (c.use_angle) {
    const double d = dot(va, vb);
    if (d * d < p.cos2_th2d * na2 * nb2 * (1.0 - REL)) return false; // |cos| < cos(th_angle)
  }
  if (c.use_overlap) {
    // compute_bioverlap (line_dists.h:190-208) with p = dot / |l2|^2 (no normalisation)
    double p1 = dot(as - bs, vb) / nb2, p2 = dot(ae - bs, vb) / nb2;
    if (p1 > p2) { const double t = p1; p1 = p2; p2 = t; }
    const double o1 = smin(p2, 1.0) - smax(p1, 0.0);
    double r1 = dot(bs - as, va) / na2, r2 = dot(be - as, va) / na2;
    if (r1 > r2) { const double t = r1; r1 = r2; r2 = t; }
    const double o2 = smin(r2, 1.0) - smax(r1, 0.0);
    const double bio = smax(o1, o2);
    if (bio < c.th_overlap - REL * (1.0 + fabs(c.th_overlap))) return false;
  }
  if (c.use_perp) {
    // squared endpoint-to-infinite-line distances (line_dists.h:105-133)
    const vec2<double> d0 = as - bs, d1 = ae - bs, d2 = bs - as, d3 = be - as;
    const double t0 = dot(d0, vb), t1 = dot(d1, vb), t2 = dot(d2, va), t3 = dot(d3, va);
    double m = dot(d0, d0) - t0 * t0 / nb2;
    m = fmax(m, dot(d1, d1) - t1 * t1 / nb2);
    m = fmax(m, dot(d2, d2) - t2 * t2 / na2);
    m = fmax(m, dot(d3, d3) - t3 * t3 / na2);
    if (m > p.th_perp2_2d * (1.0 + REL) + REL) return false;
  }
  return true;
}

// ---- node kernel (DESIGN.md §3.1) -----------------------------------------------------------------------
// Block-wide exclusive prefix of one value per thread in thread order; tot is the block's sum. Every thread of the CTA
// calls it; s_wtot is free again after the caller's next barrier.
LM_D int block_exclusive_scan(int v, int lane, int warp, int *s_wtot, int &tot) {
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) s_wtot[warp] = incl;
  __syncthreads();
  int woff = 0;
  tot = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    if (w < warp) woff += s_wtot[w];
    tot += s_wtot[w];
  }
  return woff + incl - v;
}

// Phase C: valid connections, best candidate, node record and counters (:115-153). s_nvalid is 0 on entry.
template <int NS>
LM_D void phase_c(const TriParams &p, const Slab &sl, int C, uint32_t r0, NodeRecord *rec, int tid, int lane, int warp,
                  int *s_nvalid) {
  int nvalid_local = 0;
  for (int i = tid; i < C; i += kThreads) {
    const double sc = sl.score[i];
    bool valid = sc >= p.fullscore_th; // `if (score < fullscore_th) continue;`
    if (valid && C > p.max_valid_conns) {
      // rank in the (score, tri_id) descending order of std::greater<pair<double,int>> (:128-129)
      int rank = 0;
      for (int k = 0; k < C; ++k) {
        const double sk = sl.score[k];
        rank += (sk > sc) || (sk == sc && k > i);
      }
      valid = rank < p.max_valid_conns;
    }
    p.row_state[(int64_t)r0 * NS + sl.row[i]] = valid ? 2 : 1;
    nvalid_local += valid;
    if (p.row_cand) {
      double *o = p.row_cand + ((int64_t)r0 * NS + sl.row[i]) * 10;
      o[0] = sl.sx[i]; o[1] = sl.sy[i]; o[2] = sl.sz[i]; o[3] = sl.ex[i]; o[4] = sl.ey[i]; o[5] = sl.ez[i];
      o[6] = sl.zs[i]; o[7] = sl.ze[i]; o[8] = sl.unc[i]; o[9] = sc;
    }
  }
  if (nvalid_local) atomicAdd(s_nvalid, nvalid_local);
  // best: first strict maximum from max_score = -1 (:145-153) == max score, lowest index on ties.
  if (warp == 0) {
    double bs = -1.0;
    int bi = -1;
    for (int i = lane; i < C; i += 32) {
      const double sc = sl.score[i];
      if (sc > bs) { bs = sc; bi = i; }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const double os = __shfl_down_sync(0xffffffffu, bs, d);
      const int oi = __shfl_down_sync(0xffffffffu, bi, d);
      if (oi >= 0 && (os > bs || (os == bs && (bi < 0 || oi < bi)))) { bs = os; bi = oi; }
    }
    bi = __shfl_sync(0xffffffffu, bi, 0);
    if (bi >= 0) {
      if (lane < 3) rec->line[lane] = (lane == 0) ? sl.sx[bi] : (lane == 1 ? sl.sy[bi] : sl.sz[bi]);
      else if (lane < 6) rec->line[lane] = (lane == 3) ? sl.ex[bi] : (lane == 4 ? sl.ey[bi] : sl.ez[bi]);
      else if (lane == 6) rec->line[6] = sl.zs[bi];
      else if (lane == 7) rec->line[7] = sl.ze[bi];
      else if (lane == 8) rec->line[8] = sl.unc[bi];
      else if (lane == 9) rec->score = sl.score[bi];
      else if (lane == 10) { rec->ng_view = (int32_t)(sl.ng[bi] >> 16); rec->ng_line = (int32_t)(sl.ng[bi] & 0xffffu); }
    } else {
      if (lane < 9) rec->line[lane] = (lane == 8) ? -1.0 : 0.0;
      if (lane == 9) rec->score = 0.0;
      if (lane == 10) { rec->ng_view = 0; rec->ng_line = 0; }
    }
  }
  __syncthreads();
  if (tid == 0) {
    rec->n_cand = C;
    rec->n_valid = *s_nvalid;
    if (C) atomicAdd(&p.counters[0], (unsigned long long)C);
    if (*s_nvalid) atomicAdd(&p.counters[1], (unsigned long long)*s_nvalid);
  }
  __syncthreads();
}

// One CTA per node (2D line), grid-stride over the nodes of the launch. FAST: reduced-form scorer and plane-pair
// triangulation only (the default configuration); the generic instantiation keeps the reference-structured scorer, the
// 2d margin gates and endpoint triangulation. Splitting them keeps the hot kernel's code (and instruction-cache
// footprint) small. Only phase C is a function: phase A, the fast phase B or its partner test as functions change the
// SASS of <false, false, true>, and the view staging with the generic phase B as functions change the others' spills.
template <bool SLAB, bool VP, bool FAST>
__global__ void __launch_bounds__(kThreads, (!SLAB && !VP && FAST) ? LM_TRI_MIN_BLOCKS : 4)
    tri_node_kernel(const __grid_constant__ TriParams p) {
  constexpr int NS = VP ? 3 : 1; // proposal slots per match row: [vp1, vp2, algebraic] (base_line_triangulator.cc:258-326)
  // neighbour-view staging (TMA bulk copies) on the VP instantiation only: on the headline one it measured slower than
  // the L1-cached loads it replaces (DESIGN.md §3.1)
  constexpr bool STAGE = FAST && !SLAB && VP;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int s_wtot[kWarps];
  __shared__ int s_nvalid;
  __shared__ int s_next_row;
  __shared__ Src s_src; // per-node constants of the source line: held in registers they spill in phase A
  __shared__ __align__(8) unsigned long long s_mbar; // completion of the neighbour-view bulk copies of a node
  uint32_t mbar_parity = 0;
  if constexpr (STAGE) {
    if (threadIdx.x == 0) mbar_init(&s_mbar, 1);
    __syncthreads();
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  Slab sl;
  if (SLAB) sl.carve(p.slab + (int64_t)blockIdx.x * p.slab_stride, p.cap, FAST);
  else sl.carve(reinterpret_cast<char *>(smem_raw), p.cap, FAST);
  uint32_t *list1 = FAST ? nullptr : sl.list + (size_t)(warp * 2) * (p.cap + kListExtra);
  uint32_t *list2 = FAST ? nullptr : list1 + p.cap + kListExtra;
  uint16_t *list0 = FAST ? nullptr : sl.list0 + (size_t)warp * p.cap;
  unsigned long long n1_total = 0, n2_total = 0;

  for (int64_t node = p.node_begin + blockIdx.x; node < p.node_end; node += gridDim.x) {
    const uint32_t r0 = p.node_row_off[node], r1 = p.node_row_off[node + 1];
    const int nrows = (int)(r1 - r0);
    NodeRecord *rec = &p.nodes[node];
    if (nrows == 0 || nrows * NS > p.cap) {
      if (tid < 9) rec->line[tid] = (tid == 8) ? -1.0 : 0.0;
      if (tid == 9) { rec->score = 0.0; rec->ng_view = 0; rec->ng_line = 0; rec->n_cand = 0; rec->n_valid = 0; }
      if (nrows != 0 && tid == 10) *p.overflow = 1; // staging area sized from a stale hint: the host repeats the run
      continue;
    }
    // ---------------- phase A: candidate generation with stable compaction -----------------
    // ---- neighbour views of the node -> shared memory. Rows are ordered by neighbour view, so a new view starts where
    // the view index changes; the thread that sees the change issues one 208-byte TMA bulk copy (cp.async.bulk,
    // completion on an mbarrier) into the view's slot. Phase A then reads K|R|t-derived blocks from shared memory
    // instead of chasing row -> view index -> global view record. The staging area aliases the phase-B score lists.
    const ViewD *sviews = nullptr;
    const uint8_t *slot_of_row = nullptr;
    int n_stage = 0;
    if constexpr (STAGE) {
      const int stage_off = p.cap * 4; // the depth-sort keys written by phase A come first
      ViewD *sv = reinterpret_cast<ViewD *>(reinterpret_cast<char *>(sl.psc) + stage_off);
      uint8_t *slots = reinterpret_cast<uint8_t *>(sl.sidx); // [nrows <= cap]; rewritten by the depth sort afterwards
      const int stage_cap = min(255, (int)(((size_t)kWarps * p.cap * 8 - stage_off) / sizeof(ViewD)));
      int carry = 0;
      for (int base = 0; base < nrows; base += kThreads) {
        const int r = base + tid;
        uint32_t view = 0;
        int flag = 0;
        if (r < nrows) {
          view = __ldg(&p.row_ng[r0 + r]) >> 16;
          flag = (r == 0) || ((__ldg(&p.row_ng[r0 + r - 1]) >> 16) != view);
        }
        int incl = flag;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int o = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += o;
        }
        if (lane == 31) s_wtot[warp] = incl;
        __syncthreads();
        int woff = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
          if (w < warp) woff += s_wtot[w];
          tot += s_wtot[w];
        }
        const int slot = carry + woff + incl - 1;
        if (r < nrows) slots[r] = (uint8_t)min(slot, 255);
        if (flag && slot < stage_cap) bulk_copy_g2s(sv + slot, p.views + view, (uint32_t)sizeof(ViewD), &s_mbar);
        carry += tot;
        __syncthreads();
      }
      n_stage = min(carry, stage_cap);
      if (tid == 0) mbar_arrive_expect_tx(&s_mbar, (uint32_t)(n_stage * sizeof(ViewD)));
      sviews = sv;
      slot_of_row = slots; // (the copies are awaited after the source-line constants below: their latency is hidden)
    }
    const uint32_t v1i = p.node_view[node];
    const ViewD &v1 = p.views[v1i];
    if (tid == 0) {
      Src src;
      src.l1 = ld_seg(&p.segs[node]);
      double dx = src.l1.x - src.l1.z, dy = src.l1.y - src.l1.w;
      src.ok = !(sqrt(dx * dx + dy * dy) <= p.min_length_2d); // :166
      src.w1s = mat3_mul_h(v1.M, src.l1.x, src.l1.y);
      src.w1e = mat3_mul_h(v1.M, src.l1.z, src.l1.w);
      src.ray1s = normalized(src.w1s);
      src.ray1e = normalized(src.w1e);
      src.C1 = mk3(v1.C[0], v1.C[1], v1.C[2]);
      src.n1 = normalized(cross(src.w1s, src.w1e));
      s_src = src;
    }
    __syncthreads();
    const Src &src = s_src;
    if constexpr (STAGE) {
      mbar_wait(&s_mbar, mbar_parity);
      mbar_parity ^= 1u;
    }
    int count = 0;
    for (int base = 0; base < nrows; base += kThreads) {
      const int r = base + tid;
      Cand cs[NS];
      bool oks[NS];
#pragma unroll
      for (int k = 0; k < NS; ++k) oks[k] = false;
      double4 l2 = make_double4(0, 0, 0, 0);
      uint32_t ng = 0;
      if (r < nrows && src.ok) {
        ng = __ldg(&p.row_ng[r0 + r]);
        const uint32_t ngv = ng >> 16, ngl = ng & 0xffffu;
        if (VP) {
          // Step 2 (:258-288): proposals from the VP of the source line and of the matched line; both use view 1
          const double4 l2v = ld_seg(&p.segs[p.line_off[ngv] + ngl]);
          const double ddx = l2v.x - l2v.z, ddy = l2v.y - l2v.w;
          if (!(sqrt(ddx * ddx + ddy * ddy) <= p.min_length_2d) && !p.disable_vp) {
            const ViewD *v2q = &p.views[ngv];
            if constexpr (STAGE) {
              const int slot = slot_of_row[r];
              if (slot < n_stage) v2q = &sviews[slot];
            }
            const ViewD &v2 = *v2q;
            const vec3<double> c2s = mat3_mul_h(v2.M, l2v.x, l2v.y), c2e = mat3_mul_h(v2.M, l2v.z, l2v.w);
            const int lab1 = p.vp_label[node];
            if (lab1 >= 0) {
              const double *vp = p.vps + 3 * (p.vp_off[v1i] + lab1);
              oks[0] = gen_vp_candidate(p, v1, v2, src, c2s, c2e, normalized(mat3_mul(v1.M, mk3(vp[0], vp[1], vp[2]))), cs[0]);
            }
            const int lab2 = p.vp_label[p.line_off[ngv] + ngl];
            if (lab2 >= 0) {
              const double *vp = p.vps + 3 * (p.vp_off[ngv] + lab2);
              oks[1] = gen_vp_candidate(p, v1, v2, src, c2s, c2e, normalized(mat3_mul(v1.M, mk3(vp[0], vp[1], vp[2]))), cs[1]);
            }
          }
          l2 = l2v;
        }
        const ViewD *v2p = &p.views[ngv];
        if constexpr (STAGE) {
          const int slot = slot_of_row[r];
          if (slot < n_stage) v2p = &sviews[slot];
        }
        oks[NS - 1] = gen_candidate<!FAST>(p, v1, *v2p, src, ngv, ngl, cs[NS - 1], l2);
      }
      int cnt = 0;
#pragma unroll
      for (int k = 0; k < NS; ++k) {
        if (r < nrows) p.row_state[(int64_t)(r0 + r) * NS + k] = 0;
        cnt += oks[k];
      }
      // the fast layout keeps only 1/|q|^2 of the matched segment: with |q|^2 taken before the barrier, l2 is dead
      // across it
      const double qx = l2.z - l2.x, qy = l2.w - l2.y;
      const double nq2 = qx * qx + qy * qy;
      // stable compaction: exclusive prefix of the per-row candidate counts
      int tot;
      int idx = count + block_exclusive_scan(cnt, lane, warp, s_wtot, tot);
#pragma unroll
      for (int k = 0; k < NS; ++k) {
        if (!oks[k]) continue;
        const Cand &c = cs[k];
        const vec3<double> dr = c.e - c.s;
        const double dn2 = dot(dr, dr);
        const vec3<double> d = (dn2 > 0.0) ? dr * (1.0 / sqrt(dn2)) : dr;
        sl.sx[idx] = c.s.x; sl.sy[idx] = c.s.y; sl.sz[idx] = c.s.z;
        sl.ex[idx] = c.e.x; sl.ey[idx] = c.e.y; sl.ez[idx] = c.e.z;
        sl.dx[idx] = d.x; sl.dy[idx] = d.y; sl.dz[idx] = d.z;
        sl.zs[idx] = c.zs; sl.ze[idx] = c.ze; sl.unc[idx] = c.unc;
        if (FAST) {
          const double zs1 = c.zs + consts<double>::eps(), ze1 = c.ze + consts<double>::eps();
          sl.izs2[idx] = 1.0 / (zs1 * zs1); sl.ize2[idx] = 1.0 / (ze1 * ze1); sl.inb[idx] = 1.0 / nq2;
        } else {
          sl.q0[idx] = l2.x; sl.q1[idx] = l2.y; sl.q2[idx] = l2.z; sl.q3[idx] = l2.w;
        }
        sl.ng[idx] = ng;
        sl.row[idx] = (uint32_t)r * NS + k;
        if (FAST) {
          // fp32 gate record: the endpoints as distances along the two source rays. Limits: th * (z + EPS) widened by
          // 0.5% plus 1e-5 of the larger distance (fp32 rounding of the two lambdas and of their difference is below
          // 2e-7 of it, |X_i - X_j| and |lambda_i - lambda_j| agree to 1e-15); see DESIGN.md "gates"
          const double rad = fmax(fabs(c.lam_s), fabs(c.lam_e));
          const double ls = p.l3d.th_scaleinv * (c.zs + consts<double>::eps()) * 1.005 + 1e-5 * rad;
          const double le = p.l3d.th_scaleinv * (c.ze + consts<double>::eps()) * 1.005 + 1e-5 * rad;
          GateRecF g;
          g.dx = (float)d.x; g.dy = (float)d.y; g.dz = (float)d.z; g.lam_e = (float)c.lam_e;
          g.lam_s = (float)c.lam_s; g.lim_s = (float)(ls * 1.000001); g.lim_e = (float)(le * 1.000001);
          g.img = (int)(ng >> 16);
          sl.gatef[idx] = g;
          reinterpret_cast<float *>(sl.psc)[idx] = g.lam_s; // unsorted keys of the depth sort (scratch: the score lists)
        } else {
          // fp32 gate copy, relative to the source camera centre (keeps |coord| ~ depth)
          const vec3<double> rs = c.s - src.C1, re = c.e - src.C1;
          // scale-invariance limit th * (z + EPS) widened by 0.5% plus 1e-5 of the coordinate magnitude
          // (fp32 rounding of the two endpoints is < 1e-6 of it); see DESIGN.md "gates"
          const double rad = sqrt(fmax(dot(rs, rs), dot(re, re)));
          const double ls = p.l3d.th_scaleinv * (c.zs + consts<double>::eps()) * 1.005 + 1e-5 * rad;
          const double le = p.l3d.th_scaleinv * (c.ze + consts<double>::eps()) * 1.005 + 1e-5 * rad;
          GateRec g;
          g.dx = (float)d.x; g.dy = (float)d.y; g.dz = (float)d.z; g.lims2 = (float)(ls * ls * 1.000001);
          g.sx = (float)rs.x; g.sy = (float)rs.y; g.sz = (float)rs.z; g.lime2 = (float)(le * le * 1.000001);
          g.ex = (float)re.x; g.ey = (float)re.y; g.ez = (float)re.z;
          g.pad = 0.f;
          sl.gate[idx] = g;
        }
        ++idx;
      }
      count += tot;
      __syncthreads();
    }
    const int C = count;
    if (tid == 0) { s_nvalid = 0; s_next_row = 0; }
    __syncthreads();
    // ---------------- phase B: all-pairs scoring ------------------------------------------------
    if constexpr (FAST) {
      // All candidates of the node start on one ray and end on another (GateRecF), so "l_j can score against l_i"
      // needs |lam_s(j) - lam_s(i)| <= lim_s(i): after a sort by lam_s the partners of a row are a contiguous window.
      //   B-sort   rank sort of the candidates by lam_s (ties by index), whole CTA
      //   per warp, 32 rows at a time (lane = row):
      //   B-window two binary searches per row
      //   B-gate   the other fp32 gates (end-point interval, angle, other image) over the window, twice: count, then
      //            write -- each row's partners land contiguously in the warp's pair list, no atomics, no compaction
      //   B-score  exact fp64 scores of the pair list, 32 pairs per step (lane = pair; rows found by a search over
      //            the lanes' offsets)
      //   B-sum    lane = row again: maximum per neighbour image, images added in ascending order -- the order of the
      //            reference's std::map (:105-112), so a row's total does not depend on how the work was split.
      // Pruned pairs would have scored exactly 0 (DESIGN.md "Exactness argument"); every surviving pair is scored by
      // pair_score_fast in fp64.
      const unsigned FULL = 0xffffffffu;
      {
        float *ltmp = reinterpret_cast<float *>(sl.psc);
        const int C4 = (C + 3) & ~3;
        if (tid < C4 - C) ltmp[C + tid] = __int_as_float(0x7f800000); // +inf pads: never below a key, never tie-winners
        __syncthreads();
        for (int i = tid; i < C; i += kThreads) {
          const float li = ltmp[i];
          int r = 0;
          for (int j4 = 0; j4 < C4; j4 += 4) {
            const float4 v = *reinterpret_cast<const float4 *>(ltmp + j4);
            r += (v.x < li) || (v.x == li && j4 < i);
            r += (v.y < li) || (v.y == li && j4 + 1 < i);
            r += (v.z < li) || (v.z == li && j4 + 2 < i);
            r += (v.w < li) || (v.w == li && j4 + 3 < i);
          }
          sl.slam[r] = li;
          sl.sidx[r] = (uint16_t)i;
        }
        __syncthreads(); // ltmp (= the score lists) is dead from here on
      }
      const float *slam = sl.slam;
      const uint16_t *sidx = sl.sidx;
      double *psc = sl.psc + (size_t)warp * p.cap;
      uint16_t *pent = sl.pent + (size_t)warp * p.cap;
      // rows are dealt to the warps in equal shares (C = 100: 25 rows per warp, not 32 + 32 + 32 + 4), so the warps
      // reach the barrier before phase C together
      const int n_pass = (C + 32 * kWarps - 1) / (32 * kWarps);
      const int G = (C + kWarps * n_pass - 1) / (kWarps * n_pass); // rows per warp and pass, <= 32
      for (int pass = 0; pass < n_pass; ++pass) {
        const int g0 = (pass * kWarps + warp) * G;
        if (g0 >= C) break;
        const int Gact = min(G, C - g0);
        // B-window, lane = row: two binary searches over the sorted start distances
        int lo = 0, W = 0;
        if (lane < Gact) {
          const float4 a1 = *reinterpret_cast<const float4 *>(&sl.gatef[g0 + lane].lam_s);
          int hi = C;
          if (a1.y < 3e37f) { // (false for inf / NaN limits: the whole node is the window then)
            const float wa = a1.x - a1.y, wb = a1.x + a1.y;
            int l = 0, h = C;
            while (l < h) { const int m = (l + h) >> 1; if (slam[m] < wa) l = m + 1; else h = m; }
            lo = l;
            h = C;
            while (l < h) { const int m = (l + h) >> 1; if (!(slam[m] > wb)) l = m + 1; else h = m; }
            hi = l;
          }
          W = hi - lo;
        }
        int rr = 0;
        while (rr < Gact) {
          // B-gate, one row at a time, lane = window position: the other fp32 gates (end-point interval, angle, other
          // image). The partners of a row are written in ascending candidate order (= ascending neighbour image:
          // candidates are generated image by image) at the running fill of the warp's pair list; lane r keeps the
          // offset and the count of row r of the chunk. A chunk ends when the next row would not fit the list.
          const int cb = rr;
          int fill = 0, off = 0, n = 0;
          for (; rr < Gact; ++rr) {
            const int lo_r = __shfl_sync(FULL, lo, rr), W_r = __shfl_sync(FULL, W, rr);
            const float4 a0 = *reinterpret_cast<const float4 *>(&sl.gatef[g0 + rr].dx);
            const float4 a1 = *reinterpret_cast<const float4 *>(&sl.gatef[g0 + rr].lam_s);
            int n_r = 0;
            if (W_r <= 32) {
              int j = 0x7fffffff;
              bool ok = false;
              if (lane < W_r) {
                j = sidx[lo_r + lane];
                const float4 gj = *reinterpret_cast<const float4 *>(&sl.gatef[j].dx);
                const int imgj = sl.gatef[j].img;
                ok = (imgj != __float_as_int(a1.w)) && !(fabsf(gj.w - a0.w) > a1.z) &&
                     !(fabsf(a0.x * gj.x + a0.y * gj.y + a0.z * gj.z) < p.cos_th3d_f);
              }
              unsigned m = __ballot_sync(FULL, ok);
              n_r = __popc(m);
              if (n_r) {
                if (fill + n_r > p.cap) break; // (a row has fewer than C <= cap partners: an empty list always takes it)
                int rank = 0;
                while (m) { // rank among the partners by candidate index: n_r independent shuffles
                  const int t = __ffs((int)m) - 1;
                  m &= m - 1;
                  rank += __shfl_sync(FULL, j, t) < j;
                }
                if (ok) pent[fill + rank] = (uint16_t)j;
              }
            } else {
              // wide window: partners appended unordered to scratch (the score slots of this chunk's tail are free until
              // B-score), then placed by rank
              uint16_t *tmp = reinterpret_cast<uint16_t *>(psc + fill);
              bool fits = true;
              for (int tb = 0; tb < W_r; tb += 32) {
                const int t = tb + lane;
                int j = 0;
                bool ok = false;
                if (t < W_r) {
                  j = sidx[lo_r + t];
                  const float4 gj = *reinterpret_cast<const float4 *>(&sl.gatef[j].dx);
                  const int imgj = sl.gatef[j].img;
                  ok = (imgj != __float_as_int(a1.w)) && !(fabsf(gj.w - a0.w) > a1.z) &&
                       !(fabsf(a0.x * gj.x + a0.y * gj.y + a0.z * gj.z) < p.cos_th3d_f);
                }
                const unsigned m = __ballot_sync(FULL, ok);
                if (fill + n_r + __popc(m) > p.cap) { fits = false; break; }
                if (ok) tmp[n_r + __popc(m & lt_mask)] = (uint16_t)j;
                n_r += __popc(m);
              }
              if (!fits) break;
              __syncwarp();
              // (tmp occupies 2 bytes per partner inside psc[fill ..), pent[fill ..) is a different array)
              for (int e = lane; e < n_r; e += 32) {
                const uint16_t v = tmp[e];
                int rank = 0;
                for (int x = 0; x < n_r; ++x) rank += tmp[x] < v;
                pent[fill + rank] = v;
              }
            }
            if (lane == rr) { off = fill; n = n_r; }
            fill += n_r;
          }
          const int ce = rr;
          n1_total += (unsigned long long)fill;
          __syncwarp();
          // B-score: exact reference scores, lane = pair
          for (int fb = 0; fb < fill; fb += 32) {
            const int f = fb + lane;
            int r = cb; // largest row of the chunk whose offset is <= f (rows without partners share the next offset)
#pragma unroll
            for (int step = 16; step >= 1; step >>= 1) {
              const int cand = r + step;
              const int v = __shfl_sync(FULL, off, cand & 31);
              if (cand < ce && v <= f) r = cand;
            }
            if (f < fill) {
              const int j = pent[f];
              psc[f] = pair_score_fast(p, sl, g0 + r, j, sl.ng[j]);
            }
          }
          n2_total += (unsigned long long)fill;
          __syncwarp();
          // B-sum: one image contributes its maximum once (:110-112), images in ascending order (the partners of a row
          // are sorted by candidate index, i.e. by image)
          if (lane >= cb && lane < ce) {
            double sum = 0.0, mx = 0.0;
            int cur = -1;
            for (int e = 0; e < n; ++e) {
              const int im = sl.gatef[pent[off + e]].img;
              const double sc = psc[off + e];
              if (im != cur) { sum += mx; cur = im; mx = sc; }
              else mx = (mx > sc) ? mx : sc;
            }
            sum += mx;
            sl.score[g0 + lane] = sum;
          }
          __syncwarp();
        }
      }
      __syncthreads();
    } else {
    // Warps fetch rows i dynamically. B1 prunes (i, j) pairs with the fp32 3d gates and appends the
    // survivors of several rows to a warp-private list until it holds >= kFlush entries, so that the fp64
    // stages B2 (2d margin gates) and B3 (exact reference score) run on dense 32-lane batches.
    for (int i = tid; i < C; i += kThreads) sl.score[i] = 0.0;
    // records up to the next multiple of 32 can never pass the start-point test: the prefilter loop needs no bounds
    if (tid < 32 && C + tid < ((C + 31) & ~31)) {
      GateRec z;
      z.dx = z.dy = z.dz = 0.f; z.lims2 = 0.f;
      z.sx = z.sy = z.sz = 3e18f; z.lime2 = 0.f;
      z.ex = z.ey = z.ez = 3e18f; z.pad = 0.f;
      sl.gate[C + tid] = z;
    }
    __syncthreads();
    bool more = true;
    while (more) {
      int n1 = 0;
      while (n1 < kFlush) {
        int i = 0;
        if (lane == 0) i = atomicAdd(&s_next_row, 1);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= C) { more = false; break; }
        const GateRec rf = sl.gate[i];
        const uint32_t vi = sl.ng[i] >> 16;
        // B0: start-point prefilter. The scale-invariant endpoint test (line_linker.cc:269-277, th_scaleinv of the
        // depth) is by far the most selective 3d test, so its start-point half runs first on every candidate (one
        // 16-byte load, 8 flops); the other gates only see the survivors. (A byte-hash of the log distance tested
        // four candidates per lane was measured slower: more false positives reach B1 than it saves here.)
        int n0 = 0;
        for (int jb = 0; jb < C; jb += 32) {
          const int j = jb + lane;
          const float4 b = *reinterpret_cast<const float4 *>(&sl.gate[j].sx);
          const float ax = rf.sx - b.x, ay = rf.sy - b.y, az = rf.sz - b.z;
          const bool pass = !(ax * ax + ay * ay + az * az > rf.lims2);
          const unsigned bal = __ballot_sync(0xffffffffu, pass);
          if (pass) list0[n0 + __popc(bal & lt_mask)] = (uint16_t)j;
          n0 += __popc(bal);
        }
        __syncwarp();
        // B1: the other fp32 3d gates (angle, end point) and the same-image exclusion (which also drops j == i)
        for (int kb = 0; kb < n0; kb += 32) {
          const int k = kb + lane;
          bool pass = false;
          int j = 0;
          if (k < n0) {
            j = list0[k];
            pass = (sl.ng[j] >> 16) != vi && gate3d_rest(rf, &sl.gate[j], p.cos_th3d_f);
          }
          const unsigned bal = __ballot_sync(0xffffffffu, pass);
          if (pass) list1[n1 + __popc(bal & lt_mask)] = ((uint32_t)i << 16) | (uint32_t)j;
          n1 += __popc(bal);
        }
        __syncwarp();
      }
      __syncwarp();
      n1_total += n1;
      if (n1 == 0) continue;
      // B2: fp64 margin gates of the 2d tests
      int n2 = 0;
      for (int kb = 0; kb < n1; kb += 32) {
        const int k = kb + lane;
        bool pass = false;
        uint32_t e = 0;
        if (k < n1) {
          e = list1[k];
          const int i = e >> 16, j = e & 0xffffu;
          seg<vec3<double>> Li;
          Li.s = mk3(sl.sx[i], sl.sy[i], sl.sz[i]);
          Li.e = mk3(sl.ex[i], sl.ey[i], sl.ez[i]);
          pass = gate2d(p, Li, sl, j, sl.ng[j] >> 16);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, pass);
        if (pass) list2[n2 + __popc(bal & lt_mask)] = e;
        n2 += __popc(bal);
      }
      __syncwarp();
      n2_total += n2;
      // B3: exact reference scores; maximum per (row, image), summed per row (:97-112). Entries are ordered
      // by (row, image), so both reductions are segmented warp scans with a carry across batches.
      uint32_t carry_key = 0xffffffffu, cur_row = 0xffffffffu;
      double carry_max = 0.0, cur_sum = 0.0;
      for (int kb = 0; kb < n2; kb += 32) {
        const int k = kb + lane;
        double sc = 0.0;
        uint32_t key = 0xfffffffeu, row = 0xfffffffeu; // key = row << 16 | view
        if (k < n2) {
          const uint32_t e = list2[k];
          const int i = e >> 16, j = e & 0xffffu;
          const uint32_t vj = sl.ng[j] >> 16;
          row = (uint32_t)i;
          key = (row << 16) | vj;
          seg<vec3<double>> Li;
          Li.s = mk3(sl.sx[i], sl.sy[i], sl.sz[i]);
          Li.e = mk3(sl.ex[i], sl.ey[i], sl.ez[i]);
          sc = pair_score(p, Li, mk3(sl.dx[i], sl.dy[i], sl.dz[i]), sl.zs[i], sl.ze[i], sl, j, vj);
        }
        if (key == carry_key && carry_max > sc) sc = carry_max;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const double o = __shfl_up_sync(0xffffffffu, sc, d);
          const uint32_t ok = __shfl_up_sync(0xffffffffu, key, d);
          if (lane >= d && ok == key && o > sc) sc = o;
        }
        uint32_t knext = __shfl_down_sync(0xffffffffu, key, 1);
        if (lane == 31) {
          knext = 0xfffffffdu;
          if (k + 1 < n2) { const uint32_t e2 = list2[k + 1]; knext = (e2 & 0xffff0000u) | (sl.ng[e2 & 0xffffu] >> 16); }
        }
        const bool seg_end = (k < n2) && (knext != key);
        // one image contributes its maximum once (:110-112): add the segment maxima to their row's total in
        // list order = ascending (row, image), exactly the reference's std::map order; the running
        // (row, sum) pair is warp-uniform, so the result does not depend on how rows were batched
        unsigned m = __ballot_sync(0xffffffffu, seg_end);
        while (m) {
          const int l = __ffs(m) - 1;
          const double v = __shfl_sync(0xffffffffu, sc, l);
          const uint32_t r = __shfl_sync(0xffffffffu, row, l);
          if (r != cur_row) {
            if (cur_row != 0xffffffffu && lane == 0) sl.score[cur_row] = cur_sum;
            cur_row = r;
            cur_sum = 0.0;
          }
          cur_sum += v;
          m &= m - 1;
        }
        const uint32_t k31 = __shfl_sync(0xffffffffu, key, 31);
        const double s31 = __shfl_sync(0xffffffffu, sc, 31);
        const bool end31 = __shfl_sync(0xffffffffu, (int)seg_end, 31);
        if (!end31 && kb + 31 < n2) { carry_key = k31; carry_max = s31; }
        else { carry_key = 0xffffffffu; carry_max = 0.0; }
      }
      if (cur_row != 0xffffffffu && lane == 0) sl.score[cur_row] = cur_sum;
      __syncwarp();
    }
    __syncthreads();
    } // generic phase B
    phase_c<NS>(p, sl, C, r0, rec, tid, lane, warp, &s_nvalid);
  }
  if (lane == 0 && n1_total) {
    atomicAdd(&p.counters[2], n1_total); // pairs past the fp32 3d gates
    atomicAdd(&p.counters[3], n2_total); // pairs scored exactly in fp64
  }
}

template <bool VP, bool FAST> static cudaError_t launch_tri_vf(const TriParams &p, int grid, size_t smem, cudaStream_t s) {
  if (p.use_slab) {
    tri_node_kernel<true, VP, FAST><<<grid, kThreads, 0, s>>>(p);
    return cudaGetLastError();
  }
  // the opt-in is per device (and per function): set it on every launch above the default limit
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(tri_node_kernel<false, VP, FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  if constexpr (!VP && FAST) { // five CTAs of 43 KB need the largest shared-memory carveout (228 KB on an H100)
    const cudaError_t e = cudaFuncSetAttribute(tri_node_kernel<false, VP, FAST>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                               (int)cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
  }
  tri_node_kernel<false, VP, FAST><<<grid, kThreads, smem, s>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_tri_node_kernel(const TriParams &p, int grid, size_t smem, cudaStream_t s) {
  const bool fast = tri_fast(p);
  if (p.use_vp) return fast ? launch_tri_vf<true, true>(p, grid, smem, s) : launch_tri_vf<true, false>(p, grid, smem, s);
  return fast ? launch_tri_vf<false, true>(p, grid, smem, s) : launch_tri_vf<false, false>(p, grid, smem, s);
}

} // namespace lm
