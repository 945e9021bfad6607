// oracle/orc_loc.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
// fp64 restatement of the joint point + line pose refinement (JointLocEngine / LineLocEngine):
//   optimize/hybrid_localization/cost_functions.h:28-347   Ceres_Compute2DWeight, the six line costs,
//                                                           ReprojectionLineFunctor, ReprojectionPointFunctor
//   ceresbase/point_projection.h                            PixelToWorld (Eigen q.conjugate() * v, q NOT normalised),
//                                                           WorldToPixel (ceres::QuaternionRotatePoint, normalised)
//   ceresbase/line_dists.h:8-29                             CeresComputeDist2D_sine / _cosine
//   optimize/hybrid_localization/hybrid_localization.cc     residual weights: weight_line * |l2d| / sum |l2d| of the
//                                                           3D line's group, weight_point per point; ScaledLoss
// The residuals are differentiated with ceres::Jet-style duals on the 7 ambient parameters (qvec 4, tvec 3) and chained
// through QuaternionPlusJacobian, as Ceres does. The SOLVER LOOP is PARITY UNPINNED: it is the trust-region LM of
// orc_lm.h (DESIGN.md §5) on a 6-dof tangent (quaternion 3, translation 3), with the damped normal equations solved by
// Cholesky where the reference asks Ceres for DENSE_QR (same system, different rounding). The loss functions restate
// Ceres' loss_function.cc (TrivialLoss, HuberLoss, SoftLOneLoss, CauchyLoss, ScaledLoss).
#include "orc_lm.h"
#include <cstdint>
#include <cstring>

namespace orc {

template <int N> inline Jet<N> acos(const Jet<N> &f) {
  Jet<N> h; h.a = std::acos(f.a); const double t = -1.0 / std::sqrt(1.0 - f.a * f.a);
  for (int i = 0; i < N; ++i) h.v[i] = t * f.v[i];
  return h;
}
template <int N> inline Jet<N> pow2(const Jet<N> &f) { // ceres::pow(Jet, 2): value pow(a, 2), partials 2 pow(a, 1) v
  Jet<N> h; h.a = std::pow(f.a, 2.0); const double t = 2.0 * std::pow(f.a, 1.0);
  for (int i = 0; i < N; ++i) h.v[i] = t * f.v[i];
  return h;
}
inline double acos(double x) { return std::acos(x); }
inline double pow2(double x) { return std::pow(x, 2.0); }
inline double val(double x) { return x; }
template <int N> inline double val(const Jet<N> &x) { return x.a; }

enum { kMidpoint2 = 0, kMidpointAngle3 = 1, kPerp2 = 2, kPerp4 = 3, kLineLine2 = 4, kPlaneLine2 = 5 };
inline int residual_num(int cf) { return cf == kPerp4 ? 4 : (cf == kMidpointAngle3 ? 3 : 2); } // getResidualNum

template <typename T> inline T sine2d(const T a[2], const T b[2]) { // CeresComputeDist2D_sine
  T n1 = sqrt(a[0] * a[0] + a[1] * a[1] + T(EPS)), n2 = sqrt(b[0] * b[0] + b[1] * b[1] + T(EPS));
  T s = (a[0] * b[1] - a[1] * b[0]) / (n1 * n2);
  s = abs(s);
  if (val(s) > 1.0) s = T(1.0);
  return s;
}
template <typename T> inline T cosine2d(const T a[2], const T b[2]) { // CeresComputeDist2D_cosine
  T n1 = sqrt(a[0] * a[0] + a[1] * a[1] + T(EPS)), n2 = sqrt(b[0] * b[0] + b[1] * b[1] + T(EPS));
  T c = (a[0] * b[0] + a[1] * b[1]) / (n1 * n2);
  c = abs(c);
  if (val(c) > 1.0) c = T(1.0);
  return c;
}
// ceres::UnitQuaternionRotatePoint; Eigen's Quaternion * Vector3 (_transformVector) is the same expression
template <typename T> inline void unit_rotate(const T q[4], const T p[3], T out[3]) {
  T uv0 = q[2] * p[2] - q[3] * p[1], uv1 = q[3] * p[0] - q[1] * p[2], uv2 = q[1] * p[1] - q[2] * p[0];
  uv0 = uv0 + uv0; uv1 = uv1 + uv1; uv2 = uv2 + uv2;
  out[0] = p[0] + q[0] * uv0; out[1] = p[1] + q[0] * uv1; out[2] = p[2] + q[0] * uv2;
  out[0] = out[0] + (q[2] * uv2 - q[3] * uv1);
  out[1] = out[1] + (q[3] * uv0 - q[1] * uv2);
  out[2] = out[2] + (q[1] * uv1 - q[2] * uv0);
}
template <typename T> inline void world_to_pixel(const T k[4], const T q[4], const T t[3], const T X[3], T xy[2]) {
  const T sc = T(1) / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const T u[4] = {sc * q[0], sc * q[1], sc * q[2], sc * q[3]};
  T p[3];
  unit_rotate(u, X, p);
  p[0] = p[0] + t[0]; p[1] = p[1] + t[1]; p[2] = p[2] + t[2];
  p[0] = p[0] / p[2]; p[1] = p[1] / p[2];
  xy[0] = k[0] * p[0] + k[2]; xy[1] = k[1] * p[1] + k[3];
}
template <typename T> inline void pixel_to_world(const T k[4], const T q[4], const T t[3], const T &x, const T &y,
                                                 double depth, T xyz[3]) {
  T l[3] = {(x - k[2]) / k[0], (y - k[3]) / k[1], T(1.0)};
  for (int i = 0; i < 3; ++i) l[i] = l[i] * T(depth) - t[i];
  const T qc[4] = {q[0], -q[1], -q[2], -q[3]};
  unit_rotate(qc, l, xyz);
}
template <typename T> inline void cross3(const T a[3], const T b[3], T o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
template <typename T> inline T dot3(const T a[3], const T b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

template <typename T> inline T line_line_dist(const T k[4], const T q[4], const T t[3], const T p3d[3], const T dir3d[3],
                                              const T p2d[2]) { // Ceres_3DLineLineDist
  T pa[3], pb[3];
  pixel_to_world(k, q, t, p2d[0], p2d[1], 1.0, pa);
  pixel_to_world(k, q, t, p2d[0], p2d[1], 2.0, pb);
  T dir[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]}, n[3];
  cross3(dir, dir3d, n);
  T n2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
  T d[3] = {p3d[0] - pa[0], p3d[1] - pa[1], p3d[2] - pa[2]}, c[3];
  if (val(n2) <= 1e-8) {
    cross3(dir, d, c);
    return sqrt(dot3(c, c) / dot3(dir, dir) + T(1e-8));
  }
  return dot3(n, d) / sqrt(n2);
}

// ReprojectionLineFunctor::operator() (cost_functions.h:240-286)
template <typename T> void line_residual(int cf, int wf, const double L3[6], const double L2[4], const T k[4],
                                         const T q[4], const T t[3], T res[4]) {
  T s3d[3] = {T(L3[0]), T(L3[1]), T(L3[2])}, e3d[3] = {T(L3[3]), T(L3[4]), T(L3[5])};
  T dir3d[3] = {e3d[0] - s3d[0], e3d[1] - s3d[1], e3d[2] - s3d[2]};
  T dn3 = sqrt(dot3(dir3d, dir3d) + T(1e-8));
  for (int i = 0; i < 3; ++i) dir3d[i] = dir3d[i] / dn3;
  T sr[2], er[2];
  world_to_pixel(k, q, t, s3d, sr);
  world_to_pixel(k, q, t, e3d, er);
  T s2d[2] = {T(L2[0]), T(L2[1])}, e2d[2] = {T(L2[2]), T(L2[3])};
  T dir2d[2] = {er[0] - sr[0], er[1] - sr[1]};
  T dn = sqrt(dir2d[0] * dir2d[0] + dir2d[1] * dir2d[1] + T(1e-8));
  dir2d[0] = dir2d[0] / dn; dir2d[1] = dir2d[1] / dn;
  switch (cf) {
  case kMidpoint2:
  case kMidpointAngle3: {
    T m1[2] = {T(0.5) * (sr[0] + er[0]), T(0.5) * (sr[1] + er[1])}, m2[2] = {T(0.5) * (s2d[0] + e2d[0]), T(0.5) * (s2d[1] + e2d[1])};
    res[0] = m1[0] - m2[0]; res[1] = m1[1] - m2[1];
    if (cf == kMidpointAngle3) {
      T d1[2] = {er[0] - sr[0], er[1] - sr[1]};
      T n1 = sqrt(d1[0] * d1[0] + d1[1] * d1[1] + T(1e-8));
      d1[0] = d1[0] / n1; d1[1] = d1[1] / n1;
      T d2[2] = {e2d[0] - s2d[0], e2d[1] - s2d[1]};
      T n2 = sqrt(d2[0] * d2[0] + d2[1] * d2[1] + T(1e-8));
      d2[0] = d2[0] / n2; d2[1] = d2[1] / n2;
      res[2] = n1 * sine2d(d1, d2);
    }
    break;
  }
  case kPerp2:
  case kPerp4: {
    T a[2] = {s2d[0] - sr[0], s2d[1] - sr[1]}, b[2] = {e2d[0] - sr[0], e2d[1] - sr[1]};
    T sa = sine2d(dir2d, a), sb = sine2d(dir2d, b);
    T r[4] = {a[0] * sa, a[1] * sa, b[0] * sb, b[1] * sb};
    if (cf == kPerp4) { for (int i = 0; i < 4; ++i) res[i] = r[i]; }
    else {
      res[0] = sqrt(r[0] * r[0] + r[1] * r[1] + T(1e-8));
      res[1] = sqrt(r[2] * r[2] + r[3] * r[3] + T(1e-8));
    }
    break;
  }
  case kLineLine2:
    res[0] = line_line_dist(k, q, t, s3d, dir3d, s2d);
    res[1] = line_line_dist(k, q, t, s3d, dir3d, e2d);
    break;
  case kPlaneLine2: {
    T p1a[3], p1b[3], p2a[3], p2b[3];
    pixel_to_world(k, q, t, s2d[0], s2d[1], 1.0, p1a);
    pixel_to_world(k, q, t, s2d[0], s2d[1], 2.0, p1b);
    pixel_to_world(k, q, t, e2d[0], e2d[1], 1.0, p2a);
    pixel_to_world(k, q, t, e2d[0], e2d[1], 2.0, p2b);
    T d1[3], d2[3], n[3], ds[3], de[3];
    for (int i = 0; i < 3; ++i) { d1[i] = p1b[i] - p1a[i]; d2[i] = p2b[i] - p2a[i]; }
    cross3(d1, d2, n);
    T n2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
    for (int i = 0; i < 3; ++i) { ds[i] = s3d[i] - p1a[i]; de[i] = e3d[i] - p1a[i]; }
    res[0] = dot3(n, ds) / sqrt(n2);
    res[1] = dot3(n, de) / sqrt(n2);
    break;
  }
  }
  // Ceres_Compute2DWeight(weight, dir2d, s2d, e2d), alpha = 10
  T direc[2] = {e2d[0] - s2d[0], e2d[1] - s2d[1]}, w;
  switch (wf) {
  case 1: w = exp(T(10.0) * (T(1.0) - cosine2d(dir2d, direc))); break;
  case 2: w = exp(T(10.0) * acos(cosine2d(dir2d, direc))); break;
  case 3: w = sqrt(direc[0] * direc[0] + direc[1] * direc[1] + T(1e-8)); break;
  case 4: w = T(1.0) / sqrt(direc[0] * direc[0] + direc[1] * direc[1] + T(1e-8)); break;
  default: w = T(1.0);
  }
  for (int i = 0; i < residual_num(cf); ++i) res[i] = res[i] * w;
}

// ReprojectionPointFunctor::operator() (cost_functions.h:312-340)
template <typename T> void point_residual(bool use3d, const double P3[3], const double P2[2], const T k[4], const T q[4],
                                          const T t[3], T res[2]) {
  T p2d[2] = {T(P2[0]), T(P2[1])}, p3d[3] = {T(P3[0]), T(P3[1]), T(P3[2])};
  if (use3d) {
    T pa[3], pb[3];
    pixel_to_world(k, q, t, p2d[0], p2d[1], 1.0, pa);
    pixel_to_world(k, q, t, p2d[0], p2d[1], 2.0, pb);
    T dir[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]};
    T dn = sqrt(dot3(dir, dir) + T(1e-8));
    for (int i = 0; i < 3; ++i) dir[i] = dir[i] / dn;
    T d[3] = {p3d[0] - pa[0], p3d[1] - pa[1], p3d[2] - pa[2]};
    res[0] = sqrt(dot3(d, d) - pow2(dot3(d, dir)) + T(1e-8));
    res[1] = T(0);
  } else {
    T r[2];
    world_to_pixel(k, q, t, p3d, r);
    res[0] = r[0] - T(P2[0]);
    res[1] = r[1] - T(P2[1]);
  }
}

// ceres loss_function.cc, then ScaledLoss(., a)
inline void loss_eval(int kind, double scale, double a, double s, double rho[3]) {
  const double b = scale * scale, c = 1.0 / b;
  switch (kind) {
  case 1:
    if (s > b) {
      const double r = std::sqrt(s);
      rho[0] = 2.0 * scale * r - b; rho[1] = std::max(std::numeric_limits<double>::min(), scale / r); rho[2] = -rho[1] / (2.0 * s);
    } else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
    break;
  case 2: {
    const double sum = 1.0 + s * c, tmp = std::sqrt(sum);
    rho[0] = 2.0 * b * (tmp - 1.0); rho[1] = std::max(std::numeric_limits<double>::min(), 1.0 / tmp); rho[2] = -(c * rho[1]) / (2.0 * sum);
    break;
  }
  case 3: {
    const double sum = 1.0 + s * c, inv = 1.0 / sum;
    rho[0] = b * std::log(sum); rho[1] = std::max(std::numeric_limits<double>::min(), inv); rho[2] = -c * (inv * inv);
    break;
  }
  default: rho[0] = s; rho[1] = 1.0; rho[2] = 0.0;
  }
  rho[0] *= a; rho[1] *= a; rho[2] *= a;
}

} // namespace orc

extern "C" {

// Layout shared with lm_loc_config (include/limap_b200.h).
typedef struct orc_loc_config {
  int32_t cost_function, weight_function, loss_kind, points_3d_dist;
  double loss_scale, weight_point, weight_line;
  int32_t max_num_iterations, max_num_consecutive_invalid_steps;
} orc_loc_config;

// One functor on 7-wide jets: residuals res[4] and the ambient Jacobian jac[4][7] (qvec 4, tvec 3). kind 0: line
// (data = l3d[6] then l2d[4]), kind 1: point (data = p3d[3] then p2d[2]).
void orc_loc_functor(int kind, int cf, int wf, int use3d, const double *data, const double *kvec, const double *qvec,
                     const double *tvec, double *res, double *jac) {
  typedef orc::Jet<7> J;
  J k[4] = {J(kvec[0]), J(kvec[1]), J(kvec[2]), J(kvec[3])};
  J q[4] = {J(qvec[0], 0), J(qvec[1], 1), J(qvec[2], 2), J(qvec[3], 3)}, t[3] = {J(tvec[0], 4), J(tvec[1], 5), J(tvec[2], 6)};
  J r[4];
  int m = 2;
  if (kind == 0) { orc::line_residual(cf, wf, data, data + 6, k, q, t, r); m = orc::residual_num(cf); }
  else orc::point_residual(use3d != 0, data, data + 3, k, q, t, r);
  for (int i = 0; i < 4; ++i) {
    res[i] = i < m ? r[i].a : 0.0;
    for (int j = 0; j < 7; ++j) jac[7 * i + j] = i < m ? r[i].v[j] : 0.0;
  }
}

// The loss of n blocks with squared residual norms s[n] and ScaledLoss factors a[n]: rho[n][3].
void orc_loc_loss(int kind, double scale, int64_t n, const double *a, const double *s, double *rho) {
  for (int64_t i = 0; i < n; ++i) orc::loss_eval(kind, scale, a[i], s[i], rho + 3 * i);
}

// The same functor in plain doubles (the path Ceres takes when it evaluates a cost without Jacobians).
void orc_loc_functor_value(int kind, int cf, int wf, int use3d, const double *data, const double *kvec,
                           const double *qvec, const double *tvec, double *res) {
  double r[4] = {0, 0, 0, 0};
  if (kind == 0) orc::line_residual<double>(cf, wf, data, data + 6, kvec, qvec, tvec, r);
  else orc::point_residual<double>(use3d != 0, data, data + 3, kvec, qvec, tvec, r);
  for (int i = 0; i < 4; ++i) res[i] = r[i];
}
}

namespace {

struct Block {
  int kind; // 0 line, 1 point
  double data[10];
  double a; // ScaledLoss factor
};

struct LocProblem {
  std::vector<Block> blocks;
  const orc_loc_config *cfg;
  double k[4];
  int cf() const { return cfg->cost_function; }
  int m_of(const Block &b) const { return b.kind == 0 ? orc::residual_num(cf()) : 2; }
  // cost and optionally the loss-corrected residuals / tangent Jacobian (rows of 6) at x = (qvec, tvec)
  double evaluate(const double x[7], std::vector<double> *res, std::vector<double> *jac) const {
    double cost = 0;
    double Pq[12];
    orc::QuaternionPlusJacobian(x, Pq);
    if (res) res->clear();
    if (jac) jac->clear();
    for (const Block &b : blocks) {
      const int m = m_of(b);
      double r[4], Ja[28], Jt[24] = {0};
      if (jac) {
        orc_loc_functor(b.kind, cf(), cfg->weight_function, cfg->points_3d_dist, b.data, k, x, x + 4, r, Ja);
        for (int i = 0; i < m; ++i) {
          for (int c = 0; c < 3; ++c)
            Jt[6 * i + c] = Ja[7 * i] * Pq[c] + Ja[7 * i + 1] * Pq[3 + c] + Ja[7 * i + 2] * Pq[6 + c] + Ja[7 * i + 3] * Pq[9 + c];
          for (int c = 0; c < 3; ++c) Jt[6 * i + 3 + c] = Ja[7 * i + 4 + c];
        }
      } else
        orc_loc_functor_value(b.kind, cf(), cfg->weight_function, cfg->points_3d_dist, b.data, k, x, x + 4, r);
      double s = 0;
      for (int i = 0; i < m; ++i) s += r[i] * r[i];
      double rho[3];
      orc::loss_eval(cfg->loss_kind, cfg->loss_scale, b.a, s, rho);
      cost += 0.5 * rho[0];
      if (!res && !jac) continue;
      // Corrector (ceres corrector.cc)
      const double sqrt_rho1 = std::sqrt(rho[1]);
      double residual_scaling = sqrt_rho1, alpha_sq_norm = 0.0;
      if (!(s == 0.0 || rho[2] <= 0.0)) {
        const double D = 1.0 + 2.0 * s * rho[2] / rho[1];
        const double al = 1.0 - std::sqrt(D);
        residual_scaling = sqrt_rho1 / (1 - al);
        alpha_sq_norm = al / s;
      }
      if (jac) {
        for (int c = 0; c < 6; ++c) {
          double rtj = 0;
          for (int i = 0; i < m; ++i) rtj += r[i] * Jt[6 * i + c];
          for (int i = 0; i < m; ++i)
            Jt[6 * i + c] = alpha_sq_norm == 0.0 ? sqrt_rho1 * Jt[6 * i + c] : sqrt_rho1 * (Jt[6 * i + c] - alpha_sq_norm * r[i] * rtj);
        }
        jac->insert(jac->end(), Jt, Jt + 6 * m);
      }
      if (res) for (int i = 0; i < m; ++i) res->push_back(r[i] * residual_scaling);
    }
    // a candidate whose residuals are not finite is an evaluation failure: Ceres gives it the largest cost
    if (!std::isfinite(cost)) cost = std::numeric_limits<double>::max();
    return cost;
  }
  static bool chol_solve(const double A[36], const double b[6], double x[6]) {
    double L[36] = {0};
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j <= i; ++j) {
        double s = A[6 * i + j];
        for (int k = 0; k < j; ++k) s -= L[6 * i + k] * L[6 * j + k];
        if (i == j) { if (!(s > 0)) return false; L[6 * i + i] = std::sqrt(s); }
        else L[6 * i + j] = s / L[6 * j + j];
      }
    double y[6];
    for (int i = 0; i < 6; ++i) { double s = b[i]; for (int k = 0; k < i; ++k) s -= L[6 * i + k] * y[k]; y[i] = s / L[6 * i + i]; }
    for (int i = 5; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < 6; ++k) s -= L[6 * k + i] * x[k]; x[i] = s / L[6 * i + i]; }
    return true;
  }
  // orc::LMProblem::solve (orc_lm.h) on the 6-dof tangent. term: 1 iterations, 2 radius, 3 gradient, 4 invalid steps,
  // 5 zero step, 6 zero cost change, 7 initial evaluation failed.
  void solve(double x[7], int stop_after, int32_t *iters, double *costs, int32_t *term_out) const {
    std::vector<double> r, J;
    double cost = evaluate(x, &r, &J);
    costs[0] = costs[1] = cost;
    iters[0] = iters[1] = 0;
    if (cost == std::numeric_limits<double>::max()) { *term_out = 7; return; }
    const int R = (int)r.size();
    double scale[6];
    for (int c = 0; c < 6; ++c) {
      double n2 = 0; for (int i = 0; i < R; ++i) n2 += J[6 * i + c] * J[6 * i + c];
      scale[c] = 1.0 / (1.0 + std::sqrt(n2));
    }
    auto scale_cols = [&](std::vector<double> &Jm) { for (int i = 0; i < R; ++i) for (int c = 0; c < 6; ++c) Jm[6 * i + c] *= scale[c]; };
    scale_cols(J);
    double radius = 1e4, decrease_factor = 2.0, diag[6] = {0};
    bool reuse_diagonal = false;
    int invalid = 0, it = 0, successful = 0, term = 0;
    const int max_it = stop_after >= 0 ? std::min(stop_after, cfg->max_num_iterations) : cfg->max_num_iterations;
    while (true) {
      if (it >= max_it) { term = 1; break; }
      if (radius <= 1e-32) { term = 2; break; }
      double A[36] = {0}, g[6] = {0};
      for (int i = 0; i < R; ++i) for (int a = 0; a < 6; ++a) { g[a] += J[6 * i + a] * r[i]; for (int b = 0; b < 6; ++b) A[6 * a + b] += J[6 * i + a] * J[6 * i + b]; }
      { double gmax = 0; for (int c = 0; c < 6; ++c) gmax = std::max(gmax, std::abs(g[c])); if (gmax <= 0.0) { term = 3; break; } }
      ++it;
      if (!reuse_diagonal) for (int c = 0; c < 6; ++c) diag[c] = std::min(std::max(A[7 * c], 1e-6), 1e32);
      for (int c = 0; c < 6; ++c) A[7 * c] += diag[c] / radius;
      reuse_diagonal = true;
      double step[6];
      bool ok = chol_solve(A, g, step);
      for (int c = 0; c < 6; ++c) { step[c] = -step[c]; if (!std::isfinite(step[c])) ok = false; }
      double mcc = 0;
      if (ok) for (int i = 0; i < R; ++i) { double mr = 0; for (int c = 0; c < 6; ++c) mr += J[6 * i + c] * step[c]; mcc -= mr * (r[i] + mr / 2.0); }
      if (!ok || !(mcc > 0.0)) {
        if (++invalid >= cfg->max_num_consecutive_invalid_steps) { term = 4; break; }
        radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
        continue;
      }
      invalid = 0;
      double delta[3] = {step[0] * scale[0], step[1] * scale[1], step[2] * scale[2]}, cand[7];
      orc::QuaternionPlus(x, delta, cand);
      for (int c = 0; c < 3; ++c) cand[4 + c] = x[4 + c] + step[3 + c] * scale[3 + c];
      const double cand_cost = evaluate(cand, nullptr, nullptr);
      double sn = 0; for (int c = 0; c < 7; ++c) sn += (x[c] - cand[c]) * (x[c] - cand[c]);
      if (!(std::sqrt(sn) > 0.0)) { term = 5; break; }
      if (!(std::abs(cost - cand_cost) > 0.0)) { term = 6; break; }
      const double rel = (cost - cand_cost) / mcc;
      if (rel > 1e-3) {
        for (int c = 0; c < 7; ++c) x[c] = cand[c];
        cost = evaluate(x, &r, &J);
        scale_cols(J);
        radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rel - 1.0, 3)));
        decrease_factor = 2.0; reuse_diagonal = false;
        ++successful;
      } else {
        radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
      }
    }
    iters[0] = it; iters[1] = successful;
    costs[1] = cost;
    *term_out = term;
  }
};

} // namespace

extern "C" {

// JointLocEngine::{Initialize,SetUp,Solve} for Q independent queries (arrays as lm_loc_solve). stop_after >= 0 caps the
// iterations below cfg->max_num_iterations (path tests). flags[q] bit0 solved, bit1 solution usable. term[q] as above
// (0 when not solved). Queries run in parallel over the host's cores.
void orc_loc_solve(int64_t Q, const double *kvec, const double *qvec, const double *tvec, const int64_t *pt_off,
                   const double *p3d, const double *p2d, const int64_t *grp_off, const double *l3d,
                   const int64_t *l2d_off, const double *l2d, const orc_loc_config *cfg, int32_t stop_after,
                   double *qvec_out, double *tvec_out, int32_t *iters, double *cost, uint8_t *flags, int32_t *term) {
#pragma omp parallel for schedule(dynamic, 4)
  for (int64_t q = 0; q < Q; ++q) {
    LocProblem P;
    P.cfg = cfg;
    for (int i = 0; i < 4; ++i) P.k[i] = kvec[4 * q + i];
    for (int64_t g = grp_off[q]; g < grp_off[q + 1]; ++g) {
      double sum = 0;
      for (int64_t j = l2d_off[g]; j < l2d_off[g + 1]; ++j) {
        const double *l = l2d + 4 * j;
        sum += std::sqrt((l[0] - l[2]) * (l[0] - l[2]) + (l[1] - l[3]) * (l[1] - l[3])); // Line2d::length
      }
      for (int64_t j = l2d_off[g]; j < l2d_off[g + 1]; ++j) {
        const double *l = l2d + 4 * j;
        Block b;
        b.kind = 0;
        std::memcpy(b.data, l3d + 6 * g, 48);
        std::memcpy(b.data + 6, l, 32);
        b.a = cfg->weight_line * std::sqrt((l[0] - l[2]) * (l[0] - l[2]) + (l[1] - l[3]) * (l[1] - l[3])) / sum;
        P.blocks.push_back(b);
      }
    }
    for (int64_t i = pt_off[q]; i < pt_off[q + 1]; ++i) {
      Block b;
      b.kind = 1;
      std::memcpy(b.data, p3d + 3 * i, 24);
      std::memcpy(b.data + 3, p2d + 2 * i, 16);
      b.a = cfg->weight_point;
      P.blocks.push_back(b);
    }
    double x[7];
    std::memcpy(x, qvec + 4 * q, 32);
    std::memcpy(x + 4, tvec + 3 * q, 24);
    int32_t it2[2] = {0, 0}, tm = 0;
    double c2[2] = {0, 0};
    uint8_t f = 0;
    if (!P.blocks.empty()) {
      P.solve(x, stop_after, it2, c2, &tm);
      f = 1 | ((tm != 4 && tm != 7) ? 2 : 0);
    }
    std::memcpy(qvec_out + 4 * q, x, 32);
    std::memcpy(tvec_out + 3 * q, x + 4, 24);
    iters[2 * q] = it2[0]; iters[2 * q + 1] = it2[1];
    cost[2 * q] = c2[0]; cost[2 * q + 1] = c2[1];
    flags[q] = f;
    if (term) term[q] = tm;
  }
}
}
