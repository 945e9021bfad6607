// loc_block.cuh — one residual block of the query pose refinement (ReprojectionLineFunctor for the six line costs and
// five line weights, ReprojectionPointFunctor in both point modes), the loss, Ceres' corrector and the 6x6 step solve,
// as __host__ __device__ code: loc_kernels.cu runs it on the device; tests/loc_block_host.cu builds it for the host,
// where tests/test_loc_block_host.py checks it against the reference's stored functor values and the oracle.
#pragma once
#include "loc_kernels.cuh"
#include "lm_block.cuh"
#include <cfloat>
#include <cmath>

namespace lm {
namespace loc {

typedef Dual<6> D;
LM_HD D K(double x) { return dconst<6>(x); }
LM_HD D dacos(const D &f) { // ceres acos(Jet)
  D h; h.a = acos(f.a); const double t = -1.0 / sqrt(1.0 - f.a * f.a);
#pragma unroll
  for (int i = 0; i < 6; ++i) h.v[i] = t * f.v[i];
  return h;
}
LM_HD D dpow2(const D &f) { // ceres pow(Jet, 2)
  D h; h.a = pow(f.a, 2.0); const double t = 2.0 * pow(f.a, 1.0);
#pragma unroll
  for (int i = 0; i < 6; ++i) h.v[i] = t * f.v[i];
  return h;
}

constexpr double kEps = 1e-12; // limap EPS (util/types.h)

LM_HD D sine2d(const D a[2], const D b[2]) { // CeresComputeDist2D_sine (ceresbase/line_dists.h:8-17)
  const D n1 = dsqrt(a[0] * a[0] + a[1] * a[1] + K(kEps)), n2 = dsqrt(b[0] * b[0] + b[1] * b[1] + K(kEps));
  D s = dabs((a[0] * b[1] - a[1] * b[0]) / (n1 * n2));
  if (s.a > 1.0) s = K(1.0);
  return s;
}
LM_HD D cosine2d(const D a[2], const D b[2]) { // CeresComputeDist2D_cosine (:19-29)
  const D n1 = dsqrt(a[0] * a[0] + a[1] * a[1] + K(kEps)), n2 = dsqrt(b[0] * b[0] + b[1] * b[1] + K(kEps));
  D c = dabs((a[0] * b[0] + a[1] * b[1]) / (n1 * n2));
  if (c.a > 1.0) c = K(1.0);
  return c;
}
// ceres::UnitQuaternionRotatePoint; Eigen's Quaternion * Vector3 is the same expression
LM_HD void unit_rotate(const D q[4], const D p[3], D o[3]) {
  D uv0 = q[2] * p[2] - q[3] * p[1], uv1 = q[3] * p[0] - q[1] * p[2], uv2 = q[1] * p[1] - q[2] * p[0];
  uv0 = uv0 + uv0; uv1 = uv1 + uv1; uv2 = uv2 + uv2;
  o[0] = p[0] + q[0] * uv0; o[1] = p[1] + q[0] * uv1; o[2] = p[2] + q[0] * uv2;
  o[0] = o[0] + (q[2] * uv2 - q[3] * uv1);
  o[1] = o[1] + (q[3] * uv0 - q[1] * uv2);
  o[2] = o[2] + (q[1] * uv1 - q[2] * uv0);
}
// WorldToPixel (ceresbase/point_projection.h): ceres::QuaternionRotatePoint normalises q
LM_HD void world_to_pixel(const D k[4], const D u[4], const D t[3], const D X[3], D xy[2]) {
  D p[3];
  unit_rotate(u, X, p);
  p[0] = p[0] + t[0]; p[1] = p[1] + t[1]; p[2] = p[2] + t[2];
  p[0] = p[0] / p[2]; p[1] = p[1] / p[2];
  xy[0] = k[0] * p[0] + k[2]; xy[1] = k[1] * p[1] + k[3];
}
// PixelToWorld: Eigen q.conjugate() * v, q NOT normalised; qc is the conjugate
LM_HD void pixel_to_world(const D k[4], const D qc[4], const D t[3], const D &x, const D &y, double depth, D xyz[3]) {
  D l[3] = {(x - k[2]) / k[0], (y - k[3]) / k[1], K(1.0)};
#pragma unroll
  for (int i = 0; i < 3; ++i) l[i] = l[i] * K(depth) - t[i];
  unit_rotate(qc, l, xyz);
}
LM_HD void cross3(const D a[3], const D b[3], D o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
LM_HD D dot3(const D a[3], const D b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

LM_HD D line_line_dist(const D k[4], const D qc[4], const D t[3], const D p3d[3], const D dir3d[3], const D p2d[2]) {
  D pa[3], pb[3]; // Ceres_3DLineLineDist (cost_functions.h:120-155)
  pixel_to_world(k, qc, t, p2d[0], p2d[1], 1.0, pa);
  pixel_to_world(k, qc, t, p2d[0], p2d[1], 2.0, pb);
  const D dir[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]};
  D n[3];
  cross3(dir, dir3d, n);
  const D n2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
  const D d[3] = {p3d[0] - pa[0], p3d[1] - pa[1], p3d[2] - pa[2]};
  if (n2.a <= 1e-8) {
    D c[3];
    cross3(dir, d, c);
    return dsqrt(dot3(c, c) / dot3(dir, dir) + K(1e-8));
  }
  return dot3(n, d) / dsqrt(n2);
}

// The pose x = (qvec, tvec) as duals seeded on the 6-dof tangent at delta = 0: q with the QuaternionPlusJacobian (4x3)
// columns, its conjugate qc (PixelToWorld), its normalisation u (QuaternionRotatePoint) and t with the identity; the
// intrinsics kq as constants k.
LM_HD void pose_duals(const double x[7], const double kq[4], D k[4], D q[4], D qc[4], D u[4], D t[3]) {
  const double Pq[12] = {-x[1], -x[2], -x[3], x[0], x[3], -x[2], -x[3], x[0], x[1], x[2], -x[1], x[0]};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    k[i] = K(kq[i]);
    q[i].a = x[i];
#pragma unroll
    for (int j = 0; j < 6; ++j) q[i].v[j] = j < 3 ? Pq[3 * i + j] : 0.0;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    t[i].a = x[4 + i];
#pragma unroll
    for (int j = 0; j < 6; ++j) t[i].v[j] = (j == 3 + i) ? 1.0 : 0.0;
  }
  qc[0] = q[0]; qc[1] = -q[1]; qc[2] = -q[2]; qc[3] = -q[3];
  const D sc = K(1.0) / dsqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
  for (int i = 0; i < 4; ++i) u[i] = sc * q[i];
}

template <int CF> struct NumRes { static constexpr int value = CF == 3 ? 4 : (CF == 1 ? 3 : 2); }; // getResidualNum

// ReprojectionLineFunctor::operator() (cost_functions.h:240-286)
template <int CF>
LM_HD void line_residual(const LocBlockDev &b, int wf, const D k[4], const D q[4], const D qc[4], const D u[4],
                         const D t[3], D res[4]) {
  const D s3d[3] = {K(b.v[0]), K(b.v[1]), K(b.v[2])}, e3d[3] = {K(b.v[3]), K(b.v[4]), K(b.v[5])};
  D dir3d[3] = {e3d[0] - s3d[0], e3d[1] - s3d[1], e3d[2] - s3d[2]};
  const D dn3 = dsqrt(dot3(dir3d, dir3d) + K(1e-8));
  dir3d[0] = dir3d[0] / dn3; dir3d[1] = dir3d[1] / dn3; dir3d[2] = dir3d[2] / dn3;
  D sr[2], er[2];
  world_to_pixel(k, u, t, s3d, sr);
  world_to_pixel(k, u, t, e3d, er);
  const D s2d[2] = {K(b.v[6]), K(b.v[7])}, e2d[2] = {K(b.v[8]), K(b.v[9])};
  D dir2d[2] = {er[0] - sr[0], er[1] - sr[1]};
  const D dn = dsqrt(dir2d[0] * dir2d[0] + dir2d[1] * dir2d[1] + K(1e-8));
  dir2d[0] = dir2d[0] / dn; dir2d[1] = dir2d[1] / dn;
  if (CF == 0 || CF == 1) { // Ceres_2DMidpointDist2 / Ceres_2DMidpointAngleDist3
    res[0] = K(0.5) * (sr[0] + er[0]) - K(0.5) * (s2d[0] + e2d[0]);
    res[1] = K(0.5) * (sr[1] + er[1]) - K(0.5) * (s2d[1] + e2d[1]);
    if (CF == 1) {
      D d1[2] = {er[0] - sr[0], er[1] - sr[1]};
      const D n1 = dsqrt(d1[0] * d1[0] + d1[1] * d1[1] + K(1e-8));
      d1[0] = d1[0] / n1; d1[1] = d1[1] / n1;
      D d2[2] = {e2d[0] - s2d[0], e2d[1] - s2d[1]};
      const D n2 = dsqrt(d2[0] * d2[0] + d2[1] * d2[1] + K(1e-8));
      d2[0] = d2[0] / n2; d2[1] = d2[1] / n2;
      res[2] = n1 * sine2d(d1, d2);
    }
  } else if (CF == 2 || CF == 3) { // Ceres_2DPerpendicularDist2 / 4
    const D a[2] = {s2d[0] - sr[0], s2d[1] - sr[1]}, c[2] = {e2d[0] - sr[0], e2d[1] - sr[1]};
    const D sa = sine2d(dir2d, a), sc = sine2d(dir2d, c);
    if (CF == 3) { res[0] = a[0] * sa; res[1] = a[1] * sa; res[2] = c[0] * sc; res[3] = c[1] * sc; }
    else {
      const D r0 = a[0] * sa, r1 = a[1] * sa, r2 = c[0] * sc, r3 = c[1] * sc;
      res[0] = dsqrt(r0 * r0 + r1 * r1 + K(1e-8));
      res[1] = dsqrt(r2 * r2 + r3 * r3 + K(1e-8));
    }
  } else if (CF == 4) { // Ceres_3DLineLineDist2
    res[0] = line_line_dist(k, qc, t, s3d, dir3d, s2d);
    res[1] = line_line_dist(k, qc, t, s3d, dir3d, e2d);
  } else { // Ceres_3DPlaneLineDist2
    D p1a[3], p1b[3], p2a[3], p2b[3];
    pixel_to_world(k, qc, t, s2d[0], s2d[1], 1.0, p1a);
    pixel_to_world(k, qc, t, s2d[0], s2d[1], 2.0, p1b);
    pixel_to_world(k, qc, t, e2d[0], e2d[1], 1.0, p2a);
    pixel_to_world(k, qc, t, e2d[0], e2d[1], 2.0, p2b);
    const D d1[3] = {p1b[0] - p1a[0], p1b[1] - p1a[1], p1b[2] - p1a[2]};
    const D d2[3] = {p2b[0] - p2a[0], p2b[1] - p2a[1], p2b[2] - p2a[2]};
    D n[3];
    cross3(d1, d2, n);
    const D n2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
    const D ds[3] = {s3d[0] - p1a[0], s3d[1] - p1a[1], s3d[2] - p1a[2]};
    const D de[3] = {e3d[0] - p1a[0], e3d[1] - p1a[1], e3d[2] - p1a[2]};
    res[0] = dot3(n, ds) / dsqrt(n2);
    res[1] = dot3(n, de) / dsqrt(n2);
  }
  // Ceres_Compute2DWeight(weight, dir2d, s2d, e2d), alpha = 10 (cost_functions.h:28-61)
  const D direc[2] = {e2d[0] - s2d[0], e2d[1] - s2d[1]};
  D w;
  if (wf == 1) w = dexp(K(10.0) * (K(1.0) - cosine2d(dir2d, direc)));
  else if (wf == 2) w = dexp(K(10.0) * dacos(cosine2d(dir2d, direc)));
  else if (wf == 3) w = dsqrt(direc[0] * direc[0] + direc[1] * direc[1] + K(1e-8));
  else if (wf == 4) w = K(1.0) / dsqrt(direc[0] * direc[0] + direc[1] * direc[1] + K(1e-8));
  else w = K(1.0);
#pragma unroll
  for (int i = 0; i < NumRes<CF>::value; ++i) res[i] = res[i] * w;
}

// ReprojectionPointFunctor::operator() (cost_functions.h:312-340)
LM_HD void point_residual(const LocBlockDev &b, bool use3d, const D k[4], const D qc[4], const D u[4], const D t[3],
                          D res[2]) {
  const D p2d[2] = {K(b.v[3]), K(b.v[4])}, p3d[3] = {K(b.v[0]), K(b.v[1]), K(b.v[2])};
  if (use3d) {
    D pa[3], pb[3];
    pixel_to_world(k, qc, t, p2d[0], p2d[1], 1.0, pa);
    pixel_to_world(k, qc, t, p2d[0], p2d[1], 2.0, pb);
    D dir[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]};
    const D dn = dsqrt(dot3(dir, dir) + K(1e-8));
    dir[0] = dir[0] / dn; dir[1] = dir[1] / dn; dir[2] = dir[2] / dn;
    const D d[3] = {p3d[0] - pa[0], p3d[1] - pa[1], p3d[2] - pa[2]};
    res[0] = dsqrt(dot3(d, d) - dpow2(dot3(d, dir)) + K(1e-8));
    res[1] = K(0.0);
  } else {
    D r[2];
    world_to_pixel(k, u, t, p3d, r);
    res[0] = r[0] - K(b.v[3]);
    res[1] = r[1] - K(b.v[4]);
  }
}

// ceres loss_function.cc (Trivial, Huber, SoftLOne, Cauchy), then ScaledLoss(., a)
LM_HD void loss_eval(int kind, double scale, double a, double s, double rho[3]) {
  const double b = scale * scale, c = 1.0 / b;
  if (kind == 1) {
    if (s > b) {
      const double r = sqrt(s);
      rho[0] = 2.0 * scale * r - b; rho[1] = fmax(DBL_MIN, scale / r); rho[2] = -rho[1] / (2.0 * s);
    } else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
  } else if (kind == 2) {
    const double sum = 1.0 + s * c, tmp = sqrt(sum);
    rho[0] = 2.0 * b * (tmp - 1.0); rho[1] = fmax(DBL_MIN, 1.0 / tmp); rho[2] = -(c * rho[1]) / (2.0 * sum);
  } else if (kind == 3) {
    const double sum = 1.0 + s * c, inv = 1.0 / sum;
    rho[0] = b * log(sum); rho[1] = fmax(DBL_MIN, inv); rho[2] = -c * (inv * inv);
  } else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
  rho[0] *= a; rho[1] *= a; rho[2] *= a;
}

// Ceres' Corrector (corrector.cc) for one block with squared residual norm s and loss values rho, and the corrected
// residuals and Jacobian rows it gives.
struct Corrector {
  double sqrt_rho1, residual_scaling, alpha_sq_norm;
  LM_HD Corrector(double s, const double rho[3]) {
    sqrt_rho1 = sqrt(rho[1]);
    residual_scaling = sqrt_rho1;
    alpha_sq_norm = 0.0;
    if (!(s == 0.0 || rho[2] <= 0.0)) {
      const double Dd = 1.0 + 2.0 * s * rho[2] / rho[1];
      const double al = 1.0 - sqrt(Dd);
      residual_scaling = sqrt_rho1 / (1 - al);
      alpha_sq_norm = al / s;
    }
  }
  // Entry (i, c) of the corrected Jacobian of the block's m residuals r (values and tangent derivatives), before the
  // solver's column scaling; the corrected residual i is r[i].a * residual_scaling.
  LM_HD double jacobian(const D r[4], int m, int i, int c) const {
    double v = r[i].v[c];
    if (alpha_sq_norm != 0.0) {
      double rtj = 0.0;
#pragma unroll
      for (int l = 0; l < 4; ++l) if (l < m) rtj += r[l].a * r[l].v[c];
      v = v - alpha_sq_norm * r[i].a * rtj;
    }
    return sqrt_rho1 * v;
  }
};

constexpr int kNA = 21; // packed upper triangle of the 6x6 J^T J: row a holds columns a..5

// (A + diag(dg)) x = b for the packed symmetric 6x6 system of one LM step, square-root-free L D L^T (chol_solve4 of
// lm_kernels.cu for 6 unknowns). false when a pivot is not positive.
LM_HD bool ldlt_solve6(const double Ap[kNA], const double dg[6], const double b[6], double x[6]) {
  double L[6][6], d[6], id[6];
  int idx = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = a; c < 6; ++c) { L[c][a] = Ap[idx] + (a == c ? dg[a] : 0.0); ++idx; }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double dj = L[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) dj -= L[j][k] * L[j][k] * d[k];
    if (!(dj > 0)) return false;
    d[j] = dj;
    id[j] = 1.0 / dj;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double s = L[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k] * d[k];
      L[i][j] = s * id[j];
    }
  }
  double y[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
    y[i] = s;
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double s = y[i] * id[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) s -= L[k][i] * x[k];
    x[i] = s;
  }
  return true;
}

} // namespace loc
} // namespace lm
