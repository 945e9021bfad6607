// lm_math.cuh — small fixed-size geometry for the sm_90a kernels (templated on the scalar type so
// the same code instantiates the fp64 exact path and the fp32 fast path).
// Semantics follow the reference's Eigen usage (normalized() divides only when the norm is > 0;
// std::min/std::max NaN behaviour), cited per function in the kernels that use them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define LM_HD __host__ __device__ __forceinline__
#define LM_D __device__ __forceinline__

namespace lm {

// SM count of the current device (132 on an H100 SXM): sizes the grids of the grid-stride kernels.
inline int current_device_sms() {
  int dev = 0, n = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n;
}

// Largest i in [0, n) with off[i] <= x, for ascending off with off[0] <= x (0 when n <= 1). The index type I is that
// of n. LDG: load off through the read-only data cache.
template <bool LDG = false, typename I, typename T, typename X> LM_D I last_le(const T *off, I n, X x) {
  I lo = 0, hi = n;
  while (hi - lo > 1) {
    const I mid = (lo + hi) >> 1;
    if ((LDG ? __ldg(&off[mid]) : off[mid]) <= x) lo = mid; else hi = mid;
  }
  return lo;
}

template <typename T> struct consts;
template <> struct consts<double> {
  static LM_HD double eps() { return 1e-12; } // util/types.h:34
  static LM_HD double rad2deg() { return 180.0 / 3.14159265358979323846; }
  static LM_HD double maxval() { return 1.7976931348623157e308; }
};
template <> struct consts<float> {
  static LM_HD float eps() { return 1e-12f; }
  static LM_HD float rad2deg() { return 57.29577951308232f; }
  static LM_HD float maxval() { return 3.402823466e38f; }
};

// std::min / std::max argument-order semantics (matters for NaN).
template <typename T> LM_HD T smin(T a, T b) { return (b < a) ? b : a; }
template <typename T> LM_HD T smax(T a, T b) { return (a < b) ? b : a; }

template <typename T> struct vec2 {
  T x, y;
};
template <typename T> struct vec3 {
  T x, y, z;
};
template <typename T> LM_HD vec2<T> mk2(T x, T y) { vec2<T> v; v.x = x; v.y = y; return v; }
template <typename T> LM_HD vec3<T> mk3(T x, T y, T z) { vec3<T> v; v.x = x; v.y = y; v.z = z; return v; }

template <typename T> LM_HD vec2<T> operator+(vec2<T> a, vec2<T> b) { return mk2<T>(a.x + b.x, a.y + b.y); }
template <typename T> LM_HD vec2<T> operator-(vec2<T> a, vec2<T> b) { return mk2<T>(a.x - b.x, a.y - b.y); }
template <typename T> LM_HD vec2<T> operator*(vec2<T> a, T s) { return mk2<T>(a.x * s, a.y * s); }
template <typename T> LM_HD vec2<T> operator/(vec2<T> a, T s) { return mk2<T>(a.x / s, a.y / s); }
template <typename T> LM_HD T dot(vec2<T> a, vec2<T> b) { return a.x * b.x + a.y * b.y; }

template <typename T> LM_HD vec3<T> operator+(vec3<T> a, vec3<T> b) { return mk3<T>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename T> LM_HD vec3<T> operator-(vec3<T> a, vec3<T> b) { return mk3<T>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename T> LM_HD vec3<T> operator*(vec3<T> a, T s) { return mk3<T>(a.x * s, a.y * s, a.z * s); }
template <typename T> LM_HD vec3<T> operator/(vec3<T> a, T s) { return mk3<T>(a.x / s, a.y / s, a.z / s); }
template <typename T> LM_HD T dot(vec3<T> a, vec3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> LM_HD vec3<T> cross(vec3<T> a, vec3<T> b) {
  return mk3<T>(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
template <typename V> LM_HD auto sqnorm(V a) -> decltype(dot(a, a)) { return dot(a, a); }
template <typename V> LM_HD auto norm(V a) -> decltype(dot(a, a)) { return sqrt(dot(a, a)); }
// Eigen normalized(): only divides when the squared norm is > 0.
template <typename V> LM_HD V normalized(V a) {
  auto n2 = dot(a, a);
  if (n2 > 0) return a / sqrt(n2);
  return a;
}

// 3x3 row-major matrix * vector / [x,y,1]
template <typename T> LM_HD vec3<T> mat3_mul_h(const T *M, T x, T y) {
  return mk3<T>(M[0] * x + M[1] * y + M[2], M[3] * x + M[4] * y + M[5], M[6] * x + M[7] * y + M[8]);
}
template <typename T> LM_HD vec3<T> mat3_mul(const T *M, vec3<T> v) {
  return mk3<T>(M[0] * v.x + M[1] * v.y + M[2] * v.z, M[3] * v.x + M[4] * v.y + M[5] * v.z,
                M[6] * v.x + M[7] * v.y + M[8] * v.z);
}
template <typename T> LM_HD vec3<T> mat3T_mul(const T *M, vec3<T> v) {
  return mk3<T>(M[0] * v.x + M[3] * v.y + M[6] * v.z, M[1] * v.x + M[4] * v.y + M[7] * v.z,
                M[2] * v.x + M[5] * v.y + M[8] * v.z);
}
// P (3x4 row-major) * [X;1]
template <typename T> LM_HD vec3<T> proj_h(const T *P, vec3<T> X) {
  return mk3<T>(P[0] * X.x + P[1] * X.y + P[2] * X.z + P[3], P[4] * X.x + P[5] * X.y + P[6] * X.z + P[7],
                P[8] * X.x + P[9] * X.y + P[10] * X.z + P[11]);
}
// util/types.h:40-42
template <typename T> LM_HD vec2<T> dehom(vec3<T> v) {
  T d = v.z + consts<T>::eps();
  return mk2<T>(v.x / d, v.y / d);
}

// Solve [a b c] * lambda = rhs for lambda.x via the cofactor inverse (Eigen's fixed 3x3 inverse()).
// Returns the full solution vector.
template <typename T> LM_HD vec3<T> solve3_cols(vec3<T> a, vec3<T> b, vec3<T> c, vec3<T> r) {
  // matrix m[i][j]: column j in {a,b,c}
  T m00 = a.x, m01 = b.x, m02 = c.x, m10 = a.y, m11 = b.y, m12 = c.y, m20 = a.z, m21 = b.z, m22 = c.z;
  T c00 = m11 * m22 - m12 * m21;
  T c01 = m12 * m20 - m10 * m22;
  T c02 = m10 * m21 - m11 * m20;
  T det = m00 * c00 + m01 * c01 + m02 * c02;
  T id = T(1) / det;
  T i00 = c00 * id, i01 = (m02 * m21 - m01 * m22) * id, i02 = (m01 * m12 - m02 * m11) * id;
  T i10 = c01 * id, i11 = (m00 * m22 - m02 * m20) * id, i12 = (m02 * m10 - m00 * m12) * id;
  T i20 = c02 * id, i21 = (m01 * m20 - m00 * m21) * id, i22 = (m00 * m11 - m01 * m10) * id;
  return mk3<T>(i00 * r.x + i01 * r.y + i02 * r.z, i10 * r.x + i11 * r.y + i12 * r.z,
                i20 * r.x + i21 * r.y + i22 * r.z);
}

// compute_epipolar_IoU (triangulation/functions.cc:76-98) of a source line in the segment l2 = (x1, y1, x2, y2) of a
// second view. The epipolar lines of the source endpoints come from ep: ep.start() / ep.end() = F x1 up to scale. A value
// within 1e-7 of th is recomputed in the reference's normalised form, so that the caller's own comparison with th decides
// as the reference's does. A zero-length l2 gives NaN, as in the reference. s2, e2: the endpoints of l2, v2d = e2 - s2,
// len2sq = |v2d|^2. dehomogeneous() of the cross product of two normalised line vectors == raw.xy / (raw.z + EPS |a| |b|).
template <typename EP>
LM_D double epipolar_iou(const EP &ep, double4 l2, vec2<double> s2, vec2<double> e2, vec2<double> v2d, double len2sq,
                         const double &th) {
  const vec3<double> l2h = cross(mk3(l2.x, l2.y, 1.0), mk3(l2.z, l2.w, 1.0));
  const double nl2 = dot(l2h, l2h);
  const vec3<double> eps_ = ep.start();
  const vec3<double> hs = cross(l2h, eps_);
  const double ws = 1.0 / (hs.z + consts<double>::eps() * sqrt(nl2 * dot(eps_, eps_)));
  const vec3<double> epe_ = ep.end();
  const vec3<double> he = cross(l2h, epe_);
  const double we = 1.0 / (he.z + consts<double>::eps() * sqrt(nl2 * dot(epe_, epe_)));
  const vec2<double> cs = mk2(hs.x * ws, hs.y * ws), ce = mk2(he.x * we, he.y * we);
  const double il2 = 1.0 / len2sq;
  double c1 = dot(cs - s2, v2d) * il2;
  double c2 = dot(ce - s2, v2d) * il2;
  if (c1 > c2) { double t = c1; c1 = c2; c2 = t; }
  double IoU = (smin(c2, 1.0) - smax(c1, 0.0)) / (smax(c2, 1.0) - smin(c1, 0.0));
  if (fabs(IoU - th) < 1e-7) {
    // too close to the threshold: evaluate in the reference's normalised form
    const vec3<double> coor_l2 = normalized(l2h);
    const vec2<double> cs2 = dehom(cross(coor_l2, normalized(eps_)));
    const vec2<double> ce2 = dehom(cross(coor_l2, normalized(epe_)));
    const vec2<double> dir2 = normalized(v2d);
    const double len2 = norm(s2 - e2);
    c1 = dot(cs2 - s2, dir2) / len2;
    c2 = dot(ce2 - s2, dir2) / len2;
    if (c1 > c2) { double t = c1; c1 = c2; c2 = t; }
    IoU = (smin(c2, 1.0) - smax(c1, 0.0)) / (smax(c2, 1.0) - smin(c1, 0.0));
  }
  return IoU;
}
template <typename EP> LM_D double epipolar_iou(const EP &ep, double4 l2, double th) {
  const vec2<double> s2 = mk2(l2.x, l2.y), e2 = mk2(l2.z, l2.w);
  const vec2<double> v2d = e2 - s2;
  return epipolar_iou(ep, l2, s2, e2, v2d, dot(v2d, v2d), th);
}
// The epipolar lines from the source rays where they are used: F x1 = M2^T ((C1 - C2) x (M1 x1)) exactly
// (F = K2^-T [t]x R2 R1^T K1^-1 with t = R2 (C1 - C2)). M2 = R2^T K2^-1 of the second view, base = C1 - C2, w1s / w1e =
// M1 [p; 1] of the source endpoints, held by reference so that the node kernel loads them from shared memory where it
// always did.
struct EpipolarFromRays {
  const double *M2;
  vec3<double> base;
  const vec3<double> &w1s, &w1e;
  LM_D vec3<double> start() const { return mat3T_mul(M2, cross(base, w1s)); }
  LM_D vec3<double> end() const { return mat3T_mul(M2, cross(base, w1e)); }
};
// The same lines computed once for every target line of a (source line, second view) pair.
struct EpipolarLines {
  vec3<double> s, e;
  LM_D EpipolarLines(const double *M2, vec3<double> base, vec3<double> w1s, vec3<double> w1e)
      : s(mat3T_mul(M2, cross(base, w1s))), e(mat3T_mul(M2, cross(base, w1e))) {}
  LM_D vec3<double> start() const { return s; }
  LM_D vec3<double> end() const { return e; }
};

// ------------------------------------------------------------------------------------------------
// Segment helpers shared by the 2d and 3d linkers (base/line_dists.h).
template <typename V> struct seg {
  V s, e;
};
template <typename V> LM_HD V direction(const seg<V> &l) { return normalized(l.e - l.s); }
template <typename V> LM_HD auto length(const seg<V> &l) -> decltype(norm(l.s)) { return norm(l.s - l.e); }

// line_dists.h:190-201 compute_overlap
template <typename T, typename V> LM_HD T compute_overlap(const seg<V> &l1, const seg<V> &l2) {
  T len = length(l2);
  V v = direction(l2);
  T p1 = dot(l1.s - l2.s, v) / len;
  T p2 = dot(l1.e - l2.s, v) / len;
  if (p1 > p2) { T t = p1; p1 = p2; p2 = t; }
  return smin<T>(p2, T(1)) - smax<T>(p1, T(0));
}
// line_dists.h:203-208
template <typename T, typename V> LM_HD T compute_bioverlap(const seg<V> &l1, const seg<V> &l2) {
  T v1 = compute_overlap<T, V>(l1, l2);
  T v2 = compute_overlap<T, V>(l2, l1);
  return smax<T>(v1, v2);
}
// line_dists.h:105-133: max of the four endpoint-to-infinite-line distances
template <typename T, typename V> LM_HD T dist_perp_oneway_max(const seg<V> &l1, const seg<V> &l2) {
  V v2 = direction(l2);
  V ds = l1.s - l2.s;
  T a = dot(ds, v2);
  T d12s = sqrt(smax<T>(sqnorm(ds) - a * a, T(0)));
  V de = l1.e - l2.s;
  T b = dot(de, v2);
  T d12e = sqrt(smax<T>(sqnorm(de) - b * b, T(0)));
  return (d12s < d12e) ? d12e : d12s; // used inside a max_element over 4 values
}
template <typename T, typename V> LM_HD T dist_endpoints_perpendicular(const seg<V> &l1, const seg<V> &l2) {
  // std::max_element over {d12s,d12e,d21s,d21e}: first maximal element; value is what matters.
  V v2 = direction(l2);
  V ds = l1.s - l2.s;
  T a = dot(ds, v2);
  T d0 = sqrt(smax<T>(sqnorm(ds) - a * a, T(0)));
  V de = l1.e - l2.s;
  T b = dot(de, v2);
  T d1 = sqrt(smax<T>(sqnorm(de) - b * b, T(0)));
  V v1 = direction(l1);
  V es = l2.s - l1.s;
  T c = dot(es, v1);
  T d2 = sqrt(smax<T>(sqnorm(es) - c * c, T(0)));
  V ee = l2.e - l1.s;
  T d = dot(ee, v1);
  T d3 = sqrt(smax<T>(sqnorm(ee) - d * d, T(0)));
  T m = d0;
  if (m < d1) m = d1;
  if (m < d2) m = d2;
  if (m < d3) m = d3;
  return m;
}
// line_dists.h:160-187
template <typename T, typename V> LM_HD bool get_innerseg(const seg<V> &l1, const seg<V> &l2, seg<V> &inner) {
  V l1_dir = direction(l1);
  V d2 = l2.e - l2.s;
  T denom = dot(d2, l1_dir);
  T t1 = dot(l1.s - l2.s, l1_dir) / (denom + consts<T>::eps());
  T t2 = dot(l1.e - l2.s, l1_dir) / (denom + consts<T>::eps());
  if (t1 > t2) { T t = t1; t1 = t2; t2 = t; }
  if (t1 >= T(1) || t2 <= T(0)) return false;
  inner.s = l2.s + d2 * smax<T>(t1, T(0));
  inner.e = l2.s + d2 * smin<T>(t2, T(1));
  return true;
}
template <typename T, typename V> LM_HD T dist_innerseg(const seg<V> &l1, const seg<V> &l2) {
  seg<V> a, b;
  if (!get_innerseg<T, V>(l2, l1, a)) return consts<T>::maxval();
  if (!get_innerseg<T, V>(l1, l2, b)) return consts<T>::maxval();
  return dist_endpoints_perpendicular<T, V>(a, b);
}

// ------------------------------------------------------------------------------------------------
// Linker configuration as the kernels see it (base/line_linker.h). mult = 1/sqrt(-2 ln score_th).
template <typename T> struct LinkerDev {
  T score_th, th_angle, th_overlap, th_smartoverlap, th_smartangle, th_perp, th_innerseg, th_scaleinv, mult;
  int use_angle, use_overlap, use_smartangle, use_perp, use_innerseg, use_scaleinv;
};

// line_linker.cc:15-17
template <typename T> LM_HD T expscore(T val, T sigma) {
  T q = val / sigma;
  return exp(-(q * q) / T(2));
}
template <typename T> LM_HD T thresh0(T s, T th) { return (s < th) ? T(0) : s; }

// line_dists.h:53-66
template <typename T, typename V> LM_HD T compute_angle(const seg<V> &l1, const seg<V> &l2) {
  T c = fabs(dot(direction(l1), direction(l2)));
  return acos(c) * consts<T>::rad2deg();
}

// LineLinker{2d,3d}::compute_score (line_linker.cc:139-160, :306-331). unc = 1 for 2d,
// min(uncertainty) for 3d (line_linker.cc:239-262). depth_s/e are l1's depths for scale-invariance
// (line_dists.cc:55-60).
template <typename T, typename V>
LM_HD T linker_score(const LinkerDev<T> &c, const seg<V> &l1, const seg<V> &l2, T unc, bool is3d, T depth_s, T depth_e) {
  T score = T(1);
  T angle = T(0);
  if (c.use_angle) {
    angle = compute_angle<T, V>(l1, l2);
    score = smin<T>(score, thresh0(expscore(angle, c.th_angle * c.mult), c.score_th));
  }
  if (score < c.score_th) return score;
  T bio = T(0);
  if (c.use_overlap) {
    bio = compute_bioverlap<T, V>(l1, l2);
    score = smin<T>(score, (bio > c.th_overlap) ? T(1) : T(0));
  }
  if (score < c.score_th) return score;
  if (c.use_angle && c.use_overlap && c.use_smartangle) {
    T th_angle = c.th_angle;
    if (bio < c.th_smartoverlap) {
      T ratio = (c.th_smartoverlap - bio) / (c.th_smartoverlap - c.th_overlap);
      ratio = smin<T>(ratio, T(1));
      th_angle = c.th_angle - ratio * (c.th_angle - c.th_smartangle);
    }
    score = smin<T>(score, thresh0(expscore(angle, th_angle * c.mult), c.score_th));
  }
  if (score < c.score_th) return score;
  if (c.use_perp) {
    T dist = dist_endpoints_perpendicular<T, V>(l1, l2);
    score = smin<T>(score, thresh0(expscore(dist, c.th_perp * unc * c.mult), c.score_th));
  }
  if (score < c.score_th) return score;
  if (c.use_innerseg) {
    T dist = dist_innerseg<T, V>(l1, l2);
    score = smin<T>(score, thresh0(expscore(dist, c.th_innerseg * unc * c.mult), c.score_th));
  }
  if (is3d) {
    if (score < c.score_th) return score;
    if (c.use_scaleinv) {
      T ds = norm(l1.s - l2.s), de = norm(l1.e - l2.e);
      T dist = smax<T>(ds / (depth_s + consts<T>::eps()), de / (depth_e + consts<T>::eps()));
      score = smin<T>(score, thresh0(expscore(dist, c.th_scaleinv * c.mult), c.score_th));
    }
  }
  return score;
}

} // namespace lm
