// Host build of limap_b200/csrc/loc_block.cuh for tests/test_loc_block_host.py: the query pose refinement's residual
// blocks, loss, corrector and step solve, exported as batch functions over flat double arrays (ctypes). No device code
// runs; the test compiles this file with nvcc into a temporary directory.
#include "../limap_b200/csrc/loc_block.cuh"

using namespace lm;
using namespace lm::loc;

namespace {
template <int CF>
void eval_block(int kind, int wf, int use3d, const double *data, const double *kvec, const double *x, double *res,
                double *jac) {
  D k[4], q[4], qc[4], u[4], t[3], r[4];
  pose_duals(x, kvec, k, q, qc, u, t);
  LocBlockDev B;
  for (int i = 0; i < 10; ++i) B.v[i] = data[i];
  B.a = 1.0;
  B.kind = kind;
  B.pad = 0;
  int m = 2;
  if (kind == 0) { line_residual<CF>(B, wf, k, q, qc, u, t, r); m = NumRes<CF>::value; }
  else point_residual(B, use3d != 0, k, qc, u, t, r);
  for (int i = 0; i < 4; ++i) {
    res[i] = i < m ? r[i].a : 0.0;
    for (int c = 0; c < 6; ++c) jac[6 * i + c] = i < m ? r[i].v[c] : 0.0;
  }
}
} // namespace

extern "C" {

// kind[n] (0 line: data = l3d[6] + l2d[4]; 1 point: data = p3d[3] + p2d[2]), data[n][10], kvec[n][4], x[n][7] (qvec,
// tvec) -> res[n][4], jac[n][4][6] (tangent columns: quaternion 3, translation 3), zero past the block's residuals
void loch_block(int64_t n, int cf, int wf, int use3d, const int32_t *kind, const double *data, const double *kvec,
                const double *x, double *res, double *jac) {
  for (int64_t t = 0; t < n; ++t) {
    const double *d = data + 10 * t, *k = kvec + 4 * t, *xx = x + 7 * t;
    double *r = res + 4 * t, *j = jac + 24 * t;
    switch (cf) {
    case 0: eval_block<0>(kind[t], wf, use3d, d, k, xx, r, j); break;
    case 1: eval_block<1>(kind[t], wf, use3d, d, k, xx, r, j); break;
    case 2: eval_block<2>(kind[t], wf, use3d, d, k, xx, r, j); break;
    case 3: eval_block<3>(kind[t], wf, use3d, d, k, xx, r, j); break;
    case 4: eval_block<4>(kind[t], wf, use3d, d, k, xx, r, j); break;
    default: eval_block<5>(kind[t], wf, use3d, d, k, xx, r, j); break;
    }
  }
}

// s[n], a[n] -> rho[n][3] (loss_eval, ScaledLoss factor a)
void loch_loss(int64_t n, int kind, double scale, const double *a, const double *s, double *rho) {
  for (int64_t t = 0; t < n; ++t) loss_eval(kind, scale, a[t], s[t], rho + 3 * t);
}

// A block of m residuals res[n][4] with tangent Jacobian jac[n][4][6], under loss (kind, scale) with factor a[n]: rho
// of its squared norm, then the corrector's residuals rc[n][4] and Jacobian jc[n][4][6], as loc_eval forms them
void loch_corrector(int64_t n, int m, int kind, double scale, const double *a, const double *res, const double *jac,
                    double *rho, double *rc, double *jc) {
  for (int64_t t = 0; t < n; ++t) {
    D r[4];
    for (int i = 0; i < 4; ++i) {
      r[i].a = i < m ? res[4 * t + i] : 0.0;
      for (int c = 0; c < 6; ++c) r[i].v[c] = i < m ? jac[24 * t + 6 * i + c] : 0.0;
    }
    const double s = r[0].a * r[0].a + r[1].a * r[1].a + r[2].a * r[2].a + r[3].a * r[3].a;
    double *rh = rho + 3 * t;
    loss_eval(kind, scale, a[t], s, rh);
    const Corrector corr(s, rh);
    for (int i = 0; i < 4; ++i) {
      rc[4 * t + i] = i < m ? r[i].a * corr.residual_scaling : 0.0;
      for (int c = 0; c < 6; ++c) jc[24 * t + 6 * i + c] = i < m ? corr.jacobian(r, m, i, c) : 0.0;
    }
  }
}

// (A + diag(dg)) x = b with A packed[n][21] (row a holds columns a..5) -> x[n][6], ok[n]
void loch_ldlt(int64_t n, const double *Ap, const double *dg, const double *b, double *x, int32_t *ok) {
  for (int64_t t = 0; t < n; ++t) ok[t] = ldlt_solve6(Ap + kNA * t, dg + 6 * t, b + 6 * t, x + 6 * t) ? 1 : 0;
}

} // extern "C"
