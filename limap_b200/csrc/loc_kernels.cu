// loc_kernels.cu — batched joint point + line pose refinement of query images for sm_90a.
//
// Replaces the Ceres problems of
//   LineLocEngine / JointLocEngine::{SetUp,Solve}   (optimize/hybrid_localization/hybrid_localization.cc:11-130)
// which the reference builds and solves one query after another. Every query is an independent 6-dof problem: qvec on
// the QuaternionManifold, tvec free, the PINHOLE intrinsics constant.
//
// One warp owns one query for the whole solve; persistent warps fetch queries from a counter, because solves end after
// very different iteration counts. A query's residual blocks are digested once (loc_prepare_kernel); lanes stride over
// them and accumulate the loss-corrected normal equations (J^T J 21, J^T r 6, cost, 6 column norms) in block order; the
// lanes' partial sums are then reduced by a fixed butterfly, so a query's result does not depend on which other queries
// share the launch.
//
// Residuals (loc_block.cuh): ReprojectionLineFunctor / ReprojectionPointFunctor (cost_functions.h:204-347), value path
// operation for operation with the reference's Jets (a Jet quotient multiplies by the reciprocal; Dual<6> does the
// same). Derivatives are carried as 6-wide duals seeded on the tangent at delta = 0 (QuaternionPlusJacobian columns on
// qvec, identity on tvec), which is Ceres' ambient Jacobian chained through the plus Jacobian. The cost function is a
// template parameter (six straight-line instantiations); weight and loss are per-launch constants. The solver is the
// trust-region LM of lm_kernels.cu (DESIGN.md §5) on the 6-dof tangent, with a 6x6 L D L^T solve.
#include "loc_block.cuh"
#include <algorithm>
#include <cfloat>

namespace lm {

namespace {

using namespace loc;

LM_D double warp_sum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d); // a + b == b + a: every lane ends equal
  return v;
}

struct LocNormal {
  double A[kNA], g[6], cost, cn2[6];
};

// All blocks of one query at x (qvec, tvec): cost and the loss-corrected normal equations, with the Jacobi column
// scaling applied when scale != NULL. The result is written to *out by lane 0 (shared memory) after the reduction.
template <int CF>
LM_D void loc_eval(const LocParams &p, const LocBlockDev *blocks, int64_t nb, const double *xs, const double *kq,
                   const double *scale, LocNormal *out) {
  const int lane = threadIdx.x & 31;
  D k[4], q[4], qc[4], u[4], t[3];
  {
    double x[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) x[i] = xs[i];
    pose_duals(x, kq, k, q, qc, u, t);
  }
  double A[kNA], g[6], cn2[6], cost = 0.0;
#pragma unroll
  for (int i = 0; i < kNA; ++i) A[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) { g[i] = 0.0; cn2[i] = 0.0; }
  for (int64_t kb = lane; kb < nb; kb += 32) {
    const LocBlockDev &B = blocks[kb];
    D r[4];
    int m;
    if (B.kind == 0) {
      line_residual<CF>(B, p.weight_function, k, q, qc, u, t, r);
      m = NumRes<CF>::value;
    } else {
      point_residual(B, p.points_3d_dist != 0, k, qc, u, t, r);
      m = 2;
    }
    if (m < 4) r[3] = K(0.0);
    if (m < 3) r[2] = K(0.0);
    const double s = r[0].a * r[0].a + r[1].a * r[1].a + r[2].a * r[2].a + r[3].a * r[3].a;
    double rho[3];
    loss_eval(p.loss_kind, p.loss_scale, B.a, s, rho);
    cost += 0.5 * rho[0];
    const Corrector corr(s, rho);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i >= m) break;
      double J[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const double v = corr.jacobian(r, m, i, c);
        cn2[c] += v * v;
        J[c] = scale ? v * scale[c] : v;
      }
      const double ri = r[i].a * corr.residual_scaling;
      int idx = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        g[a] += J[a] * ri;
#pragma unroll
        for (int c = a; c < 6; ++c) A[idx++] += J[a] * J[c];
      }
    }
  }
  // fixed-order reduction over the warp
#pragma unroll
  for (int i = 0; i < kNA; ++i) A[i] = warp_sum(A[i]);
#pragma unroll
  for (int i = 0; i < 6; ++i) { g[i] = warp_sum(g[i]); cn2[i] = warp_sum(cn2[i]); }
  cost = warp_sum(cost);
  __syncwarp();
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kNA; ++i) out->A[i] = A[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) { out->g[i] = g[i]; out->cn2[i] = cn2[i]; }
    // an evaluation with non-finite residuals fails: Ceres gives the candidate the largest cost
    out->cost = isfinite(cost) ? cost : DBL_MAX;
  }
  __syncwarp();
}

struct LocWarpState {
  double x[7], cand[7], scale[6], diag[6], kq[4];
  LocNormal N, Nc;
};

template <int CF> __global__ void __launch_bounds__(128) loc_refine_kernel(const __grid_constant__ LocParams p) {
  __shared__ LocWarpState s_ws[4];
  LocWarpState &ws = s_ws[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  for (;;) {
    long long qi = 0;
    if (lane == 0) qi = (long long)atomicAdd(p.next_query, 1ull);
    qi = __shfl_sync(0xffffffffu, qi, 0);
    if (qi >= p.Q) break;
    const int64_t b0 = p.blk_off[qi], nb = p.blk_off[qi + 1] - b0;
    const LocBlockDev *blocks = p.blocks + b0;
    __syncwarp();
    if (lane < 7) ws.x[lane] = p.x0[7 * qi + lane];
    if (lane < 4) ws.kq[lane] = p.kvec[4 * qi + lane];
    __syncwarp();
    int it = 0, successful = 0, term = 0;
    double cost0 = 0.0, cost = 0.0;
    if (nb > 0) {
      loc_eval<CF>(p, blocks, nb, ws.x, ws.kq, nullptr, &ws.N);
      cost0 = cost = ws.N.cost;
      if (cost0 == DBL_MAX) term = 7; // the initial evaluation failed
    }
    if (nb > 0 && term == 0) {
      // Jacobi scaling 1/(1 + ||J_col||), fixed at iteration 0
      if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 6; ++c) ws.scale[c] = 1.0 / (1.0 + sqrt(ws.N.cn2[c]));
        int idx = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          ws.N.g[a] *= ws.scale[a];
#pragma unroll
          for (int c = a; c < 6; ++c) ws.N.A[idx++] *= ws.scale[a] * ws.scale[c];
        }
      }
      __syncwarp();
      double radius = 1e4, decrease_factor = 2.0;
      bool reuse_diagonal = false;
      int invalid = 0;
      for (;;) {
        if (it >= p.max_num_iterations) { term = 1; break; }
        if (radius <= 1e-32) { term = 2; break; }
        {
          double gmax = 0;
#pragma unroll
          for (int c = 0; c < 6; ++c) gmax = fmax(gmax, fabs(ws.N.g[c]));
          if (gmax <= 0.0) { term = 3; break; }
        }
        ++it;
        if (!reuse_diagonal) {
          __syncwarp();
          if (lane == 0) {
            const int di[6] = {0, 6, 11, 15, 18, 20};
#pragma unroll
            for (int c = 0; c < 6; ++c) ws.diag[c] = fmin(fmax(ws.N.A[di[c]], 1e-6), 1e32);
          }
          __syncwarp();
        }
        reuse_diagonal = true;
        // the 6x6 solve is warp-uniform: every lane computes it from the shared state
        double step[6], mcc = 0.0;
        bool ok;
        {
          double An[kNA], gn[6], dg[6];
#pragma unroll
          for (int c = 0; c < kNA; ++c) An[c] = ws.N.A[c];
#pragma unroll
          for (int c = 0; c < 6; ++c) { gn[c] = ws.N.g[c]; dg[c] = ws.diag[c] / radius; }
          ok = ldlt_solve6(An, dg, gn, step);
#pragma unroll
          for (int c = 0; c < 6; ++c) { step[c] = -step[c]; if (!isfinite(step[c])) ok = false; }
          if (ok) { // model_cost_change = -(step . g + step^T (J^T J) step / 2)
            double sg = 0, sAs = 0;
            int idx = 0;
#pragma unroll
            for (int a = 0; a < 6; ++a) {
              sg += step[a] * gn[a];
#pragma unroll
              for (int c = a; c < 6; ++c) { sAs += ((a == c) ? 1.0 : 2.0) * step[a] * step[c] * An[idx]; ++idx; }
            }
            mcc = -(sg + 0.5 * sAs);
          }
        }
        if (!ok || !(mcc > 0.0)) {
          if (++invalid >= p.max_invalid) { term = 4; break; }
          radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
          continue;
        }
        invalid = 0;
        double sn = 0.0;
        {
          double xr[7], delta[3], cand[7];
#pragma unroll
          for (int c = 0; c < 7; ++c) xr[c] = ws.x[c];
#pragma unroll
          for (int c = 0; c < 3; ++c) delta[c] = step[c] * ws.scale[c];
          quat_plus(xr, delta, cand);
#pragma unroll
          for (int c = 0; c < 3; ++c) cand[4 + c] = xr[4 + c] + step[3 + c] * ws.scale[3 + c];
#pragma unroll
          for (int c = 0; c < 7; ++c) sn += (xr[c] - cand[c]) * (xr[c] - cand[c]);
          __syncwarp();
          if (lane == 0) {
#pragma unroll
            for (int c = 0; c < 7; ++c) ws.cand[c] = cand[c];
          }
          __syncwarp();
        }
        // one evaluation per iteration: the candidate with its Jacobian, kept when the step is accepted
        loc_eval<CF>(p, blocks, nb, ws.cand, ws.kq, ws.scale, &ws.Nc);
        const double cost_c = ws.Nc.cost;
        if (!(sqrt(sn) > 0.0)) { term = 5; break; }
        if (!(fabs(cost - cost_c) > 0.0)) { term = 6; break; }
        const double rel = (cost - cost_c) / mcc;
        if (rel > 1e-3) {
          __syncwarp();
          if (lane < 7) ws.x[lane] = ws.cand[lane];
          if (lane < kNA) ws.N.A[lane] = ws.Nc.A[lane];
          if (lane < 6) ws.N.g[lane] = ws.Nc.g[lane];
          __syncwarp();
          cost = cost_c;
          const double tq = 2.0 * rel - 1.0;
          radius = fmin(1e16, radius / fmax(1.0 / 3.0, 1.0 - tq * tq * tq));
          decrease_factor = 2.0; reuse_diagonal = false;
          ++successful;
        } else {
          radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
        }
      }
    }
    __syncwarp();
    if (lane < 7) p.x_out[7 * qi + lane] = ws.x[lane];
    if (lane == 0) {
      p.iters[2 * qi] = it; p.iters[2 * qi + 1] = successful;
      p.cost[2 * qi] = cost0; p.cost[2 * qi + 1] = cost;
      // Summary::IsSolutionUsable: not after a failed initial evaluation or too many invalid steps
      p.flags[qi] = nb > 0 ? (uint8_t)(1 | ((term != 4 && term != 7) ? 2 : 0)) : (uint8_t)0;
    }
  }
}

// One thread per block: the line blocks of 2D line j (with the group's length sum) and point i, at their slot
// blk_off[q] + position in the query (lines first, in group order, then points)
__global__ void loc_prepare_kernel(const int64_t *__restrict__ grp_off, const double *__restrict__ l3d,
                                   const int64_t *__restrict__ l2d_off, const double *__restrict__ l2d,
                                   const int64_t *__restrict__ pt_off, const double *__restrict__ p3d,
                                   const double *__restrict__ p2d, const int64_t *__restrict__ blk_off, int64_t Q,
                                   int64_t G, int64_t n_l2d, int64_t n_pts, double weight_line, double weight_point,
                                   LocBlockDev *__restrict__ out) {
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (k >= n_l2d + n_pts) return;
  LocBlockDev B;
  B.pad = 0;
  if (k < n_l2d) {
    const int64_t g = last_le<true>(l2d_off, G + 1, k);
    const int64_t q = last_le<true>(grp_off, Q + 1, g);
    double sum = 0.0; // JointLocEngine::AddResiduals: sum of Line2d::length() over the group, in order
    for (int64_t j = l2d_off[g]; j < l2d_off[g + 1]; ++j) {
      const double dx = l2d[4 * j] - l2d[4 * j + 2], dy = l2d[4 * j + 1] - l2d[4 * j + 3];
      sum += sqrt(dx * dx + dy * dy);
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) B.v[i] = l3d[6 * g + i];
#pragma unroll
    for (int i = 0; i < 4; ++i) B.v[6 + i] = l2d[4 * k + i];
    const double dx = B.v[6] - B.v[8], dy = B.v[7] - B.v[9];
    B.a = weight_line * sqrt(dx * dx + dy * dy) / sum;
    B.kind = 0;
    out[blk_off[q] + (k - l2d_off[grp_off[q]])] = B;
  } else {
    const int64_t i = k - n_l2d;
    const int64_t q = last_le<true>(pt_off, Q + 1, i);
#pragma unroll
    for (int c = 0; c < 3; ++c) B.v[c] = p3d[3 * i + c];
    B.v[3] = p2d[2 * i];
    B.v[4] = p2d[2 * i + 1];
#pragma unroll
    for (int c = 5; c < 10; ++c) B.v[c] = 0.0;
    B.a = weight_point;
    B.kind = 1;
    const int64_t n_lines_q = l2d_off[grp_off[q + 1]] - l2d_off[grp_off[q]];
    out[blk_off[q] + n_lines_q + (i - pt_off[q])] = B;
  }
}

} // namespace

void launch_loc_prepare(const int64_t *grp_off, const double *l3d, const int64_t *l2d_off, const double *l2d,
                        const int64_t *pt_off, const double *p3d, const double *p2d, const int64_t *blk_off, int64_t Q,
                        int64_t G, int64_t n_l2d, int64_t n_pts, double weight_line, double weight_point,
                        LocBlockDev *out, cudaStream_t s) {
  const int64_t n = n_l2d + n_pts;
  if (n <= 0) return;
  loc_prepare_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(grp_off, l3d, l2d_off, l2d, pt_off, p3d, p2d, blk_off, Q, G,
                                                            n_l2d, n_pts, weight_line, weight_point, out);
}

void launch_loc_refine(const LocParams &p, int cost_function, cudaStream_t s) {
  if (p.Q <= 0) return;
  const int warps = 4;
  const int grid = (int)std::min<int64_t>((p.Q + warps - 1) / warps, (int64_t)current_device_sms() * 8);
  switch (cost_function) {
  case 0: loc_refine_kernel<0><<<grid, warps * 32, 0, s>>>(p); break;
  case 1: loc_refine_kernel<1><<<grid, warps * 32, 0, s>>>(p); break;
  case 2: loc_refine_kernel<2><<<grid, warps * 32, 0, s>>>(p); break;
  case 3: loc_refine_kernel<3><<<grid, warps * 32, 0, s>>>(p); break;
  case 4: loc_refine_kernel<4><<<grid, warps * 32, 0, s>>>(p); break;
  default: loc_refine_kernel<5><<<grid, warps * 32, 0, s>>>(p); break;
  }
}

} // namespace lm
