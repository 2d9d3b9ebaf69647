// Robust pose-graph optimisation (tzr_pose_graph_optimize, DESIGN.md §3.16): Open3D's multiway-registration step with
// GNC-TLS in place of its line process, written out as this project's own definition in include/teaser_b200.h.  One
// graph per call; the host runs the GNC-TLS iterations and reads back PgState once per iteration, and every inner
// Levenberg-Marquardt iteration is enqueued without a synchronisation:
//
//   pg_edge_kernel      one thread per edge: the residual e = (log R_E, t_E) of E = T_d^-1 T_s T_sd^-1 at the current or
//                       the candidate poses, e^T Lambda e, r-bar, and the Jacobian terms A^T Lambda A and A^T Lambda e
//                       with A = Ad(T_d^-1).
//   pg_cost_kernel      one warp: the weighted cost sum w_e e^T Lambda e in a fixed order; starts the inner solve (mode
//                       0) or decides on a candidate step (mode 1: accept or reject, the damping, the stop test).
//   pg_assemble_kernel  one warp per listed 6 x 6 block of H (lower triangle) or 6-row block of the right-hand side:
//                       its contributions in ascending edge index, in the order the host planned, so no atomics and no
//                       dependence on scheduling; the diagonal carries the damping.
//   (cuSOLVER)          cusolverDnDpotrf + cusolverDnDpotrs on the dense (K - 1) 6-row system.
//   pg_update_kernel    one thread per node: the candidate pose Exp(delta_k) T_k.
//   pg_gnc_kernel       one warp: the GNC-TLS weight update of the uncertain edges from r-bar, the rotation stage's
//                       schedule.
//
// Everything is IEEE float64 with no FMA contraction (the library's -fmad=false).
#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr double kPgLambda0 = 1e-4;      // initial damping of every inner solve
constexpr double kPgLambdaMax = 1e8;     // a rejection that raises the damping past this ends the inner solve
constexpr double kPgRelTol = 1e-10;      // |cost - candidate cost| <= kPgRelTol cost + floor ends the inner solve

// c = a b for 3 x 3 column-major matrices; entry (r, k): (a(r,0) b(0,k) + a(r,1) b(1,k)) + a(r,2) b(2,k)
__device__ __forceinline__ void m33(const double* a, const double* b, double* c) {
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) c[3 * k + r] = (a[r] * b[3 * k] + a[3 + r] * b[3 * k + 1]) + a[6 + r] * b[3 * k + 2];
}
// c = a^T b
__device__ __forceinline__ void m33_tn(const double* a, const double* b, double* c) {
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r)
      c[3 * k + r] = (a[3 * r] * b[3 * k] + a[3 * r + 1] * b[3 * k + 1]) + a[3 * r + 2] * b[3 * k + 2];
}
// c = a b^T
__device__ __forceinline__ void m33_nt(const double* a, const double* b, double* c) {
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) c[3 * k + r] = (a[r] * b[k] + a[3 + r] * b[3 + k]) + a[6 + r] * b[6 + k];
}
// y = a x, y = a^T x
__device__ __forceinline__ void mv3(const double* a, const double* x, double* y) {
#pragma unroll
  for (int r = 0; r < 3; ++r) y[r] = (a[r] * x[0] + a[3 + r] * x[1]) + a[6 + r] * x[2];
}
__device__ __forceinline__ void mtv3(const double* a, const double* x, double* y) {
#pragma unroll
  for (int r = 0; r < 3; ++r) y[r] = (a[3 * r] * x[0] + a[3 * r + 1] * x[1]) + a[3 * r + 2] * x[2];
}

// omega = log(R) (column-major R), include/teaser_b200.h: v = vee(R - R^T) / 2, c = (tr R - 1) / 2,
// theta = atan2(|v|, c); theta < 1e-5: omega = (1 + theta^2 / 6) v; c < -0.9: the axis from the symmetric part
// (its largest diagonal's column) with the sign of v; otherwise omega = (theta / |v|) v
__device__ void so3_log(const double* R, double w[3]) {
  const double v[3] = {0.5 * (R[5] - R[7]), 0.5 * (R[6] - R[2]), 0.5 * (R[1] - R[3])};
  const double s = sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
  const double c = 0.5 * (((R[0] + R[4]) + R[8]) - 1.0);
  const double th = atan2(s, c);
  if (th < 1e-5) {
    const double f = 1.0 + th * th / 6.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = f * v[k];
  } else if (c < -0.9) {
    double B[9];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int r = 0; r < 3; ++r) B[3 * k + r] = 0.5 * (R[3 * k + r] + R[3 * r + k]) - (r == k ? c : 0.0);
    int k = 0;
    if (B[4] > B[0]) k = 1;
    if (B[8] > B[4 * k]) k = 2;
    const double nrm = sqrt(B[4 * k] * (1.0 - c));
    double a[3] = {B[3 * k] / nrm, B[3 * k + 1] / nrm, B[3 * k + 2] / nrm};
    if ((a[0] * v[0] + a[1] * v[1]) + a[2] * v[2] < 0.0)
#pragma unroll
      for (int r = 0; r < 3; ++r) a[r] = -a[r];
#pragma unroll
    for (int r = 0; r < 3; ++r) w[r] = th * a[r];
  } else {
    const double f = th / s;
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = f * v[k];
  }
}

// (R, t) = Exp(w, tau) in SE(3): R = I + b [w]x + a' [w]x^2 (Rodrigues), t = V tau with V = I + b' [w]x + c' [w]x^2;
// theta = |w| < 1e-5 takes the series a' = 1/2 - theta^2/24, b = 1 - theta^2/6, b' = 1/2 - theta^2/24,
// c' = 1/6 - theta^2/120
__device__ void se3_exp(const double w[3], const double tau[3], double R[9], double t[3]) {
  const double th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2];
  const double th = sqrt(th2);
  double A, Bq, Vb, Vc;
  if (th < 1e-5) {
    A = 1.0 - th2 / 6.0;
    Bq = 0.5 - th2 / 24.0;
    Vb = 0.5 - th2 / 24.0;
    Vc = 1.0 / 6.0 - th2 / 120.0;
  } else {
    const double sn = sin(th), cs = cos(th);
    A = sn / th;
    Bq = (1.0 - cs) / th2;
    Vb = Bq;
    Vc = (th - sn) / (th2 * th);
  }
  // W = [w]x, W2 = W W (column-major)
  const double W[9] = {0.0, w[2], -w[1], -w[2], 0.0, w[0], w[1], -w[0], 0.0};
  double W2[9];
  m33(W, W, W2);
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const double I = (k == 0 || k == 4 || k == 8) ? 1.0 : 0.0;
    R[k] = (I + A * W[k]) + Bq * W2[k];
  }
  double V[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const double I = (k == 0 || k == 4 || k == 8) ? 1.0 : 0.0;
    V[k] = (I + Vb * W[k]) + Vc * W2[k];
  }
  mv3(V, tau, t);
}

__device__ __forceinline__ double* pose_at(const PgDev& dv, int K, int buf, int k) {
  return dv.poses + 12 * ((size_t)buf * K + k);
}
__device__ __forceinline__ double* term_at(const PgDev& dv, int E, int buf, int e) {
  return dv.eterm + kPgTermStride * ((size_t)buf * E + e);
}

// Edge e's terms at the poses in buffer buf into that buffer's terms (pg_edge_kernel and the batched solve share it)
__device__ __forceinline__ void pg_edge_terms(const PgDev& dv, int K, int E, int buf, int e) {
  const PgEdge& ed = dv.edges[e];
  const double* Ts = pose_at(dv, K, buf, ed.s);
  const double* Td = pose_at(dv, K, buf, ed.d);
  // R_E = R_d^T (R_s R_sd^T), t_E = R_d^T ((t_s - t_d) - (R_s R_sd^T) t_sd)
  double Q[9], RE[9], u[3], w[3], tE[3];
  m33_nt(Ts, ed.R, Q);
  m33_tn(Td, Q, RE);
  mv3(Q, ed.t, u);
#pragma unroll
  for (int r = 0; r < 3; ++r) w[r] = (Ts[9 + r] - Td[9 + r]) - u[r];
  mtv3(Td, w, tE);
  double err[6];
  so3_log(RE, err);
  err[3] = tE[0];
  err[4] = tE[1];
  err[5] = tE[2];
  // Le = Lambda e, c = e^T Lambda e
  double Le[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) a = a + ed.L[6 * r + k] * err[k];
    Le[r] = a;
  }
  double c = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) c = c + err[k] * Le[k];
  // A = Ad(T_d^-1) = [[Rt, 0], [[p]x Rt, Rt]] with Rt = R_d^T, p = -R_d^T t_d
  double p[3], Rt[9];
  mtv3(Td, Td + 9, p);
#pragma unroll
  for (int r = 0; r < 3; ++r) p[r] = -p[r];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) Rt[3 * k + r] = Td[3 * r + k];
  const double P[9] = {0.0, p[2], -p[1], -p[2], 0.0, p[0], p[1], -p[0], 0.0};
  double PR[9];
  m33(P, Rt, PR);
  double A[6][6];  // A[row][col]
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      A[r][k] = Rt[3 * k + r];
      A[r][3 + k] = 0.0;
      A[3 + r][k] = PR[3 * k + r];
      A[3 + r][3 + k] = Rt[3 * k + r];
    }
  double* out = term_at(dv, E, buf, e);
  // LA = Lambda A; M = A^T (Lambda A), v = A^T Le
  double LA[6][6];
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double a = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) a = a + ed.L[6 * r + q] * A[q][k];
      LA[r][k] = a;
    }
#pragma unroll
  for (int r = 0; r < 6; ++r) {
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double a = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) a = a + A[q][r] * LA[q][k];
      out[6 * r + k] = a;
    }
    double a = 0.0;
#pragma unroll
    for (int q = 0; q < 6; ++q) a = a + A[q][r] * Le[q];
    out[36 + r] = a;
  }
  out[42] = c;
  out[43] = c * ed.inv_norm;
}

// which = 0: the current poses into the current terms; 1: the candidate poses (the other buffer), skipped once the
// inner solve has stopped
__global__ void pg_edge_kernel(PgDev dv, int K, int E, int which) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const PgState& st = *dv.state;
  if (which == 1 && st.done) return;
  pg_edge_terms(dv, K, E, which == 0 ? st.cur : 1 - st.cur, e);
}

// The fixed-order weighted sum over one warp: lane l adds w_e x_e for e = l, l + 32, ... in turn, then a butterfly
__device__ double pg_warp_sum(const PgDev& dv, int E, int buf) {
  double a = 0.0;
  for (int e = threadIdx.x; e < E; e += 32) a = a + dv.weight[e] * term_at(dv, E, buf, e)[42];
  for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  return a;
}

// pg_cost_kernel's two modes on the state st, run by one warp.  Start: the inner solve at the current poses' cost.
__device__ __forceinline__ void pg_cost_start(const PgDev& dv, PgState& st, int E) {
  const double cost = pg_warp_sum(dv, E, st.cur);
  if (threadIdx.x != 0) return;
  st.cost = cost;
  st.lambda = kPgLambda0;
  st.done = 0;
  st.inner = 0;
}

// Step: the decision on the candidate poses' cost (include/teaser_b200.h states the rule)
__device__ __forceinline__ void pg_cost_step(const PgDev& dv, PgState& st, int E, double cost_floor) {
  if (st.done) return;
  const double cand = pg_warp_sum(dv, E, 1 - st.cur);
  if (threadIdx.x != 0) return;
  st.cand_cost = cand;
  st.inner += 1;
  const bool ok = st.info[0] == 0 && st.info[1] == 0 && isfinite(cand);
  if (ok && fabs(st.cost - cand) <= kPgRelTol * st.cost + cost_floor) {
    if (cand < st.cost) {
      st.cur = 1 - st.cur;
      st.cost = cand;
    }
    st.done = 1;
  } else if (ok && cand < st.cost) {
    st.cur = 1 - st.cur;
    st.cost = cand;
    st.lambda = st.lambda * 0.1;
  } else {
    st.lambda = st.lambda * 10.0;
    if (st.lambda > kPgLambdaMax) st.done = 1;
  }
}

// mode 0: start the inner solve at the current poses; mode 1: decide on the candidate
__global__ void pg_cost_kernel(PgDev dv, int E, int mode, double cost_floor) {
  PgState& st = *dv.state;
  if (mode == 0) {
    pg_cost_start(dv, st, E);
    return;
  }
  pg_cost_step(dv, st, E, cost_floor);
}

// One warp's share of pg_assemble_kernel: listed block bl of H (lower triangle; entry (r, k) = sum of sign * (w_e
// M_e(r, k)) in the listed order, then on a diagonal block's diagonal a + lambda (a + 1)) or the right-hand side block
// -(sum of sign * (w_e v_e(r))) into g
__device__ __forceinline__ void pg_assemble_block(const PgDev& dv, const PgState& st, int E, int n, int cur,
                                                  const PgBlock bl, int lane, double* g) {
  if (bl.bj < 0) {
    if (lane >= 6) return;
    double a = 0.0;
    for (int q = bl.lo; q < bl.hi; ++q) {
      const PgTerm tm = dv.terms[q];
      a = a + (double)tm.sign * (dv.weight[tm.e] * term_at(dv, E, cur, tm.e)[36 + lane]);
    }
    g[6 * bl.bi + lane] = -a;
    return;
  }
  for (int l = lane; l < 36; l += 32) {
    const int r = l / 6, k = l % 6;
    double a = 0.0;
    for (int q = bl.lo; q < bl.hi; ++q) {
      const PgTerm tm = dv.terms[q];
      a = a + (double)tm.sign * (dv.weight[tm.e] * term_at(dv, E, cur, tm.e)[6 * r + k]);
    }
    if (bl.bi == bl.bj && r == k) a = a + st.lambda * (a + 1.0);
    dv.H[(size_t)(6 * bl.bi + r) + (size_t)(6 * bl.bj + k) * (size_t)n] = a;
  }
}

// One warp per listed block.  H block (bi, bj), bi >= bj: entry (r, k) = sum over its terms of sign * (w_e M_e(r, k))
// in the listed order, then on a diagonal block's diagonal a + lambda (a + 1): the additive part keeps the damped system
// positive definite when a node's every edge has weight 0 (its block of H is then 0); H is column-major n x n and
// only its lower triangle is read.  Right-hand-side block bi (bj = -1): -(sum of sign * (w_e v_e(r))).
__global__ void pg_assemble_kernel(PgDev dv, int E, int n, int nblocks) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= nblocks) return;
  const PgState& st = *dv.state;
  if (st.done) return;
  pg_assemble_block(dv, st, E, n, st.cur, dv.blocks[b], lane, dv.g);
}

// The candidate Tn = Exp(x) T (R' = R_x R, t' = R_x t + t_x) from the node's 6 entries x of the step
__device__ __forceinline__ void pg_candidate(const double* T, const double* x, double* Tn) {
  double Rx[9], tx[3], u[3];
  se3_exp(x, x + 3, Rx, tx);
  m33(Rx, T, Tn);
  mv3(Rx, T + 9, u);
#pragma unroll
  for (int r = 0; r < 3; ++r) Tn[9 + r] = u[r] + tx[r];
}

// One thread per node: the candidate T_k' = Exp(delta_k) T_k; the reference node keeps its pose
__global__ void pg_update_kernel(PgDev dv, int K, int ref) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const PgState& st = *dv.state;
  if (st.done) return;
  const double* T = pose_at(dv, K, st.cur, k);
  double* Tn = pose_at(dv, K, 1 - st.cur, k);
  if (k == ref) {
    for (int q = 0; q < 12; ++q) Tn[q] = T[q];
    return;
  }
  pg_candidate(T, dv.g + 6 * (k < ref ? k : k - 1), Tn);
}

// GNC-TLS after GNC iteration `iter` (the rotation stage's schedule on r-bar, include/teaser_b200.h), run by one warp
// (lane = threadIdx.x) on the state st.  The weight formula is a copy of gnc_tls_block's (rot_trans.cu), not a shared
// function: sharing it would move the rotation kernels' code, which must stay as it is, and this one reads a
// normalised residual (noise bound 1) from one warp.
__device__ __forceinline__ void pg_gnc_rule(const PgDev& dv, PgState& st, int E, int iter, double gnc_factor,
                                            double cost_threshold) {
  const int lane = threadIdx.x;
  const int cur = st.cur;
  int n_unc = 0;
  double rmax = 0.0;
  for (int e = lane; e < E; e += 32)
    if (dv.edges[e].uncertain) {
      ++n_unc;
      rmax = fmax(rmax, term_at(dv, E, cur, e)[43]);
    }
  for (int o = 16; o; o >>= 1) {
    n_unc += __shfl_xor_sync(0xffffffffu, n_unc, o);
    rmax = fmax(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
  }
  if (n_unc == 0) {  // every edge certain: no GNC step
    if (lane == 0) st.stop = 1;
    return;
  }
  double mu = st.mu;
  if (iter == 0) {
    // stop unless mu is finite and positive: 2 max r-bar - 1 <= 0 means every uncertain edge is an inlier, and at
    // max r-bar = 1/2 exactly mu would be +inf and every weight NaN
    mu = 1.0 / (2.0 * rmax - 1.0);
    if (!(mu > 0.0) || isinf(mu)) {
      if (lane == 0) {
        st.mu = mu;
        st.stop = 1;
      }
      return;
    }
  }
  const double th1 = (mu + 1.0) / mu;
  const double th2 = mu / (mu + 1.0);
  double c = 0.0;
  for (int e = lane; e < E; e += 32) {
    if (!dv.edges[e].uncertain) continue;
    const double r = term_at(dv, E, cur, e)[43];
    c = c + dv.weight[e] * r;
    double wn;
    if (r >= th1)
      wn = 0.0;
    else if (r <= th2)
      wn = 1.0;
    else
      wn = sqrt(mu * (mu + 1.0) / r) - mu;
    dv.weight[e] = wn;
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane != 0) return;
  const double diff = fabs(c - st.gnc_cost);
  st.mu = mu * gnc_factor;
  st.gnc_cost = c;
  if (diff < cost_threshold) st.stop = 1;
}

__global__ void pg_gnc_kernel(PgDev dv, int E, int iter, double gnc_factor, double cost_threshold) {
  pg_gnc_rule(dv, *dv.state, E, iter, gnc_factor, cost_threshold);
}

}  // namespace

int launch_pose_graph_begin(const PgPlan& plan, const PgDev& dv, double cost_floor, cudaStream_t st) {
  pg_edge_kernel<<<(plan.E + 127) / 128, 128, 0, st>>>(dv, plan.K, plan.E, 0);
  pg_cost_kernel<<<1, 32, 0, st>>>(dv, plan.E, 0, cost_floor);
  return 2;
}

int launch_pose_graph_assemble(const PgPlan& plan, const PgDev& dv, cudaStream_t st) {
  pg_assemble_kernel<<<(plan.blocks + 3) / 4, 128, 0, st>>>(dv, plan.E, plan.n, plan.blocks);
  return 1;
}

int launch_pose_graph_step(const PgPlan& plan, const PgDev& dv, int ref, double cost_floor, cudaStream_t st) {
  pg_update_kernel<<<(plan.K + 127) / 128, 128, 0, st>>>(dv, plan.K, ref);
  pg_edge_kernel<<<(plan.E + 127) / 128, 128, 0, st>>>(dv, plan.K, plan.E, 1);
  pg_cost_kernel<<<1, 32, 0, st>>>(dv, plan.E, 1, cost_floor);
  return 3;
}

int launch_pose_graph_gnc(const PgPlan& plan, const PgDev& dv, int iter, cudaStream_t st) {
  pg_gnc_kernel<<<1, 32, 0, st>>>(dv, plan.E, iter, plan.gnc_factor, plan.cost_threshold);
  return 1;
}

// ---- Open3D's line process (tzr_pose_graph_optimize_line_process, DESIGN.md §3.22) -------------------------------------
//   lp_edge_kernel      one thread per edge: M = X^-1 T_d^-1 T_s, zeta = lin(M), J_s from the generator products,
//                       J_s^T Lambda J_s, J_s^T Lambda zeta and zeta^T Lambda zeta at the current, candidate or returned
//                       poses.
//   lp_begin_kernel     one block: F with the incoming confidences, then the confidence update; starts the pass.
//   lp_assemble_kernel  one warp per listed block: H (undamped) and b = -sum sign l_e v_e, as pg_assemble_kernel.
//   lp_stats_kernel     one block: max(b), |x|; at the start lambda = 1e-5 max diag(H); after an accepted trial the
//                       end of the outer iteration (min_right_term, min_residual, max_iteration).
//   lp_damp_kernel      H + lambda I (lower triangle) and b into the factor buffer, which potrf overwrites.
//   (cuSOLVER)          cusolverDnDpotrf + cusolverDnDpotrs on the 6 K rows.
//   lp_step_kernel      one block: |delta|, delta . (lambda delta + b) and the min_relative_increment rule.
//   lp_update_kernel    one thread per node: the candidate V(delta_k) T_k.
//   lp_decide_kernel    one block: F' with the old confidences, rho, accept / reject, the lambda / nu schedule and the
//                       trial rules; an accepted candidate updates the confidences.
// Every kernel returns at once when the pass has stopped.  Reductions run in one block in a fixed order: thread t adds
// the entries t, t + blockDim, ... in turn, then a shared-memory tree (tests/line_process_reference.py: block_sum).
namespace {

constexpr int kLpSmall = 256;   // threads of the edge-sum kernels (begin, decide)
constexpr int kLpLarge = 1024;  // threads of the kernels that reduce over 6 K entries or K nodes (step, stats)

struct Pose12 {
  double v[12];
};

__device__ __forceinline__ double* lp_pose(const LpDev& dv, int K, int buf, int k) {
  return dv.poses + 12 * ((size_t)buf * K + k);
}
__device__ __forceinline__ double* lp_terms(const LpDev& dv, int E, int buf, int e) {
  return dv.eterm + kPgTermStride * ((size_t)buf * E + e);
}

// the block's fixed-order sum / max of one value per thread (blockDim a power of two)
__device__ double lp_block_sum(double a, double* sh) {
  const int t = threadIdx.x;
  sh[t] = a;
  __syncthreads();
  for (int s = blockDim.x >> 1; s; s >>= 1) {
    if (t < s) sh[t] = sh[t] + sh[t + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}
__device__ double lp_block_max(double a, double* sh) {
  const int t = threadIdx.x;
  sh[t] = a;
  __syncthreads();
  for (int s = blockDim.x >> 1; s; s >>= 1) {
    if (t < s) sh[t] = fmax(sh[t], sh[t + s]);
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// F = sum_e l_e c_e + mu (sqrt(l_e) - 1)^2 over edge-term buffer buf
__device__ double lp_residual(const LpDev& dv, int E, int buf, double mu, double* sh) {
  double a = 0.0;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const double l = dv.conf[e], q = sqrt(l) - 1.0;
    a = a + (l * lp_terms(dv, E, buf, e)[42] + mu * (q * q));
  }
  return lp_block_sum(a, sh);
}

// the confidence update of the uncertain edges from edge-term buffer buf: l = (mu / (mu + c))^2
__device__ void lp_confidences(const LpDev& dv, int E, int buf, double mu) {
  for (int e = threadIdx.x; e < E; e += blockDim.x)
    if (dv.edges[e].uncertain) {
      const double q = mu / (mu + lp_terms(dv, E, buf, e)[42]);
      dv.conf[e] = q * q;
    }
}

// lin(N) of the top 3 x 4 of a 4 x 4 matrix: N column-major 3 x 3 and its translation column
__device__ __forceinline__ void lp_lin(const double* N, const double* t, double* z) {
  z[0] = 0.5 * (N[5] - N[7]);
  z[1] = 0.5 * (N[6] - N[2]);
  z[2] = 0.5 * (N[1] - N[3]);
  z[3] = t[0];
  z[4] = t[1];
  z[5] = t[2];
}

// One edge's terms at poses Ts, Td into out (kPgTermStride doubles; lp_edge_kernel and the batched pass share it)
__device__ __forceinline__ void lp_edge_terms(const PgEdge& ed, const double* Ts, const double* Td, double* out) {
  // P = X^-1 T_d^-1: R_P = (R_d R_X)^T, t_P = -R_X^T (R_d^T t_d + t_X); M = P T_s
  double RdX[9], RP[9], u[3], tP[3], RM[9], tM[3];
  m33(Td, ed.R, RdX);
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) RP[3 * k + r] = RdX[3 * r + k];
  mtv3(Td, Td + 9, u);
#pragma unroll
  for (int r = 0; r < 3; ++r) u[r] = u[r] + ed.t[r];
  mtv3(ed.R, u, tP);
#pragma unroll
  for (int r = 0; r < 3; ++r) tP[r] = -tP[r];
  m33(RP, Ts, RM);
  mv3(RP, Ts + 9, tM);
#pragma unroll
  for (int r = 0; r < 3; ++r) tM[r] = tM[r] + tP[r];
  double z[6];
  lp_lin(RM, tM, z);
  // J_s[:, i] = lin(P G_i T_s): G_0..2 the skew generators, G_3..5 the unit translations
  double J[6][6];  // J[row][col]
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double G[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    // skew(e_i), column-major: (i=0) (2,1) = 1, (1,2) = -1; (i=1) (0,2) = 1, (2,0) = -1; (i=2) (1,0) = 1, (0,1) = -1
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    G[3 * j + k] = 1.0;
    G[3 * k + j] = -1.0;
    double Q[9], N[9], tN[3], col[6];
    m33(RP, G, Q);
    m33(Q, Ts, N);
    mv3(Q, Ts + 9, tN);
    lp_lin(N, tN, col);
#pragma unroll
    for (int r = 0; r < 6; ++r) J[r][i] = col[r];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int r = 0; r < 3; ++r) J[r][3 + i] = 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) J[3 + r][3 + i] = RP[3 * i + r];
  }
  // Lz = Lambda zeta, c = zeta^T Lambda zeta
  double Lz[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) a = a + ed.L[6 * r + k] * z[k];
    Lz[r] = a;
  }
  double c = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) c = c + z[k] * Lz[k];
  double LJ[6][6];
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double a = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) a = a + ed.L[6 * r + q] * J[q][k];
      LJ[r][k] = a;
    }
#pragma unroll
  for (int r = 0; r < 6; ++r) {
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double a = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) a = a + J[q][r] * LJ[q][k];
      out[6 * r + k] = a;
    }
    double a = 0.0;
#pragma unroll
    for (int q = 0; q < 6; ++q) a = a + J[q][r] * Lz[q];
    out[36 + r] = a;
  }
  out[42] = c;
}

// which = 0: the current poses into the current terms; 1: the candidate poses (the other buffer), skipped once the pass
// has stopped or the trial formed no candidate; 2: the other buffer, always (the compensated poses)
__global__ void lp_edge_kernel(LpDev dv, int K, int E, int which) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const LpState& st = *dv.state;
  if (which == 1 && (st.done || st.skip)) return;
  const int buf = which == 0 ? st.cur : 1 - st.cur;
  const PgEdge& ed = dv.edges[e];
  lp_edge_terms(ed, lp_pose(dv, K, buf, ed.s), lp_pose(dv, K, buf, ed.d), lp_terms(dv, E, buf, e));
}

// The start of a pass: F with the incoming confidences, then their update; H and b follow
__global__ void lp_begin_kernel(LpDev dv, LpPlan p) {
  __shared__ double sh[kLpSmall];
  LpState& st = *dv.state;
  const double F = lp_residual(dv, p.E, st.cur, p.mu, sh);
  lp_confidences(dv, p.E, st.cur, p.mu);
  if (threadIdx.x != 0) return;
  st.F = F;
  st.Fc = 0.0;
  st.nu = 2.0;
  st.done = st.reason = st.skip = 0;
  st.accepted = 1;
  st.iter = st.lm = st.trials = 0;
}

// One warp per listed block: H block (bi, bj), bi >= bj: sum of sign * (l_e A_e(r, k)) in the listed order (column-major
// n x n, lower blocks only); b block bi (bj = -1): -(sum of sign * (l_e v_e(r))).  Only after the start or an accepted
// trial.
// Entry j of a block: sum of sign * (l_e term_e[j]) over its terms in the listed order, as lp_assemble_kernel sums it
// (that kernel keeps its own loop, whose machine code this helper would move)
__device__ __forceinline__ double lp_block_entry(const LpDev& dv, int E, int cur, const PgBlock& bl, int j) {
  double a = 0.0;
  for (int q = bl.lo; q < bl.hi; ++q) {
    const PgTerm tm = dv.terms[q];
    a = a + (double)tm.sign * (dv.conf[tm.e] * lp_terms(dv, E, cur, tm.e)[j]);
  }
  return a;
}

__global__ void lp_assemble_kernel(LpDev dv, int E, int n, int nblocks) {
  const int bk = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (bk >= nblocks) return;
  const LpState& st = *dv.state;
  if (st.done || !st.accepted) return;
  const PgBlock bl = dv.blocks[bk];
  const int cur = st.cur;
  if (bl.bj < 0) {
    if (lane >= 6) return;
    double a = 0.0;
    for (int q = bl.lo; q < bl.hi; ++q) {
      const PgTerm tm = dv.terms[q];
      a = a + (double)tm.sign * (dv.conf[tm.e] * lp_terms(dv, E, cur, tm.e)[36 + lane]);
    }
    dv.b[6 * bl.bi + lane] = -a;
    return;
  }
  for (int l = lane; l < 36; l += 32) {
    const int r = l / 6, k = l % 6;
    double a = 0.0;
    for (int q = bl.lo; q < bl.hi; ++q) {
      const PgTerm tm = dv.terms[q];
      a = a + (double)tm.sign * (dv.conf[tm.e] * lp_terms(dv, E, cur, tm.e)[6 * r + k]);
    }
    dv.H[(size_t)(6 * bl.bi + r) + (size_t)(6 * bl.bj + k) * (size_t)n] = a;
  }
}

// Open3D's TransformMatrix4dToVector6d of a pose (R column-major): ZYX Euler angles, then t; its squared norm in order
__device__ double lp_euler_sq(const double* T) {
  const double sy = sqrt(T[0] * T[0] + T[1] * T[1]);
  double x, y, z;
  if (!(sy < 1e-6)) {
    x = atan2(T[5], T[8]);
    y = atan2(-T[2], sy);
    z = atan2(T[1], T[0]);
  } else {
    x = atan2(-T[7], T[4]);
    y = atan2(-T[2], sy);
    z = 0.0;
  }
  return ((((x * x + y * y) + z * z) + T[9] * T[9]) + T[10] * T[10]) + T[11] * T[11];
}

// The rules of lp_stats_kernel once max(b) = bm, max diag(H) = hm (mode 0) and |x|^2 = xs are known, for the batched
// pass (lp_stats_kernel keeps its own copy, whose machine code calling this helper would move)
__device__ __forceinline__ void lp_stats_rule(LpState& st, const LpPlan& p, int mode, double bm, double hm, double xs) {
  st.xnorm = sqrt(xs);
  if (mode == 0) st.lambda = 1e-5 * hm;
  if (bm < p.min_right_term) {
    st.done = 1;
    st.reason = TZR_LP_STOP_RIGHT_TERM;
  }
  if (mode == 0) return;
  st.lm = 0;
  if (!st.done && st.F < p.min_residual) {
    st.done = 1;
    st.reason = TZR_LP_STOP_MIN_RESIDUAL;
  }
  if (!st.done && st.iter >= p.max_iteration) {
    st.done = 1;
    st.reason = TZR_LP_STOP_MAX_ITERATION;
  }
}

// mode 0: the start of a pass (lambda = 1e-5 max diag H, nu = 2); mode 1: after an accepted trial, the end of the outer
// iteration.  Both: max(b) against min_right_term and |x| of the current poses.
__global__ void lp_stats_kernel(LpDev dv, LpPlan p, int mode) {
  __shared__ double sh[kLpLarge];
  LpState& st = *dv.state;
  if (st.done || !st.accepted) return;
  double bm = -INFINITY, hm = -INFINITY;
  for (int i = threadIdx.x; i < p.n; i += blockDim.x) {
    bm = fmax(bm, dv.b[i]);
    if (mode == 0) hm = fmax(hm, dv.H[(size_t)i * p.n + i]);
  }
  bm = lp_block_max(bm, sh);
  if (mode == 0) hm = lp_block_max(hm, sh);
  double xs = 0.0;
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) xs = xs + lp_euler_sq(lp_pose(dv, p.K, st.cur, k));
  xs = lp_block_sum(xs, sh);
  if (threadIdx.x != 0) return;
  st.xnorm = sqrt(xs);
  if (mode == 0) st.lambda = 1e-5 * hm;
  if (bm < p.min_right_term) {
    st.done = 1;
    st.reason = TZR_LP_STOP_RIGHT_TERM;
  }
  if (mode == 0) return;
  st.lm = 0;
  if (!st.done && st.F < p.min_residual) {
    st.done = 1;
    st.reason = TZR_LP_STOP_MIN_RESIDUAL;
  }
  if (!st.done && st.iter >= p.max_iteration) {
    st.done = 1;
    st.reason = TZR_LP_STOP_MAX_ITERATION;
  }
}

// H + lambda I (lower triangle; A's upper triangle is not read) into A and b into delta.  Grid (ceil(n / 256), n): one
// thread per row of column blockIdx.y.
__global__ void lp_damp_kernel(LpDev dv, int n) {
  const LpState& st = *dv.state;
  if (st.done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n) return;
  if (j == 0) dv.delta[i] = dv.b[i];
  if (i < j) return;
  const size_t o = (size_t)i + (size_t)j * n;
  dv.A[o] = i == j ? dv.H[o] + st.lambda : dv.H[o];
}

// The trial's outcome before any candidate from |delta|^2 = s2 and pd = delta . (lambda delta + b)
__device__ __forceinline__ void lp_step_rule(LpState& st, const LpPlan& p, double s2, double pd) {
  const double dn = sqrt(s2);
  st.dnorm = dn;
  st.pred = pd;
  if (st.info[0] != 0 || st.info[1] != 0 || !isfinite(s2) || !isfinite(pd))
    st.skip = 2;
  else if (dn < p.min_rel_inc * (st.xnorm + p.min_rel_inc))
    st.skip = 1;
  else
    st.skip = 0;
}

// |delta|, delta . (lambda delta + b) and the trial's outcome before any candidate: skip 2 when the factorisation failed
// or delta is not finite, 1 when |delta| < min_relative_increment (|x| + min_relative_increment)
__global__ void lp_step_kernel(LpDev dv, LpPlan p) {
  __shared__ double sh[kLpLarge];
  LpState& st = *dv.state;
  if (st.done) return;
  const double lam = st.lambda;
  double s2 = 0.0, pd = 0.0;
  for (int i = threadIdx.x; i < p.n; i += blockDim.x) {
    const double d = dv.delta[i];
    s2 = s2 + d * d;
    pd = pd + d * (lam * d + dv.b[i]);
  }
  s2 = lp_block_sum(s2, sh);
  pd = lp_block_sum(pd, sh);
  if (threadIdx.x != 0) return;
  lp_step_rule(st, p, s2, pd);
}

// The candidate Tn = V(d) T, V(d) = [R_z(d_2) R_y(d_1) R_x(d_0) | (d_3, d_4, d_5)]
__device__ __forceinline__ void lp_candidate(const double* T, const double* d, double* Tn) {
  const double cx = cos(d[0]), sx = sin(d[0]), cy = cos(d[1]), sy = sin(d[1]), cz = cos(d[2]), sz = sin(d[2]);
  const double Rz[9] = {cz, sz, 0.0, -sz, cz, 0.0, 0.0, 0.0, 1.0};
  const double Ry[9] = {cy, 0.0, -sy, 0.0, 1.0, 0.0, sy, 0.0, cy};
  const double Rx[9] = {1.0, 0.0, 0.0, 0.0, cx, sx, 0.0, -sx, cx};
  double Rzy[9], V[9], u[3];
  m33(Rz, Ry, Rzy);
  m33(Rzy, Rx, V);
  m33(V, T, Tn);
  mv3(V, T + 9, u);
#pragma unroll
  for (int r = 0; r < 3; ++r) Tn[9 + r] = u[r] + d[3 + r];
}

// One thread per node: the candidate V(delta_k) T_k
__global__ void lp_update_kernel(LpDev dv, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const LpState& st = *dv.state;
  if (st.done || st.skip) return;
  lp_candidate(lp_pose(dv, K, st.cur, k), dv.delta + 6 * (size_t)k, lp_pose(dv, K, 1 - st.cur, k));
}

// The trial's decision from F' = Fc (include/teaser_b200.h states the rules in order); returns 1 when the candidate
// is accepted
__device__ __forceinline__ int lp_decide_rule(LpState& st, const LpPlan& p, int skip, double Fc) {
  if (st.lm == 0) st.iter += 1;
  st.lm += 1;
  st.trials += 1;
  st.Fc = Fc;
  int a = 0;
  if (skip == 1) {
    st.done = 1;
    st.reason = TZR_LP_STOP_REL_INCREMENT;
  } else {
    const double dF = st.F - Fc;
    const double rho = skip ? -1.0 : dF / (st.pred + 1e-3);
    if (rho > 0.0 && dF < p.min_rel_res_inc * st.F) {
      st.done = 1;
      st.reason = TZR_LP_STOP_REL_RESIDUAL;
    } else if (rho > 0.0) {
      const double q = 2.0 * rho - 1.0;
      st.lambda = st.lambda * fmax(p.lower, fmin(p.upper, 1.0 - (q * q) * q));
      st.nu = 2.0;
      st.F = Fc;
      st.cur = 1 - st.cur;
      a = 1;
    } else {
      st.lambda = st.lambda * st.nu;
      st.nu = 2.0 * st.nu;
    }
  }
  if (!st.done && st.lm >= p.max_lm) {
    st.done = 1;
    st.reason = TZR_LP_STOP_LM_TRIALS;
  }
  st.accepted = a;
  return a;
}

// The trial's decision
__global__ void lp_decide_kernel(LpDev dv, LpPlan p) {
  __shared__ double sh[kLpSmall];
  __shared__ int acc;
  LpState& st = *dv.state;
  if (st.done) return;
  const int skip = st.skip;
  const double Fc = skip ? 0.0 : lp_residual(dv, p.E, 1 - st.cur, p.mu, sh);
  if (threadIdx.x == 0) acc = lp_decide_rule(st, p, skip, Fc);
  __syncthreads();
  if (acc) lp_confidences(dv, p.E, st.cur, p.mu);
}

// Tn = C T with C = T0 (T_ref)^-1 (each caller forms C in the same order)
__device__ __forceinline__ void lp_compensate_pose(const double* T0, const double* Tr, const double* T, double* Tn) {
  // C: R_C = R0 R_ref^T, t_C = t0 - R_C t_ref
  double RC[9], tC[3], u[3];
  m33_nt(T0, Tr, RC);
  mv3(RC, Tr + 9, u);
#pragma unroll
  for (int r = 0; r < 3; ++r) tC[r] = T0[9 + r] - u[r];
  m33(RC, T, Tn);
  mv3(RC, T + 9, u);
#pragma unroll
  for (int r = 0; r < 3; ++r) Tn[9 + r] = u[r] + tC[r];
}

// The compensation T_k <- C T_k with C = T0 (T_ref)^-1 into the other buffer
__global__ void lp_compensate_kernel(LpDev dv, int K, int ref, Pose12 T0) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const LpState& st = *dv.state;
  lp_compensate_pose(T0.v, lp_pose(dv, K, st.cur, ref), lp_pose(dv, K, st.cur, k), lp_pose(dv, K, 1 - st.cur, k));
}

// ---- many graphs in one call (tzr_pose_graph_optimize_line_process_batch, DESIGN.md §3.23) ----------------------------
// lp_batch_kernel: one CTA of kLbThreads per graph runs a whole pass of the line process: the edge terms, F and the
// confidence update, H and b over the host's block plan, the start's statistics, then every trial (H + lambda I, a dense
// Cholesky of the 6 K rows, the two substitutions, |delta| and delta . (lambda delta + b), the candidate and its edge
// terms, the decision, and after an accepted trial the rebuilt H and b) until the pass stops, with the pass's state in
// shared memory.  The rules are the single entry's helpers above (lp_edge_terms, lp_candidate, lp_step_rule,
// lp_decide_rule, lp_stats_rule, lp_block_entry, lp_residual, lp_confidences, lp_compensate_pose).  Every reduction is
// a fixed-shape block reduction over kLbThreads, so a graph's result depends on nothing but the graph.
constexpr int kLbThreads = 256;  // threads per graph
constexpr int kLbNb = 32;        // Cholesky panel width
constexpr int kLbDt = 33;        // row stride of the diagonal tile in shared memory

// Dense Cholesky A = L L^T of the lower triangle of the column-major n x n A, in place, right-looking in panels of 32
// columns: the diagonal tile is factored in shared memory (Dt), the rows below it are solved against it one thread per
// row and kept in shared memory (Ps: column k of the panel at Ps + k ldp), then the trailing lower triangle is updated
// in 64 x 64 tiles, 4 x 4 entries per thread, by FP64 FMAs in ascending k.  The strict upper triangle is neither read
// nor written.  Returns 0, or 1 + the first column whose pivot is not > 0 (NaN included); every thread returns the same.
__device__ int lb_cholesky(double* A, int n, double* Ps, int ldp, double* Dt) {
  const int t = threadIdx.x;
  for (int j0 = 0; j0 < n; j0 += kLbNb) {
    const int nb = min(kLbNb, n - j0), p = j0 + nb, m = n - p;
    for (int w = t; w < nb * nb; w += kLbThreads) {
      const int r = w % nb, c = w / nb;
      if (r >= c) Dt[r * kLbDt + c] = A[(size_t)(j0 + r) + (size_t)(j0 + c) * n];
    }
    __syncthreads();
    for (int k = 0; k < nb; ++k) {
      const double piv = Dt[k * kLbDt + k];
      if (!(piv > 0.0)) return j0 + k + 1;
      const double lkk = sqrt(piv);
      if (t > k && t < nb) Dt[t * kLbDt + k] = Dt[t * kLbDt + k] / lkk;
      __syncthreads();
      if (t == 0) Dt[k * kLbDt + k] = lkk;
      const int q = nb - 1 - k;
      for (int w = t; w < q * q; w += kLbThreads) {
        const int r = k + 1 + w % q, c = k + 1 + w / q;
        if (r >= c) Dt[r * kLbDt + c] = Dt[r * kLbDt + c] - Dt[r * kLbDt + k] * Dt[c * kLbDt + k];
      }
      __syncthreads();
    }
    for (int w = t; w < nb * nb; w += kLbThreads) {
      const int r = w % nb, c = w / nb;
      if (r >= c) A[(size_t)(j0 + r) + (size_t)(j0 + c) * n] = Dt[r * kLbDt + c];
    }
    if (m == 0) break;  // the last panel; any panel with rows below it is 32 wide
    // L21 = A21 L11^-T: row i solves x L11^T = a by forward substitution
    for (int i = p + t; i < n; i += kLbThreads) {
      double x[kLbNb];
#pragma unroll
      for (int k = 0; k < kLbNb; ++k) {
        double s = A[(size_t)i + (size_t)(j0 + k) * n];
#pragma unroll
        for (int q = 0; q < k; ++q) s = fma(-x[q], Dt[k * kLbDt + q], s);
        x[k] = s / Dt[k * kLbDt + k];
        A[(size_t)i + (size_t)(j0 + k) * n] = x[k];
        Ps[k * ldp + (i - p)] = x[k];
      }
    }
    __syncthreads();
    // A22 -= L21 L21^T on the lower 64 x 64 tiles; thread (tr, tc) owns rows tr + 16 a and columns tc + 16 c of a tile
    const int T = (m + 63) / 64, tr = t & 15, tc = t >> 4;
    for (int ti = 0; ti < T; ++ti)
      for (int tj = 0; tj <= ti; ++tj) {
        int ri[4], cj[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          ri[a] = 64 * ti + tr + 16 * a;
          cj[a] = 64 * tj + tc + 16 * a;
        }
        double acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
#pragma unroll 4
        for (int k = 0; k < kLbNb; ++k) {
          const double* col = Ps + k * ldp;
          double u[4], v[4];
#pragma unroll
          for (int a = 0; a < 4; ++a) {
            u[a] = col[min(ri[a], m - 1)];
            v[a] = col[min(cj[a], m - 1)];
          }
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[a][c] = fma(u[a], v[c], acc[a][c]);
        }
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (ri[a] < m && ri[a] >= cj[c]) {
              double* e = A + (size_t)(p + ri[a]) + (size_t)(p + cj[c]) * n;
              *e = *e - acc[a][c];
            }
      }
    __syncthreads();
  }
  return 0;
}

// x <- (L L^T)^-1 x with the factor of lb_cholesky (x in shared memory).  Each 32-row block's triangle is solved by
// warp 0 (one row per lane, the solved entry broadcast by a shuffle); the forward sweep then updates the rows below one
// thread per row, and the backward sweep first forms each block's sum over the rows below it, one warp per column, the
// lanes' partial sums added by a butterfly.
__device__ void lb_solve(const double* A, int n, double* x, double* tmp) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int j0 = 0; j0 < n; j0 += kLbNb) {
    const int nb = min(kLbNb, n - j0);
    if (warp == 0) {
      double v = lane < nb ? x[j0 + lane] : 0.0;
      for (int k = 0; k < nb; ++k) {
        if (lane == k) v = v / A[(size_t)(j0 + k) * (n + 1)];
        const double yk = __shfl_sync(0xffffffffu, v, k);
        if (lane > k && lane < nb) v = v - A[(size_t)(j0 + lane) + (size_t)(j0 + k) * n] * yk;
      }
      if (lane < nb) x[j0 + lane] = v;
    }
    __syncthreads();
    for (int i = j0 + nb + t; i < n; i += kLbThreads) {
      double s = x[i];
      for (int k = 0; k < nb; ++k) s = s - A[(size_t)i + (size_t)(j0 + k) * n] * x[j0 + k];
      x[i] = s;
    }
    __syncthreads();
  }
  for (int j0 = ((n - 1) / kLbNb) * kLbNb; j0 >= 0; j0 -= kLbNb) {
    const int nb = min(kLbNb, n - j0), p = j0 + nb;
    for (int c = warp; c < nb; c += kLbThreads / 32) {
      double s = 0.0;
      for (int i = p + lane; i < n; i += 32) s = s + A[(size_t)i + (size_t)(j0 + c) * n] * x[i];
      for (int o = 16; o; o >>= 1) s = s + __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) tmp[c] = s;
    }
    __syncthreads();
    if (warp == 0) {
      double v = lane < nb ? x[j0 + lane] - tmp[lane] : 0.0;
      for (int k = nb - 1; k >= 0; --k) {
        if (lane == k) v = v / A[(size_t)(j0 + k) * (n + 1)];
        const double xk = __shfl_sync(0xffffffffu, v, k);
        if (lane < k) v = v - A[(size_t)(j0 + k) + (size_t)(j0 + lane) * n] * xk;
      }
      if (lane < nb) x[j0 + lane] = v;
    }
    __syncthreads();
  }
}

// H (listed lower blocks) and b from the terms in buffer cur, one thread per block entry
__device__ void lb_assemble(const LpDev& dv, const LpPlan& p, int cur) {
  for (int w = threadIdx.x; w < p.blocks * 36; w += kLbThreads) {
    const PgBlock bl = dv.blocks[w / 36];
    const int j = w % 36;
    if (bl.bj < 0) {
      if (j < 6) dv.b[6 * bl.bi + j] = -lp_block_entry(dv, p.E, cur, bl, 36 + j);
    } else {
      dv.H[(size_t)(6 * bl.bi + j / 6) + (size_t)(6 * bl.bj + j % 6) * (size_t)p.n] = lp_block_entry(dv, p.E, cur, bl, j);
    }
  }
  __syncthreads();
}

// max(b), max diag(H) (mode 0) and |x| of the current poses, then lp_stats_rule
__device__ void lb_stats(const LpDev& dv, const LpPlan& p, int mode, LpState& st, double* red) {
  double bm = -INFINITY, hm = -INFINITY;
  for (int i = threadIdx.x; i < p.n; i += kLbThreads) {
    bm = fmax(bm, dv.b[i]);
    if (mode == 0) hm = fmax(hm, dv.H[(size_t)i * p.n + i]);
  }
  bm = lp_block_max(bm, red);
  if (mode == 0) hm = lp_block_max(hm, red);
  double xs = 0.0;
  for (int k = threadIdx.x; k < p.K; k += kLbThreads) xs = xs + lp_euler_sq(lp_pose(dv, p.K, st.cur, k));
  xs = lp_block_sum(xs, red);
  if (threadIdx.x == 0) lp_stats_rule(st, p, mode, bm, hm, xs);
  __syncthreads();
}

// the terms of every edge at the poses in buffer buf
__device__ void lb_edges(const LpDev& dv, int K, int E, int buf) {
  for (int e = threadIdx.x; e < E; e += kLbThreads) {
    const PgEdge& ed = dv.edges[e];
    lp_edge_terms(ed, lp_pose(dv, K, buf, ed.s), lp_pose(dv, K, buf, ed.d), lp_terms(dv, E, buf, e));
  }
  __syncthreads();
}

// One pass of graph blockIdx.x.  pass 0 starts from the graph's starting poses; pass 1 continues from the poses pass 0
// left (its state's cur), then compensates and evaluates every edge of pass 1's table at the returned poses.  Both
// write the state and the confidences to the graph's output slice, pass 1 also the poses and the residuals.
__global__ void __launch_bounds__(kLbThreads) lp_batch_kernel(const LpBatchGraph* graphs, int pass, int ldp) {
  extern __shared__ double smem[];
  double* Ps = smem;                   // kLbNb x ldp: the Cholesky panel
  double* Dt = Ps + kLbNb * ldp;       // kLbNb x kLbDt: its diagonal tile
  double* x = Dt + kLbNb * kLbDt;      // ldp: b, then delta
  double* red = x + ldp;               // kLbThreads: block reductions
  double* tmp = red + kLbThreads;      // kLbNb: the backward sweep's sums
  __shared__ LpState st;
  const LpBatchGraph& g = graphs[blockIdx.x];
  const LpDev dv = g.dv;
  const LpPlan p = g.plan;
  const int K = p.K, E = p.E, n = p.n, t = threadIdx.x;
  if (pass == 0)
    for (int w = t; w < 12 * K; w += kLbThreads) dv.poses[w] = g.init[w];
  if (t == 0) st.cur = pass == 0 ? 0 : dv.state->cur;
  for (size_t w = t; w < (size_t)n * n; w += kLbThreads) dv.H[w] = 0.0;
  for (int i = t; i < n; i += kLbThreads) dv.b[i] = 0.0;
  __syncthreads();
  // the start (lp_begin_kernel, lp_assemble_kernel, lp_stats_kernel mode 0)
  lb_edges(dv, K, E, st.cur);
  const double F = lp_residual(dv, E, st.cur, p.mu, red);
  lp_confidences(dv, E, st.cur, p.mu);
  if (t == 0) {
    st.F = F;
    st.Fc = 0.0;
    st.nu = 2.0;
    st.done = st.reason = st.skip = 0;
    st.accepted = 1;
    st.iter = st.lm = st.trials = 0;
    st.info[0] = st.info[1] = 0;
  }
  __syncthreads();
  lb_assemble(dv, p, st.cur);
  lb_stats(dv, p, 0, st, red);
  while (!st.done) {
    // H + lambda I and b (lp_damp_kernel), the factorisation and the solve
    const double lam = st.lambda;
    for (int j = 0; j < n; ++j)
      for (int i = j + t; i < n; i += kLbThreads) {
        const size_t o = (size_t)i + (size_t)j * n;
        dv.A[o] = i == j ? dv.H[o] + lam : dv.H[o];
      }
    for (int i = t; i < n; i += kLbThreads) x[i] = dv.b[i];
    __syncthreads();
    const int bad = lb_cholesky(dv.A, n, Ps, ldp, Dt);
    __syncthreads();
    if (!bad) lb_solve(dv.A, n, x, tmp);
    // lp_step_kernel
    double s2 = 0.0, pd = 0.0;
    for (int i = t; i < n; i += kLbThreads) {
      const double d = x[i];
      s2 = s2 + d * d;
      pd = pd + d * (lam * d + dv.b[i]);
    }
    s2 = lp_block_sum(s2, red);
    pd = lp_block_sum(pd, red);
    if (t == 0) {
      st.info[0] = bad;
      lp_step_rule(st, p, s2, pd);
    }
    __syncthreads();
    // the candidate and its terms (lp_update_kernel, lp_edge_kernel), then lp_decide_kernel
    const int skip = st.skip, cur = st.cur;
    double Fc = 0.0;
    if (!skip) {
      for (int k = t; k < K; k += kLbThreads) lp_candidate(lp_pose(dv, K, cur, k), x + 6 * k, lp_pose(dv, K, 1 - cur, k));
      __syncthreads();
      lb_edges(dv, K, E, 1 - cur);
      Fc = lp_residual(dv, E, 1 - cur, p.mu, red);
    }
    if (t == 0) lp_decide_rule(st, p, skip, Fc);
    __syncthreads();
    if (st.accepted) {
      lp_confidences(dv, E, st.cur, p.mu);
      __syncthreads();
      if (!st.done) {
        lb_assemble(dv, p, st.cur);
        lb_stats(dv, p, 1, st, red);
      }
    }
  }
  for (int e = t; e < E; e += kLbThreads) g.out[e] = dv.conf[e];
  if (pass == 1) {
    // lp_compensate_kernel, then every edge of pass 1's table at the returned poses (lp_edge_kernel's last launch)
    int buf = st.cur;
    if (g.ref >= 0) {
      for (int k = t; k < K; k += kLbThreads)
        lp_compensate_pose(g.T0, lp_pose(dv, K, buf, g.ref), lp_pose(dv, K, buf, k), lp_pose(dv, K, 1 - buf, k));
      buf = 1 - buf;
      __syncthreads();
    }
    double* out_pose = g.out + g.E1;
    double* out_res = out_pose + 12 * K;
    for (int w = t; w < 12 * K; w += kLbThreads) out_pose[w] = dv.poses[(size_t)buf * 12 * K + w];
    for (int e = t; e < g.E1; e += kLbThreads) {
      const PgEdge& ed = g.edges1[e];
      double term[kPgTermStride];
      lp_edge_terms(ed, lp_pose(dv, K, buf, ed.s), lp_pose(dv, K, buf, ed.d), term);
      out_res[e] = term[42];
    }
  }
  if (t == 0) *dv.state = st;
}

// ---- many GNC-TLS graphs in one call (tzr_pose_graph_optimize_batch, DESIGN.md §3.24) ---------------------------------
// pg_batch_kernel: one CTA of kLbThreads per graph runs the whole GNC-TLS solve with its state in shared memory: per
// GNC iteration the edge terms and the cost (pg_edge_kernel, pg_cost_kernel mode 0), then per inner iteration H
// cleared, assembled and damped (pg_assemble_kernel), lb_cholesky and lb_solve in place of potrf / potrs, the candidate
// and its terms and the decision (pg_update_kernel, pg_edge_kernel, pg_cost_kernel mode 1), then the weight update
// (pg_gnc_kernel).  The rules are the single entry's helpers, and warp 0 runs the cost sums and the weight update as
// the single entry's one-warp kernels do, so with the same edge terms the costs, mu and the weights are the same bits.

// the terms of every edge at the poses in buffer buf
__device__ void pb_edges(const PgDev& dv, int K, int E, int buf) {
  for (int e = threadIdx.x; e < E; e += kLbThreads) pg_edge_terms(dv, K, E, buf, e);
  __syncthreads();
}

__global__ void __launch_bounds__(kLbThreads) pg_batch_kernel(const PgBatchGraph* graphs, int ldp) {
  extern __shared__ double smem[];
  double* Ps = smem;                   // kLbNb x ldp: the Cholesky panel
  double* Dt = Ps + kLbNb * ldp;       // kLbNb x kLbDt: its diagonal tile
  double* x = Dt + kLbNb * kLbDt;      // ldp: -g, then the step
  // x + ldp: kLbThreads doubles that only lp_batch_kernel uses (its reductions; the two share
  // line_process_batch_smem's layout)
  double* tmp = x + ldp + kLbThreads;  // kLbNb: the backward sweep's sums
  __shared__ PgState st;
  const PgBatchGraph& g = graphs[blockIdx.x];
  const PgDev dv = g.dv;
  const PgPlan p = g.plan;
  const int K = p.K, E = p.E, n = p.n, ref = g.ref, t = threadIdx.x;
  for (int w = t; w < 12 * K; w += kLbThreads) dv.poses[w] = g.init[w];
  if (t == 0) st = *dv.state;
  __syncthreads();
  // the terms of the buffer that holds no candidate yet are zeroed, so that the cost sum after a failed factorisation
  // (pg_cost_step sums the candidate buffer whatever its status) reads defined values
  double* cand_terms = dv.eterm + (size_t)(1 - st.cur) * E * kPgTermStride;
  for (int w = t; w < E * kPgTermStride; w += kLbThreads) cand_terms[w] = 0.0;
  int outer = 0, inner_total = 0;
  for (int it = 0; it < g.max_iterations; ++it) {
    pb_edges(dv, K, E, st.cur);
    if (t < 32) pg_cost_start(dv, st, E);
    __syncthreads();
    // the single entry enqueues max_inner iterations, and every one after the stop is a no-op
    for (int j = 0; j < p.max_inner && !st.done; ++j) {
      // H's lower triangle cleared (the factor of the previous iteration fills blocks the plan does not list), then
      // the listed blocks with the damping, one warp per block as pg_assemble_kernel, and -g into x
      for (int w = t; w < n * n; w += kLbThreads)
        if (w % n >= w / n) dv.H[w] = 0.0;
      __syncthreads();
      const int cur = st.cur;
      for (int b = t >> 5; b < p.blocks; b += kLbThreads / 32)
        pg_assemble_block(dv, st, E, n, cur, dv.blocks[b], t & 31, x);
      __syncthreads();
      const int bad = lb_cholesky(dv.H, n, Ps, ldp, Dt);
      __syncthreads();
      if (!bad) {
        lb_solve(dv.H, n, x, tmp);
        for (int k = t; k < K; k += kLbThreads) {
          const double* T = pose_at(dv, K, cur, k);
          double* Tn = pose_at(dv, K, 1 - cur, k);
          if (k == ref)
            for (int q = 0; q < 12; ++q) Tn[q] = T[q];
          else
            pg_candidate(T, x + 6 * (k < ref ? k : k - 1), Tn);
        }
        __syncthreads();
        pb_edges(dv, K, E, 1 - cur);
      }
      // a failed factorisation is a rejection, as a non-zero potrf status is; pg_cost_step then sums the candidate
      // buffer's terms from an earlier candidate (or the zeros written above) and discards the sum
      if (t == 0) {
        st.info[0] = bad;
        st.info[1] = 0;
      }
      if (t < 32) pg_cost_step(dv, st, E, g.cost_floor);
      __syncthreads();
    }
    outer = it + 1;
    inner_total += st.inner;
    if (t < 32) pg_gnc_rule(dv, st, E, it, p.gnc_factor, p.cost_threshold);
    __syncthreads();
    if (st.stop) break;
  }
  // the outputs: poses and r-bar at the current buffer, the weights, the summary
  const int cur = st.cur;
  double* out_pose = g.out;
  double* out_w = out_pose + 12 * K;
  double* out_res = out_w + E;
  for (int w = t; w < 12 * K; w += kLbThreads) out_pose[w] = dv.poses[(size_t)cur * 12 * K + w];
  for (int e = t; e < E; e += kLbThreads) {
    out_w[e] = dv.weight[e];
    out_res[e] = term_at(dv, E, cur, e)[43];
  }
  if (t == 0) {
    g.summary->iterations = outer;
    g.summary->inner_iterations = inner_total;
    g.summary->cost = st.cost;
    *dv.state = st;
  }
}

// ---- the batch kernels' factorisation on given matrices (tzr_dense_cholesky_batch, DESIGN.md §3.23) ------------------
// dc_batch_kernel: one CTA of kLbThreads per matrix, with the two batch kernels' shared-memory layout and panel stride
// ldp = n_max: lb_cholesky on the matrix in place, then, when it succeeds, lb_solve on x = b in the slot where those
// kernels keep their right-hand side.
__global__ void __launch_bounds__(kLbThreads) dc_batch_kernel(const DcMatrix* mats, int ldp) {
  extern __shared__ double smem[];
  double* Ps = smem;                   // kLbNb x ldp: the Cholesky panel
  double* Dt = Ps + kLbNb * ldp;       // kLbNb x kLbDt: its diagonal tile
  double* x = Dt + kLbNb * kLbDt;      // ldp: b, then the solution
  double* tmp = x + ldp + kLbThreads;  // kLbNb: the backward sweep's sums
  const DcMatrix m = mats[blockIdx.x];
  const int n = m.n, t = threadIdx.x;
  for (int i = t; i < n; i += kLbThreads) x[i] = m.x[i];
  __syncthreads();
  const int bad = lb_cholesky(m.A, n, Ps, ldp, Dt);
  __syncthreads();
  if (!bad) {
    lb_solve(m.A, n, x, tmp);
    for (int i = t; i < n; i += kLbThreads) m.x[i] = x[i];
  }
  if (t == 0) *m.info = bad;
}

}  // namespace

int launch_line_process_begin(const LpPlan& plan, const LpDev& dv, cudaStream_t st) {
  lp_edge_kernel<<<(std::max(plan.E, 1) + 127) / 128, 128, 0, st>>>(dv, plan.K, plan.E, 0);
  lp_begin_kernel<<<1, kLpSmall, 0, st>>>(dv, plan);
  lp_assemble_kernel<<<(std::max(plan.blocks, 1) + 3) / 4, 128, 0, st>>>(dv, plan.E, plan.n, plan.blocks);
  lp_stats_kernel<<<1, kLpLarge, 0, st>>>(dv, plan, 0);
  return 4;
}

int launch_line_process_damp(const LpPlan& plan, const LpDev& dv, cudaStream_t st) {
  lp_damp_kernel<<<dim3((plan.n + 255) / 256, plan.n), 256, 0, st>>>(dv, plan.n);
  return 1;
}

int launch_line_process_trial(const LpPlan& plan, const LpDev& dv, cudaStream_t st) {
  lp_step_kernel<<<1, kLpLarge, 0, st>>>(dv, plan);
  lp_update_kernel<<<(plan.K + 127) / 128, 128, 0, st>>>(dv, plan.K);
  lp_edge_kernel<<<(std::max(plan.E, 1) + 127) / 128, 128, 0, st>>>(dv, plan.K, plan.E, 1);
  lp_decide_kernel<<<1, kLpSmall, 0, st>>>(dv, plan);
  lp_assemble_kernel<<<(std::max(plan.blocks, 1) + 3) / 4, 128, 0, st>>>(dv, plan.E, plan.n, plan.blocks);
  lp_stats_kernel<<<1, kLpLarge, 0, st>>>(dv, plan, 1);
  return 6;
}

int launch_line_process_finish(const LpPlan& plan, const LpDev& dv, int ref, const double* T0, cudaStream_t st) {
  int n = 0;
  if (ref >= 0) {
    Pose12 t0;
    for (int q = 0; q < 12; ++q) t0.v[q] = T0[q];
    lp_compensate_kernel<<<(plan.K + 127) / 128, 128, 0, st>>>(dv, plan.K, ref, t0);
    ++n;
  }
  lp_edge_kernel<<<(std::max(plan.E, 1) + 127) / 128, 128, 0, st>>>(dv, plan.K, plan.E, ref >= 0 ? 2 : 0);
  return n + 1;
}

size_t line_process_batch_smem(int n_max) {
  return sizeof(double) * ((size_t)(kLbNb + 1) * n_max + kLbNb * kLbDt + kLbThreads + kLbNb);
}

int launch_line_process_batch(const LpBatchGraph* graphs, int G, int n_max, int pass, cudaStream_t st) {
  const size_t smem = line_process_batch_smem(n_max);
  cudaFuncSetAttribute(lp_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  lp_batch_kernel<<<G, kLbThreads, smem, st>>>(graphs, pass, n_max);
  return 1;
}

int launch_pose_graph_batch(const PgBatchGraph* graphs, int G, int n_max, cudaStream_t st) {
  const size_t smem = line_process_batch_smem(n_max);
  cudaFuncSetAttribute(pg_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  pg_batch_kernel<<<G, kLbThreads, smem, st>>>(graphs, n_max);
  return 1;
}

int launch_dense_cholesky_batch(const DcMatrix* mats, int G, int n_max, cudaStream_t st) {
  const size_t smem = line_process_batch_smem(n_max);
  cudaFuncSetAttribute(dc_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dc_batch_kernel<<<G, kLbThreads, smem, st>>>(mats, n_max);
  return 1;
}

}  // namespace tzr
