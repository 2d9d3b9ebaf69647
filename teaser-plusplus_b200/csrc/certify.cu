// Certification downstream of solve(): teaser::DRSCertifier::certify (reference teaser/src/certification.cc:40-190)
// on the device, FP64 throughout, for B problems in one launch sequence; tzr_certify and the single building blocks
// are the case B = 1.  Problem b has n = 4N + 4; its matrices are dense, column-major, padded to the group's nmax.
//
//   cbt_blocks_kernel    per measurement k: the 4x4 blocks of Q_cost (getQCost, :233-291) already rotated by the
//                        block-diagonal Omega (:293-314: Q_bar = D^T Q D acts block-wise), the 4x4 block of the initial
//                        multiplier guess (getLambdaGuess, :448-529) and the terms of mu = x^T Q x (:92).
//   cbt_reduce_kernel    sums those per-k terms (top-left lambda block, mu).
//   cbt_fill_kernel      assembles M_init = Q_bar - mu J_bar - lambda_bar_init (:100).
//   cbt_sym_kernel       B = (M + M^T) / 2 (getNearestPSD linalg.h:90; computeSubOptimalityGap :193).
//   [eigendecomposition of B: cusolverDnDsyevd per problem, or cusolverDnXsyevBatched over 8 or more, loaded lazily
//    with dlopen — the one library call of this stage, in the role cuBLAS has for plain GEMMs; see DESIGN.md 3.10]
//   cbt_psd_kernel       M_PSD = V diag(max(w, 0)) V^T over the positive eigenpairs only (linalg.h:93-98), from the first
//                        positive eigenvalue that cbt_first_pos_kernel finds; FP64 tensor cores.
//   cbt_affine_kernel    W = 2 M_PSD - M - M_init (:139); M_affine = M_init + W_dual (:153);
//                        M += gamma_tau (M_affine - M_PSD) (:181).
//   cbt_dual_bw_kernel .. cbt_dual_mean_kernel   getOptimalDualProjection (:316-446) with the sparse inverse map A_inv
//                        (getLinearProjection, :531-655: (N(N+1)/2)^2 entries in the reference) applied in closed form:
//                        out[a,b] = (x+2y) B[a,b] + y (th_a (Rs[b]-Cs[b]) - th_b (Rs[a]-Cs[a])) with two O(N^2) sums.
//   cbt_gap_kernel       the sub-optimality gap (:192-231), the trajectory and the stop rule.
#include <cusolverDn.h>
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "tzr_internal.cuh"

namespace tzr {

namespace {

// ---- lazily bound cuSOLVER entry points (keeps libteaser_b200.so loadable without libcusolver) ----------------
struct Cusolver {
  void* lib = nullptr;
  cusolverStatus_t (*create)(cusolverDnHandle_t*) = nullptr;
  cusolverStatus_t (*destroy)(cusolverDnHandle_t) = nullptr;
  cusolverStatus_t (*set_stream)(cusolverDnHandle_t, cudaStream_t) = nullptr;
  cusolverStatus_t (*syevd_buf)(cusolverDnHandle_t, cusolverEigMode_t, cublasFillMode_t, int, const double*, int,
                                const double*, int*) = nullptr;
  cusolverStatus_t (*syevd)(cusolverDnHandle_t, cusolverEigMode_t, cublasFillMode_t, int, double*, int, double*,
                            double*, int, int*) = nullptr;
  // batched route of tzr_certify_batch (optional: without them the batch loops syevd)
  cusolverStatus_t (*create_params)(cusolverDnParams_t*) = nullptr;
  cusolverStatus_t (*destroy_params)(cusolverDnParams_t) = nullptr;
  cusolverStatus_t (*syev_batched_buf)(cusolverDnHandle_t, cusolverDnParams_t, cusolverEigMode_t, cublasFillMode_t,
                                       int64_t, cudaDataType, const void*, int64_t, cudaDataType, const void*,
                                       cudaDataType, size_t*, size_t*, int64_t) = nullptr;
  cusolverStatus_t (*syev_batched)(cusolverDnHandle_t, cusolverDnParams_t, cusolverEigMode_t, cublasFillMode_t,
                                   int64_t, cudaDataType, void*, int64_t, cudaDataType, void*, cudaDataType, void*,
                                   size_t, void*, size_t, int*, int64_t) = nullptr;
  // dense Cholesky of the pose graph's normal equations (pose_graph.cu, DESIGN.md §3.16)
  cusolverStatus_t (*potrf_buf)(cusolverDnHandle_t, cublasFillMode_t, int, double*, int, int*) = nullptr;
  cusolverStatus_t (*potrf)(cusolverDnHandle_t, cublasFillMode_t, int, double*, int, double*, int, int*) = nullptr;
  cusolverStatus_t (*potrs)(cusolverDnHandle_t, cublasFillMode_t, int, int, const double*, int, double*, int,
                            int*) = nullptr;
  bool cholesky = false;
  bool batched = false;
  bool ok = false;
  std::string err;
};

Cusolver& cusolver() {
  static Cusolver c = [] {
    Cusolver s;
    const char* names[] = {"libcusolver.so.11", "libcusolver.so", "/usr/local/cuda/lib64/libcusolver.so.11"};
    for (const char* nme : names) {
      s.lib = dlopen(nme, RTLD_NOW | RTLD_LOCAL);
      if (s.lib) break;
    }
    if (!s.lib) {
      s.err = std::string("cannot load libcusolver: ") + dlerror();
      return s;
    }
    s.create = (decltype(s.create))dlsym(s.lib, "cusolverDnCreate");
    s.destroy = (decltype(s.destroy))dlsym(s.lib, "cusolverDnDestroy");
    s.set_stream = (decltype(s.set_stream))dlsym(s.lib, "cusolverDnSetStream");
    s.syevd_buf = (decltype(s.syevd_buf))dlsym(s.lib, "cusolverDnDsyevd_bufferSize");
    s.syevd = (decltype(s.syevd))dlsym(s.lib, "cusolverDnDsyevd");
    s.create_params = (decltype(s.create_params))dlsym(s.lib, "cusolverDnCreateParams");
    s.destroy_params = (decltype(s.destroy_params))dlsym(s.lib, "cusolverDnDestroyParams");
    s.syev_batched_buf = (decltype(s.syev_batched_buf))dlsym(s.lib, "cusolverDnXsyevBatched_bufferSize");
    s.syev_batched = (decltype(s.syev_batched))dlsym(s.lib, "cusolverDnXsyevBatched");
    s.batched = s.create_params && s.destroy_params && s.syev_batched_buf && s.syev_batched;
    s.potrf_buf = (decltype(s.potrf_buf))dlsym(s.lib, "cusolverDnDpotrf_bufferSize");
    s.potrf = (decltype(s.potrf))dlsym(s.lib, "cusolverDnDpotrf");
    s.potrs = (decltype(s.potrs))dlsym(s.lib, "cusolverDnDpotrs");
    s.cholesky = s.potrf_buf && s.potrf && s.potrs;
    s.ok = s.create && s.destroy && s.set_stream && s.syevd_buf && s.syevd;
    if (!s.ok) s.err = "libcusolver lacks the Dsyevd entry points";
    return s;
  }();
  return c;
}

// ---- small dense helpers ---------------------------------------------------------------------------------------
__device__ __forceinline__ void mat4_mul(const double* A, const double* B, double* C) {  // column-major 4x4
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += A[r + 4 * k] * B[k + 4 * c];
      C[r + 4 * c] = s;
    }
}

// Omega^T X Omega for a column-major 4x4 X
__device__ void rotate_block(const double* om, const double* X, double* out) {
  double omT[16], t[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) omT[r + 4 * c] = om[c + 4 * r];
  mat4_mul(omT, X, t);
  mat4_mul(t, om, out);
}

__constant__ signed char kP[9][16] = {  // certification.cc:242-252
    {1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1},  {0, 1, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 1, 0},
    {0, 0, 1, 0, 0, 0, 0, -1, 1, 0, 0, 0, 0, -1, 0, 0},  {0, 1, 0, 0, 1, 0, 0, 0, 0, 0, 0, -1, 0, 0, -1, 0},
    {-1, 0, 0, 0, 0, 1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1},  {0, 0, 0, 1, 0, 0, 1, 0, 0, 1, 0, 0, 1, 0, 0, 0},
    {0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1, 0, 0},    {0, 0, 0, -1, 0, 0, 1, 0, 0, 1, 0, 0, -1, 0, 0, 0},
    {-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};

__device__ __forceinline__ void hat(const double* u, double* H) {  // column-major 3x3 (linalg.h:20-29)
  H[0] = 0;      H[3] = -u[2];  H[6] = u[1];
  H[1] = u[2];   H[4] = 0;      H[7] = -u[0];
  H[2] = -u[1];  H[5] = u[0];   H[8] = 0;
}

// per-k outputs, 16 doubles each (column-major 4x4): offA (rotated first-row/column block), diagB (rotated diagonal
// block), lam (the un-negated "current_block" of getLambdaGuess); terms[k] = theta-weighted contribution to mu
__device__ __forceinline__ void cert_block(int k, const double* __restrict__ src, const double* __restrict__ dst,
                                           const double* __restrict__ theta, const double* __restrict__ Rcm,
                                           const double* __restrict__ q_xyzw, double nbs, double* offA, double* diagB,
                                           double* lam, double* mu_terms) {
  const double v1[3] = {src[3 * k], src[3 * k + 1], src[3 * k + 2]};
  const double v2[3] = {dst[3 * k], dst[3 * k + 1], dst[3 * k + 2]};
  // P_k = reshape(P' vec(v2 v1'), [4,4]) (column-major vec and reshape, :268-271)
  double A9[9];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) A9[r + 3 * c] = v2[r] * v1[c];
  double Pk[16];
  for (int e = 0; e < 16; ++e) {
    double s = 0;
    for (int m = 0; m < 9; ++m) s += (double)kP[m][e] * A9[m];
    Pk[e] = s;
  }
  const double nn = (v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2]) + (v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2]);
  const double ck = 0.5 * (nn - nbs), ck2 = 0.5 * (nn + nbs);
  double Ak[16], Bk[16];
  for (int e = 0; e < 16; ++e) {
    const double id = (e % 5 == 0) ? 1.0 : 0.0;
    Ak[e] = -0.5 * Pk[e] + ck / 2 * id;
    Bk[e] = -Pk[e] + ck2 * id;
  }
  const double x = q_xyzw[0], y = q_xyzw[1], z = q_xyzw[2], w = q_xyzw[3];
  const double om[16] = {w, z, -y, -x, -z, w, x, -y, y, -x, w, -z, x, y, z, w};  // getOmega1 (:293-303), column-major
  rotate_block(om, Ak, offA + 16 * (size_t)k);
  rotate_block(om, Bk, diagB + 16 * (size_t)k);
  // mu = x^T Q x, x = kron([1, theta], q): blocks (0,k), (k,0) hold A_k, (k,k) holds B_k
  const double qv[4] = {x, y, z, w};
  double qAq = 0, qBq = 0;
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r) {
      qAq += qv[r] * Ak[r + 4 * c] * qv[c];
      qBq += qv[r] * Bk[r + 4 * c] * qv[c];
    }
  const double th = theta[k];
  mu_terms[k] = 2.0 * th * qAq + th * th * qBq;
  // getLambdaGuess (:448-529)
  double R[9];
  for (int e = 0; e < 9; ++e) R[e] = Rcm[e];  // column-major
  double Rs[3], d[3], xi[3];
  for (int r = 0; r < 3; ++r) Rs[r] = R[r] * v1[0] + R[r + 3] * v1[1] + R[r + 6] * v1[2];
  for (int r = 0; r < 3; ++r) d[r] = v2[r] - Rs[r];
  for (int r = 0; r < 3; ++r) xi[r] = R[3 * r] * d[0] + R[3 * r + 1] * d[1] + R[3 * r + 2] * d[2];  // R^T d
  double sh[9], xh[9], shsh[9], xhsh[9];
  hat(v1, sh);
  hat(xi, xh);
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) {
      double a = 0, b = 0;
      for (int m = 0; m < 3; ++m) {
        a += sh[r + 3 * m] * sh[m + 3 * c];
        b += xh[r + 3 * m] * sh[m + 3 * c];
      }
      shsh[r + 3 * c] = a;
      xhsh[r + 3 * c] = b;
    }
  const double sxi = v1[0] * xi[0] + v1[1] * xi[1] + v1[2] * xi[2];
  const double xx = xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2];
  const bool inl = th > 0;
  const double c44 = inl ? (-0.75 * xx - 0.25 * nbs) : (-0.25 * xx - 0.75 * nbs);
  const double cxx = inl ? 0.75 : 0.25, cvec = inl ? -1.5 : -0.5;
  double blk[16];
  for (int e = 0; e < 16; ++e) blk[e] = 0;
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) {
      const double id = r == c ? 1.0 : 0.0;
      blk[r + 4 * c] = shsh[r + 3 * c] - 0.5 * sxi * id + 0.5 * xhsh[r + 3 * c] + 0.5 * xi[r] * v1[c] - cxx * xx * id -
                       0.25 * nbs * id;
    }
  for (int r = 0; r < 3; ++r) {
    const double v = cvec * (xh[r] * v1[0] + xh[r + 3] * v1[1] + xh[r + 6] * v1[2]);
    blk[r + 12] = v;  // column 3
    blk[3 + 4 * r] = v;  // row 3
  }
  blk[15] = c44;
  for (int e = 0; e < 16; ++e) lam[16 * (size_t)k + e] = blk[e];
}

// one CTA: top[16] = sum_k lam_k, *mu = sum_k mu_terms[k] (k ascending per thread, then a fixed tree: deterministic)
__device__ __forceinline__ void cert_reduce_cta(const double* lam, const double* mu_terms, int N, double* top,
                                                double* mu) {
  __shared__ double sh[256];
  for (int e = 0; e <= 16; ++e) {
    double s = 0;
    for (int k = threadIdx.x; k < N; k += 256) s += (e < 16) ? lam[16 * (size_t)k + e] : mu_terms[k];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
      if (threadIdx.x < off) sh[threadIdx.x] += sh[threadIdx.x + off];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      if (e < 16) top[e] = sh[0];
      else *mu = sh[0];
    }
    __syncthreads();
  }
}

// M_init = Q_bar - mu J_bar - lambda_bar_init, one thread per entry
__device__ __forceinline__ double cert_fill_value(int r, int c, const double* offA, const double* diagB,
                                                  const double* lam, const double* top, const double* mu) {
  const int bi = r >> 2, bj = c >> 2, lr = r & 3, lc = c & 3;
  double v = 0;
  if (bi == 0 && bj == 0) {
    v = -((lr == lc) ? *mu : 0.0) - top[lr + 4 * lc];  // Q_bar(0,0) = 0; -mu J; lambda(0,0) = +sum of blocks
  } else if (bi == 0) {
    v = offA[16 * (size_t)(bj - 1) + lr + 4 * lc];
  } else if (bj == 0) {
    v = offA[16 * (size_t)(bi - 1) + lr + 4 * lc];
  } else if (bi == bj) {
    v = diagB[16 * (size_t)(bi - 1) + lr + 4 * lc] + lam[16 * (size_t)(bi - 1) + lr + 4 * lc];  // lambda = -blk
  }
  return v;
}

// ---- getOptimalDualProjection -----------------------------------------------------------------------------------
// pair (i, j), 0 <= i < j <= N, running index as in the reference's double loop (:342-343)
__device__ __forceinline__ long long pair_id(int i, int j, int N1) {  // N1 = N + 1 blocks
  return (long long)i * N1 - (long long)i * (i + 1) / 2 + (j - i - 1);
}

#define WAT(r, c) W[(size_t)(c) * n + (r)]

// The bodies below take the leading dimension n of W / Wd as an argument: the padded size of a certify batch.
// bW[p][0..2] = -th_ij C + D - E + th_ij F (:349-368)
__device__ __forceinline__ void dual_bw_at(const double* __restrict__ W, int n, const double* __restrict__ thp, int N,
                                           int i, int j, double* __restrict__ bW) {
  const int N1 = N + 1;
  if (i >= N || j <= i || j >= N1) return;
  const double tij = thp[i] * thp[j];
  const long long p = pair_id(i, j, N1);
  for (int c = 0; c < 3; ++c) {
    const double Cc = WAT(4 * i + 3, 4 * i + c), Dc = WAT(4 * j + 3, 4 * i + c);
    const double Ec = WAT(4 * i + 3, 4 * j + c), Fc = WAT(4 * j + 3, 4 * j + c);
    bW[3 * p + c] = ((-tij * Cc + Dc) + (-1.0) * Ec) + tij * Fc;
  }
}

// D[v][c] = Rs[v][c] - Cs[v][c]: Rs[v] = sum_{j>v} th_j B[v,j], Cs[v] = sum_{i<v} th_i B[i,v]   (one thread per (v,c))
__device__ __forceinline__ void dual_sums_at(const double* __restrict__ bW, const double* __restrict__ thp, int N,
                                             int t, double* __restrict__ D) {
  const int N1 = N + 1;
  if (t >= 3 * N1) return;
  const int v = t / 3, c = t % 3;
  double rs = 0, cs = 0;
  for (int j = v + 1; j < N1; ++j) rs += thp[j] * bW[3 * pair_id(v, j, N1) + c];
  for (int i = 0; i < v; ++i) cs += thp[i] * bW[3 * pair_id(i, v, N1) + c];
  D[t] = rs - cs;
}

// off-diagonal blocks of W_dual (both triangles) (:381-415), A_inv applied in closed form
__device__ __forceinline__ void dual_off_at(const double* __restrict__ W, int n, const double* __restrict__ thp,
                                            const double* __restrict__ bW, const double* __restrict__ D, int N, int i,
                                            int j, double* __restrict__ Wd) {
  const int N1 = N + 1;
  if (i >= N || j <= i || j >= N1) return;
  const double y = 1.0 / (2.0 * N + 6.0), x = (N + 1.0) * y;
  const long long p = pair_id(i, j, N1);
  double yd[3];
  for (int c = 0; c < 3; ++c)
    yd[c] = (x + 2 * y) * bW[3 * p + c] + y * (thp[i] * D[3 * j + c] - thp[j] * D[3 * i + c]);
  double blk[16];
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r) blk[r + 4 * c] = (WAT(4 * i + r, 4 * j + c) - WAT(4 * i + c, 4 * j + r)) / 2;
  for (int r = 0; r < 3; ++r) {
    blk[r + 12] = yd[r];
    blk[3 + 4 * r] = -yd[r];
  }
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r) {
      Wd[(size_t)(4 * j + c) * n + 4 * i + r] = blk[r + 4 * c];
      Wd[(size_t)(4 * i + r) * n + 4 * j + c] = blk[r + 4 * c];  // transpose (:416-417)
    }
}

// diagonal blocks (:419-434): one warp per block row; then diag3[i][9] holds the 3x3 corner for the mean
__device__ __forceinline__ void dual_diag_at(const double* __restrict__ W, int n, const double* __restrict__ thp,
                                             int N, int i, int lane, double* __restrict__ Wd,
                                             double* __restrict__ diag3) {
  const int N1 = N + 1;
  if (i >= N1) return;
  double rs[4] = {0, 0, 0, 0};
  for (int j = lane; j < N1; j += 32) {
    if (j == i) continue;  // the diagonal block is still zero when the reference sums the block row
    const double tj = thp[j];
    for (int r = 0; r < 4; ++r) rs[r] += tj * Wd[(size_t)(4 * j + 3) * n + 4 * i + r];
  }
  for (int r = 0; r < 4; ++r)
    for (int off = 16; off > 0; off >>= 1) rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], off);
  if (lane == 0) {
    const double ti = thp[i];
    double blk[16];
    for (int c = 0; c < 4; ++c)
      for (int r = 0; r < 4; ++r) blk[r + 4 * c] = WAT(4 * i + r, 4 * i + c);
    for (int r = 0; r < 4; ++r) blk[r + 12] = -ti * rs[r];
    for (int c = 0; c < 4; ++c) blk[3 + 4 * c] = -ti * rs[c];
    for (int c = 0; c < 4; ++c)
      for (int r = 0; r < 4; ++r) Wd[(size_t)(4 * i + c) * n + 4 * i + r] = blk[r + 4 * c];
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r) diag3[9 * (size_t)i + r + 3 * c] = blk[r + 4 * c];
  }
}

// one CTA: mean of the 3x3 corners, subtracted from every diagonal block (:435-445)
__device__ __forceinline__ void dual_mean_cta(const double* __restrict__ diag3, int n, int N,
                                              double* __restrict__ Wd) {
  __shared__ double sh[256];
  __shared__ double mean[9];
  const int N1 = N + 1;
  for (int e = 0; e < 9; ++e) {
    double s = 0;
    for (int i = threadIdx.x; i < N1; i += 256) s += diag3[9 * (size_t)i + e];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
      if (threadIdx.x < off) sh[threadIdx.x] += sh[threadIdx.x + off];
      __syncthreads();
    }
    if (threadIdx.x == 0) mean[e] = sh[0] / (double)N1;
    __syncthreads();
  }
  for (int t = threadIdx.x; t < 9 * N1; t += 256) {
    const int i = t / 9, e = t % 9, r = e % 3, c = e / 3;
    Wd[(size_t)(4 * i + c) * n + 4 * i + r] -= mean[e];
  }
}

inline int grid1(long long items, int threads) { return (int)((items + threads - 1) / threads); }

// ---- certify batch (tzr_certify_batch): B problems in one launch sequence ----------------------------------------
// Every problem's matrices are nmax x nmax (nmax = 4 max N + 4 of the group), column-major, leading dimension nmax, at
// b * nmax^2; the real block is the top-left n x n.  Per-measurement arrays lie back to back (first measurement k_off),
// block-row arrays likewise (first block row v_off = k_off + b).  Every kernel skips problems whose active flag is 0.
struct CertBatchProb {
  int N, n;            // measurements, 4N + 4
  int k_off, v_off;    // first measurement; first block row (thp, D, diag3)
  long long p_off;     // first block pair of bW
  int active;          // 1 while the iteration runs
  int iters;           // iterations done (length of the trajectory)
  int first_pos;       // first eigen column with a positive eigenvalue
  unsigned long long pad_bits;  // largest |entry| of the starting matrix (M_init), as its bit pattern
  double mu, best;
  double nbs;          // cbar2 * noise_bound^2 of this problem
};

// Eigenvalue of the pad block (the identity times it) of a padded problem: block diagonal, so the padded matrix has the
// real block's eigenpairs plus (c, e_k) with e_k zero on the real rows; see DESIGN.md 3.9.  c is the largest power of
// two not above the largest |entry| of the problem's starting matrix (1 if that is 0): it follows the problem's scale,
// so the padded matrix has the real block's norm at any scale, and scaling a problem by 2^k scales c exactly.
__device__ __forceinline__ double cert_pad(unsigned long long bits) {
  const double m = __longlong_as_double(bits);
  return m > 0 ? ldexp(1.0, ilogb(m)) : 1.0;
}

__global__ void cbt_blocks_kernel(const CertBatchProb* __restrict__ pr, const double* __restrict__ src,
                                  const double* __restrict__ dst, const double* __restrict__ theta,
                                  const double* __restrict__ R, const double* __restrict__ q, double* offA,
                                  double* diagB, double* lam, double* mu_terms) {
  const CertBatchProb p = pr[blockIdx.y];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p.N) return;
  const size_t o = p.k_off;
  cert_block(k, src + 3 * o, dst + 3 * o, theta + o, R + 9 * blockIdx.y, q + 4 * blockIdx.y, p.nbs, offA + 16 * o,
             diagB + 16 * o, lam + 16 * o, mu_terms + o);
}

// The measurements of a retained solve's problem (one CTA of kRTThreads per problem of the group), written where the
// host path would have copied them: src/dst/theta at k_off, thp (1, theta) at v_off.  The TIMs are the rotation stage's,
// bit for bit (rot_trans.cu): CHAIN TIM i runs from clique point i to point i+1 (the last one back to point 0), its dst
// side times 1/scale; COMPLETE walks the clique points with for_each_tim.  A problem with a non-finite measurement is
// marked inactive, so no later kernel or eigensolver call touches it; active[g] receives the flag.
__global__ void __launch_bounds__(kRTThreads) cbt_solve_gather_kernel(const CertGatherProb* __restrict__ gt,
                                                                      CertBatchProb* pr, double* src, double* dst,
                                                                      double* theta, double* thp, int* active) {
  __shared__ double s_a[3 * 128], s_b[3 * 128];  // COMPLETE clique points (4N + 4 <= 32768 keeps m <= 128)
  const CertGatherProb g = gt[blockIdx.x];
  const int m = g.m, tid = threadIdx.x;
  const double inv_scale = 1.0 / g.scale;
  double* s = src + 3 * (size_t)g.k_off;
  double* d = dst + 3 * (size_t)g.k_off;
  double* th = theta + g.k_off;
  double* tp = thp + g.v_off + 1;
  bool bad = false;
  auto put = [&](long long k, double x0, double x1, double x2, double y0, double y1, double y2) {
    s[3 * k] = x0; s[3 * k + 1] = x1; s[3 * k + 2] = x2;
    d[3 * k] = y0; d[3 * k + 1] = y1; d[3 * k + 2] = y2;
    const double t = g.rmask[k] ? 1.0 : -1.0;
    th[k] = t;
    tp[k] = t;
    bad |= !(isfinite(x0) && isfinite(x1) && isfinite(x2) && isfinite(y0) && isfinite(y1) && isfinite(y2));
  };
  if (!g.complete) {
    for (int i = tid; i < m; i += kRTThreads) {
      const int root = g.clq[i];
      const int leaf = (i != m - 1) ? g.clq[i + 1] : g.clq[0];
      const double* sr = g.src + 3 * (size_t)root;
      const double* sl = g.src + 3 * (size_t)leaf;
      const double* dr = g.dst + 3 * (size_t)root;
      const double* dl = g.dst + 3 * (size_t)leaf;
      put(i, sl[0] - sr[0], sl[1] - sr[1], sl[2] - sr[2], (dl[0] - dr[0]) * inv_scale, (dl[1] - dr[1]) * inv_scale,
          (dl[2] - dr[2]) * inv_scale);
    }
  } else {
    for (int i = tid; i < m; i += kRTThreads)
      for (int r = 0; r < 3; ++r) {
        s_a[3 * i + r] = g.src[3 * (size_t)g.clq[i] + r];
        s_b[3 * i + r] = g.dst[3 * (size_t)g.clq[i] + r];
      }
    __syncthreads();
    TimSrc ts;
    ts.complete = 1;
    ts.m = m;
    ts.count = (long long)m * (m - 1) / 2;
    ts.a = s_a;
    ts.b = s_b;
    ts.inv_scale = inv_scale;
    for_each_tim(ts, put);
  }
  bad = __syncthreads_or(bad) != 0;
  if (tid == 0) {
    thp[g.v_off] = 1.0;
    pr[blockIdx.x].active = bad ? 0 : 1;
    active[blockIdx.x] = bad ? 0 : 1;
  }
}

__global__ void __launch_bounds__(256) cbt_reduce_kernel(CertBatchProb* pr, const double* lam,
                                                        const double* mu_terms, double* top) {
  const int b = blockIdx.x;
  const size_t o = pr[b].k_off;
  __shared__ double mu;
  cert_reduce_cta(lam + 16 * o, mu_terms + o, pr[b].N, top + 16 * b, &mu);
  if (threadIdx.x == 0) pr[b].mu = mu;
}

// M_init of every problem, the pad region zero; the largest |entry| into pad_bits (non-negative doubles order like
// their bit patterns; one atomic per warp)
__global__ void cbt_fill_kernel(CertBatchProb* __restrict__ pr, int nmax, const double* offA, const double* diagB,
                                const double* lam, const double* top, double* M_init) {
  const int b = blockIdx.y;
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  CertBatchProb& p = pr[b];
  double v = 0;
  if (e < (long long)nmax * nmax) {
    const int r = (int)(e % nmax), c = (int)(e / nmax);
    const size_t o = p.k_off;
    if (r < p.n && c < p.n)
      v = cert_fill_value(r, c, offA + 16 * o, diagB + 16 * o, lam + 16 * o, top + 16 * b, &p.mu);
    M_init[(size_t)b * nmax * nmax + e] = v;
  }
  unsigned long long m = (unsigned long long)__double_as_longlong(fabs(v));
  for (int off = 16; off > 0; off >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(&p.pad_bits, m);
}

// B = (M + M^T) / 2 on the real block, cert_pad * I on the pad block
__global__ void cbt_sym_kernel(const CertBatchProb* __restrict__ pr, int nmax, const double* __restrict__ M,
                               double* __restrict__ Bm) {
  const int b = blockIdx.y;
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)nmax * nmax || !pr[b].active) return;
  const int n = pr[b].n;
  const int r = (int)(e % nmax), c = (int)(e / nmax);
  const size_t base = (size_t)b * nmax * nmax;
  Bm[base + e] =
      (r < n && c < n) ? (M[base + e] + M[base + (size_t)r * nmax + c]) / 2 : (r == c ? cert_pad(pr[b].pad_bits) : 0.0);
}

// first eigen column with w > 0 (w ascending); ne_full: the eigensolver ran on the padded nmax (else on n)
__global__ void cbt_first_pos_kernel(CertBatchProb* pr, int B, int nmax, int ne_full, const double* __restrict__ w) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !pr[b].active) return;
  const double* wb = w + (size_t)b * nmax;
  int lo = 0, hi = ne_full ? nmax : pr[b].n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (wb[mid] > 0) hi = mid;
    else lo = mid + 1;
  }
  pr[b].first_pos = lo;
}

// C = V[:, k0:ne] diag(w[k0:ne]) V[:, k0:ne]^T on the real block, FP64 tensor cores (DMMA, mma.sync m8n8k4).  64 x 64
// output tile per CTA, 8 warps of 32 x 16 (4 x 2 MMA tiles); k in slabs of 16 staged in shared memory, the eigenvalue
// scaling applied to the A operand on the way in.  Row pitch 68 doubles: the fragment loads (row = k, 8 consecutive
// columns per k) are conflict-free in each half-warp.
constexpr int kPT = 64, kPK = 16, kPS = kPT + 4;
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(256) cbt_psd_kernel(const CertBatchProb* __restrict__ pr, int nmax, int ne_full,
                                                     const double* __restrict__ V, const double* __restrict__ w,
                                                     double* __restrict__ C) {
  __shared__ double As[kPK][kPS], Bs[kPK][kPS];
  const int b = blockIdx.z;
  const int n = pr[b].n, r0 = blockIdx.x * kPT, c0 = blockIdx.y * kPT;
  if (!pr[b].active || r0 >= n || c0 >= n) return;
  const int ne = ne_full ? nmax : n, k0 = pr[b].first_pos;
  const size_t base = (size_t)b * nmax * nmax;
  V += base;
  C += base;
  w += (size_t)b * nmax;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gid = lane >> 2, tig = lane & 3;
  const int wr = (warp & 1) * 32, wc = (warp >> 1) * 16;
  double acc[4][2][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j][0] = acc[i][j][1] = 0;
  for (int kb = k0; kb < ne; kb += kPK) {
    for (int e = threadIdx.x; e < kPK * kPT; e += 256) {
      const int kk = e / kPT, i = e % kPT;
      const int k = kb + kk;
      const double wk = k < ne ? w[k] : 0.0;
      As[kk][i] = (k < ne && r0 + i < n && wk > 0) ? V[(size_t)k * nmax + r0 + i] * wk : 0.0;
      Bs[kk][i] = (k < ne && c0 + i < n) ? V[(size_t)k * nmax + c0 + i] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kPK; kk += 4) {
      double a[4], bb[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk + tig][wr + 8 * i + gid];
#pragma unroll
      for (int j = 0; j < 2; ++j) bb[j] = Bs[kk + tig][wc + 8 * j + gid];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i], bb[j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + wr + 8 * i + gid, c = c0 + wc + 8 * j + 2 * tig + h;
        if (r < n && c < n) C[(size_t)c * nmax + r] = acc[i][j][h];
      }
}

// op 0: W = 2 Mpsd - M - Minit (affine-in), 1: Maff = Minit + Wd (affine-out), 2: M += gamma_tau (Maff - Mpsd)
// (update); real block of every active problem
__global__ void cbt_affine_kernel(const CertBatchProb* __restrict__ pr, int nmax, int op, const double* __restrict__ X,
                                  const double* __restrict__ Y, double* __restrict__ Z, const double* __restrict__ Minit,
                                  double gamma_tau) {
  const int b = blockIdx.y;
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)nmax * nmax || !pr[b].active) return;
  const int n = pr[b].n;
  if ((int)(e % nmax) >= n || (int)(e / nmax) >= n) return;
  const size_t i = (size_t)b * nmax * nmax + e;
  if (op == 0) Z[i] = 2 * X[i] - Y[i] - Minit[i];
  else if (op == 1) Z[i] = Minit[i] + X[i];
  else Z[i] += gamma_tau * (X[i] - Y[i]);
}

__global__ void cbt_dual_bw_kernel(const CertBatchProb* __restrict__ pr, int nmax, const double* __restrict__ W,
                                   const double* __restrict__ thp, double* __restrict__ bW) {
  const CertBatchProb& p = pr[blockIdx.z];
  if (!p.active) return;
  dual_bw_at(W + (size_t)blockIdx.z * nmax * nmax, nmax, thp + p.v_off, p.N, blockIdx.y,
             blockIdx.x * blockDim.x + threadIdx.x, bW + 3 * p.p_off);
}

__global__ void cbt_dual_sums_kernel(const CertBatchProb* __restrict__ pr, const double* __restrict__ bW,
                                     const double* __restrict__ thp, double* __restrict__ D) {
  const CertBatchProb& p = pr[blockIdx.y];
  if (!p.active) return;
  dual_sums_at(bW + 3 * p.p_off, thp + p.v_off, p.N, blockIdx.x * blockDim.x + threadIdx.x, D + 3 * (size_t)p.v_off);
}

__global__ void cbt_dual_off_kernel(const CertBatchProb* __restrict__ pr, int nmax, const double* __restrict__ W,
                                    const double* __restrict__ thp, const double* __restrict__ bW,
                                    const double* __restrict__ D, double* __restrict__ Wd) {
  const CertBatchProb& p = pr[blockIdx.z];
  if (!p.active) return;
  const size_t base = (size_t)blockIdx.z * nmax * nmax;
  dual_off_at(W + base, nmax, thp + p.v_off, bW + 3 * p.p_off, D + 3 * (size_t)p.v_off, p.N, blockIdx.y,
              blockIdx.x * blockDim.x + threadIdx.x, Wd + base);
}

__global__ void cbt_dual_diag_kernel(const CertBatchProb* __restrict__ pr, int nmax, const double* __restrict__ W,
                                     const double* __restrict__ thp, double* __restrict__ Wd,
                                     double* __restrict__ diag3) {
  const CertBatchProb& p = pr[blockIdx.y];
  if (!p.active) return;
  const size_t base = (size_t)blockIdx.y * nmax * nmax;
  dual_diag_at(W + base, nmax, thp + p.v_off, p.N, blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5),
               threadIdx.x & 31, Wd + base, diag3 + 9 * (size_t)p.v_off);
}

__global__ void __launch_bounds__(256) cbt_dual_mean_kernel(const CertBatchProb* __restrict__ pr, int nmax,
                                                           const double* __restrict__ diag3, double* __restrict__ Wd) {
  const CertBatchProb& p = pr[blockIdx.x];
  if (!p.active) return;
  dual_mean_cta(diag3 + 9 * (size_t)p.v_off, nmax, p.N, Wd + (size_t)blockIdx.x * nmax * nmax);
}

// Compact batch of the eigensolver once some problems have finished: slot s holds problem idx[s].  Gather copies the
// matrices into the compact buffer; scatter copies back the eigenvalues, info and (vectors = 1) the eigenvectors.
__global__ void cbt_gather_kernel(const int* __restrict__ idx, int nmax, const double* __restrict__ Bm,
                                  double* __restrict__ Bc) {
  const long long nn = (long long)nmax * nmax, e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < nn) Bc[blockIdx.y * nn + e] = Bm[idx[blockIdx.y] * nn + e];
}

__global__ void cbt_scatter_kernel(const int* __restrict__ idx, int nmax, int vectors, const double* __restrict__ Bc,
                                   const double* __restrict__ wc, const int* __restrict__ infoc, double* __restrict__ Bm,
                                   double* __restrict__ w, int* __restrict__ info) {
  const int s = blockIdx.y, b = idx[s];
  const long long nn = (long long)nmax * nmax, e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (vectors && e < nn) Bm[b * nn + e] = Bc[s * nn + e];
  if (e < nmax) w[(size_t)b * nmax + e] = wc[(size_t)s * nmax + e];
  if (e == 0) info[b] = infoc[s];
}

// The gap rule per active problem (info != 0 -> inf, min_eig > 0 -> 0, else -min_eig (N+1) / mu), the
// trajectory entry, the best gap, and the stop rule (gap < sub_optimality or the iteration cap); active_out: the flags
__global__ void cbt_gap_kernel(CertBatchProb* pr, int B, int nmax, const double* __restrict__ w,
                               const int* __restrict__ info, int iter, double sub_optimality, double max_iterations,
                               double* traj, int traj_cap, int* active_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  CertBatchProb& p = pr[b];
  if (p.active) {
    const double min_eig = w[(size_t)b * nmax];  // ascending: w[0] is the minimum
    double gap;
    if (info[b] != 0) gap = INFINITY;
    else if (min_eig > 0) gap = 0;
    else gap = (-min_eig * (p.N + 1)) / p.mu;
    if (iter < traj_cap) traj[(size_t)b * traj_cap + iter] = gap;
    p.iters = iter + 1;
    if (gap < p.best) p.best = gap;
    if (gap < sub_optimality || (double)(iter + 1) >= max_iterations) p.active = 0;
  }
  active_out[b] = p.active;
}


}  // namespace

// quaternion of R (Eigen::Quaterniond(R).normalize(), :66-69) on the host: 20 flops
static void quaternion_xyzw(const double* R_cm, double q[4]) {
  const double* R = R_cm;  // column-major: R(r,c) = R[r + 3c]
  auto Rm = [&](int r, int c) { return R[r + 3 * c]; };
  const double t = Rm(0, 0) + Rm(1, 1) + Rm(2, 2);
  double x, y, z, ww;
  if (t > 0) {
    double s = std::sqrt(t + 1.0);
    ww = 0.5 * s;
    s = 0.5 / s;
    x = (Rm(2, 1) - Rm(1, 2)) * s;
    y = (Rm(0, 2) - Rm(2, 0)) * s;
    z = (Rm(1, 0) - Rm(0, 1)) * s;
  } else {
    int i = 0;
    if (Rm(1, 1) > Rm(0, 0)) i = 1;
    if (Rm(2, 2) > Rm(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = std::sqrt(Rm(i, i) - Rm(j, j) - Rm(k, k) + 1.0);
    double v[3];
    v[i] = 0.5 * s;
    s = 0.5 / s;
    ww = (Rm(k, j) - Rm(j, k)) * s;
    v[j] = (Rm(j, i) + Rm(i, j)) * s;
    v[k] = (Rm(k, i) + Rm(i, k)) * s;
    x = v[0]; y = v[1]; z = v[2];
  }
  const double nrm = std::sqrt(x * x + y * y + z * z + ww * ww);
  q[0] = x / nrm; q[1] = y / nrm; q[2] = z / nrm; q[3] = ww / nrm;
}

// ---- tzr_certify_batch ---------------------------------------------------------------------------------------------
// Fewest active problems for which an eigen step takes cusolverDnXsyevBatched; below, one cusolverDnDsyevd per active
// problem.  The batched call has a large fixed cost: per DRS iteration (two eigen steps) 12-16 ms at n = 204 for 16
// and for 64 problems, against 3.4 ms per problem on Dsyevd; 45 ms for 16 at n = 404 (7.3 per problem), 140 ms for 16
// at n = 1004 (21 per problem).  That puts the crossover at about 5-7 problems; at 8 the batched call was faster at
// every measured size (DESIGN.md 3.9).
constexpr int kCertBatchedMinActive = 8;

namespace {
struct CertBatchWork {
  double *src, *dst, *theta, *thp, *R, *q, *offA, *diagB, *lam, *mu_terms, *top, *bW, *D, *diag3, *w;
  double *M_init, *M, *Bm, *M_psd, *W, *Wd, *M_aff, *traj, *wc;
  CertBatchProb* pr;
  int *info, *active, *infoc, *idx;
  void* work;
  CertGatherProb* gt;  // device inputs of the group (gather: certify_batch_device's device input mode), else null
};

// Device bytes of a group of G problems with K measurements, P block pairs, padded size nmax and T trajectory columns,
// plus `work` bytes of eigensolver workspace (and the group's gather table); carve() of the same arguments lays them out.
size_t cbt_carve(void* base, int G, long long K, long long P, int nmax, int T, size_t work, CertBatchWork* out,
                 bool gather = false) {
  char* p = (char*)base;
  auto take = [&](size_t bytes) {
    void* r = p;
    p += (bytes + 255) / 256 * 256;
    return r;
  };
  const size_t V = (size_t)K + G, nn = (size_t)nmax * nmax, d = sizeof(double);
  CertBatchWork w;
  w.src = (double*)take(3 * K * d); w.dst = (double*)take(3 * K * d); w.theta = (double*)take(K * d);
  w.thp = (double*)take(V * d); w.R = (double*)take(9 * (size_t)G * d); w.q = (double*)take(4 * (size_t)G * d);
  w.offA = (double*)take(16 * K * d); w.diagB = (double*)take(16 * K * d); w.lam = (double*)take(16 * K * d);
  w.mu_terms = (double*)take(K * d); w.top = (double*)take(16 * (size_t)G * d);
  w.bW = (double*)take(3 * (size_t)P * d); w.D = (double*)take(3 * V * d); w.diag3 = (double*)take(9 * V * d);
  w.w = (double*)take((size_t)G * nmax * d);
  w.M_init = (double*)take(G * nn * d); w.M = (double*)take(G * nn * d); w.Bm = (double*)take(G * nn * d);
  w.M_psd = (double*)take(G * nn * d); w.W = (double*)take(G * nn * d); w.Wd = (double*)take(G * nn * d);
  w.M_aff = (double*)take(G * nn * d); w.traj = (double*)take((size_t)G * T * d);
  w.pr = (CertBatchProb*)take(G * sizeof(CertBatchProb));
  w.info = (int*)take(G * sizeof(int)); w.active = (int*)take(G * sizeof(int));
  w.wc = (double*)take((size_t)G * nmax * d); w.infoc = (int*)take(G * sizeof(int)); w.idx = (int*)take(G * sizeof(int));
  w.work = take(work);
  w.gt = gather ? (CertGatherProb*)take(G * sizeof(CertGatherProb)) : nullptr;
  if (out) *out = w;
  return (size_t)(p - (char*)base);
}
}  // namespace

int certify_batch_device(CertMode mode, const tzr_certifier_params& prm, int B, const int32_t* N, const double* R_cm,
                         const double* const* src, const double* const* dst, const double* const* theta,
                         const CertGatherProb* gather, int32_t* gathered,
                         tzr_certification_result* results, double* const* traj, const int32_t* traj_cap,
                         const double* const* X_in, double* const* X_out, double* const* w_out, double* mu_out,
                         bool loop_eig, void** scratch, size_t* scratch_cap, void** solver_handle, int64_t* launches,
                         cudaStream_t st, std::string* err) {
  const bool certify = mode == CertMode::kCertify;
  const bool dev_in = certify && gather;  // measurements gathered on the device from a retained solve
  const bool eigen = certify || mode == CertMode::kPsd;  // the modes that run the eigensolver
  const bool setup = certify || mode == CertMode::kSetup;  // the modes that build M_init
  int nmax_all = 0;
  for (int b = 0; b < B; ++b) {
    if (4 * (size_t)N[b] + 4 > 32768) {
      *err = "problem " + std::to_string(b) + ": 4N+4 = " + std::to_string(4 * (size_t)N[b] + 4) + " exceeds 32768";
      return TZR_ERR_TOO_LARGE;
    }
    nmax_all = std::max(nmax_all, 4 * N[b] + 4);
  }
  // cuSOLVER is loaded, and the handle created, only where the eigensolver runs: the setup and dual-projection modes
  // work without the library
  Cusolver* cs = nullptr;
  cusolverDnHandle_t& handle = *reinterpret_cast<cusolverDnHandle_t*>(solver_handle);  // owned by the context
  if (eigen) {
    cs = &cusolver();
    if (!cs->ok) {
      *err = cs->err;
      return TZR_ERR_UNSUPPORTED;
    }
    if (!handle && cs->create(&handle) != CUSOLVER_STATUS_SUCCESS) {
      *err = "cusolverDnCreate failed";
      return TZR_ERR_CUDA;
    }
    cs->set_stream(handle, st);
  }
  cusolverDnParams_t sp = nullptr;
  bool batched = eigen && !loop_eig && cs->batched && B > 1 && cs->create_params(&sp) == CUSOLVER_STATUS_SUCCESS;
  struct ParamsGuard {
    Cusolver* cs;
    cusolverDnParams_t& p;
    ~ParamsGuard() { if (p) cs->destroy_params(p); }
  } guard{cs, sp};
  // eigensolver workspace of `G` problems padded to `nmax`: (device bytes, host bytes); {0, 0} when the batched call
  // refuses the size
  auto batched_ws = [&](int nmax, int G, size_t* host) -> size_t {
    size_t dmax = 0, hmax = 0;
    for (cusolverEigMode_t jobz : {CUSOLVER_EIG_MODE_VECTOR, CUSOLVER_EIG_MODE_NOVECTOR}) {
      size_t dv = 0, hv = 0;
      if (cs->syev_batched_buf(handle, sp, jobz, CUBLAS_FILL_MODE_LOWER, nmax, CUDA_R_64F, nullptr, nmax, CUDA_R_64F,
                               nullptr, CUDA_R_64F, &dv, &hv, G) != CUSOLVER_STATUS_SUCCESS)
        return 0;
      dmax = std::max(dmax, dv);
      hmax = std::max(hmax, hv);
    }
    *host = hmax;
    return std::max<size_t>(dmax, 1);
  };
  // Dsyevd workspace bytes at `nmax`: 0 when the query fails, and in the modes without an eigensolver
  auto syevd_ws = [&](int nmax) -> size_t {
    int lwork = 0;
    if (!eigen || cs->syevd_buf(handle, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, nmax, nullptr, nmax, nullptr,
                                &lwork) != CUSOLVER_STATUS_SUCCESS)
      return 0;
    return (size_t)lwork * sizeof(double);
  };
  const size_t loop_ws_all = syevd_ws(nmax_all);
  if (eigen && !loop_ws_all) {
    *err = "cusolverDnDsyevd_bufferSize failed";
    return TZR_ERR_CUDA;
  }
  size_t host_ws = 0;
  const size_t ws1 = batched ? batched_ws(nmax_all, 1, &host_ws) : 0;
  if (batched && !ws1) batched = false;  // the batched call refuses nmax: loop route
  // trajectory columns kept on the device: what the caller can receive, at most the iteration cap
  const double maxit = prm.max_iterations;
  int T = 0;
  for (int b = 0; traj && traj_cap && b < B; ++b)
    if (traj[b]) T = std::max(T, (int)traj_cap[b]);
  T = (int)std::min<double>(T, std::max(0.0, std::ceil(maxit)));
  size_t fr = 0, tot = 0;
  cudaMemGetInfo(&fr, &tot);
  const size_t budget = (size_t)(0.9 * (double)(fr + *scratch_cap));
  const double nbs = prm.cbar2 * prm.noise_bound * prm.noise_bound;

  // groups of consecutive problems that fit the device, each run to completion in one launch sequence
  for (int b0 = 0; b0 < B;) {
    int b1 = b0, nmax = 0;
    long long K = 0, P = 0;
    size_t need = 0;
    while (b1 < B && b1 - b0 < 65535) {
      const int nm2 = std::max(nmax, 4 * N[b1] + 4), G2 = b1 - b0 + 1;
      const long long K2 = K + N[b1], P2 = P + (long long)N[b1] * (N[b1] + 1) / 2;
      const size_t ws = std::max(loop_ws_all, batched ? ws1 * (size_t)G2 : 0);
      const size_t need2 = cbt_carve(nullptr, G2, K2, P2, nm2, T, ws, nullptr, dev_in);
      if (need2 > budget && b1 > b0) break;
      if (need2 > budget) {
        *err = "the certifier batch workspace of " + std::to_string(need2) + " bytes (one problem, 4N+4 = " +
               std::to_string(nm2) + ") does not fit the device";
        return TZR_ERR_ALLOC;
      }
      nmax = nm2; K = K2; P = P2; need = need2;
      ++b1;
    }
    // The estimate above scales the one-problem workspace; the group's own query decides.  Halve the group until the
    // workspace it really needs fits.
    bool bat = false;
    size_t hws = 0, dws = 0, lwork_bytes = 0;
    for (;;) {
      bat = batched && b1 - b0 >= kCertBatchedMinActive;
      hws = dws = 0;
      if (bat) {
        dws = batched_ws(nmax, b1 - b0, &hws);
        if (!dws) bat = false;
      }
      lwork_bytes = syevd_ws(nmax);
      need = cbt_carve(nullptr, b1 - b0, K, P, nmax, T, std::max(dws, lwork_bytes), nullptr, dev_in);
      if (need <= budget || b1 - b0 == 1) break;
      b1 = b0 + (b1 - b0) / 2;
      nmax = 0; K = 0; P = 0;
      for (int b = b0; b < b1; ++b) {
        nmax = std::max(nmax, 4 * N[b] + 4);
        K += N[b];
        P += (long long)N[b] * (N[b] + 1) / 2;
      }
    }
    const int G = b1 - b0;
    if (need > *scratch_cap) {
      if (*scratch) cudaFree(*scratch);
      *scratch = nullptr;
      *scratch_cap = 0;
      if (cudaMalloc(scratch, need) != cudaSuccess) {
        cudaGetLastError();
        *err = "cudaMalloc of " + std::to_string(need) + " bytes for the certifier batch failed";
        return TZR_ERR_ALLOC;
      }
      *scratch_cap = need;
    }
    CertBatchWork w;
    cbt_carve(*scratch, G, K, P, nmax, T, std::max(dws, lwork_bytes), &w, dev_in);
    std::vector<char> host_work(std::max<size_t>(hws, 1));
    // host tables (device input mode: only the rotations and the gather table; the kernel below writes the rest)
    std::vector<CertBatchProb> tab(G);
    const long long Kh = dev_in ? 0 : K;
    std::vector<double> h_src(3 * Kh), h_dst(3 * Kh), h_th(Kh), h_thp(dev_in ? 0 : K + G), h_R(9 * (size_t)G),
        h_q(4 * (size_t)G);
    std::vector<CertGatherProb> h_gt(dev_in ? G : 0);
    int maxN = 0;
    for (int g = 0, k = 0; g < G; ++g) {
      const int b = b0 + g, Nb = N[b];
      CertBatchProb& t = tab[g];
      t.N = Nb; t.n = 4 * Nb + 4; t.k_off = k; t.v_off = k + g;
      t.p_off = g ? tab[g - 1].p_off + (long long)tab[g - 1].N * (tab[g - 1].N + 1) / 2 : 0;
      t.active = 1; t.iters = 0; t.first_pos = 0; t.pad_bits = 0; t.mu = 0; t.best = INFINITY;
      t.nbs = dev_in ? gather[b].nbs : nbs;
      if (mode == CertMode::kPsd) {  // the PSD building block starts from X_in[b]: its pad follows that matrix
        double m = 0;
        for (size_t e = 0; e < (size_t)t.n * t.n; ++e) m = std::max(m, std::fabs(X_in[b][e]));
        std::memcpy(&t.pad_bits, &m, sizeof m);
      }
      if (setup) {
        if (dev_in) {
          h_gt[g] = gather[b];
          h_gt[g].k_off = t.k_off;
          h_gt[g].v_off = t.v_off;
        } else {
          std::copy(src[b], src[b] + 3 * (size_t)Nb, h_src.begin() + 3 * (size_t)k);
          std::copy(dst[b], dst[b] + 3 * (size_t)Nb, h_dst.begin() + 3 * (size_t)k);
          std::copy(theta[b], theta[b] + Nb, h_th.begin() + k);
        }
        std::copy(R_cm + 9 * (size_t)b, R_cm + 9 * (size_t)b + 9, h_R.begin() + 9 * (size_t)g);
        quaternion_xyzw(R_cm + 9 * (size_t)b, &h_q[4 * (size_t)g]);
      }
      if (!dev_in) {
        h_thp[k + g] = 1.0;
        if (mode != CertMode::kPsd) std::copy(theta[b], theta[b] + Nb, h_thp.begin() + k + g + 1);
      }
      maxN = std::max(maxN, Nb);
      k += Nb;
    }
    if (!dev_in) {
      cudaMemcpyAsync(w.src, h_src.data(), h_src.size() * sizeof(double), cudaMemcpyHostToDevice, st);
      cudaMemcpyAsync(w.dst, h_dst.data(), h_dst.size() * sizeof(double), cudaMemcpyHostToDevice, st);
      cudaMemcpyAsync(w.theta, h_th.data(), h_th.size() * sizeof(double), cudaMemcpyHostToDevice, st);
      cudaMemcpyAsync(w.thp, h_thp.data(), h_thp.size() * sizeof(double), cudaMemcpyHostToDevice, st);
    }
    cudaMemcpyAsync(w.R, h_R.data(), h_R.size() * sizeof(double), cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(w.q, h_q.data(), h_q.size() * sizeof(double), cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(w.pr, tab.data(), G * sizeof(CertBatchProb), cudaMemcpyHostToDevice, st);
    if (dev_in) {
      cudaMemcpyAsync(w.gt, h_gt.data(), G * sizeof(CertGatherProb), cudaMemcpyHostToDevice, st);
      cbt_solve_gather_kernel<<<G, kRTThreads, 0, st>>>(w.gt, w.pr, w.src, w.dst, w.theta, w.thp, w.active);
      *launches += 1;
    }
    const long long nn = (long long)nmax * nmax;
    const dim3 ge(grid1(nn, 256), G), gp(grid1(maxN + 1, 128), maxN, G), gt((nmax + kPT - 1) / kPT, (nmax + kPT - 1) / kPT, G);
    if (setup) {
      cbt_blocks_kernel<<<dim3(grid1(maxN, 128), G), 128, 0, st>>>(w.pr, w.src, w.dst, w.theta, w.R, w.q, w.offA,
                                                                    w.diagB, w.lam, w.mu_terms);
      cbt_reduce_kernel<<<G, 256, 0, st>>>(w.pr, w.lam, w.mu_terms, w.top);
      cbt_fill_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, w.offA, w.diagB, w.lam, w.top, w.M_init);
      *launches += 3;
      if (certify) cudaMemcpyAsync(w.M, w.M_init, (size_t)G * nn * sizeof(double), cudaMemcpyDeviceToDevice, st);
    }
    std::vector<int> act(G, 1), idx;  // active flags of the last read-back; their indices (compact batch)
    if (dev_in) {  // the gather's flags: a problem with a non-finite measurement starts (and stays) inactive
      cudaMemcpyAsync(act.data(), w.active, G * sizeof(int), cudaMemcpyDeviceToHost, st);
      if (cudaStreamSynchronize(st) != cudaSuccess) {
        *err = cudaGetErrorString(cudaGetLastError());
        return TZR_ERR_CUDA;
      }
      for (int g = 0; g < G; ++g) gathered[b0 + g] = act[g];
    }
    int n_act = (int)std::count(act.begin(), act.end(), 1), idx_for = -1;  // idx_for: the n_act whose idx is on the device
    bool full_step = bat;                // the step's eigen columns cover nmax (batched call) or n (Dsyevd)
    // one eigendecomposition of every active problem's Bm, and nothing for the finished ones: the batched call over the
    // padded matrices (in place while every problem is active, else over the active ones gathered into W, which is dead
    // at both eigen steps) while at least kCertBatchedMinActive are active, else cusolverDnDsyevd on each active real
    // block.  If the batched call
    // refuses, the Dsyevd loop serves the rest of the call.  Every eigensolver call counts as one launch.
    auto eig = [&](cusolverEigMode_t jobz) -> int {
      full_step = bat && n_act >= kCertBatchedMinActive;
      if (full_step) {
        size_t dws_a = dws, hws_a = hws;
        if (n_act < G) {
          dws_a = batched_ws(nmax, n_act, &hws_a);
          if (idx_for != n_act) {
            idx.clear();
            for (int g = 0; g < G; ++g)
              if (act[g]) idx.push_back(g);
            cudaMemcpyAsync(w.idx, idx.data(), n_act * sizeof(int), cudaMemcpyHostToDevice, st);
            idx_for = n_act;
          }
        }
        if (dws_a && dws_a <= dws && hws_a <= hws) {
          const bool all = n_act == G;
          const dim3 gc(grid1(nn, 256), n_act);
          if (!all) cbt_gather_kernel<<<gc, 256, 0, st>>>(w.idx, nmax, w.Bm, w.W);
          if (cs->syev_batched(handle, sp, jobz, CUBLAS_FILL_MODE_LOWER, nmax, CUDA_R_64F, all ? w.Bm : w.W, nmax,
                               CUDA_R_64F, all ? w.w : w.wc, CUDA_R_64F, w.work, dws_a, host_work.data(), hws_a,
                               all ? w.info : w.infoc, n_act) == CUSOLVER_STATUS_SUCCESS) {
            if (!all)
              cbt_scatter_kernel<<<gc, 256, 0, st>>>(w.idx, nmax, jobz == CUSOLVER_EIG_MODE_VECTOR ? 1 : 0, w.W, w.wc,
                                                     w.infoc, w.Bm, w.w, w.info);
            *launches += all ? 1 : 3;
            return TZR_OK;
          }
          if (!all) *launches += 1;
        }
        bat = full_step = false;
      }
      for (int g = 0; g < G; ++g) {
        if (!act[g]) continue;
        if (cs->syevd(handle, jobz, CUBLAS_FILL_MODE_LOWER, tab[g].n, w.Bm + (size_t)g * nn, nmax,
                      w.w + (size_t)g * nmax, (double*)w.work, (int)(lwork_bytes / sizeof(double)),
                      w.info + g) != CUSOLVER_STATUS_SUCCESS) {
          *err = "cusolverDnDsyevd failed";
          return TZR_ERR_CUDA;
        }
        *launches += 1;
      }
      return TZR_OK;
    };
    if (!certify) {
      // one building block on the group, in the layout and on the eigen route of the iteration below: each problem's
      // n x n input into the real block of M (PSD) or W (dual); the real block of M_init (setup), M_psd or Wd back
      const size_t ld = (size_t)nmax * sizeof(double);
      if (mode != CertMode::kSetup) {
        double* in = mode == CertMode::kPsd ? w.M : w.W;
        for (int g = 0; g < G; ++g) {
          const size_t nb = (size_t)tab[g].n * sizeof(double);
          cudaMemcpy2DAsync(in + (size_t)g * nn, ld, X_in[b0 + g], nb, nb, tab[g].n, cudaMemcpyHostToDevice, st);
        }
      }
      if (mode == CertMode::kPsd) {
        cbt_sym_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, w.M, w.Bm);
        if (int rc = eig(CUSOLVER_EIG_MODE_VECTOR)) return rc;
        cbt_first_pos_kernel<<<grid1(G, 128), 128, 0, st>>>(w.pr, G, nmax, full_step ? 1 : 0, w.w);
        cbt_psd_kernel<<<gt, 256, 0, st>>>(w.pr, nmax, full_step ? 1 : 0, w.Bm, w.w, w.M_psd);
        *launches += 3;
      } else if (mode == CertMode::kDual) {
        cbt_dual_bw_kernel<<<gp, 128, 0, st>>>(w.pr, nmax, w.W, w.thp, w.bW);
        cbt_dual_sums_kernel<<<dim3(grid1(3 * (maxN + 1), 128), G), 128, 0, st>>>(w.pr, w.bW, w.thp, w.D);
        cbt_dual_off_kernel<<<gp, 128, 0, st>>>(w.pr, nmax, w.W, w.thp, w.bW, w.D, w.Wd);
        cbt_dual_diag_kernel<<<dim3(grid1(maxN + 1, 4), G), 128, 0, st>>>(w.pr, nmax, w.W, w.thp, w.Wd, w.diag3);
        cbt_dual_mean_kernel<<<G, 256, 0, st>>>(w.pr, nmax, w.diag3, w.Wd);
        *launches += 5;
      }
      const double* out = mode == CertMode::kSetup ? w.M_init : mode == CertMode::kPsd ? w.M_psd : w.Wd;
      for (int g = 0; g < G; ++g) {
        const size_t nb = (size_t)tab[g].n * sizeof(double);
        cudaMemcpy2DAsync(X_out[b0 + g], nb, out + (size_t)g * nn, ld, nb, tab[g].n, cudaMemcpyDeviceToHost, st);
        if (w_out && w_out[b0 + g])
          cudaMemcpyAsync(w_out[b0 + g], w.w + (size_t)g * nmax, nb, cudaMemcpyDeviceToHost, st);
      }
      std::vector<int> info(G, 0);
      if (mode == CertMode::kPsd) cudaMemcpyAsync(info.data(), w.info, G * sizeof(int), cudaMemcpyDeviceToHost, st);
      if (mode == CertMode::kSetup)
        cudaMemcpyAsync(tab.data(), w.pr, G * sizeof(CertBatchProb), cudaMemcpyDeviceToHost, st);
      if (cudaStreamSynchronize(st) != cudaSuccess) {
        *err = cudaGetErrorString(cudaGetLastError());
        return TZR_ERR_CUDA;
      }
      for (int g = 0; g < G; ++g) {
        if (info[g] != 0) {
          *err = "problem " + std::to_string(b0 + g) + ": the eigensolver reported info " + std::to_string(info[g]);
          return TZR_ERR_CUDA;
        }
        if (mode == CertMode::kSetup) mu_out[b0 + g] = tab[g].mu;
      }
      b0 = b1;
      continue;
    }
    for (int iter = 0; n_act > 0 && (double)iter < maxit; ++iter) {
      cbt_sym_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, w.M, w.Bm);
      if (int rc = eig(CUSOLVER_EIG_MODE_VECTOR)) return rc;
      cbt_first_pos_kernel<<<grid1(G, 128), 128, 0, st>>>(w.pr, G, nmax, full_step ? 1 : 0, w.w);
      cbt_psd_kernel<<<gt, 256, 0, st>>>(w.pr, nmax, full_step ? 1 : 0, w.Bm, w.w, w.M_psd);
      cbt_affine_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, 0, w.M_psd, w.M, w.W, w.M_init, 0.0);
      cbt_dual_bw_kernel<<<gp, 128, 0, st>>>(w.pr, nmax, w.W, w.thp, w.bW);
      cbt_dual_sums_kernel<<<dim3(grid1(3 * (maxN + 1), 128), G), 128, 0, st>>>(w.pr, w.bW, w.thp, w.D);
      cbt_dual_off_kernel<<<gp, 128, 0, st>>>(w.pr, nmax, w.W, w.thp, w.bW, w.D, w.Wd);
      cbt_dual_diag_kernel<<<dim3(grid1(maxN + 1, 4), G), 128, 0, st>>>(w.pr, nmax, w.W, w.thp, w.Wd, w.diag3);
      cbt_dual_mean_kernel<<<G, 256, 0, st>>>(w.pr, nmax, w.diag3, w.Wd);
      cbt_affine_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, 1, w.Wd, nullptr, w.M_aff, w.M_init, 0.0);
      cbt_sym_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, w.M_aff, w.Bm);
      if (int rc = eig(CUSOLVER_EIG_MODE_NOVECTOR)) return rc;
      cbt_gap_kernel<<<grid1(G, 128), 128, 0, st>>>(w.pr, G, nmax, w.w, w.info, iter, prm.sub_optimality, maxit,
                                                     w.traj, T, w.active);
      *launches += 13;
      cudaMemcpyAsync(act.data(), w.active, G * sizeof(int), cudaMemcpyDeviceToHost, st);
      if (cudaStreamSynchronize(st) != cudaSuccess) {
        *err = cudaGetErrorString(cudaGetLastError());
        return TZR_ERR_CUDA;
      }
      n_act = (int)std::count(act.begin(), act.end(), 1);
      if (n_act == 0) break;
      cbt_affine_kernel<<<ge, 256, 0, st>>>(w.pr, nmax, 2, w.M_aff, w.M_psd, w.M, nullptr, prm.gamma_tau);
      *launches += 1;
    }
    std::vector<double> h_traj((size_t)G * T);
    cudaMemcpyAsync(tab.data(), w.pr, G * sizeof(CertBatchProb), cudaMemcpyDeviceToHost, st);
    if (T) cudaMemcpyAsync(h_traj.data(), w.traj, h_traj.size() * sizeof(double), cudaMemcpyDeviceToHost, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) {
      *err = cudaGetErrorString(cudaGetLastError());
      return TZR_ERR_CUDA;
    }
    for (int g = 0; g < G; ++g) {
      const int b = b0 + g;
      results[b].is_optimal = tab[g].best < prm.sub_optimality ? 1 : 0;
      results[b].n_iterations = tab[g].iters;
      results[b].best_suboptimality = tab[g].best;
      if (traj && traj_cap && traj[b]) {
        const int m = std::min(std::min(tab[g].iters, (int)traj_cap[b]), T);
        std::copy(h_traj.begin() + (size_t)g * T, h_traj.begin() + (size_t)g * T + m, traj[b]);
      }
    }
    b0 = b1;
  }
  return TZR_OK;
}

int dense_cholesky_setup(void** solver_handle, int n, double* A, int* lwork, cudaStream_t st, std::string* err) {
  Cusolver& cs = cusolver();
  if (!cs.ok || !cs.cholesky) {
    *err = cs.ok ? "libcusolver lacks the Dpotrf / Dpotrs entry points" : cs.err;
    return TZR_ERR_UNSUPPORTED;
  }
  cusolverDnHandle_t& handle = *reinterpret_cast<cusolverDnHandle_t*>(solver_handle);  // owned by the context
  if (!handle && cs.create(&handle) != CUSOLVER_STATUS_SUCCESS) {
    *err = "cusolverDnCreate failed";
    return TZR_ERR_CUDA;
  }
  cs.set_stream(handle, st);
  if (cs.potrf_buf(handle, CUBLAS_FILL_MODE_LOWER, n, A, n, lwork) != CUSOLVER_STATUS_SUCCESS) {
    *err = "cusolverDnDpotrf_bufferSize failed";
    return TZR_ERR_CUDA;
  }
  return TZR_OK;
}

int dense_cholesky_solve(void* solver_handle, int n, double* A, double* b, double* work, int lwork, int* info,
                         std::string* err) {
  Cusolver& cs = cusolver();
  cusolverDnHandle_t handle = (cusolverDnHandle_t)solver_handle;
  if (cs.potrf(handle, CUBLAS_FILL_MODE_LOWER, n, A, n, work, lwork, info) != CUSOLVER_STATUS_SUCCESS ||
      cs.potrs(handle, CUBLAS_FILL_MODE_LOWER, n, 1, A, n, b, n, info + 1) != CUSOLVER_STATUS_SUCCESS) {
    *err = "cusolverDnDpotrf / cusolverDnDpotrs failed";
    return TZR_ERR_CUDA;
  }
  return TZR_OK;
}

void certify_release(void* solver_handle) {
  if (solver_handle && cusolver().ok) cusolver().destroy((cusolverDnHandle_t)solver_handle);
}

}  // namespace tzr
