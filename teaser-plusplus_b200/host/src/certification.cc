// teaser::DRSCertifier façade: forwards to the C-ABI (no CPU implementation behind it).
#include "teaser/certification.h"

#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread

namespace {
tzr_certifier_params to_c(const DRSCertifier::Params& p) {
  tzr_certifier_params c;
  tzr_certifier_params_default(&c);
  c.noise_bound = p.noise_bound;
  c.cbar2 = p.cbar2;
  c.sub_optimality = p.sub_optimality;
  c.max_iterations = p.max_iterations;
  c.gamma_tau = p.gamma_tau;
  c.eig_decomposition_solver = static_cast<int>(p.eig_decomposition_solver);
  return c;
}
[[noreturn]] void fail(const char* what, int rc, tzr_ctx* ctx) {
  throw std::runtime_error(std::string(what) + ": " + tzr_status_string(rc) + " (" + tzr_last_error(ctx) + ")");
}
}  // namespace

CertificationResult DRSCertifier::certify(const Eigen::Matrix3d& R_solution,
                                          const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                                          const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                                          const Eigen::Matrix<bool, 1, Eigen::Dynamic>& theta) {
  // certification.cc:27-37: true -> 1, false -> -1
  Eigen::Matrix<double, 1, Eigen::Dynamic> theta_double(1, theta.cols());
  for (Eigen::Index i = 0; i < theta.cols(); ++i) theta_double(i) = theta(i) ? 1 : -1;
  return certify(R_solution, src, dst, theta_double);
}

CertificationResult DRSCertifier::certify(const Eigen::Matrix3d& R_solution,
                                          const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                                          const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                                          const Eigen::Matrix<double, 1, Eigen::Dynamic>& theta) {
  const int n = static_cast<int>(src.cols());
  if (dst.cols() != src.cols() || theta.cols() != src.cols() || n == 0)
    throw std::invalid_argument("teaser::DRSCertifier::certify: src, dst and theta must have the same, non-zero width");
  tzr_ctx* ctx = b200_context();
  const tzr_certifier_params p = to_c(params_);
  const int cap = static_cast<int>(std::max(1.0, std::ceil(params_.max_iterations)));
  CertificationResult out;
  out.suboptimality_traj.resize(cap);
  tzr_certification_result r;
  const int rc = tzr_certify(ctx, &p, R_solution.data(), src.data(), dst.data(), theta.data(), n, &r,
                             out.suboptimality_traj.data(), cap);
  if (rc != TZR_OK) fail("teaser::DRSCertifier (GPU)", rc, ctx);
  out.suboptimality_traj.resize(r.n_iterations);
  out.is_optimal = r.is_optimal != 0;
  out.best_suboptimality = r.best_suboptimality;
  return out;
}

std::vector<CertificationResult> DRSCertifier::certifyBatch(
    const std::vector<Eigen::Matrix3d>& R_solutions, const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& src,
    const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& dst,
    const std::vector<Eigen::Matrix<bool, 1, Eigen::Dynamic>>& theta) {
  std::vector<Eigen::Matrix<double, 1, Eigen::Dynamic>> theta_double;
  theta_double.reserve(theta.size());
  for (const auto& t : theta) {
    Eigen::Matrix<double, 1, Eigen::Dynamic> td(1, t.cols());
    for (Eigen::Index i = 0; i < t.cols(); ++i) td(i) = t(i) ? 1 : -1;
    theta_double.push_back(td);
  }
  return certifyBatch(R_solutions, src, dst, theta_double);
}

std::vector<CertificationResult> DRSCertifier::certifyBatch(
    const std::vector<Eigen::Matrix3d>& R_solutions, const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& src,
    const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& dst,
    const std::vector<Eigen::Matrix<double, 1, Eigen::Dynamic>>& theta) {
  const size_t B = R_solutions.size();
  if (B == 0 || src.size() != B || dst.size() != B || theta.size() != B)
    throw std::invalid_argument("teaser::DRSCertifier::certifyBatch: the four vectors must have the same, non-zero size");
  std::vector<int32_t> n(B), caps(B);
  std::vector<double> R(9 * B);
  std::vector<const double*> s(B), d(B), t(B);
  std::vector<double*> traj(B);
  std::vector<CertificationResult> out(B);
  const int cap = static_cast<int>(std::max(1.0, std::ceil(params_.max_iterations)));
  for (size_t b = 0; b < B; ++b) {
    n[b] = static_cast<int32_t>(src[b].cols());
    if (dst[b].cols() != src[b].cols() || theta[b].cols() != src[b].cols() || n[b] == 0)
      throw std::invalid_argument("teaser::DRSCertifier::certifyBatch: problem " + std::to_string(b) +
                                  ": src, dst and theta must have the same, non-zero width");
    std::copy(R_solutions[b].data(), R_solutions[b].data() + 9, R.begin() + 9 * b);
    s[b] = src[b].data();
    d[b] = dst[b].data();
    t[b] = theta[b].data();
    out[b].suboptimality_traj.resize(cap);
    traj[b] = out[b].suboptimality_traj.data();
    caps[b] = cap;
  }
  tzr_ctx* ctx = b200_context();
  const tzr_certifier_params p = to_c(params_);
  std::vector<tzr_certification_result> r(B);
  const int rc = tzr_certify_batch(ctx, &p, static_cast<int>(B), n.data(), R.data(), s.data(), d.data(), t.data(),
                                   r.data(), traj.data(), caps.data());
  if (rc != TZR_OK) fail("teaser::DRSCertifier::certifyBatch (GPU)", rc, ctx);
  for (size_t b = 0; b < B; ++b) {
    out[b].suboptimality_traj.resize(r[b].n_iterations);
    out[b].is_optimal = r[b].is_optimal != 0;
    out[b].best_suboptimality = r[b].best_suboptimality;
  }
  return out;
}

Eigen::Matrix4d DRSCertifier::getOmega1(double x, double y, double z, double w) {
  Eigen::Matrix4d o;
  const double v[4][4] = {{w, -z, y, x}, {z, w, -x, y}, {-y, x, w, z}, {-x, -y, -z, w}};
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) o(r, c) = v[r][c];
  return o;
}

void DRSCertifier::getBlockDiagOmega(int Npm, double qx, double qy, double qz, double qw, Eigen::MatrixXd* D_omega) {
  D_omega->resize(Npm, Npm);
  D_omega->setZero();
  const Eigen::Matrix4d o = getOmega1(qx, qy, qz, qw);
  for (int i = 0; i < Npm / 4; ++i)
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) (*D_omega)(4 * i + r, 4 * i + c) = o(r, c);
}

void DRSCertifier::getOptimalDualProjection(const Eigen::MatrixXd& W,
                                            const Eigen::Matrix<double, 1, Eigen::Dynamic>& theta_prepended,
                                            Eigen::MatrixXd* W_dual) {
  const int n = static_cast<int>(theta_prepended.cols()) - 1;
  if (n <= 0 || W.rows() != 4 * n + 4 || W.cols() != 4 * n + 4)
    throw std::invalid_argument("teaser::DRSCertifier::getOptimalDualProjection: W must be (4N+4) x (4N+4)");
  W_dual->resize(W.rows(), W.cols());
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_certifier_dual_projection(ctx, W.data(), theta_prepended.data() + 1, n, W_dual->data());
  if (rc != TZR_OK) fail("teaser::DRSCertifier::getOptimalDualProjection (GPU)", rc, ctx);
}

void DRSCertifier::getInitialMatrix(const Eigen::Matrix3d& R_solution,
                                    const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                                    const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                                    const Eigen::Matrix<double, 1, Eigen::Dynamic>& theta, Eigen::MatrixXd* M_init,
                                    double* mu) {
  const int n = static_cast<int>(src.cols());
  M_init->resize(4 * n + 4, 4 * n + 4);
  tzr_ctx* ctx = b200_context();
  const tzr_certifier_params p = to_c(params_);
  const int rc = tzr_certifier_initial_matrix(ctx, &p, R_solution.data(), src.data(), dst.data(), theta.data(), n,
                                              M_init->data(), mu);
  if (rc != TZR_OK) fail("teaser::DRSCertifier::getInitialMatrix (GPU)", rc, ctx);
}

}  // namespace teaser
