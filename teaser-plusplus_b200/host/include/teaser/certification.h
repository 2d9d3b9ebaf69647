// Certifier classes of the TEASER++ public API (mirrors teaser/include/teaser/certification.h:19-237 of the
// reference).  DRSCertifier::certify runs on the GPU through tzr_certify (include/teaser_b200.h); the building blocks
// the reference exposes for its unit tests are available where they make sense without Eigen's sparse module:
// getOmega1, getBlockDiagOmega, getOptimalDualProjection (the inverse map of getLinearProjection is applied in closed
// form on the device, so no A_inv argument), getInitialMatrix (= D^T Q_cost D - mu J - lambda_guess).
#pragma once
#include <vector>

#include "teaser/eigen_lite.h"

namespace teaser {

struct CertificationResult {
  bool is_optimal = false;
  double best_suboptimality = -1;
  std::vector<double> suboptimality_traj;
};

/** Abstract virtual class representing certification of registration results (certification.h:31-52). */
class AbstractRotationCertifier {
 public:
  virtual ~AbstractRotationCertifier() {}
  virtual CertificationResult certify(const Eigen::Matrix3d& rotation_solution,
                                      const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                                      const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                                      const Eigen::Matrix<bool, 1, Eigen::Dynamic>& theta) = 0;
};

/** Douglas–Rachford Splitting certifier (certification.h:57-237). */
class DRSCertifier : public AbstractRotationCertifier {
 public:
  enum class EIG_SOLVER_TYPE {
    EIGEN = 0,    ///< accepted for source compatibility; the device eigensolver is used for both values
    SPECTRA = 1,
  };

  struct Params {
    double noise_bound = 0.01;
    double cbar2 = 1;
    double sub_optimality = 1e-3;
    double max_iterations = 2e2;
    double gamma_tau = 1.999999;
    EIG_SOLVER_TYPE eig_decomposition_solver = EIG_SOLVER_TYPE::EIGEN;
  };

  DRSCertifier() = delete;
  DRSCertifier(const Params& params) : params_(params) {}
  DRSCertifier(double noise_bound, double cbar2) {
    params_.noise_bound = noise_bound;
    params_.cbar2 = cbar2;
  }

  CertificationResult certify(const Eigen::Matrix3d& R_solution, const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                              const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                              const Eigen::Matrix<bool, 1, Eigen::Dynamic>& theta) override;

  CertificationResult certify(const Eigen::Matrix3d& R_solution, const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                              const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                              const Eigen::Matrix<double, 1, Eigen::Dynamic>& theta);

  /// certify on every problem of the vectors in one device call (tzr_certify_batch); result b is what certify gives
  /// for problem b alone.  All four vectors have the same, non-zero length.
  std::vector<CertificationResult> certifyBatch(const std::vector<Eigen::Matrix3d>& R_solutions,
                                                const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& src,
                                                const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& dst,
                                                const std::vector<Eigen::Matrix<bool, 1, Eigen::Dynamic>>& theta);

  std::vector<CertificationResult> certifyBatch(const std::vector<Eigen::Matrix3d>& R_solutions,
                                                const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& src,
                                                const std::vector<Eigen::Matrix<double, 3, Eigen::Dynamic>>& dst,
                                                const std::vector<Eigen::Matrix<double, 1, Eigen::Dynamic>>& theta);

  /// certification.cc:293-303; q given as (x, y, z, w)
  Eigen::Matrix4d getOmega1(double qx, double qy, double qz, double qw);

  /// certification.cc:305-314
  void getBlockDiagOmega(int Npm, double qx, double qy, double qz, double qw, Eigen::MatrixXd* D_omega);

  /// certification.cc:316-446 (theta_prepended has N+1 entries, the first one 1)
  void getOptimalDualProjection(const Eigen::MatrixXd& W, const Eigen::Matrix<double, 1, Eigen::Dynamic>& theta_prepended,
                                Eigen::MatrixXd* W_dual);

  /// M_init of certification.cc:100 and mu of :92
  void getInitialMatrix(const Eigen::Matrix3d& R_solution, const Eigen::Matrix<double, 3, Eigen::Dynamic>& src,
                        const Eigen::Matrix<double, 3, Eigen::Dynamic>& dst,
                        const Eigen::Matrix<double, 1, Eigen::Dynamic>& theta, Eigen::MatrixXd* M_init, double* mu);

  const Params& getParams() const { return params_; }

 private:
  Params params_;
};

}  // namespace teaser
