// GPU build of the reference's C++ quick-start (examples/teaser_cpp_ply/teaser_cpp_ply.cc): the solver-facing
// lines (PLYReader, Params, constructor, solve, getSolution) are written exactly as a TEASER++ user writes them.
//   usage: example_cpp_ply <bun_zipper_res3.ply>
#include <chrono>
#include <cmath>
#include <fstream>
#include <iostream>
#include <random>
#include <sstream>
#include <string>

#include <teaser/ply_io.h>
#include <teaser/registration.h>

constexpr double NOISE_BOUND = 0.001;
constexpr int N_OUTLIERS = 1700;
constexpr double OUTLIER_TRANSLATION_LB = 5;
constexpr double OUTLIER_TRANSLATION_UB = 10;

int main(int argc, char** argv) {
  if (argc < 2) {
    std::cerr << "usage: " << argv[0] << " bun_zipper_res3.ply\n";
    return 2;
  }
  // Load the .ply file (teaser_cpp_ply.cc:44-55)
  teaser::PLYReader reader;
  teaser::PointCloud src_cloud;
  auto status = reader.read(argv[1], src_cloud);
  if (status != 0) {
    std::cerr << "cannot read " << argv[1] << "\n";
    return 2;
  }
  const int N = static_cast<int>(src_cloud.size());
  // Convert the point cloud to Eigen
  teaser::Mat3X src(3, N);
  for (int i = 0; i < N; ++i) {
    src(0, i) = src_cloud[i].x;
    src(1, i) = src_cloud[i].y;
    src(2, i) = src_cloud[i].z;
  }
  Eigen::Matrix3d R;
  R << 9.96926560e-01, 6.68735757e-02, -4.06664421e-02,
      -6.61289946e-02, 9.97617877e-01, 1.94008687e-02,
       4.18675510e-02, -1.66517807e-02, 9.98977765e-01;
  Eigen::Vector3d t(-1.15576939e-01, -3.87705398e-02, 1.14874890e-01);
  teaser::Mat3X tgt(3, N);
  std::mt19937 gen(1889);
  std::uniform_real_distribution<double> noise(-1.0, 1.0);
  for (int i = 0; i < N; ++i)
    for (int r = 0; r < 3; ++r)
      tgt(r, i) = R(r, 0) * src(0, i) + R(r, 1) * src(1, i) + R(r, 2) * src(2, i) + t(r) + noise(gen) * NOISE_BOUND / 2;
  std::uniform_int_distribution<int> pick(0, N - 1);
  std::uniform_int_distribution<int> shift(static_cast<int>(OUTLIER_TRANSLATION_LB), static_cast<int>(OUTLIER_TRANSLATION_UB));
  for (int k = 0; k < N_OUTLIERS; ++k) {
    const int c = pick(gen);
    const int d = shift(gen);
    for (int r = 0; r < 3; ++r) tgt(r, c) += d;
  }

  // ---- exactly the reference's solver-facing code (teaser_cpp_ply.cc:79-95)
  teaser::RobustRegistrationSolver::Params params;
  params.noise_bound = NOISE_BOUND;
  params.cbar2 = 1;
  params.estimate_scaling = false;
  params.rotation_max_iterations = 100;
  params.rotation_gnc_factor = 1.4;
  params.rotation_estimation_algorithm = teaser::RobustRegistrationSolver::ROTATION_ESTIMATION_ALGORITHM::GNC_TLS;
  params.rotation_cost_threshold = 0.005;

  teaser::RobustRegistrationSolver solver(params);
  solver.solve(src, tgt);  // warm-up: CUDA context + workspace
  std::chrono::steady_clock::time_point begin = std::chrono::steady_clock::now();
  solver.solve(src, tgt);
  std::chrono::steady_clock::time_point end = std::chrono::steady_clock::now();
  auto solution = solver.getSolution();

  const double c = ((R.transpose() * solution.rotation).trace() - 1) / 2;
  std::cout << "clique size: " << solver.getInlierMaxClique().size() << "\n";
  std::cout << "rotation error (rad): " << std::abs(std::acos(std::fmin(std::fmax(c, -1.0), 1.0))) << "\n";
  std::cout << "translation error (m): " << (t - solution.translation).norm() << "\n";
  std::cout << "time (s): "
            << std::chrono::duration_cast<std::chrono::microseconds>(end - begin).count() / 1000000.0 << "\n";
  return solution.valid ? 0 : 1;
}
