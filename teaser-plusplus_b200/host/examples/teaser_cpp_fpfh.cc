// GPU build of the reference's feature-matching example (examples/teaser_cpp_fpfh/teaser_cpp_fpfh.cc:41-131):
// Matcher::calculateCorrespondences -> RobustRegistrationSolver::solve(src_cloud, tgt_cloud, correspondences), with
// the solver- and matcher-facing lines written as a TEASER++ user writes them.  PCL (FPFH estimation) is not part of
// the GPU path, so the descriptors come from a file: the reference's own fixture test/teaser/data/bunny_fpfh.csv
// (PCL FPFH of bunny.pcd); the target cloud is the transformed, shuffled, noisy source with 30 % of its descriptors
// replaced by other points' descriptors (wrong matches).
// With only the .pcd argument the descriptors of both clouds are computed with teaser::FPFHEstimation, exactly as the
// reference example does (teaser_cpp_fpfh.cc:86-89).
//   usage: example_cpp_fpfh <bunny.pcd> [<bunny_fpfh.csv>]
#include <chrono>
#include <cmath>
#include <fstream>
#include <iostream>
#include <numeric>
#include <random>
#include <sstream>
#include <string>

#include <teaser/matcher.h>
#include <teaser/registration.h>

constexpr double NOISE_BOUND = 0.001;

int main(int argc, char** argv) {
  if (argc < 2) {
    std::cerr << "usage: " << argv[0] << " bunny.pcd [bunny_fpfh.csv]\n";
    return 2;
  }
  const bool from_file = argc >= 3;
  teaser::PointCloud src_cloud;
  {
    std::ifstream f(argv[1]);
    std::string line;
    bool data = false;
    while (std::getline(f, line)) {
      if (data) {
        std::istringstream is(line);
        teaser::PointXYZ p;
        if (is >> p.x >> p.y >> p.z) src_cloud.push_back(p);
      } else if (line.rfind("DATA", 0) == 0) {
        data = true;
      }
    }
  }
  const int N = static_cast<int>(src_cloud.size());
  teaser::FPFHCloud obj_descriptors;
  if (from_file) {
    std::ifstream f(argv[2]);
    obj_descriptors.resize(N);
    for (int i = 0; i < N; ++i)
      for (int k = 0; k < 33; ++k) f >> obj_descriptors[i].histogram[k];
    if (!f) {
      std::cerr << "descriptor file too short\n";
      return 2;
    }
  }

  Eigen::Matrix3d R;
  R << 9.96926560e-01, 6.68735757e-02, -4.06664421e-02,
      -6.61289946e-02, 9.97617877e-01, 1.94008687e-02,
       4.18675510e-02, -1.66517807e-02, 9.98977765e-01;
  Eigen::Vector3d t(-1.15576939e-01, -3.87705398e-02, 1.14874890e-01);
  std::mt19937 gen(397);
  std::uniform_real_distribution<double> noise(-1.0, 1.0);
  std::vector<int> perm(N);
  std::iota(perm.begin(), perm.end(), 0);
  std::shuffle(perm.begin(), perm.end(), gen);
  teaser::PointCloud tgt_cloud;
  teaser::FPFHCloud scene_descriptors;
  std::uniform_int_distribution<int> pick(0, N - 1);
  for (int j = 0; j < N; ++j) {
    const teaser::PointXYZ& p = src_cloud[perm[j]];
    double q[3];
    for (int r = 0; r < 3; ++r) q[r] = R(r, 0) * p.x + R(r, 1) * p.y + R(r, 2) * p.z + t(r) + noise(gen) * NOISE_BOUND / 2;
    tgt_cloud.push_back({static_cast<float>(q[0]), static_cast<float>(q[1]), static_cast<float>(q[2])});
    if (from_file) {
      const bool wrong = j % 10 < 3;
      teaser::FPFHSignature33 d = obj_descriptors[wrong ? pick(gen) : perm[j]];
      if (wrong) d.histogram[j % 33] += 0.5f;  // keep the wrong descriptor from being an exact duplicate
      scene_descriptors.push_back(d);
    }
  }
  if (!from_file) {
    // Compute FPFH (teaser_cpp_fpfh.cc:86-89; radii scaled to this 397-point cloud)
    teaser::FPFHEstimation fpfh;
    obj_descriptors = *fpfh.computeFPFHFeatures(src_cloud, 0.03, 0.05);
    scene_descriptors = *fpfh.computeFPFHFeatures(tgt_cloud, 0.03, 0.05);
  }

  // ---- the reference's matcher- and solver-facing code (teaser_cpp_fpfh.cc:91-113)
  teaser::Matcher matcher;
  auto correspondences =
      matcher.calculateCorrespondences(src_cloud, tgt_cloud, obj_descriptors, scene_descriptors, false, true, false, 0.95);

  teaser::RobustRegistrationSolver::Params params;
  params.noise_bound = NOISE_BOUND;
  params.cbar2 = 1;
  params.estimate_scaling = false;
  params.rotation_max_iterations = 100;
  params.rotation_gnc_factor = 1.4;
  params.rotation_estimation_algorithm = teaser::RobustRegistrationSolver::ROTATION_ESTIMATION_ALGORITHM::GNC_TLS;
  params.rotation_cost_threshold = 0.005;

  teaser::RobustRegistrationSolver solver(params);
  std::chrono::steady_clock::time_point begin = std::chrono::steady_clock::now();
  solver.solve(src_cloud, tgt_cloud, correspondences);
  std::chrono::steady_clock::time_point end = std::chrono::steady_clock::now();
  auto solution = solver.getSolution();

  int right = 0;
  for (auto& c : correspondences) right += perm[c.second] == c.first;
  const double c = ((R.transpose() * solution.rotation).trace() - 1) / 2;
  std::cout << "correspondences: " << correspondences.size() << "\n";
  std::cout << "correct correspondences: " << right << "\n";
  std::cout << "clique size: " << solver.getInlierMaxClique().size() << "\n";
  std::cout << "rotation error (rad): " << std::abs(std::acos(std::fmin(std::fmax(c, -1.0), 1.0))) << "\n";
  std::cout << "translation error (m): " << (t - solution.translation).norm() << "\n";
  std::cout << "time (s): "
            << std::chrono::duration_cast<std::chrono::microseconds>(end - begin).count() / 1000000.0 << "\n";
  return solution.valid ? 0 : 1;
}
