// pybind11 module `teaserpp_python._teaserpp` for the GPU path.  Same module / class / method / property names
// as the reference binding (python/teaserpp_python/teaserpp_python.cc:25-291) so existing Python callers keep
// working; arrays cross the boundary as numpy (3,N) float64 exactly like the reference's pybind11/eigen.h casters
// (copied if not Fortran-contiguous).  Fixes of the reference's copy-paste slips (SURVEY Q4): the dst_* properties
// return the dst getters, Params exposes max_clique_num_threads, the ctor default time limit is 3600.
// The certifier classes (EigSolverType, CertificationResult, DRSCertifier + Params, :71-74,249-291) are bound too.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <array>
#include <cstring>
#include <sstream>

#include "teaser/certification.h"
#include "teaser/icp.h"
#include "teaser/pose_graph.h"
#include "teaser/normals.h"
#include "teaser/registration.h"
#include "teaser/voxel.h"

namespace py = pybind11;
using Solver = teaser::RobustRegistrationSolver;

namespace {

using ArrD = py::array_t<double, py::array::f_style | py::array::forcecast>;

teaser::Mat3X to_mat3x(const ArrD& a) {
  if (a.ndim() != 2 || a.shape(0) != 3) throw std::invalid_argument("expected a (3, N) float64 array");
  teaser::Mat3X m(3, a.shape(1));
  std::memcpy(m.data(), a.data(), sizeof(double) * 3 * static_cast<size_t>(a.shape(1)));
  return m;
}

template <typename T, int R, int C>
py::array_t<T> to_numpy(const Eigen::Matrix<T, R, C>& m) {
  py::array_t<T, py::array::f_style> out({static_cast<py::ssize_t>(m.rows()), static_cast<py::ssize_t>(m.cols())});
  if (m.size()) std::memcpy(out.mutable_data(), m.data(), sizeof(T) * static_cast<size_t>(m.size()));
  return out;
}
template <typename T, int R>
py::array_t<T> vec_to_numpy(const Eigen::Matrix<T, R, 1>& m) {
  py::array_t<T> out(static_cast<py::ssize_t>(m.rows()));
  if (m.size()) std::memcpy(out.mutable_data(), m.data(), sizeof(T) * static_cast<size_t>(m.size()));
  return out;
}
py::array_t<bool> row_to_numpy(const teaser::BoolRow& m) {
  py::array_t<bool> out(static_cast<py::ssize_t>(m.cols()));
  for (Eigen::Index i = 0; i < m.cols(); ++i) out.mutable_data()[i] = m(i);
  return out;
}
py::array_t<int> irow_to_numpy(const Eigen::Matrix<int, 1, Eigen::Dynamic>& m) {
  py::array_t<int> out(static_cast<py::ssize_t>(m.cols()));
  for (Eigen::Index i = 0; i < m.cols(); ++i) out.mutable_data()[i] = m(i);
  return out;
}

using CloudArray = py::array_t<float, py::array::c_style | py::array::forcecast>;

teaser::PointCloud cloud_of(const CloudArray& a) {
  if (a.ndim() != 2 || a.shape(1) != 3) throw std::invalid_argument("clouds must be (n,3) arrays");
  teaser::PointCloud pc;
  const float* d = a.data();
  pc.reserve(static_cast<size_t>(a.shape(0)));
  for (py::ssize_t i = 0; i < a.shape(0); ++i) pc.push_back({d[3 * i], d[3 * i + 1], d[3 * i + 2]});
  return pc;
}

py::array_t<float> cloud_to_numpy(const teaser::PointCloud& pc) {
  py::array_t<float> out({static_cast<py::ssize_t>(pc.size()), static_cast<py::ssize_t>(3)});
  float* d = out.mutable_data();
  for (size_t i = 0; i < pc.size(); ++i) {
    d[3 * i] = pc[i].x;
    d[3 * i + 1] = pc[i].y;
    d[3 * i + 2] = pc[i].z;
  }
  return out;
}

// (n,3) or (n,4) float normals (a fourth column is the curvature, which ICP ignores)
teaser::NormalCloud normals_of(const CloudArray& a) {
  if (a.ndim() != 2 || (a.shape(1) != 3 && a.shape(1) != 4))
    throw std::invalid_argument("normals must be (n,3) or (n,4) arrays");
  const py::ssize_t w = a.shape(1);
  teaser::NormalCloud nc(static_cast<size_t>(a.shape(0)));
  const float* d = a.data();
  for (py::ssize_t i = 0; i < a.shape(0); ++i)
    nc[i] = {d[w * i], d[w * i + 1], d[w * i + 2], w == 4 ? d[w * i + 3] : 0.f};
  return nc;
}

py::array_t<float> normals_to_numpy(const teaser::NormalCloud& nc) {
  py::array_t<float> out({static_cast<py::ssize_t>(nc.size()), static_cast<py::ssize_t>(4)});
  if (!nc.empty()) std::memcpy(out.mutable_data(), &nc[0].normal_x, sizeof(float) * 4 * nc.size());
  return out;
}

teaser::ColorCloud colors_of(const CloudArray& a) {
  if (a.ndim() != 2 || a.shape(1) != 3) throw std::invalid_argument("colours must be (n,3) arrays");
  teaser::ColorCloud cc(static_cast<size_t>(a.shape(0)));
  if (!cc.empty()) std::memcpy(&cc[0].r, a.data(), sizeof(float) * 3 * cc.size());
  return cc;
}

py::array_t<float> colors_to_numpy(const teaser::ColorCloud& cc) {
  py::array_t<float> out({static_cast<py::ssize_t>(cc.size()), static_cast<py::ssize_t>(3)});
  if (!cc.empty()) std::memcpy(out.mutable_data(), &cc[0].r, sizeof(float) * 3 * cc.size());
  return out;
}

py::array_t<double> gradients_to_numpy(const std::vector<std::array<double, 3>>& g) {
  py::array_t<double> out({static_cast<py::ssize_t>(g.size()), static_cast<py::ssize_t>(3)});
  if (!g.empty()) std::memcpy(out.mutable_data(), g[0].data(), sizeof(double) * 3 * g.size());
  return out;
}

py::dict icp_dict(const teaser::PointToPointICPResult& r) {
  return py::dict(py::arg("solution") = r.solution, py::arg("fitness") = r.fitness,
                  py::arg("inlier_rmse") = r.inlier_rmse, py::arg("iterations") = r.iterations,
                  py::arg("converged") = r.converged, py::arg("correspondences") = r.correspondences);
}

// (4,4) float64 matrices <-> Eigen::Matrix4d, (6,6) <-> teaser::Matrix6d
template <int N>
Eigen::Matrix<double, N, N> square_of(const py::array_t<double, py::array::c_style | py::array::forcecast>& a) {
  if (a.ndim() != 2 || a.shape(0) != N || a.shape(1) != N) throw std::invalid_argument("expected a square matrix");
  Eigen::Matrix<double, N, N> M;
  for (int r = 0; r < N; ++r)
    for (int c = 0; c < N; ++c) M(r, c) = a.at(r, c);
  return M;
}
template <int N>
py::array_t<double> square_to_numpy(const Eigen::Matrix<double, N, N>& M) {
  py::array_t<double> out({static_cast<py::ssize_t>(N), static_cast<py::ssize_t>(N)});
  for (int r = 0; r < N; ++r)
    for (int c = 0; c < N; ++c) out.mutable_at(r, c) = M(r, c);
  return out;
}
using SqArr = py::array_t<double, py::array::c_style | py::array::forcecast>;

// MultiScaleICP's scales from Python: (voxel_size, max_correspondence_distance, max_iteration[, normal_search_radius[,
// relative_fitness[, relative_rmse]]]) tuples or dicts with those keys; the normal radius defaults to 2 voxel_size
std::vector<teaser::ICPScale> scales_of(const py::list& scales) {
  static const char* keys[] = {"voxel_size", "max_correspondence_distance", "max_iteration", "normal_search_radius",
                               "relative_fitness", "relative_rmse"};
  std::vector<teaser::ICPScale> out;
  for (const py::handle& h : scales) {
    std::vector<py::object> v(6);
    if (py::isinstance<py::dict>(h)) {
      const py::dict d = py::reinterpret_borrow<py::dict>(h);
      for (auto kv : d) {
        const std::string k = py::str(kv.first);
        int i = 0;
        while (i < 6 && k != keys[i]) ++i;
        if (i == 6) throw std::invalid_argument("MultiScaleICP: unknown scale field " + k);
        v[i] = py::reinterpret_borrow<py::object>(kv.second);
      }
    } else {
      const py::sequence q = py::reinterpret_borrow<py::sequence>(h);
      if (q.size() > 6) throw std::invalid_argument("MultiScaleICP: a scale tuple has at most 6 entries");
      for (size_t i = 0; i < q.size(); ++i) v[i] = q[i];
    }
    for (int i = 0; i < 3; ++i)
      if (!v[i]) throw std::invalid_argument(std::string("MultiScaleICP: a scale needs ") + keys[i]);
    teaser::ICPScale sc(v[0].cast<double>(), v[1].cast<double>(), v[2].cast<int>());
    if (v[3]) sc.normal_search_radius = v[3].cast<double>();
    if (v[4]) sc.relative_fitness = v[4].cast<double>();
    if (v[5]) sc.relative_rmse = v[5].cast<double>();
    out.push_back(sc);
  }
  return out;
}

teaser::MultiScaleICP::Method method_of(const std::string& m) {
  if (m == "point_to_point") return teaser::MultiScaleICP::kPointToPoint;
  if (m == "point_to_plane") return teaser::MultiScaleICP::kPointToPlane;
  if (m == "generalized") return teaser::MultiScaleICP::kGeneralized;
  if (m == "colored") return teaser::MultiScaleICP::kColored;
  throw std::invalid_argument("MultiScaleICP: unknown method " + m);
}

py::dict multiscale_dict(const teaser::MultiScaleICP::Result& r) {
  py::list records, info;
  for (const auto& pr : r.records) {
    py::list row;
    for (const auto& x : pr) row.append(icp_dict(x));
    records.append(row);
  }
  for (const auto& M : r.information) info.append(square_to_numpy<6>(M));
  return py::dict(py::arg("records") = records, py::arg("n_down") = r.n_down, py::arg("status") = r.status,
                  py::arg("too_large") = r.too_large, py::arg("information") = info,
                  py::arg("info_counts") = r.info_counts);
}

py::dict multiscale_run(const teaser::MultiScaleICP& icp, const std::vector<CloudArray>& clouds,
                        const std::vector<std::pair<int, int>>& pairs,
                        const std::vector<teaser::RegistrationSolution>& init, const py::object& colors,
                        bool information) {
  std::vector<teaser::PointCloud> pcs;
  std::vector<teaser::ColorCloud> ccs;
  for (const auto& a : clouds) pcs.push_back(cloud_of(a));
  if (!colors.is_none())
    for (const auto& a : colors.cast<std::vector<CloudArray>>()) ccs.push_back(colors_of(a));
  teaser::MultiScaleICP::Result r;
  {
    py::gil_scoped_release release;
    r = icp.refineBatch(pcs, ccs, pairs, init, information);
  }
  return multiscale_dict(r);
}

}  // namespace

PYBIND11_MODULE(_teaserpp, m) {
  m.doc() = "Python binding for TEASER++ (GPU-native solve() path)";

  py::class_<teaser::RegistrationSolution>(m, "RegistrationSolution")
      .def(py::init([]() {  // identity (seeds for PointToPointICP.refine)
        teaser::RegistrationSolution s;
        s.rotation.setIdentity();
        s.translation.setZero();
        return s;
      }))
      .def_readwrite("valid", &teaser::RegistrationSolution::valid)
      .def_readwrite("scale", &teaser::RegistrationSolution::scale)
      .def_property(
          "translation", [](const teaser::RegistrationSolution& s) { return vec_to_numpy(s.translation); },
          [](teaser::RegistrationSolution& s, py::array_t<double> v) {
            for (int k = 0; k < 3; ++k) s.translation(k) = v.at(k);
          })
      .def_property(
          "rotation", [](const teaser::RegistrationSolution& s) { return to_numpy(s.rotation); },
          [](teaser::RegistrationSolution& s, ArrD v) { std::memcpy(s.rotation.data(), v.data(), 9 * sizeof(double)); })
      .def("__repr__", [](const teaser::RegistrationSolution& a) {
        std::ostringstream os;
        os << "<RegistrationSolution with scale=" << a.scale << "\ntranslation=\n";
        for (int k = 0; k < 3; ++k) os << a.translation(k) << "\n";
        os << "rotation=\n";
        for (int r = 0; r < 3; ++r) os << a.rotation(r, 0) << " " << a.rotation(r, 1) << " " << a.rotation(r, 2) << "\n";
        os << ">";
        return os.str();
      });

  // GPU extra: the refinement step of the reference's FPFH + TEASER++ + ICP tutorial (teaser::PointToPointICP)
  py::class_<teaser::PointToPointICP>(m, "PointToPointICP")
      .def(py::init([](double max_correspondence_distance, int max_iteration, double relative_fitness,
                       double relative_rmse) {
             teaser::PointToPointICP::Params p;
             p.max_correspondence_distance = max_correspondence_distance;
             p.max_iteration = max_iteration;
             p.relative_fitness = relative_fitness;
             p.relative_rmse = relative_rmse;
             return teaser::PointToPointICP(p);
           }),
           py::arg("max_correspondence_distance"), py::arg("max_iteration") = 30, py::arg("relative_fitness") = 1e-6,
           py::arg("relative_rmse") = 1e-6)
      .def("refine",
           [](const teaser::PointToPointICP& icp, const CloudArray& src, const CloudArray& dst,
              const teaser::RegistrationSolution& init) {
             const teaser::PointCloud s = cloud_of(src), d = cloud_of(dst);
             teaser::PointToPointICP::Result r;
             {
               py::gil_scoped_release release;
               r = icp.refine(s, d, init);
             }
             return icp_dict(r);
           },
           py::arg("src"), py::arg("dst"), py::arg("init"))
      .def("refine_batch",
           [](const teaser::PointToPointICP& icp, const std::vector<CloudArray>& src, const std::vector<CloudArray>& dst,
              const std::vector<teaser::RegistrationSolution>& init) {
             std::vector<teaser::PointCloud> s, d;
             for (const auto& a : src) s.push_back(cloud_of(a));
             for (const auto& a : dst) d.push_back(cloud_of(a));
             std::vector<teaser::PointToPointICP::Result> res;
             {
               py::gil_scoped_release release;
               res = icp.refineBatch(s, d, init);
             }
             py::list out;
             for (const auto& r : res) out.append(icp_dict(r));
             return out;
           },
           py::arg("src"), py::arg("dst"), py::arg("init"));

  // GPU extra: robust kernels for point-to-plane and generalized ICP (teaser::RobustKernel): RobustKernel("tukey", k)
  // or RobustKernel(RobustKernel.Type.TUKEY, k); L2 by default
  py::class_<teaser::RobustKernel> rk(m, "RobustKernel");
  py::enum_<teaser::RobustKernel::Type>(rk, "Type")
      .value("L2", teaser::RobustKernel::kL2)
      .value("L1", teaser::RobustKernel::kL1)
      .value("HUBER", teaser::RobustKernel::kHuber)
      .value("CAUCHY", teaser::RobustKernel::kCauchy)
      .value("GM", teaser::RobustKernel::kGM)
      .value("TUKEY", teaser::RobustKernel::kTukey);
  rk.def(py::init<>())
      .def(py::init<teaser::RobustKernel::Type, double>(), py::arg("type"), py::arg("k") = 1.0)
      .def(py::init([](const std::string& name, double k) {
             static const char* names[] = {"l2", "l1", "huber", "cauchy", "gm", "tukey"};
             for (int t = 0; t < 6; ++t)
               if (name == names[t]) return teaser::RobustKernel(static_cast<teaser::RobustKernel::Type>(t), k);
             throw std::invalid_argument("RobustKernel: unknown kernel \"" + name + "\"");
           }),
           py::arg("type"), py::arg("k") = 1.0)
      .def_readwrite("type", &teaser::RobustKernel::type)
      .def_readwrite("k", &teaser::RobustKernel::k);

  // GPU extra: multiway registration (teaser/pose_graph.h): information matrices and the GNC-TLS pose graph
  m.def(
      "information_matrix",
      [](const CloudArray& src, const CloudArray& dst, const teaser::RegistrationSolution& T,
         double max_correspondence_distance) {
        teaser::PointCloud s = cloud_of(src), d = cloud_of(dst);
        int count = 0;
        teaser::Matrix6d L;
        {
          py::gil_scoped_release release;
          L = teaser::informationMatrix(s, d, T, max_correspondence_distance, &count);
        }
        return py::make_tuple(square_to_numpy<6>(L), count);
      },
      py::arg("src"), py::arg("dst"), py::arg("transform"), py::arg("max_correspondence_distance"));
  m.def(
      "information_matrix_batch",
      [](const std::vector<CloudArray>& src, const std::vector<CloudArray>& dst,
         const std::vector<teaser::RegistrationSolution>& T, double max_correspondence_distance) {
        std::vector<teaser::PointCloud> s, d;
        for (const auto& a : src) s.push_back(cloud_of(a));
        for (const auto& a : dst) d.push_back(cloud_of(a));
        std::vector<int> counts;
        std::vector<teaser::Matrix6d> L;
        {
          py::gil_scoped_release release;
          L = teaser::informationMatrixBatch(s, d, T, max_correspondence_distance, &counts);
        }
        py::list out;
        for (const auto& M : L) out.append(square_to_numpy<6>(M));
        return py::make_tuple(out, counts);
      },
      py::arg("src"), py::arg("dst"), py::arg("transforms"), py::arg("max_correspondence_distance"));
  py::class_<teaser::PoseGraph>(m, "PoseGraph")
      .def(py::init([](double max_correspondence_distance, double gnc_factor, double cost_threshold,
                       int max_iterations, int max_inner_iterations, int reference_node) {
             teaser::PoseGraph::Params p;
             p.max_correspondence_distance = max_correspondence_distance;
             p.gnc_factor = gnc_factor;
             p.cost_threshold = cost_threshold;
             p.max_iterations = max_iterations;
             p.max_inner_iterations = max_inner_iterations;
             p.reference_node = reference_node;
             return teaser::PoseGraph(p);
           }),
           py::arg("max_correspondence_distance"), py::arg("gnc_factor") = 1.4, py::arg("cost_threshold") = 1e-6,
           py::arg("max_iterations") = 100, py::arg("max_inner_iterations") = 10, py::arg("reference_node") = 0)
      .def(
          "optimize",
          [](const teaser::PoseGraph& g, int num_nodes, const std::vector<std::pair<int, int>>& edges,
             const std::vector<SqArr>& transforms, const std::vector<SqArr>& information,
             const std::vector<bool>& uncertain, const py::object& initial_poses) {
            if (transforms.size() != edges.size() || information.size() != edges.size() ||
                (!uncertain.empty() && uncertain.size() != edges.size()))
              throw std::invalid_argument("one transform, information matrix (and uncertain flag) per edge");
            std::vector<teaser::PoseGraph::Edge> E(edges.size());
            for (size_t e = 0; e < edges.size(); ++e) {
              E[e].source = edges[e].first;
              E[e].target = edges[e].second;
              E[e].transform = square_of<4>(transforms[e]);
              E[e].information = square_of<6>(information[e]);
              E[e].uncertain = !uncertain.empty() && uncertain[e];
            }
            std::vector<Eigen::Matrix4d> init;
            if (!initial_poses.is_none())
              for (const auto& a : initial_poses.cast<std::vector<SqArr>>()) init.push_back(square_of<4>(a));
            teaser::PoseGraph::Result r;
            {
              py::gil_scoped_release release;
              r = g.optimize(num_nodes, E, initial_poses.is_none() ? nullptr : &init);
            }
            py::list poses;
            for (const auto& T : r.poses) poses.append(square_to_numpy<4>(T));
            return py::dict(py::arg("poses") = poses, py::arg("weights") = r.weights, py::arg("inliers") = r.inliers,
                            py::arg("residuals") = r.residuals, py::arg("iterations") = r.iterations,
                            py::arg("inner_iterations") = r.inner_iterations, py::arg("cost") = r.cost);
          },
          py::arg("num_nodes"), py::arg("edges"), py::arg("transforms"), py::arg("information"),
          py::arg("uncertain") = std::vector<bool>(), py::arg("initial_poses") = py::none());

  // GPU extra: point-to-plane ICP (teaser::PointToPlaneICP), given the target normals
  py::class_<teaser::PointToPlaneICP>(m, "PointToPlaneICP")
      .def(py::init([](double max_correspondence_distance, int max_iteration, double relative_fitness,
                       double relative_rmse, const teaser::RobustKernel& kernel) {
             teaser::PointToPlaneICP::Params p;
             p.max_correspondence_distance = max_correspondence_distance;
             p.max_iteration = max_iteration;
             p.relative_fitness = relative_fitness;
             p.relative_rmse = relative_rmse;
             return teaser::PointToPlaneICP(p, kernel);
           }),
           py::arg("max_correspondence_distance"), py::arg("max_iteration") = 30, py::arg("relative_fitness") = 1e-6,
           py::arg("relative_rmse") = 1e-6, py::arg("kernel") = teaser::RobustKernel())
      .def_property("kernel", &teaser::PointToPlaneICP::getKernel, &teaser::PointToPlaneICP::setKernel)
      .def("refine",
           [](const teaser::PointToPlaneICP& icp, const CloudArray& src, const CloudArray& dst,
              const CloudArray& dst_normals, const teaser::RegistrationSolution& init) {
             const teaser::PointCloud s = cloud_of(src), d = cloud_of(dst);
             const teaser::NormalCloud n = normals_of(dst_normals);
             teaser::PointToPlaneICP::Result r;
             {
               py::gil_scoped_release release;
               r = icp.refine(s, d, n, init);
             }
             return icp_dict(r);
           },
           py::arg("src"), py::arg("dst"), py::arg("dst_normals"), py::arg("init"))
      .def("refine_batch",
           [](const teaser::PointToPlaneICP& icp, const std::vector<CloudArray>& src, const std::vector<CloudArray>& dst,
              const std::vector<CloudArray>& dst_normals, const std::vector<teaser::RegistrationSolution>& init) {
             std::vector<teaser::PointCloud> s, d;
             std::vector<teaser::NormalCloud> n;
             for (const auto& a : src) s.push_back(cloud_of(a));
             for (const auto& a : dst) d.push_back(cloud_of(a));
             for (const auto& a : dst_normals) n.push_back(normals_of(a));
             std::vector<teaser::PointToPlaneICP::Result> res;
             {
               py::gil_scoped_release release;
               res = icp.refineBatch(s, d, n, init);
             }
             py::list out;
             for (const auto& r : res) out.append(icp_dict(r));
             return out;
           },
           py::arg("src"), py::arg("dst"), py::arg("dst_normals"), py::arg("init"));

  // GPU extra: generalized ICP (teaser::GeneralizedICP), given both clouds' normals
  py::class_<teaser::GeneralizedICP>(m, "GeneralizedICP")
      .def(py::init([](double max_correspondence_distance, int max_iteration, double relative_fitness,
                       double relative_rmse, double epsilon, const teaser::RobustKernel& kernel) {
             teaser::GeneralizedICP::Params p;
             p.max_correspondence_distance = max_correspondence_distance;
             p.max_iteration = max_iteration;
             p.relative_fitness = relative_fitness;
             p.relative_rmse = relative_rmse;
             p.epsilon = epsilon;
             return teaser::GeneralizedICP(p, kernel);
           }),
           py::arg("max_correspondence_distance"), py::arg("max_iteration") = 30, py::arg("relative_fitness") = 1e-6,
           py::arg("relative_rmse") = 1e-6, py::arg("epsilon") = 1e-3, py::arg("kernel") = teaser::RobustKernel())
      .def_property("kernel", &teaser::GeneralizedICP::getKernel, &teaser::GeneralizedICP::setKernel)
      .def("refine",
           [](const teaser::GeneralizedICP& icp, const CloudArray& src, const CloudArray& dst,
              const CloudArray& src_normals, const CloudArray& dst_normals, const teaser::RegistrationSolution& init) {
             const teaser::PointCloud s = cloud_of(src), d = cloud_of(dst);
             const teaser::NormalCloud sn = normals_of(src_normals), dn = normals_of(dst_normals);
             teaser::GeneralizedICP::Result r;
             {
               py::gil_scoped_release release;
               r = icp.refine(s, d, sn, dn, init);
             }
             return icp_dict(r);
           },
           py::arg("src"), py::arg("dst"), py::arg("src_normals"), py::arg("dst_normals"), py::arg("init"))
      .def("refine_batch",
           [](const teaser::GeneralizedICP& icp, const std::vector<CloudArray>& src, const std::vector<CloudArray>& dst,
              const std::vector<CloudArray>& src_normals, const std::vector<CloudArray>& dst_normals,
              const std::vector<teaser::RegistrationSolution>& init) {
             std::vector<teaser::PointCloud> s, d;
             std::vector<teaser::NormalCloud> sn, dn;
             for (const auto& a : src) s.push_back(cloud_of(a));
             for (const auto& a : dst) d.push_back(cloud_of(a));
             for (const auto& a : src_normals) sn.push_back(normals_of(a));
             for (const auto& a : dst_normals) dn.push_back(normals_of(a));
             std::vector<teaser::GeneralizedICP::Result> res;
             {
               py::gil_scoped_release release;
               res = icp.refineBatch(s, d, sn, dn, init);
             }
             py::list out;
             for (const auto& r : res) out.append(icp_dict(r));
             return out;
           },
           py::arg("src"), py::arg("dst"), py::arg("src_normals"), py::arg("dst_normals"), py::arg("init"));

  // GPU extra: coloured ICP (teaser::ColoredICP), given the target normals and both clouds' (n,3) colours
  py::class_<teaser::ColoredICP>(m, "ColoredICP")
      .def(py::init([](double max_correspondence_distance, int max_iteration, double relative_fitness,
                       double relative_rmse, double lambda_geometric, const teaser::RobustKernel& kernel) {
             teaser::ColoredICP::Params p;
             p.max_correspondence_distance = max_correspondence_distance;
             p.max_iteration = max_iteration;
             p.relative_fitness = relative_fitness;
             p.relative_rmse = relative_rmse;
             p.lambda_geometric = lambda_geometric;
             return teaser::ColoredICP(p, kernel);
           }),
           py::arg("max_correspondence_distance"), py::arg("max_iteration") = 30, py::arg("relative_fitness") = 1e-6,
           py::arg("relative_rmse") = 1e-6, py::arg("lambda_geometric") = 0.968,
           py::arg("kernel") = teaser::RobustKernel())
      .def_property("kernel", &teaser::ColoredICP::getKernel, &teaser::ColoredICP::setKernel)
      .def("refine",
           [](const teaser::ColoredICP& icp, const CloudArray& src, const CloudArray& dst, const CloudArray& dst_normals,
              const CloudArray& src_colors, const CloudArray& dst_colors, const teaser::RegistrationSolution& init) {
             const teaser::PointCloud s = cloud_of(src), d = cloud_of(dst);
             const teaser::NormalCloud n = normals_of(dst_normals);
             const teaser::ColorCloud sc = colors_of(src_colors), dc = colors_of(dst_colors);
             teaser::ColoredICP::Result r;
             {
               py::gil_scoped_release release;
               r = icp.refine(s, d, n, sc, dc, init);
             }
             return icp_dict(r);
           },
           py::arg("src"), py::arg("dst"), py::arg("dst_normals"), py::arg("src_colors"), py::arg("dst_colors"),
           py::arg("init"))
      .def("refine_batch",
           [](const teaser::ColoredICP& icp, const std::vector<CloudArray>& src, const std::vector<CloudArray>& dst,
              const std::vector<CloudArray>& dst_normals, const std::vector<CloudArray>& src_colors,
              const std::vector<CloudArray>& dst_colors, const std::vector<teaser::RegistrationSolution>& init) {
             std::vector<teaser::PointCloud> s, d;
             std::vector<teaser::NormalCloud> n;
             std::vector<teaser::ColorCloud> sc, dc;
             for (const auto& a : src) s.push_back(cloud_of(a));
             for (const auto& a : dst) d.push_back(cloud_of(a));
             for (const auto& a : dst_normals) n.push_back(normals_of(a));
             for (const auto& a : src_colors) sc.push_back(colors_of(a));
             for (const auto& a : dst_colors) dc.push_back(colors_of(a));
             std::vector<teaser::ColoredICP::Result> res;
             {
               py::gil_scoped_release release;
               res = icp.refineBatch(s, d, n, sc, dc, init);
             }
             py::list out;
             for (const auto& r : res) out.append(icp_dict(r));
             return out;
           },
           py::arg("src"), py::arg("dst"), py::arg("dst_normals"), py::arg("src_colors"), py::arg("dst_colors"),
           py::arg("init"));

  // GPU extra: multi-scale ICP (teaser::MultiScaleICP) over a cloud table; refine_batch returns a dict: records
  // (per pair, per scale, icp dicts without correspondences), n_down and status (per cloud, per scale), too_large, and
  // with information the last scale's information matrices and counts
  py::class_<teaser::MultiScaleICP>(m, "MultiScaleICP")
      .def(py::init([](const py::list& scales, const std::string& method, double lambda_geometric, double epsilon,
                       const teaser::RobustKernel& kernel) {
             teaser::MultiScaleICP::Params p;
             p.scales = scales_of(scales);
             p.method = method_of(method);
             p.lambda_geometric = lambda_geometric;
             p.epsilon = epsilon;
             p.kernel = kernel;
             return teaser::MultiScaleICP(p);
           }),
           py::arg("scales"), py::arg("method") = "point_to_plane", py::arg("lambda_geometric") = 0.968,
           py::arg("epsilon") = 1e-3, py::arg("kernel") = teaser::RobustKernel())
      .def("refine_batch", &multiscale_run, py::arg("clouds"), py::arg("pairs"), py::arg("init"),
           py::arg("colors") = py::none(), py::arg("information") = false);
  m.def(
      "multiscale_icp",
      [](const std::vector<CloudArray>& clouds, const std::vector<std::pair<int, int>>& pairs, const py::list& scales,
         const std::vector<teaser::RegistrationSolution>& init, const std::string& method, const py::object& colors,
         double lambda_geometric, double epsilon, const teaser::RobustKernel& kernel, bool information) {
        teaser::MultiScaleICP::Params p;
        p.scales = scales_of(scales);
        p.method = method_of(method);
        p.lambda_geometric = lambda_geometric;
        p.epsilon = epsilon;
        p.kernel = kernel;
        return multiscale_run(teaser::MultiScaleICP(p), clouds, pairs, init, colors, information);
      },
      py::arg("clouds"), py::arg("pairs"), py::arg("scales"), py::arg("init"), py::arg("method") = "point_to_plane",
      py::arg("colors") = py::none(), py::arg("lambda_geometric") = 0.968, py::arg("epsilon") = 1e-3,
      py::arg("kernel") = teaser::RobustKernel(), py::arg("information") = false);

  // GPU extra: coloured ICP's colour gradients (teaser::estimateColorGradients), as (n,3) float64
  m.def("estimate_color_gradients",
        [](const CloudArray& points, const CloudArray& normals, const CloudArray& colors, double radius) {
          const teaser::PointCloud pc = cloud_of(points);
          const teaser::NormalCloud nc = normals_of(normals);
          const teaser::ColorCloud cc = colors_of(colors);
          std::vector<std::array<double, 3>> g;
          {
            py::gil_scoped_release release;
            g = teaser::estimateColorGradients(pc, nc, cc, radius);
          }
          return gradients_to_numpy(g);
        },
        py::arg("points"), py::arg("normals"), py::arg("colors"), py::arg("radius"));
  m.def("estimate_color_gradients_batch",
        [](const std::vector<CloudArray>& points, const std::vector<CloudArray>& normals,
           const std::vector<CloudArray>& colors, double radius) {
          std::vector<teaser::PointCloud> pcs;
          std::vector<teaser::NormalCloud> ncs;
          std::vector<teaser::ColorCloud> ccs;
          for (const auto& a : points) pcs.push_back(cloud_of(a));
          for (const auto& a : normals) ncs.push_back(normals_of(a));
          for (const auto& a : colors) ccs.push_back(colors_of(a));
          std::vector<std::vector<std::array<double, 3>>> res;
          {
            py::gil_scoped_release release;
            res = teaser::estimateColorGradientsBatch(pcs, ncs, ccs, radius);
          }
          py::list out;
          for (const auto& g : res) out.append(gradients_to_numpy(g));
          return out;
        },
        py::arg("points"), py::arg("normals"), py::arg("colors"), py::arg("radius"));

  // GPU extra: FPFHEstimation's normals alone (teaser::estimateNormals), as (n,4) float32 (nx, ny, nz, curvature)
  m.def("estimate_normals",
        [](const CloudArray& points, double normal_search_radius) {
          const teaser::PointCloud pc = cloud_of(points);
          teaser::NormalCloud out;
          {
            py::gil_scoped_release release;
            out = teaser::estimateNormals(pc, normal_search_radius);
          }
          return normals_to_numpy(out);
        },
        py::arg("points"), py::arg("normal_search_radius") = 0.03);
  m.def("estimate_normals_batch",
        [](const std::vector<CloudArray>& points, double normal_search_radius) {
          std::vector<teaser::PointCloud> pcs;
          for (const auto& a : points) pcs.push_back(cloud_of(a));
          std::vector<teaser::NormalCloud> res;
          {
            py::gil_scoped_release release;
            res = teaser::estimateNormalsBatch(pcs, normal_search_radius);
          }
          py::list out;
          for (const auto& nc : res) out.append(normals_to_numpy(nc));
          return out;
        },
        py::arg("points"), py::arg("normal_search_radius") = 0.03);

  // GPU extra: the first step of the same tutorial, Open3D's voxel_down_sample (teaser::voxelDownSample); with colors
  // ((n,3)) it returns (points, colour means)
  m.def("voxel_down_sample",
        [](const CloudArray& points, double voxel_size, const py::object& colors) -> py::object {
          const teaser::PointCloud pc = cloud_of(points);
          if (colors.is_none()) {
            teaser::PointCloud out;
            {
              py::gil_scoped_release release;
              out = teaser::voxelDownSample(pc, voxel_size);
            }
            return cloud_to_numpy(out);
          }
          const teaser::ColorCloud cc = colors_of(colors.cast<CloudArray>());
          teaser::PointCloud out;
          teaser::ColorCloud cout;
          {
            py::gil_scoped_release release;
            out = teaser::voxelDownSample(pc, cc, voxel_size, &cout);
          }
          return py::make_tuple(cloud_to_numpy(out), colors_to_numpy(cout));
        },
        py::arg("points"), py::arg("voxel_size"), py::arg("colors") = py::none());
  m.def("voxel_down_sample_batch",
        [](const std::vector<CloudArray>& points, double voxel_size, const py::object& colors) -> py::object {
          std::vector<teaser::PointCloud> pcs;
          for (const auto& a : points) pcs.push_back(cloud_of(a));
          std::vector<teaser::PointCloud> res;
          std::vector<teaser::ColorCloud> cres;
          if (colors.is_none()) {
            py::gil_scoped_release release;
            res = teaser::voxelDownSampleBatch(pcs, voxel_size);
          } else {
            std::vector<teaser::ColorCloud> ccs;
            for (const auto& a : colors.cast<std::vector<CloudArray>>()) ccs.push_back(colors_of(a));
            py::gil_scoped_release release;
            res = teaser::voxelDownSampleBatch(pcs, ccs, voxel_size, &cres);
          }
          py::list out;
          for (const auto& pc : res) out.append(cloud_to_numpy(pc));
          if (colors.is_none()) return out;
          py::list cout;
          for (const auto& cc : cres) cout.append(colors_to_numpy(cc));
          return py::make_tuple(out, cout);
        },
        py::arg("points"), py::arg("voxel_size"), py::arg("colors") = py::none());

  m.attr("OMP_MAX_THREADS") = 0;  // the GPU path ignores max_clique_num_threads

  py::enum_<Solver::ROTATION_ESTIMATION_ALGORITHM>(m, "RotationEstimationAlgorithm")
      .value("GNC_TLS", Solver::ROTATION_ESTIMATION_ALGORITHM::GNC_TLS)
      .value("FGR", Solver::ROTATION_ESTIMATION_ALGORITHM::FGR)
      .value("QUATRO", Solver::ROTATION_ESTIMATION_ALGORITHM::QUATRO);
  py::enum_<Solver::INLIER_GRAPH_FORMULATION>(m, "InlierGraphFormulation")
      .value("CHAIN", Solver::INLIER_GRAPH_FORMULATION::CHAIN)
      .value("COMPLETE", Solver::INLIER_GRAPH_FORMULATION::COMPLETE);
  py::enum_<Solver::INLIER_SELECTION_MODE>(m, "InlierSelectionMode")
      .value("PMC_EXACT", Solver::INLIER_SELECTION_MODE::PMC_EXACT)
      .value("PMC_HEU", Solver::INLIER_SELECTION_MODE::PMC_HEU)
      .value("KCORE_HEU", Solver::INLIER_SELECTION_MODE::KCORE_HEU)
      .value("NONE", Solver::INLIER_SELECTION_MODE::NONE);

  py::class_<Solver> solver(m, "RobustRegistrationSolver", py::dynamic_attr());

  solver.def(py::init<const Solver::Params&>())
      .def(py::init<double, double, bool, Solver::ROTATION_ESTIMATION_ALGORITHM, double, size_t, double,
                    Solver::INLIER_GRAPH_FORMULATION, Solver::INLIER_SELECTION_MODE, double, bool, bool, double, int>(),
           py::arg("noise_bound") = 0.01, py::arg("cbar2") = 1, py::arg("estimate_scaling") = true,
           py::arg("rotation_estimation_algorithm") = Solver::ROTATION_ESTIMATION_ALGORITHM::GNC_TLS,
           py::arg("rotation_gnc_factor") = 1.4, py::arg("rotation_max_iterations") = 100,
           py::arg("rotation_cost_threshold") = 1e-6,
           py::arg("rotation_tim_graph") = Solver::INLIER_GRAPH_FORMULATION::CHAIN,
           py::arg("inlier_selection_mode") = Solver::INLIER_SELECTION_MODE::PMC_EXACT,
           py::arg("kcore_heuristic_threshold") = 0.5, py::arg("use_max_clique") = true,
           py::arg("max_clique_exact_solution") = true, py::arg("max_clique_time_limit") = 3600,
           py::arg("max_clique_num_threads") = 0)
      .def("getParams", &Solver::getParams)
      .def("reset", py::overload_cast<const Solver::Params&>(&Solver::reset))
      .def("solve", [](Solver& s, const ArrD& src, const ArrD& dst) {
             teaser::Mat3X a = to_mat3x(src), b = to_mat3x(dst);
             py::gil_scoped_release release;  // the reference holds the GIL; nothing here touches Python
             return s.solve(a, b);
           })
      .def("solve_batch",
           [](Solver& s, const std::vector<ArrD>& src, const std::vector<ArrD>& dst, const std::vector<int>& devices) {
             // GPU extra: many independent problems in one call, sharded over the GPUs of the node inside the library
             std::vector<teaser::Mat3X> a, b;
             for (const auto& x : src) a.push_back(to_mat3x(x));
             for (const auto& x : dst) b.push_back(to_mat3x(x));
             std::vector<std::vector<int>> cliques;
             std::vector<teaser::RegistrationSolution> sols;
             {
               py::gil_scoped_release release;
               sols = s.solveBatch(a, b, &cliques, devices);
             }
             return py::make_tuple(sols, cliques);
           },
           py::arg("src"), py::arg("dst"), py::arg("devices") = std::vector<int>{})
      .def("solve_and_certify_batch",
           [](Solver& s, const std::vector<ArrD>& src, const std::vector<ArrD>& dst,
              const teaser::DRSCertifier::Params& cert_params) {
             // GPU extra: one batched solve and one batched certification of its retained results, one device
             std::vector<teaser::Mat3X> a, b;
             for (const auto& x : src) a.push_back(to_mat3x(x));
             for (const auto& x : dst) b.push_back(to_mat3x(x));
             std::vector<Solver::SolveCertifyResult> res;
             {
               py::gil_scoped_release release;
               res = s.solveAndCertifyBatch(a, b, cert_params);
             }
             py::list out;
             for (const auto& r : res)
               out.append(py::dict(py::arg("solution") = r.solution, py::arg("max_clique") = r.max_clique,
                                   py::arg("rotation_inliers_mask") = row_to_numpy(r.rotation_inliers_mask),
                                   py::arg("translation_inliers_mask") = row_to_numpy(r.translation_inliers_mask),
                                   py::arg("certified") = r.certified, py::arg("certification") = r.certification));
             return out;
           },
           py::arg("src"), py::arg("dst"), py::arg("cert_params"))
      .def("solve_cloud_pairs",
           [](Solver& s, const std::vector<py::array_t<float, py::array::c_style | py::array::forcecast>>& clouds,
              const std::vector<std::pair<int, int>>& pairs, double normal_search_radius, double fpfh_search_radius,
              bool use_absolute_scale, bool use_crosscheck, bool use_tuple_test, float tuple_scale,
              uint64_t tuple_seed) {
             // GPU extra: FPFH, matching and the solve of many cloud pairs in one device call (solveCloudPairs)
             std::vector<teaser::PointCloud> pcs(clouds.size());
             for (size_t c = 0; c < clouds.size(); ++c) {
               const auto& a = clouds[c];
               if (a.ndim() != 2 || a.shape(1) != 3) throw std::invalid_argument("clouds must be (n,3) arrays");
               const float* d = a.data();
               pcs[c].reserve(static_cast<size_t>(a.shape(0)));
               for (py::ssize_t i = 0; i < a.shape(0); ++i) pcs[c].push_back({d[3 * i], d[3 * i + 1], d[3 * i + 2]});
             }
             Solver::CloudPairParams cp;
             cp.normal_search_radius = normal_search_radius;
             cp.fpfh_search_radius = fpfh_search_radius;
             cp.use_absolute_scale = use_absolute_scale;
             cp.use_crosscheck = use_crosscheck;
             cp.use_tuple_test = use_tuple_test;
             cp.tuple_scale = tuple_scale;
             cp.tuple_seed = tuple_seed;
             std::vector<Solver::CloudPairResult> res;
             {
               py::gil_scoped_release release;
               res = s.solveCloudPairs(pcs, pairs, cp);
             }
             py::list out;
             for (const auto& r : res)
               out.append(py::dict(py::arg("status") = r.status, py::arg("correspondences") = r.correspondences,
                                   py::arg("solution") = r.solution, py::arg("max_clique") = r.max_clique,
                                   py::arg("global_scale") = r.global_scale));
             return out;
           },
           py::arg("clouds"), py::arg("pairs"), py::arg("normal_search_radius") = 0.03,
           py::arg("fpfh_search_radius") = 0.05, py::arg("use_absolute_scale") = true, py::arg("use_crosscheck") = true,
           py::arg("use_tuple_test") = true, py::arg("tuple_scale") = 0.0f, py::arg("tuple_seed") = 0x7ea5e2ull)
      .def("solve_cloud_pairs_icp",
           [](Solver& s, const std::vector<CloudArray>& clouds, const std::vector<std::pair<int, int>>& pairs,
              double max_correspondence_distance, int max_iteration, double relative_fitness, double relative_rmse,
              double normal_search_radius, double fpfh_search_radius, bool use_absolute_scale, bool use_crosscheck,
              bool use_tuple_test, float tuple_scale, uint64_t tuple_seed, const std::string& method, double epsilon,
              const py::object& kernel, const py::object& colors, double lambda_geometric) {
             // GPU extra: solve_cloud_pairs, then point-to-point (point-to-plane, generalized, coloured) ICP of every
             // pair with a valid solution, in one call
             if (method != "point_to_point" && method != "point_to_plane" && method != "generalized" &&
                 method != "colored")
               throw std::invalid_argument(
                   "method must be \"point_to_point\", \"point_to_plane\", \"generalized\" or \"colored\"");
             // colours: one (n,3) array per cloud, for method="colored" and no other
             if (colors.is_none() != (method != "colored"))
               throw std::invalid_argument("colors are required by method=\"colored\" and by no other method");
             // a robust kernel (point-to-plane and generalized only; None keeps the unweighted entries)
             if (!kernel.is_none() && method == "point_to_point")
               throw std::invalid_argument("point-to-point ICP takes no robust kernel");
             const bool robust = !kernel.is_none();
             const teaser::RobustKernel rk = robust ? kernel.cast<teaser::RobustKernel>() : teaser::RobustKernel();
             std::vector<teaser::PointCloud> pcs;
             for (const auto& a : clouds) pcs.push_back(cloud_of(a));
             std::vector<teaser::ColorCloud> ccs;
             if (!colors.is_none())
               for (const auto& a : colors.cast<std::vector<CloudArray>>()) ccs.push_back(colors_of(a));
             Solver::CloudPairParams cp;
             cp.normal_search_radius = normal_search_radius;
             cp.fpfh_search_radius = fpfh_search_radius;
             cp.use_absolute_scale = use_absolute_scale;
             cp.use_crosscheck = use_crosscheck;
             cp.use_tuple_test = use_tuple_test;
             cp.tuple_scale = tuple_scale;
             cp.tuple_seed = tuple_seed;
             teaser::GeneralizedICP::Params ip;
             ip.max_correspondence_distance = max_correspondence_distance;
             ip.max_iteration = max_iteration;
             ip.relative_fitness = relative_fitness;
             ip.relative_rmse = relative_rmse;
             ip.epsilon = epsilon;
             std::vector<Solver::CloudPairICPResult> res;
             {
               py::gil_scoped_release release;
               if (method == "colored") {
                 teaser::ColoredICPParams cip;
                 static_cast<teaser::PointToPointICPParams&>(cip) = ip;
                 cip.lambda_geometric = lambda_geometric;
                 res = s.solveCloudPairsColoredICP(pcs, ccs, pairs, cp, cip, rk);
               } else if (robust)
                 res = method == "generalized" ? s.solveCloudPairsGeneralizedICP(pcs, pairs, cp, ip, rk)
                                               : s.solveCloudPairsPointToPlane(pcs, pairs, cp, ip, rk);
               else
                 res = method == "generalized"      ? s.solveCloudPairsGeneralizedICP(pcs, pairs, cp, ip)
                       : method == "point_to_plane" ? s.solveCloudPairsPointToPlane(pcs, pairs, cp, ip)
                                                    : s.solveCloudPairs(pcs, pairs, cp, ip);
             }
             py::list out;
             for (const auto& r : res)
               out.append(py::dict(py::arg("status") = r.status, py::arg("correspondences") = r.correspondences,
                                   py::arg("solution") = r.solution, py::arg("max_clique") = r.max_clique,
                                   py::arg("global_scale") = r.global_scale, py::arg("refined") = r.refined,
                                   py::arg("icp") = r.refined ? py::object(icp_dict(r.icp)) : py::object(py::none())));
             return out;
           },
           py::arg("clouds"), py::arg("pairs"), py::arg("max_correspondence_distance"), py::arg("max_iteration") = 30,
           py::arg("relative_fitness") = 1e-6, py::arg("relative_rmse") = 1e-6, py::arg("normal_search_radius") = 0.03,
           py::arg("fpfh_search_radius") = 0.05, py::arg("use_absolute_scale") = true, py::arg("use_crosscheck") = true,
           py::arg("use_tuple_test") = true, py::arg("tuple_scale") = 0.0f, py::arg("tuple_seed") = 0x7ea5e2ull,
           py::arg("method") = "point_to_point", py::arg("epsilon") = 1e-3, py::arg("kernel") = py::none(),
           py::arg("colors") = py::none(), py::arg("lambda_geometric") = 0.968)
      .def(
          "solve_multiway",
          [](Solver& s, const std::vector<CloudArray>& clouds, const std::vector<std::pair<int, int>>& pairs,
             double max_correspondence_distance, const py::object& uncertain, int max_iteration,
             double relative_fitness, double relative_rmse, double normal_search_radius, double fpfh_search_radius,
             bool use_absolute_scale, bool use_crosscheck, bool use_tuple_test, float tuple_scale,
             uint64_t tuple_seed, double gnc_factor, double cost_threshold, int max_iterations,
             int max_inner_iterations, int reference_node, const py::object& colors, double lambda_geometric,
             const py::object& kernel) {
            // GPU extra: solve_cloud_pairs_icp(method="point_to_plane"), information matrices and the GNC-TLS pose
            // graph in one call (solveMultiway); uncertain None: pair (k, k + 1) certain, every other pair uncertain.
            // colors (one (n,3) array per cloud): method="colored" instead, with lambda_geometric and kernel (None: L2)
            if (!kernel.is_none() && colors.is_none())
              throw std::invalid_argument("a robust kernel needs colors (coloured ICP)");
            const teaser::RobustKernel rk = kernel.is_none() ? teaser::RobustKernel() : kernel.cast<teaser::RobustKernel>();
            std::vector<teaser::PointCloud> pcs;
            for (const auto& a : clouds) pcs.push_back(cloud_of(a));
            std::vector<teaser::ColorCloud> ccs;
            if (!colors.is_none())
              for (const auto& a : colors.cast<std::vector<CloudArray>>()) ccs.push_back(colors_of(a));
            Solver::CloudPairParams cp;
            cp.normal_search_radius = normal_search_radius;
            cp.fpfh_search_radius = fpfh_search_radius;
            cp.use_absolute_scale = use_absolute_scale;
            cp.use_crosscheck = use_crosscheck;
            cp.use_tuple_test = use_tuple_test;
            cp.tuple_scale = tuple_scale;
            cp.tuple_seed = tuple_seed;
            teaser::PointToPointICPParams ip;
            ip.max_correspondence_distance = max_correspondence_distance;
            ip.max_iteration = max_iteration;
            ip.relative_fitness = relative_fitness;
            ip.relative_rmse = relative_rmse;
            teaser::PoseGraphParams pg;
            pg.max_correspondence_distance = max_correspondence_distance;
            pg.gnc_factor = gnc_factor;
            pg.cost_threshold = cost_threshold;
            pg.max_iterations = max_iterations;
            pg.max_inner_iterations = max_inner_iterations;
            pg.reference_node = reference_node;
            const bool given = !uncertain.is_none();
            const std::vector<bool> unc = given ? uncertain.cast<std::vector<bool>>() : std::vector<bool>();
            Solver::MultiwayResult r;
            {
              py::gil_scoped_release release;
              if (!colors.is_none()) {
                teaser::ColoredICPParams cip;
                static_cast<teaser::PointToPointICPParams&>(cip) = ip;
                cip.lambda_geometric = lambda_geometric;
                r = given ? s.solveMultiway(pcs, ccs, pairs, cp, cip, pg, unc, rk)
                          : s.solveMultiway(pcs, ccs, pairs, cp, cip, pg, rk);
              } else {
                r = given ? s.solveMultiway(pcs, pairs, cp, ip, pg, unc) : s.solveMultiway(pcs, pairs, cp, ip, pg);
              }
            }
            py::list pair_out, info, poses;
            for (const auto& q : r.pairs)
              pair_out.append(py::dict(py::arg("status") = q.status, py::arg("solution") = q.solution,
                                       py::arg("refined") = q.refined,
                                       py::arg("icp") = q.refined ? py::object(icp_dict(q.icp)) : py::object(py::none())));
            for (const auto& M : r.information) info.append(square_to_numpy<6>(M));
            for (const auto& T : r.poses) poses.append(square_to_numpy<4>(T));
            return py::dict(py::arg("pairs") = pair_out, py::arg("information") = info,
                            py::arg("information_counts") = r.information_counts,
                            py::arg("edge_weights") = r.edge_weights, py::arg("edge_inliers") = r.edge_inliers,
                            py::arg("poses") = poses, py::arg("pose_graph_status") = r.pose_graph_status,
                            py::arg("iterations") = r.iterations, py::arg("inner_iterations") = r.inner_iterations,
                            py::arg("cost") = r.cost);
          },
          py::arg("clouds"), py::arg("pairs"), py::arg("max_correspondence_distance"), py::arg("uncertain") = py::none(),
          py::arg("max_iteration") = 30, py::arg("relative_fitness") = 1e-6, py::arg("relative_rmse") = 1e-6,
          py::arg("normal_search_radius") = 0.03, py::arg("fpfh_search_radius") = 0.05,
          py::arg("use_absolute_scale") = true, py::arg("use_crosscheck") = true, py::arg("use_tuple_test") = true,
          py::arg("tuple_scale") = 0.0f, py::arg("tuple_seed") = 0x7ea5e2ull, py::arg("gnc_factor") = 1.4,
          py::arg("cost_threshold") = 1e-6, py::arg("max_iterations") = 100, py::arg("max_inner_iterations") = 10,
          py::arg("reference_node") = 0, py::arg("colors") = py::none(), py::arg("lambda_geometric") = 0.968,
          py::arg("kernel") = py::none())
      .def_property_readonly("solution", &Solver::getSolution)
      .def("getSolution", &Solver::getSolution)
      .def_property_readonly("gnc_rotation_cost_at_termination", &Solver::getGNCRotationCostAtTermination)
      .def("getGNCRotationCostAtTermination", &Solver::getGNCRotationCostAtTermination)
      .def_property_readonly("scale_inliers_mask", [](Solver& s) { return row_to_numpy(s.getScaleInliersMask()); })
      .def("getScaleInliersMask", [](Solver& s) { return row_to_numpy(s.getScaleInliersMask()); })
      .def_property_readonly("scale_inliers_map", [](Solver& s) { return to_numpy(s.getScaleInliersMap()); })
      .def("getScaleInliersMap", [](Solver& s) { return to_numpy(s.getScaleInliersMap()); })
      .def_property_readonly("scale_inliers", &Solver::getScaleInliers)
      .def("getScaleInliers", &Solver::getScaleInliers)
      .def_property_readonly("rotation_inliers_mask", [](Solver& s) { return row_to_numpy(s.getRotationInliersMask()); })
      .def("getRotationInliersMask", [](Solver& s) { return row_to_numpy(s.getRotationInliersMask()); })
      .def("getRotationInliersMap", [](Solver& s) { return irow_to_numpy(s.getRotationInliersMap()); })
      .def_property_readonly("rotation_inliers", &Solver::getRotationInliers)
      .def("getRotationInliers", &Solver::getRotationInliers)
      .def_property_readonly("translation_inliers_mask",
                             [](Solver& s) { return row_to_numpy(s.getTranslationInliersMask()); })
      .def("getTranslationInliersMask", [](Solver& s) { return row_to_numpy(s.getTranslationInliersMask()); })
      .def_property_readonly("translation_inliers_map",
                             [](Solver& s) { return irow_to_numpy(s.getTranslationInliersMap()); })
      .def("getTranslationInliersMap", [](Solver& s) { return irow_to_numpy(s.getTranslationInliersMap()); })
      .def_property_readonly("translation_inliers", &Solver::getTranslationInliers)
      .def("getTranslationInliers", &Solver::getTranslationInliers)
      .def("getInputOrderedTranslationInliers", &Solver::getInputOrderedTranslationInliers)
      .def_property_readonly("inlier_max_clique", &Solver::getInlierMaxClique)
      .def("getInlierMaxClique", &Solver::getInlierMaxClique)
      .def_property_readonly("inlier_graph", &Solver::getInlierGraph)
      .def("getInlierGraph", &Solver::getInlierGraph)
      .def_property_readonly("src_tims_map", [](Solver& s) { return to_numpy(s.getSrcTIMsMap()); })
      .def("getSrcTIMsMap", [](Solver& s) { return to_numpy(s.getSrcTIMsMap()); })
      .def_property_readonly("dst_tims_map", [](Solver& s) { return to_numpy(s.getDstTIMsMap()); })
      .def("getDstTIMsMap", [](Solver& s) { return to_numpy(s.getDstTIMsMap()); })
      .def_property_readonly("src_tims_map_for_rotation", [](Solver& s) { return to_numpy(s.getSrcTIMsMapForRotation()); })
      .def("getSrcTIMsMapForRotation", [](Solver& s) { return to_numpy(s.getSrcTIMsMapForRotation()); })
      .def_property_readonly("dst_tims_map_for_rotation", [](Solver& s) { return to_numpy(s.getDstTIMsMapForRotation()); })
      .def("getDstTIMsMapForRotation", [](Solver& s) { return to_numpy(s.getDstTIMsMapForRotation()); })
      .def_property_readonly("max_clique_src_tims", [](Solver& s) { return to_numpy(s.getMaxCliqueSrcTIMs()); })
      .def("getMaxCliqueSrcTIMs", [](Solver& s) { return to_numpy(s.getMaxCliqueSrcTIMs()); })
      .def_property_readonly("max_clique_dst_tims", [](Solver& s) { return to_numpy(s.getMaxCliqueDstTIMs()); })
      .def("getMaxCliqueDstTIMs", [](Solver& s) { return to_numpy(s.getMaxCliqueDstTIMs()); })
      .def_property_readonly("src_tims", [](Solver& s) { return to_numpy(s.getSrcTIMs()); })
      .def("getSrcTIMs", [](Solver& s) { return to_numpy(s.getSrcTIMs()); })
      .def_property_readonly("dst_tims", [](Solver& s) { return to_numpy(s.getDstTIMs()); })
      .def("getDstTIMs", [](Solver& s) { return to_numpy(s.getDstTIMs()); })
      // GPU extras
      .def("isMaxCliqueProvenOptimal", &Solver::isMaxCliqueProvenOptimal)
      .def("getNumInlierGraphEdges", &Solver::getNumInlierGraphEdges)
      .def("getGNCRotationIterations", &Solver::getGNCRotationIterations);

  py::class_<Solver::Params>(solver, "Params")
      .def(py::init<>())
      .def_readwrite("noise_bound", &Solver::Params::noise_bound)
      .def_readwrite("cbar2", &Solver::Params::cbar2)
      .def_readwrite("estimate_scaling", &Solver::Params::estimate_scaling)
      .def_readwrite("rotation_estimation_algorithm", &Solver::Params::rotation_estimation_algorithm)
      .def_readwrite("rotation_gnc_factor", &Solver::Params::rotation_gnc_factor)
      .def_readwrite("rotation_max_iterations", &Solver::Params::rotation_max_iterations)
      .def_readwrite("rotation_tim_graph", &Solver::Params::rotation_tim_graph)
      .def_readwrite("inlier_selection_mode", &Solver::Params::inlier_selection_mode)
      .def_readwrite("kcore_heuristic_threshold", &Solver::Params::kcore_heuristic_threshold)
      .def_readwrite("rotation_cost_threshold", &Solver::Params::rotation_cost_threshold)
      .def_readwrite("use_max_clique", &Solver::Params::use_max_clique)
      .def_readwrite("max_clique_exact_solution", &Solver::Params::max_clique_exact_solution)
      .def_readwrite("max_clique_time_limit", &Solver::Params::max_clique_time_limit)
      .def_readwrite("max_clique_num_threads", &Solver::Params::max_clique_num_threads)
      .def("__repr__", [](const Solver::Params& a) {
        std::ostringstream os;
        const char* rot[] = {"GNC_TLS", "FGR", "QUATRO"};
        const char* sel[] = {"PMC_EXACT", "PMC_HEU", "KCORE_HEU", "NONE"};
        os << "<Params with noise_bound=" << a.noise_bound << "\ncbar2=" << a.cbar2
           << "\nestimate_scaling=" << a.estimate_scaling
           << "\nrotation_estimation_algorithm=" << rot[static_cast<int>(a.rotation_estimation_algorithm)]
           << "\nrotation_gnc_factor=" << a.rotation_gnc_factor
           << "\nrotation_max_iterations=" << a.rotation_max_iterations
           << "\nrotation_cost_threshold=" << a.rotation_cost_threshold
           << "\ninlier_selection_mode=" << sel[static_cast<int>(a.inlier_selection_mode)]
           << "\nkcore_heuristic_threshold=" << a.kcore_heuristic_threshold
           << "\nmax_clique_time_limit=" << a.max_clique_time_limit << "\n>";
        return os.str();
      });

  // ---- certifier (reference teaserpp_python.cc:71-74, 249-291)
  using Cert = teaser::DRSCertifier;
  py::enum_<Cert::EIG_SOLVER_TYPE>(m, "EigSolverType")
      .value("EIGEN", Cert::EIG_SOLVER_TYPE::EIGEN)
      .value("SPECTRA", Cert::EIG_SOLVER_TYPE::SPECTRA);

  py::class_<teaser::CertificationResult>(m, "CertificationResult")
      .def_readwrite("is_optimal", &teaser::CertificationResult::is_optimal)
      .def_readwrite("best_suboptimality", &teaser::CertificationResult::best_suboptimality)
      .def_readwrite("suboptimality_traj", &teaser::CertificationResult::suboptimality_traj)
      .def("__repr__", [](const teaser::CertificationResult& a) {
        std::ostringstream os;
        os << "<CertificationResult \n"
           << "Is optimal:" << a.is_optimal << "\n"
           << "Best suboptimality:" << a.best_suboptimality << "\n"
           << "Iterations: " << a.suboptimality_traj.size() << "\n"
           << ">";
        return os.str();
      });

  py::class_<Cert> certifier(m, "DRSCertifier");
  auto to_r3 = [](const ArrD& R) {
    if (R.ndim() != 2 || R.shape(0) != 3 || R.shape(1) != 3) throw std::invalid_argument("expected a (3, 3) rotation");
    Eigen::Matrix3d m3;
    std::memcpy(m3.data(), R.data(), sizeof(double) * 9);
    return m3;
  };
  certifier.def(py::init<const Cert::Params>())
      // one entry point for both reference overloads (bool mask / +-1 doubles): dispatching on the dtype here keeps
      // pybind11's implicit array conversions from sending a float theta to the bool overload
      .def("certify", [to_r3](Cert& c, const ArrD& R, const ArrD& src, const ArrD& dst, const py::array& theta) {
        if (theta.dtype().kind() == 'b') {
          auto tb = py::array_t<bool, py::array::c_style | py::array::forcecast>::ensure(theta);
          Eigen::Matrix<bool, 1, Eigen::Dynamic> th(1, tb.size());
          for (py::ssize_t i = 0; i < tb.size(); ++i) th(i) = tb.data()[i];
          return c.certify(to_r3(R), to_mat3x(src), to_mat3x(dst), th);
        }
        auto td = py::array_t<double, py::array::c_style | py::array::forcecast>::ensure(theta);
        if (!td) throw std::invalid_argument("theta must be a bool or float array");
        Eigen::Matrix<double, 1, Eigen::Dynamic> th(1, td.size());
        std::memcpy(th.data(), td.data(), sizeof(double) * static_cast<size_t>(td.size()));
        return c.certify(to_r3(R), to_mat3x(src), to_mat3x(dst), th);
      })
      // lists of rotations, (3,N) arrays and thetas; all-bool thetas take the bool overload, otherwise every theta is
      // taken as +-1 doubles (a bool one mapped true -> 1, false -> -1)
      .def("certify_batch", [to_r3](Cert& c, const std::vector<ArrD>& Rs, const std::vector<ArrD>& srcs,
                                    const std::vector<ArrD>& dsts, const std::vector<py::array>& thetas) {
        std::vector<Eigen::Matrix3d> R;
        std::vector<teaser::Mat3X> s, d;
        for (const auto& x : Rs) R.push_back(to_r3(x));
        for (const auto& x : srcs) s.push_back(to_mat3x(x));
        for (const auto& x : dsts) d.push_back(to_mat3x(x));
        bool all_bool = !thetas.empty();
        for (const auto& t : thetas) all_bool = all_bool && t.dtype().kind() == 'b';
        if (all_bool) {
          std::vector<Eigen::Matrix<bool, 1, Eigen::Dynamic>> th;
          for (const auto& t : thetas) {
            auto tb = py::array_t<bool, py::array::c_style | py::array::forcecast>::ensure(t);
            Eigen::Matrix<bool, 1, Eigen::Dynamic> m(1, tb.size());
            for (py::ssize_t i = 0; i < tb.size(); ++i) m(i) = tb.data()[i];
            th.push_back(m);
          }
          py::gil_scoped_release release;
          return c.certifyBatch(R, s, d, th);
        }
        std::vector<Eigen::Matrix<double, 1, Eigen::Dynamic>> th;
        for (const auto& t : thetas) {
          auto td = py::array_t<double, py::array::c_style | py::array::forcecast>::ensure(t);
          if (!td) throw std::invalid_argument("theta must be a bool or float array");
          Eigen::Matrix<double, 1, Eigen::Dynamic> m(1, td.size());
          for (py::ssize_t i = 0; i < td.size(); ++i)
            m(i) = t.dtype().kind() == 'b' ? (td.data()[i] != 0 ? 1.0 : -1.0) : td.data()[i];
          th.push_back(m);
        }
        py::gil_scoped_release release;
        return c.certifyBatch(R, s, d, th);
      });

  py::class_<Cert::Params>(certifier, "Params")
      .def(py::init<>())
      .def_readwrite("noise_bound", &Cert::Params::noise_bound)
      .def_readwrite("cbar2", &Cert::Params::cbar2)
      .def_readwrite("sub_optimality", &Cert::Params::sub_optimality)
      .def_readwrite("max_iterations", &Cert::Params::max_iterations)
      .def_readwrite("gamma_tau", &Cert::Params::gamma_tau)
      .def_readwrite("eig_decomposition_solver", &Cert::Params::eig_decomposition_solver);
}
