// pybind11 module `teaserpp_python._teaserpp` for the GPU path.  Same module / class / method / property names
// as the reference binding (python/teaserpp_python/teaserpp_python.cc:25-291) so existing Python callers keep
// working; arrays cross the boundary as numpy (3,N) float64 exactly like the reference's pybind11/eigen.h casters
// (copied if not Fortran-contiguous).  Fixes of the reference's copy-paste slips (SURVEY Q4): the dst_* properties
// return the dst getters, Params exposes max_clique_num_threads, the ctor default time limit is 3600.
// The certifier classes (EigSolverType, CertificationResult, DRSCertifier + Params, :71-74,249-291) are bound too.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <sstream>

#include "teaser/certification.h"
#include "teaser/registration.h"

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

}  // namespace

PYBIND11_MODULE(_teaserpp, m) {
  m.doc() = "Python binding for TEASER++ (GPU-native solve() path)";

  py::class_<teaser::RegistrationSolution>(m, "RegistrationSolution")
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
