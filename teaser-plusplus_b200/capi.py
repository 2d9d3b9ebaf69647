"""ctypes binding of the C-ABI product library (csrc/libteaser_b200.so, include/teaser_b200.h).

There is no CPU fallback: every entry point raises if the library is missing or no CUDA device is
usable.  Points are (N,3) float64 C-contiguous numpy arrays (== the reference's column-major 3xN).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC_DIR = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(CSRC_DIR, "libteaser_b200.so")


class TzrError(RuntimeError):
    pass


class Params(C.Structure):
    """tzr_params == teaser::RobustRegistrationSolver::Params (registration.h:419-514)."""
    _fields_ = [
        ("noise_bound", C.c_double),
        ("cbar2", C.c_double),
        ("estimate_scaling", C.c_int32),
        ("rotation_estimation_algorithm", C.c_int32),
        ("rotation_gnc_factor", C.c_double),
        ("rotation_max_iterations", C.c_uint64),
        ("rotation_cost_threshold", C.c_double),
        ("rotation_tim_graph", C.c_int32),
        ("inlier_selection_mode", C.c_int32),
        ("kcore_heuristic_threshold", C.c_double),
        ("use_max_clique", C.c_int32),
        ("max_clique_exact_solution", C.c_int32),
        ("max_clique_time_limit", C.c_double),
        ("max_clique_num_threads", C.c_int32),
        ("reserved", C.c_int32),
    ]


class Solution(C.Structure):
    """tzr_solution == teaser::RegistrationSolution (registration.h:32-39) + diagnostics."""
    _fields_ = [
        ("valid", C.c_int32),
        ("clique_size", C.c_int32),
        ("scale", C.c_double),
        ("translation", C.c_double * 3),
        ("rotation", C.c_double * 9),
        ("clique_proven_optimal", C.c_int32),
        ("gnc_iterations", C.c_int32),
        ("gnc_cost", C.c_double),
        ("n_rotation_inliers", C.c_int32),
        ("n_translation_inliers", C.c_int32),
        ("n_edges", C.c_int64),
        ("stage_ms", C.c_double * 8),
    ]

    @property
    def R(self):
        return np.array(self.rotation[:]).reshape(3, 3).T.copy()

    @property
    def t(self):
        return np.array(self.translation[:])


SOLUTION_DTYPE = np.dtype([
    ("valid", np.int32), ("clique_size", np.int32), ("scale", np.float64), ("translation", np.float64, (3,)),
    ("rotation", np.float64, (9,)), ("clique_proven_optimal", np.int32), ("gnc_iterations", np.int32),
    ("gnc_cost", np.float64), ("n_rotation_inliers", np.int32), ("n_translation_inliers", np.int32),
    ("n_edges", np.int64), ("stage_ms", np.float64, (8,))], align=True)
assert SOLUTION_DTYPE.itemsize == C.sizeof(Solution), (SOLUTION_DTYPE.itemsize, C.sizeof(Solution))

_lib = None

class CertifierParams(C.Structure):
    """tzr_certifier_params == DRSCertifier::Params (certification.h:70-108)."""
    _fields_ = [("noise_bound", C.c_double), ("cbar2", C.c_double), ("sub_optimality", C.c_double),
                ("max_iterations", C.c_double), ("gamma_tau", C.c_double), ("eig_decomposition_solver", C.c_int32),
                ("reserved", C.c_int32)]


class CertificationResult(C.Structure):
    _fields_ = [("is_optimal", C.c_int32), ("n_iterations", C.c_int32), ("best_suboptimality", C.c_double)]


class FrontendParams(C.Structure):
    """tzr_frontend_params: FPFHEstimation::computeFPFHFeatures' radii and Matcher::calculateCorrespondences' flags."""
    _fields_ = [("normal_search_radius", C.c_double), ("fpfh_search_radius", C.c_double),
                ("use_absolute_scale", C.c_int32), ("use_crosscheck", C.c_int32), ("use_tuple_test", C.c_int32),
                ("tuple_scale", C.c_float)]


class IcpParams(C.Structure):
    """tzr_icp_params: Open3D's registration_icp distance and ICPConvergenceCriteria."""
    _fields_ = [("max_correspondence_distance", C.c_double), ("relative_fitness", C.c_double),
                ("relative_rmse", C.c_double), ("max_iteration", C.c_int32), ("reserved", C.c_int32)]


class Similarity(C.Structure):
    """tzr_similarity: scale, column-major rotation, translation."""
    _fields_ = [("scale", C.c_double), ("rotation", C.c_double * 9), ("translation", C.c_double * 3)]


class IcpResult(C.Structure):
    """tzr_icp_result."""
    _fields_ = [("transform", Similarity), ("fitness", C.c_double), ("inlier_rmse", C.c_double),
                ("iterations", C.c_int32), ("n_correspondences", C.c_int32), ("converged", C.c_int32),
                ("reserved", C.c_int32)]


SIMILARITY_DTYPE = np.dtype([("scale", np.float64), ("rotation", np.float64, (9,)), ("translation", np.float64, (3,))],
                            align=True)
ICP_RESULT_DTYPE = np.dtype([
    ("transform", SIMILARITY_DTYPE), ("fitness", np.float64), ("inlier_rmse", np.float64), ("iterations", np.int32),
    ("n_correspondences", np.int32), ("converged", np.int32), ("reserved", np.int32)], align=True)


class IcpScale(C.Structure):
    """tzr_icp_scale: one scale of tzr_icp_multiscale_batch's schedule."""
    _fields_ = [("voxel_size", C.c_double), ("max_correspondence_distance", C.c_double),
                ("normal_search_radius", C.c_double), ("relative_fitness", C.c_double), ("relative_rmse", C.c_double),
                ("max_iteration", C.c_int32), ("reserved", C.c_int32)]


# tzr_icp_multiscale_batch's methods (TZR_ICP_*), by the names Context.icp_multiscale accepts
ICP_METHODS = {"point_to_point": 0, "point_to_plane": 1, "generalized": 2, "colored": 3}
# the fields of a scale in the order a tuple gives them, and the defaults of the optional ones
ICP_SCALE_FIELDS = ("voxel_size", "max_correspondence_distance", "max_iteration", "normal_search_radius",
                    "relative_fitness", "relative_rmse")


def icp_scale(scale) -> IcpScale:
    """A tzr_icp_scale from an IcpScale (as given), a dict or a tuple in ICP_SCALE_FIELDS order.  voxel_size,
    max_correspondence_distance and max_iteration are required; normal_search_radius defaults to 2 voxel_size (Open3D's
    tutorials) and the criteria to 1e-6.  The library checks the values."""
    if isinstance(scale, IcpScale):
        return scale
    if isinstance(scale, dict):
        unknown = set(scale) - set(ICP_SCALE_FIELDS)
        if unknown:
            raise TzrError(f"icp_scale: unknown field(s) {sorted(unknown)} (fields: {ICP_SCALE_FIELDS})")
        d = dict(scale)
    else:
        t = tuple(scale)
        if len(t) > len(ICP_SCALE_FIELDS):
            raise TzrError(f"icp_scale: a tuple has at most {len(ICP_SCALE_FIELDS)} entries {ICP_SCALE_FIELDS}")
        d = dict(zip(ICP_SCALE_FIELDS, t))
    missing = [k for k in ICP_SCALE_FIELDS[:3] if k not in d]
    if missing:
        raise TzrError(f"icp_scale: {missing} required")
    v = float(d["voxel_size"])
    return IcpScale(v, float(d["max_correspondence_distance"]), float(d.get("normal_search_radius", 2.0 * v)),
                    float(d.get("relative_fitness", 1e-6)), float(d.get("relative_rmse", 1e-6)),
                    int(d["max_iteration"]), 0)


class RobustKernel(C.Structure):
    """tzr_robust_kernel: type (LOSS_*) and k (finite and > 0 for HUBER, CAUCHY, GM and TUKEY)."""
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("k", C.c_double)]


class FgrParams(C.Structure):
    """tzr_fgr_params: Fast Global Registration's options (Open3D's FastGlobalRegistrationOption)."""
    _fields_ = [("division_factor", C.c_double), ("use_absolute_scale", C.c_int32), ("decrease_mu", C.c_int32),
                ("maximum_correspondence_distance", C.c_double), ("iteration_number", C.c_int32),
                ("reserved", C.c_int32)]


class RansacParams(C.Structure):
    """tzr_ransac_params: correspondence RANSAC's options (Open3D's ransac_n, RANSACConvergenceCriteria and its three
    correspondence checkers, each with an enable flag)."""
    _fields_ = [("max_correspondence_distance", C.c_double), ("ransac_n", C.c_int32), ("max_iteration", C.c_int32),
                ("confidence", C.c_double), ("check_edge_length", C.c_int32), ("check_distance", C.c_int32),
                ("edge_length_similarity", C.c_double), ("distance_threshold", C.c_double),
                ("check_normal", C.c_int32), ("reserved", C.c_int32), ("normal_angle_threshold", C.c_double)]


class RansacInfo(C.Structure):
    """tzr_ransac_info: one problem's loop summary."""
    _fields_ = [("drawn", C.c_int32), ("passed", C.c_int32), ("winner", C.c_int32), ("inliers", C.c_int32),
                ("usable", C.c_int32), ("reserved", C.c_int32), ("rmse", C.c_double)]


RANSAC_INFO_DTYPE = np.dtype([("drawn", np.int32), ("passed", np.int32), ("winner", np.int32), ("inliers", np.int32),
                              ("usable", np.int32), ("reserved", np.int32), ("rmse", np.float64)])


class PoseGraphParams(C.Structure):
    """tzr_pose_graph_params: the GNC-TLS pose graph's distance c, schedule and reference node."""
    _fields_ = [("max_correspondence_distance", C.c_double), ("gnc_factor", C.c_double),
                ("cost_threshold", C.c_double), ("max_iterations", C.c_int32), ("max_inner_iterations", C.c_int32),
                ("reference_node", C.c_int32), ("reserved", C.c_int32)]


class PoseGraphSummary(C.Structure):
    """tzr_pose_graph_summary."""
    _fields_ = [("iterations", C.c_int32), ("inner_iterations", C.c_int32), ("cost", C.c_double)]


class LineProcessParams(C.Structure):
    """tzr_line_process_params: Open3D's GlobalOptimizationOption and ConvergenceCriteria for the line process."""
    _fields_ = [("max_correspondence_distance", C.c_double), ("edge_prune_threshold", C.c_double),
                ("preference_loop_closure", C.c_double), ("min_relative_increment", C.c_double),
                ("min_relative_residual_increment", C.c_double), ("min_right_term", C.c_double),
                ("min_residual", C.c_double), ("upper_scale_factor", C.c_double), ("lower_scale_factor", C.c_double),
                ("reference_node", C.c_int32), ("max_iteration", C.c_int32), ("max_iteration_lm", C.c_int32),
                ("reserved", C.c_int32)]


class LineProcessSummary(C.Structure):
    """tzr_line_process_summary: per pass (iterations, trials, stop reason, mu), the pruned count and the final F."""
    _fields_ = [("iterations", C.c_int32 * 2), ("trials", C.c_int32 * 2), ("stop_reason", C.c_int32 * 2),
                ("pruned", C.c_int32), ("reserved", C.c_int32), ("residual", C.c_double), ("mu", C.c_double * 2)]


# TZR_LP_STOP_*: the rule that stopped a line-process pass
LP_STOP = {1: "right_term", 2: "relative_increment", 3: "relative_residual", 4: "lm_trials", 5: "min_residual",
           6: "max_iteration"}

# robust kernel types (TZR_LOSS_*), by the names robust_kernel() accepts
LOSS_TYPES = {"l2": 0, "l1": 1, "huber": 2, "cauchy": 3, "gm": 4, "tukey": 5}
assert C.sizeof(IcpParams) == 32, C.sizeof(IcpParams)
assert C.sizeof(PoseGraphParams) == 40 and PoseGraphParams.reference_node.offset == 32, C.sizeof(PoseGraphParams)
assert C.sizeof(PoseGraphSummary) == 16 and PoseGraphSummary.cost.offset == 8, C.sizeof(PoseGraphSummary)
assert C.sizeof(LineProcessParams) == 88 and LineProcessParams.reference_node.offset == 72, C.sizeof(LineProcessParams)
assert C.sizeof(LineProcessSummary) == 56 and LineProcessSummary.residual.offset == 32, C.sizeof(LineProcessSummary)
assert C.sizeof(IcpScale) == 48 and IcpScale.max_iteration.offset == 40, C.sizeof(IcpScale)
assert C.sizeof(FgrParams) == 32 and FgrParams.maximum_correspondence_distance.offset == 16, C.sizeof(FgrParams)
assert C.sizeof(RansacParams) == 64 and RansacParams.normal_angle_threshold.offset == 56, C.sizeof(RansacParams)
assert RANSAC_INFO_DTYPE.itemsize == C.sizeof(RansacInfo) == 32, C.sizeof(RansacInfo)
assert C.sizeof(RobustKernel) == 16 and RobustKernel.k.offset == 8, C.sizeof(RobustKernel)
assert SIMILARITY_DTYPE.itemsize == C.sizeof(Similarity) == 104, C.sizeof(Similarity)
assert ICP_RESULT_DTYPE.itemsize == C.sizeof(IcpResult) == 136, (ICP_RESULT_DTYPE.itemsize, C.sizeof(IcpResult))


_SYMBOLS = [
    "tzr_abi_version", "tzr_status_string", "tzr_last_error", "tzr_params_default", "tzr_ctx_create",
    "tzr_ctx_destroy", "tzr_ctx_set_stream", "tzr_ctx_synchronize", "tzr_ctx_kernel_launches", "tzr_words_per_row",
    "tzr_graph_build", "tzr_max_clique", "tzr_max_clique_batch", "tzr_gnc_tls_rotation", "tzr_rotation_solve", "tzr_tls_translation", "tzr_scalar_tls",
    "tzr_solve", "tzr_solve_batch", "tzr_solve_batch_dev", "tzr_solve_batch_ragged_dev", "tzr_last_graph", "tzr_last_filter_consts", "tzr_last_stage_ms",
    "tzr_ctx_set_flags", "tzr_ctx_filter_mismatches", "tzr_ctx_filter_rechecks", "tzr_ctx_debug_counters",
    "tzr_match_correspondences", "tzr_feature_nn", "tzr_compute_fpfh", "tzr_certifier_params_default", "tzr_certify",
    "tzr_certifier_initial_matrix", "tzr_certifier_dual_projection", "tzr_last_graph_info", "tzr_ctx_stage_log",
    "tzr_ctx_stage_log_read", "tzr_solve_batch_multi", "tzr_ctx_clique_info", "tzr_compute_fpfh_batch",
    "tzr_match_correspondences_batch", "tzr_ctx_set_max_n", "tzr_ctx_clique_route", "tzr_certify_batch",
    "tzr_certifier_psd_projection", "tzr_certifier_batch_psd_projection", "tzr_certifier_batch_dual_projection",
    "tzr_fpfh_pair_features", "tzr_fpfh_smallest_eigenpair", "tzr_last_inliers", "tzr_certify_last_solve",
    "tzr_frontend_params_default", "tzr_register_cloud_pairs", "tzr_icp_params_default", "tzr_icp", "tzr_icp_batch",
    "tzr_register_cloud_pairs_icp", "tzr_voxel_downsample", "tzr_voxel_downsample_batch", "tzr_estimate_normals",
    "tzr_estimate_normals_batch", "tzr_icp_point_to_plane", "tzr_icp_point_to_plane_batch",
    "tzr_register_cloud_pairs_icp_point_to_plane", "tzr_icp_generalized", "tzr_icp_generalized_batch",
    "tzr_register_cloud_pairs_icp_generalized", "tzr_icp_point_to_plane_robust_batch", "tzr_icp_generalized_robust_batch",
    "tzr_register_cloud_pairs_icp_robust", "tzr_ctx_last_strip_blocks", "tzr_graph_strip_schedule",
    "tzr_ctx_set_scale_chunk", "tzr_ctx_last_scale_chunks",
    "tzr_information_matrix", "tzr_information_matrix_batch", "tzr_pose_graph_params_default", "tzr_pose_graph_optimize",
    "tzr_pose_graph_optimize_batch",
    "tzr_register_cloud_pairs_multiway", "tzr_estimate_color_gradients", "tzr_estimate_color_gradients_batch",
    "tzr_icp_colored", "tzr_icp_colored_batch", "tzr_voxel_downsample_colors", "tzr_voxel_downsample_colors_batch",
    "tzr_register_cloud_pairs_icp_colored", "tzr_register_cloud_pairs_multiway_colored", "tzr_icp_multiscale_batch",
    "tzr_fgr_params_default", "tzr_fgr", "tzr_fgr_batch", "tzr_register_cloud_pairs_fgr",
    "tzr_ransac_params_default", "tzr_ransac", "tzr_ransac_batch", "tzr_register_cloud_pairs_ransac",
    "tzr_line_process_params_default", "tzr_pose_graph_optimize_line_process",
    "tzr_pose_graph_optimize_line_process_batch", "tzr_dense_cholesky_batch",
    "tzr_register_cloud_pairs_multiway_line_process",
    "tzr_register_cloud_pairs_multiway_batch", "tzr_register_cloud_pairs_multiway_line_process_batch",
]

# status codes (tzr_status)
TZR_OK = 0
TZR_ERR_INVALID_ARG = -1
TZR_ERR_TOO_LARGE = -6

# debug flag bits 28-31 of tzr_ctx_set_flags: the default graph kernel's strip length (0: chosen from the batch)
FLAG_STRIP_SHIFT = 28


def strip_flags(L: int) -> int:
    """The debug flag bits that force strips of L = 1 ... 15 blocks in the default graph kernel (0: its own choice)."""
    if not 0 <= L <= 15:
        raise ValueError(f"strip length {L} outside 0 ... 15")
    return L << FLAG_STRIP_SHIFT


def strip_schedule(nt: int, L: int):
    """tzr_graph_strip_schedule: (I, J0) int32 arrays of the default graph kernel's strips over nt row blocks, strips of
    L blocks, in the device's order (host only)."""
    count = lib().tzr_graph_strip_schedule(nt, L, None, None)
    if count < 0:
        raise TzrError(f"tzr_graph_strip_schedule({nt}, {L}): {lib().tzr_status_string(count).decode()}")
    I, J0 = np.zeros(count, dtype=np.int32), np.zeros(count, dtype=np.int32)
    lib().tzr_graph_strip_schedule(nt, L, _p(I, C.c_int32), _p(J0, C.c_int32))
    return I, J0


# debug flags of tzr_ctx_set_flags that choose tzr_compute_fpfh(_batch)'s radius search for every cloud
FLAG_FPFH_BRUTE_FORCE = 4194304
FLAG_FPFH_GRID = 8388608
# ... and tzr_icp(_batch)'s nearest-neighbour search for every target
FLAG_ICP_BRUTE_FORCE = 33554432
FLAG_ICP_GRID = 67108864


def build(verbose: bool = False):
    """Compile csrc/*.cu for sm_90a with nvcc (cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC_DIR] + ([] if verbose else ["-s"])
    subprocess.check_call(cmd)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TzrError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    dp, u8p, i32p, i64p, u64p = (C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_int32),
                                 C.POINTER(C.c_int64), C.POINTER(C.c_uint64))
    vp = C.c_void_p
    L.tzr_abi_version.restype = C.c_int
    L.tzr_status_string.restype = C.c_char_p
    L.tzr_status_string.argtypes = [C.c_int]
    L.tzr_last_error.restype = C.c_char_p
    L.tzr_last_error.argtypes = [vp]
    L.tzr_params_default.argtypes = [C.POINTER(Params)]
    L.tzr_params_default.restype = None
    L.tzr_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.tzr_ctx_destroy.argtypes = [vp]
    L.tzr_ctx_set_stream.argtypes = [vp, vp]
    L.tzr_ctx_synchronize.argtypes = [vp]
    L.tzr_ctx_kernel_launches.argtypes = [vp]
    L.tzr_ctx_kernel_launches.restype = C.c_int64
    L.tzr_words_per_row.argtypes = [C.c_int]
    L.tzr_graph_build.argtypes = [vp, dp, dp, C.c_int, C.c_double, u64p, i32p, i64p]
    L.tzr_max_clique.argtypes = [vp, u64p, C.c_int, C.c_int, C.c_double, C.c_double, i32p, i32p, i32p]
    L.tzr_max_clique_batch.argtypes = [vp, C.c_int, C.c_int, u64p, C.c_int, C.c_double, C.c_double, i32p, i32p, i32p,
                                       i32p]
    L.tzr_gnc_tls_rotation.argtypes = [vp, dp, dp, C.c_int, C.c_double, C.c_double, C.c_uint64, C.c_double, dp, u8p,
                                       dp, i32p]
    L.tzr_rotation_solve.argtypes = [vp, C.c_int, dp, dp, C.c_int, C.c_double, C.c_double, C.c_uint64, C.c_double, dp,
                                     u8p, dp, i32p]
    L.tzr_tls_translation.argtypes = [vp, dp, dp, C.c_int, C.c_double, C.c_double, dp, u8p]
    L.tzr_scalar_tls.argtypes = [vp, dp, dp, C.c_int64, dp, u8p]
    L.tzr_solve.argtypes = [vp, C.POINTER(Params), dp, dp, C.c_int, C.POINTER(Solution), i32p, u8p, u8p]
    L.tzr_solve_batch.argtypes = [vp, C.POINTER(Params), C.c_int, i32p, C.POINTER(dp), C.POINTER(dp),
                                  C.POINTER(Solution), i32p, C.c_int]
    L.tzr_solve_batch_dev.argtypes = [vp, C.POINTER(Params), C.c_int, C.c_int, vp, vp, vp, vp]
    L.tzr_solve_batch_ragged_dev.argtypes = [vp, C.POINTER(Params), C.c_int, i32p, vp, vp, vp, vp]
    L.tzr_last_graph.argtypes = [vp, C.c_int, u64p, i32p]
    L.tzr_last_filter_consts.argtypes = [vp, C.c_int, dp, C.POINTER(C.c_float), i32p]
    L.tzr_last_stage_ms.argtypes = [vp, dp, dp, dp, dp]
    L.tzr_last_graph_info.argtypes = [vp, i32p, i32p, i32p, u64p]
    L.tzr_ctx_stage_log.argtypes = [vp, C.c_int]
    L.tzr_ctx_stage_log_read.argtypes = [vp, dp, i32p]
    L.tzr_solve_batch_multi.argtypes = [i32p, C.c_int, C.POINTER(Params), C.c_int, i32p, C.POINTER(dp), C.POINTER(dp),
                                        C.POINTER(Solution), i32p, C.c_int]
    L.tzr_ctx_set_flags.argtypes = [vp, C.c_uint32]
    L.tzr_ctx_filter_mismatches.argtypes = [vp]
    L.tzr_ctx_filter_mismatches.restype = C.c_int64
    L.tzr_ctx_filter_rechecks.argtypes = [vp]
    L.tzr_ctx_filter_rechecks.restype = C.c_int64
    L.tzr_ctx_debug_counters.argtypes = [vp, i64p]
    L.tzr_ctx_last_strip_blocks.argtypes = [vp]
    L.tzr_ctx_set_scale_chunk.argtypes = [vp, C.c_longlong]
    L.tzr_ctx_last_scale_chunks.argtypes = [vp]
    L.tzr_graph_strip_schedule.argtypes = [C.c_int, C.c_int, i32p, i32p]
    L.tzr_ctx_clique_info.argtypes = [vp, i32p, i32p]
    L.tzr_ctx_set_max_n.argtypes = [vp, C.c_int]
    L.tzr_ctx_clique_route.argtypes = [vp, i32p]
    fp = C.POINTER(C.c_float)
    L.tzr_match_correspondences.argtypes = [vp, fp, C.c_int, fp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_float, C.c_uint64, i32p, C.c_int64, i64p, fp]
    L.tzr_feature_nn.argtypes = [vp, fp, C.c_int, fp, C.c_int, C.c_int, i32p, fp]
    L.tzr_compute_fpfh.argtypes = [vp, fp, C.c_int, C.c_double, C.c_double, fp, fp]
    fpp = C.POINTER(fp)
    L.tzr_compute_fpfh_batch.argtypes = [vp, C.c_int, i32p, fpp, C.c_double, C.c_double, fpp, fpp, i32p]
    L.tzr_fpfh_pair_features.argtypes = [vp, C.c_int, fp, fp, fp, fp, fp, i32p]
    L.tzr_fpfh_smallest_eigenpair.argtypes = [vp, C.c_int, fp, fp, fp]
    L.tzr_match_correspondences_batch.argtypes = [vp, C.c_int, i32p, fpp, i32p, fpp, fpp, fpp, C.c_int, C.c_int,
                                                  C.c_int, C.c_int, C.c_float, u64p, C.POINTER(i32p), i64p, i64p, fp]
    L.tzr_certifier_params_default.argtypes = [C.POINTER(CertifierParams)]
    L.tzr_certifier_params_default.restype = None
    L.tzr_certify.argtypes = [vp, C.POINTER(CertifierParams), dp, dp, dp, dp, C.c_int, C.POINTER(CertificationResult),
                              dp, C.c_int]
    L.tzr_certify_batch.argtypes = [vp, C.POINTER(CertifierParams), C.c_int, i32p, dp, C.POINTER(dp), C.POINTER(dp),
                                    C.POINTER(dp), C.POINTER(CertificationResult), C.POINTER(dp), i32p]
    L.tzr_certifier_initial_matrix.argtypes = [vp, C.POINTER(CertifierParams), dp, dp, dp, dp, C.c_int, dp, dp]
    L.tzr_certifier_dual_projection.argtypes = [vp, dp, dp, C.c_int, dp]
    L.tzr_certifier_psd_projection.argtypes = [vp, dp, C.c_int, dp, dp]
    L.tzr_certifier_batch_psd_projection.argtypes = [vp, C.c_int, i32p, C.POINTER(dp), C.POINTER(dp)]
    L.tzr_certifier_batch_dual_projection.argtypes = [vp, C.c_int, i32p, C.POINTER(dp), C.POINTER(dp), C.POINTER(dp)]
    L.tzr_last_inliers.argtypes = [vp, C.c_int, u8p, u8p, i64p, i32p]
    L.tzr_certify_last_solve.argtypes = [vp, C.POINTER(CertifierParams), C.c_int, i32p, C.POINTER(CertificationResult),
                                         i32p, C.POINTER(dp), i32p]
    L.tzr_frontend_params_default.argtypes = [C.POINTER(FrontendParams)]
    L.tzr_frontend_params_default.restype = None
    L.tzr_register_cloud_pairs.argtypes = [vp, C.POINTER(FrontendParams), C.POINTER(Params), C.c_int, i32p, fpp,
                                           C.c_int, i32p, u64p, C.POINTER(Solution), i32p, i32p, i64p,
                                           C.POINTER(i32p), C.POINTER(i32p), fp]
    L.tzr_icp_params_default.argtypes = [C.POINTER(IcpParams)]
    L.tzr_icp_params_default.restype = None
    L.tzr_icp.argtypes = [vp, C.POINTER(IcpParams), fp, C.c_int, fp, C.c_int, C.POINTER(Similarity),
                          C.POINTER(IcpResult), i32p]
    L.tzr_icp_batch.argtypes = [vp, C.POINTER(IcpParams), C.c_int, i32p, fpp, i32p, fpp, C.POINTER(Similarity),
                                C.POINTER(IcpResult), C.POINTER(i32p)]
    L.tzr_register_cloud_pairs_icp.argtypes = L.tzr_register_cloud_pairs.argtypes + [C.POINTER(IcpParams),
                                                                                    C.POINTER(IcpResult)]
    L.tzr_estimate_normals.argtypes = [vp, fp, C.c_int, C.c_double, fp]
    L.tzr_estimate_normals_batch.argtypes = [vp, C.c_int, i32p, fpp, C.c_double, fpp, i32p]
    L.tzr_icp_point_to_plane.argtypes = [vp, C.POINTER(IcpParams), fp, C.c_int, fp, C.c_int, fp, C.POINTER(Similarity),
                                         C.POINTER(IcpResult), i32p]
    L.tzr_icp_point_to_plane_batch.argtypes = [vp, C.POINTER(IcpParams), C.c_int, i32p, fpp, i32p, fpp, fpp,
                                               C.POINTER(Similarity), C.POINTER(IcpResult), C.POINTER(i32p)]
    L.tzr_register_cloud_pairs_icp_point_to_plane.argtypes = L.tzr_register_cloud_pairs_icp.argtypes
    L.tzr_icp_generalized.argtypes = [vp, C.POINTER(IcpParams), C.c_double, fp, C.c_int, fp, fp, C.c_int, fp,
                                      C.POINTER(Similarity), C.POINTER(IcpResult), i32p]
    L.tzr_icp_generalized_batch.argtypes = [vp, C.POINTER(IcpParams), C.c_double, C.c_int, i32p, fpp, fpp, i32p, fpp,
                                            fpp, C.POINTER(Similarity), C.POINTER(IcpResult), C.POINTER(i32p)]
    L.tzr_register_cloud_pairs_icp_generalized.argtypes = L.tzr_register_cloud_pairs.argtypes + [
        C.POINTER(IcpParams), C.c_double, C.POINTER(IcpResult)]
    L.tzr_icp_point_to_plane_robust_batch.argtypes = L.tzr_icp_point_to_plane_batch.argtypes + [C.POINTER(RobustKernel)]
    L.tzr_icp_generalized_robust_batch.argtypes = L.tzr_icp_generalized_batch.argtypes + [C.POINTER(RobustKernel)]
    L.tzr_register_cloud_pairs_icp_robust.argtypes = L.tzr_register_cloud_pairs.argtypes + [
        C.POINTER(IcpParams), C.c_int32, C.c_double, C.POINTER(RobustKernel), C.POINTER(IcpResult)]
    L.tzr_information_matrix.argtypes = [vp, fp, C.c_int, fp, C.c_int, C.POINTER(Similarity), C.c_double, dp, i32p]
    L.tzr_information_matrix_batch.argtypes = [vp, C.c_int, i32p, fpp, i32p, fpp, C.POINTER(Similarity), C.c_double,
                                               dp, i32p]
    L.tzr_pose_graph_params_default.argtypes = [C.POINTER(PoseGraphParams)]
    L.tzr_pose_graph_params_default.restype = None
    L.tzr_pose_graph_optimize.argtypes = [vp, C.POINTER(PoseGraphParams), C.c_int, C.c_int, i32p,
                                          C.POINTER(Similarity), dp, i32p, C.POINTER(Similarity),
                                          C.POINTER(Similarity), dp, u8p, dp, C.POINTER(PoseGraphSummary)]
    L.tzr_pose_graph_optimize_batch.argtypes = [
        vp, C.POINTER(PoseGraphParams), C.c_int, i32p, i32p, C.POINTER(i32p), C.POINTER(C.POINTER(Similarity)),
        C.POINTER(dp), C.POINTER(i32p), C.POINTER(C.POINTER(Similarity)), C.POINTER(C.POINTER(Similarity)),
        C.POINTER(dp), C.POINTER(u8p), C.POINTER(dp), C.POINTER(PoseGraphSummary), i32p]
    L.tzr_register_cloud_pairs_multiway.argtypes = L.tzr_register_cloud_pairs_icp.argtypes + [
        i32p, C.POINTER(PoseGraphParams), dp, i32p, dp, u8p, C.POINTER(Similarity), C.POINTER(PoseGraphSummary), i32p]
    L.tzr_estimate_color_gradients.argtypes = [vp, fp, C.c_int, fp, fp, C.c_double, dp]
    L.tzr_estimate_color_gradients_batch.argtypes = [vp, C.c_int, i32p, fpp, fpp, fpp, C.c_double, C.POINTER(dp), i32p]
    L.tzr_icp_colored.argtypes = L.tzr_icp_point_to_plane.argtypes + [fp, fp, C.c_double, C.POINTER(RobustKernel)]
    L.tzr_icp_colored_batch.argtypes = L.tzr_icp_point_to_plane_batch.argtypes + [fpp, fpp, C.c_double,
                                                                                   C.POINTER(RobustKernel)]
    L.tzr_register_cloud_pairs_icp_colored.argtypes = L.tzr_register_cloud_pairs.argtypes + [
        C.POINTER(IcpParams), fpp, C.c_double, C.POINTER(RobustKernel), C.POINTER(IcpResult)]
    L.tzr_register_cloud_pairs_multiway_colored.argtypes = L.tzr_register_cloud_pairs_icp_colored.argtypes + \
        L.tzr_register_cloud_pairs_multiway.argtypes[len(L.tzr_register_cloud_pairs_icp.argtypes):]
    L.tzr_voxel_downsample.argtypes = [vp, fp, C.c_int, C.c_double, fp, i32p, i32p]
    L.tzr_voxel_downsample_batch.argtypes = [vp, C.c_int, i32p, fpp, C.c_double, fpp, i32p, C.POINTER(i32p), i32p]
    L.tzr_voxel_downsample_colors.argtypes = L.tzr_voxel_downsample.argtypes + [fp, fp]
    L.tzr_voxel_downsample_colors_batch.argtypes = L.tzr_voxel_downsample_batch.argtypes + [fpp, fpp]
    L.tzr_icp_multiscale_batch.argtypes = [vp, C.c_int, C.c_int, C.POINTER(IcpScale), C.c_int, i32p, fpp, fpp,
                                           C.c_int, i32p, C.POINTER(Similarity), C.c_double, C.c_double,
                                           C.POINTER(RobustKernel), C.POINTER(IcpResult), i32p, i32p, dp, i32p]
    L.tzr_fgr_params_default.argtypes = [C.POINTER(FgrParams)]
    L.tzr_fgr_params_default.restype = None
    L.tzr_fgr.argtypes = [vp, C.POINTER(FgrParams), fp, C.c_int, fp, C.c_int, C.c_int, i32p, C.POINTER(IcpResult), i32p]
    L.tzr_fgr_batch.argtypes = [vp, C.POINTER(FgrParams), C.c_int, i32p, fpp, i32p, fpp, i32p, C.POINTER(i32p),
                                C.POINTER(IcpResult), C.POINTER(i32p)]
    L.tzr_register_cloud_pairs_fgr.argtypes = [vp, C.POINTER(FrontendParams), C.POINTER(FgrParams), C.c_int, i32p, fpp,
                                               C.c_int, i32p, u64p, i32p, i64p, C.POINTER(i32p), fp,
                                               C.POINTER(IcpResult)]
    L.tzr_ransac_params_default.argtypes = [C.POINTER(RansacParams)]
    L.tzr_ransac_params_default.restype = None
    L.tzr_ransac.argtypes = [vp, C.POINTER(RansacParams), fp, C.c_int, fp, C.c_int, C.c_int, i32p, C.c_uint64, fp, fp,
                             C.POINTER(IcpResult), C.POINTER(RansacInfo), i32p]
    L.tzr_ransac_batch.argtypes = [vp, C.POINTER(RansacParams), C.c_int, i32p, fpp, i32p, fpp, i32p, C.POINTER(i32p),
                                   u64p, fpp, fpp, C.POINTER(IcpResult), C.POINTER(RansacInfo), C.POINTER(i32p)]
    L.tzr_register_cloud_pairs_ransac.argtypes = [vp, C.POINTER(FrontendParams), C.POINTER(RansacParams), C.c_int,
                                                  i32p, fpp, C.c_int, i32p, u64p, u64p, i32p, i64p, C.POINTER(i32p),
                                                  fp, C.POINTER(IcpResult), C.POINTER(RansacInfo)]
    L.tzr_line_process_params_default.argtypes = [C.POINTER(LineProcessParams)]
    L.tzr_line_process_params_default.restype = None
    L.tzr_pose_graph_optimize_line_process.argtypes = [vp, C.POINTER(LineProcessParams)] + \
        L.tzr_pose_graph_optimize.argtypes[2:-1] + [C.POINTER(LineProcessSummary)]
    L.tzr_pose_graph_optimize_line_process_batch.argtypes = [
        vp, C.POINTER(LineProcessParams), C.c_int, i32p, i32p, C.POINTER(i32p), C.POINTER(C.POINTER(Similarity)),
        C.POINTER(dp), C.POINTER(i32p), C.POINTER(C.POINTER(Similarity)), C.POINTER(C.POINTER(Similarity)),
        C.POINTER(dp), C.POINTER(u8p), C.POINTER(dp), C.POINTER(LineProcessSummary), i32p]
    L.tzr_dense_cholesky_batch.argtypes = [vp, C.c_int, i32p, C.POINTER(dp), C.POINTER(dp), C.POINTER(dp),
                                           C.POINTER(dp), i32p]
    L.tzr_register_cloud_pairs_multiway_line_process.argtypes = L.tzr_register_cloud_pairs_icp_colored.argtypes + [
        i32p, C.POINTER(LineProcessParams), dp, i32p, dp, u8p, C.POINTER(Similarity), C.POINTER(LineProcessSummary),
        i32p]
    mw_batch = [C.c_int, i32p, C.c_double, fpp, i32p, fpp]  # G, graph_offsets and the fused map
    L.tzr_register_cloud_pairs_multiway_batch.argtypes = L.tzr_register_cloud_pairs_icp_colored.argtypes + \
        L.tzr_register_cloud_pairs_multiway.argtypes[len(L.tzr_register_cloud_pairs_icp.argtypes):] + mw_batch
    L.tzr_register_cloud_pairs_multiway_line_process_batch.argtypes = \
        L.tzr_register_cloud_pairs_multiway_line_process.argtypes + mw_batch
    for s in _SYMBOLS:
        getattr(L, s)  # raises AttributeError if the header and the library disagree
    _lib = L
    return L


def default_params(**kw) -> Params:
    p = Params()
    lib().tzr_params_default(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def icp_params(max_correspondence_distance: float, **kw) -> IcpParams:
    """tzr_icp_params_default with max_correspondence_distance and any field in kw set."""
    p = IcpParams()
    lib().tzr_icp_params_default(C.byref(p))
    p.max_correspondence_distance = float(max_correspondence_distance)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def line_process_params(max_correspondence_distance: float, **kw) -> LineProcessParams:
    """tzr_line_process_params_default with max_correspondence_distance and any field in kw set."""
    p = LineProcessParams()
    lib().tzr_line_process_params_default(C.byref(p))
    p.max_correspondence_distance = float(max_correspondence_distance)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def _line_process_summary(summ):
    return dict(iterations=list(summ.iterations), trials=list(summ.trials), stop_reason=list(summ.stop_reason),
                pruned=int(summ.pruned), residual=float(summ.residual), mu=list(summ.mu))


def pose_graph_params(max_correspondence_distance: float, **kw) -> PoseGraphParams:
    """tzr_pose_graph_params_default with max_correspondence_distance and any field in kw set."""
    p = PoseGraphParams()
    lib().tzr_pose_graph_params_default(C.byref(p))
    p.max_correspondence_distance = float(max_correspondence_distance)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def fgr_params(**kw) -> FgrParams:
    """tzr_fgr_params_default (Open3D's FastGlobalRegistrationOption defaults) with any field in kw set; the library
    checks the values."""
    p = FgrParams()
    lib().tzr_fgr_params_default(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def ransac_params(max_correspondence_distance, **kw) -> RansacParams:
    """tzr_ransac_params_default (Open3D's defaults: ransac_n 3, 100000 iterations, confidence 0.999, no checkers) at
    max_correspondence_distance, with any field in kw set; the library checks the values."""
    p = RansacParams()
    lib().tzr_ransac_params_default(C.byref(p))
    p.max_correspondence_distance = float(max_correspondence_distance)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def _seeds64(seeds, n, what):
    """n 64-bit seeds as a uint64 array (None: zeros); Python integers taken modulo 2^64."""
    if seeds is None:
        return np.zeros(n, dtype=np.uint64)
    a = np.array([int(x) % (1 << 64) for x in seeds], dtype=np.uint64)
    if a.shape != (n,):
        raise TzrError(f"{what}: one seed per problem is required")
    return a


def corr_rows(corr, what="fgr"):
    """One problem's correspondences as a (K,2) int32 C-contiguous array of (source index, target index) rows: any
    (K,2) integer array or sequence of pairs, K = 0 included.  Values outside int32 are refused here; the library checks
    each index against its cloud."""
    a = np.asarray(corr)
    if a.size == 0:
        return np.zeros((0, 2), dtype=np.int32)
    if a.ndim != 2 or a.shape[1] != 2 or not np.issubdtype(a.dtype, np.integer):
        raise TzrError(f"{what}: correspondences must be a (K,2) integer array")
    if a.min() < np.iinfo(np.int32).min or a.max() > np.iinfo(np.int32).max:
        raise TzrError(f"{what}: a correspondence index does not fit int32")
    return np.ascontiguousarray(a, dtype=np.int32)


def _poses(sims):
    """(K,4,4) float64 rigid matrices from K Similarity records."""
    out = np.zeros((len(sims), 4, 4))
    for k, x in enumerate(sims):
        out[k, :3, :3] = np.asarray(x.rotation[:]).reshape(3, 3).T
        out[k, :3, 3] = x.translation[:]
        out[k, 3, 3] = 1.0
    return out


def robust_kernel(kernel) -> RobustKernel | None:
    """A tzr_robust_kernel from None (None: no kernel), a RobustKernel (as given), a name ("l2", "l1", "huber",
    "cauchy", "gm", "tukey") or a (name, k) pair, e.g. ("tukey", 0.05).  The library checks the type and k."""
    if kernel is None or isinstance(kernel, RobustKernel):
        return kernel
    name, k = (kernel, 0.0) if isinstance(kernel, str) else (kernel[0], kernel[1] if len(kernel) > 1 else 0.0)
    if str(name).lower() not in LOSS_TYPES:
        raise TzrError(f"robust_kernel: unknown kernel {name!r} (one of {sorted(LOSS_TYPES)})")
    return RobustKernel(LOSS_TYPES[str(name).lower()], 0, float(k))


def similarity(init=None) -> Similarity:
    """A tzr_similarity from None (identity), a (4,4) rigid matrix, a dict / record with scale, rotation (3x3 or
    column-major 9) and translation, or a Similarity."""
    if isinstance(init, Similarity):
        return init
    s = Similarity()
    if init is None:
        s.scale, R, t = 1.0, np.eye(3), np.zeros(3)
    elif isinstance(init, np.ndarray) and init.shape == (4, 4):
        s.scale, R, t = 1.0, init[:3, :3], init[:3, 3]
    else:
        R = np.asarray(init["rotation"], dtype=np.float64)
        R = R.reshape(3, 3).T if R.shape == (9,) else R
        s.scale, t = float(init["scale"]), np.asarray(init["translation"], dtype=np.float64)
    s.rotation[:] = [float(x) for x in np.asarray(R, dtype=np.float64).T.reshape(-1)]
    s.translation[:] = [float(x) for x in np.asarray(t, dtype=np.float64).reshape(3)]
    return s


def icp_result_dict(r) -> dict:
    """An IcpResult (or an ICP_RESULT_DTYPE record) as a dict: scale, R (3x3), t, fitness, inlier_rmse, iterations,
    n_correspondences, converged."""
    if isinstance(r, IcpResult):
        r = np.frombuffer(bytes(r), dtype=ICP_RESULT_DTYPE)[0]
    tr = r["transform"]
    return dict(scale=float(tr["scale"]), R=np.asarray(tr["rotation"]).reshape(3, 3).T.copy(),
                t=np.asarray(tr["translation"]).copy(), fitness=float(r["fitness"]),
                inlier_rmse=float(r["inlier_rmse"]), iterations=int(r["iterations"]),
                n_correspondences=int(r["n_correspondences"]), converged=bool(r["converged"]))


def _cloud32(a, what):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] != 3 or a.shape[0] == 0:
        raise TzrError(f"{what}: clouds must be non-empty (n,3) arrays")
    return a


def _normals32(a, n, what):
    """Target normals as (n,4) float32 rows (nx, ny, nz, curvature): an (n,4) array as given, an (n,3) one with a zero
    fourth column (the library ignores it)."""
    a = np.asarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[0] != n or a.shape[1] not in (3, 4):
        raise TzrError(f"{what}: normals must be (nd,3) or (nd,4) with one row per target point")
    if a.shape[1] == 3:
        a = np.concatenate([a, np.zeros((n, 1), dtype=np.float32)], axis=1)
    return np.ascontiguousarray(a)


def _colors32(a, n, what):
    """Colours as (n,3) float32 rows (r, g, b), one per point."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.shape != (n, 3):
        raise TzrError(f"{what}: colours must be (n,3) with one row per point")
    return a


def _pts(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("points must be (N,3)")
    return a


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class _GraphBatch:
    """The pointer-per-graph arrays of the batched pose-graph calls: G, K, E, edges, transforms, information,
    uncertain, initial_poses (NULL entries where a graph has none) and, per graph, the outputs poses (K), a double (E), a
    byte (E) and a double (E) array.  outs[g] = (K, E, poses, double, byte, double); status (G int32) and status_p."""

    def __init__(self, graphs, who):
        G = len(graphs)
        self.G, self.P = G, max(1, G)
        P = self.P
        self.keep = []  # the arrays the pointers refer to
        i32p, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
        simp = C.POINTER(Similarity)
        self.Ks, self.Es = np.zeros(P, dtype=np.int32), np.zeros(P, dtype=np.int32)
        self.ed_p, self.tr_p, self.info_p = (i32p * P)(), (simp * P)(), (dp * P)()
        self.unc_p, self.init_p, self.pose_p = (i32p * P)(), (simp * P)(), (simp * P)()
        self.d1_p, self.u8_p, self.d2_p = (dp * P)(), (C.POINTER(C.c_uint8) * P)(), (dp * P)()
        self.outs = []
        for g, gr in enumerate(graphs):
            K = int(gr["K"])
            ed = np.ascontiguousarray(gr["edges"], dtype=np.int32).reshape(-1, 2)
            E = ed.shape[0]
            info = np.ascontiguousarray(gr["information"], dtype=np.float64).reshape(E, 36)
            if len(gr["transforms"]) != E:
                raise TzrError(f"{who}: one transform per edge is required")
            tr = (Similarity * max(1, E))(*[similarity(x) for x in gr["transforms"]])
            self.keep.append(tr)
            self.Ks[g], self.Es[g] = K, E
            self.ed_p[g], self.info_p[g] = self._ptr(ed, C.c_int32), self._ptr(info, C.c_double)
            self.tr_p[g] = C.cast(tr, simp)
            if gr.get("uncertain") is not None:
                unc = np.ascontiguousarray(gr["uncertain"], dtype=np.int32)
                if unc.shape != (E,):
                    raise TzrError(f"{who}: uncertain needs one entry per edge")
                self.unc_p[g] = self._ptr(unc, C.c_int32)
            if gr.get("initial_poses") is not None:
                init = (Similarity * max(1, K))(*[similarity(x) for x in gr["initial_poses"]])
                self.keep.append(init)
                self.init_p[g] = C.cast(init, simp)
            poses = (Similarity * max(1, K))()
            d1, u8, d2 = np.zeros(max(1, E)), np.zeros(max(1, E), dtype=np.uint8), np.zeros(max(1, E))
            self.keep.append(poses)
            self.pose_p[g] = C.cast(poses, simp)
            self.d1_p[g], self.u8_p[g], self.d2_p[g] = (self._ptr(d1, C.c_double), self._ptr(u8, C.c_uint8),
                                                        self._ptr(d2, C.c_double))
            self.outs.append((K, E, poses, d1, u8, d2))
        self.status = np.zeros(P, dtype=np.int32)
        self.status_p = _p(self.status, C.c_int32)

    def _ptr(self, a, t):
        self.keep.append(a)
        return C.cast(a.ctypes.data, C.POINTER(t))

    def args(self):
        """G through the per-graph output arrays, in the batched calls' order."""
        return (self.G, _p(self.Ks, C.c_int32), _p(self.Es, C.c_int32), self.ed_p, self.tr_p, self.info_p, self.unc_p,
                self.init_p, self.pose_p, self.d1_p, self.u8_p, self.d2_p)

    def one(self):
        """The single calls' K through the output arrays: graph 0's entries of args()."""
        return (int(self.Ks[0]), int(self.Es[0]), self.ed_p[0], self.tr_p[0], self.info_p[0], self.unc_p[0],
                self.init_p[0], self.pose_p[0], self.d1_p[0], self.u8_p[0], self.d2_p[0])


def _pose_graph_result(out, summ):
    """One graph's dict of optimize_pose_graph(_batch) from its _GraphBatch outputs and summary."""
    K, E, poses, w, m, r = out
    return dict(poses=_poses(poses)[:K], weights=w[:E], mask=m[:E].astype(bool), residuals=r[:E],
                iterations=int(summ.iterations), inner_iterations=int(summ.inner_iterations), cost=float(summ.cost))


def _line_process_result(out, summ):
    """One graph's dict of global_optimization(_batch) from its _GraphBatch outputs and summary."""
    K, E, poses, l, m, r = out
    return dict(poses=_poses(poses)[:K], confidence=l[:E], kept=m[:E].astype(bool), residuals=r[:E],
                **_line_process_summary(summ))


def multiway_batch_table(sequences, pairs, uncertain=None, tuple_seeds=None, colors=None):
    """The flat table of register_multiway_batch: clouds, colours, pairs (global cloud indices), uncertain flags and
    tuple seeds of every sequence back to back, with offsets (the graph offsets, G + 1) and pair_offsets (each
    sequence's first pair, G + 1)."""
    G = len(sequences)
    if G == 0 or len(pairs) != G:
        raise TzrError("register_multiway_batch: one list of pairs per sequence is required")
    for name, arg in (("uncertain", uncertain), ("tuple_seeds", tuple_seeds), ("colors", colors)):
        if arg is not None and len(arg) != G:
            raise TzrError(f"register_multiway_batch: {name} needs one entry per sequence")
    clouds, cols, flat, unc, seeds, off, poff = [], [], [], [], [], [0], [0]
    for g, seq in enumerate(sequences):
        pc = np.asarray(pairs[g], dtype=np.int64).reshape(-1, 2)
        if pc.size and (pc.min() < 0 or pc.max() >= len(seq)):
            raise TzrError(f"register_multiway_batch: a pair of sequence {g} names a cloud that is not in it")
        u = [0 if b == a + 1 else 1 for a, b in pc] if uncertain is None or uncertain[g] is None else list(uncertain[g])
        t = [0] * len(pc) if tuple_seeds is None or tuple_seeds[g] is None else [int(x) for x in tuple_seeds[g]]
        if len(u) != len(pc) or len(t) != len(pc):
            raise TzrError(f"register_multiway_batch: sequence {g} needs one uncertain flag and tuple seed per pair")
        if colors is not None and len(colors[g]) != len(seq):
            raise TzrError(f"register_multiway_batch: sequence {g} needs one colour array per cloud")
        flat += [(off[-1] + int(a), off[-1] + int(b)) for a, b in pc]
        unc += u
        seeds += t
        clouds += list(seq)
        cols += [] if colors is None else list(colors[g])
        off.append(off[-1] + len(seq))
        poff.append(len(flat))
    return dict(clouds=clouds, colors=None if colors is None else cols, pairs=np.array(flat, dtype=np.int32).reshape(-1, 2),
                uncertain=np.array(unc, dtype=np.int32), tuple_seeds=seeds, offsets=np.array(off, dtype=np.int32),
                pair_offsets=poff)


def split_multiway_batch(out, pair_offsets, offsets):
    """register_multiway_batch's per-sequence results from _register_pairs' output over the flat table: each
    sequence's slice of every per-pair output, its problem indices counted within the sequence, and its dict (its
    pairs' rows of the per-pair arrays, its poses, its graph's status, summary and map)."""
    sols, status, index, corr, clq, gs, icp_res, mw = out
    res = []
    for g in range(len(pair_offsets) - 1):
        a, b = pair_offsets[g], pair_offsets[g + 1]
        idx = index[a:b].copy()
        solved = idx >= 0
        idx[solved] = np.arange(int(solved.sum()), dtype=idx.dtype)
        d = {k: v[a:b] for k, v in mw.items() if k not in ("poses", "graphs")}
        d["poses"] = mw["poses"][offsets[g]:offsets[g + 1]]
        d.update(mw["graphs"][g])
        res.append((sols[a:b], status[a:b], idx, corr[a:b], clq[a:b], gs[a:b], icp_res[a:b], d))
    return res


class Context:
    """One CUDA device + stream + workspace (tzr_ctx).  max_n: per-problem size limit, 32768 (default) ... 65536
    (tzr_ctx_set_max_n)."""

    def __init__(self, device: int = -1, max_n: int = 32768):
        self._h = C.c_void_p()
        rc = lib().tzr_ctx_create(device, C.byref(self._h))
        if rc != 0:
            raise TzrError(f"tzr_ctx_create failed: {lib().tzr_status_string(rc).decode()}")
        if max_n != 32768:
            try:
                self.set_max_n(max_n)
            except TzrError:
                self.close()
                raise

    def close(self):
        if self._h:
            lib().tzr_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise TzrError(f"{lib().tzr_status_string(rc).decode()}: {lib().tzr_last_error(self._h).decode()}")

    # -- utilities
    def set_flags(self, flags: int):
        self._ck(lib().tzr_ctx_set_flags(self._h, flags))

    def filter_mismatches(self) -> int:
        return int(lib().tzr_ctx_filter_mismatches(self._h))

    def filter_rechecks(self) -> int:
        return int(lib().tzr_ctx_filter_rechecks(self._h))

    def debug_counters(self):
        out = np.zeros(16, dtype=np.int64)
        self._ck(lib().tzr_ctx_debug_counters(self._h, _p(out, C.c_int64)))
        return dict(filter_mismatches=int(out[0]), filter_rechecks=int(out[1]), clique_nodes=int(out[2]),
                    reduce_rounds=int(out[3]), reduce_vertices=int(out[4]), colourings=int(out[5]),
                    coloured_vertices=int(out[6]), tc_problems=int(out[7]),
                    # exact clique search, per-root timing (flag 4): cycles in the root colour bound / degree rules /
                    # colourings, slowest root (ns, vertex), summed root time, roots above 1 ms
                    root_colour_cycles=int(out[8]), reduce_cycles=int(out[9]), colour_cycles=int(out[10]),
                    slowest_root_ns=int(out[11]) >> 16, slowest_root_vertex=int(out[11]) & 0xffff,
                    root_ns_total=int(out[12]), roots_over_1ms=int(out[13]), block_bound_prunes=int(out[14]),
                    # problems graph_strip2_kernel built with the Gram-form test (the rest: interval test or another kernel)
                    gram_problems=int(out[15]))

    def last_strip_blocks(self) -> int:
        """Strip length of the default graph kernel's most recent launch (0: none, or another kernel built the graph)."""
        return int(lib().tzr_ctx_last_strip_blocks(self._h))

    def set_scale_chunk(self, max_end_points: int):
        """Chunk capacity of the unknown-scale stage's regenerating route, in end points (2 per TIM): 0 automatic
        (2^27, the route above 8192 points), k >= 2048 that route above 256 points in chunks of at most k end points
        (raised when more than 4096 chunks would be needed).  Every capacity gives the same estimate."""
        self._ck(lib().tzr_ctx_set_scale_chunk(self._h, int(max_end_points)))

    def last_scale_chunks(self) -> int:
        """Largest chunk count of one problem in the most recent unknown-scale stage (1: sorted at once; 0: none, or
        the bitonic path)."""
        return int(lib().tzr_ctx_last_scale_chunks(self._h))

    def clique_info(self, B: int):
        """Geometry of the most recent max_clique(_batch) call and each problem's root-heuristic clique size."""
        geom = np.zeros(3, dtype=np.int32)
        heur = np.zeros(B, dtype=np.int32)
        self._ck(lib().tzr_ctx_clique_info(self._h, _p(geom, C.c_int32), _p(heur, C.c_int32)))
        return dict(exact_ctas=int(geom[0]), exact_conc=int(geom[1]), max_depth=int(geom[2]), heuristic_best=heur)

    def set_max_n(self, max_n: int):
        """Per-problem size limit: 32768 <= max_n <= 65536; above 32768 the clique stage takes the large route."""
        self._ck(lib().tzr_ctx_set_max_n(self._h, int(max_n)))

    def clique_route(self, B: int):
        """(B,) int32 clique route of each problem of the most recent clique stage: 0 small route, k > 0 large route
        with the core compacted to k vertices (k = clique size: no search ran), -1 core above the cap (heuristic
        clique, not proven).  k and the cap test refer to the (L-1)-core itself, never to a superset of it."""
        out = np.zeros(B, dtype=np.int32)
        self._ck(lib().tzr_ctx_clique_route(self._h, _p(out, C.c_int32)))
        return out

    def kernel_launches(self) -> int:
        return int(lib().tzr_ctx_kernel_launches(self._h))

    def synchronize(self):
        self._ck(lib().tzr_ctx_synchronize(self._h))

    def set_stream(self, cuda_stream_ptr: int):
        self._ck(lib().tzr_ctx_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    def last_stage_ms(self):
        v = [C.c_double() for _ in range(4)]
        self._ck(lib().tzr_last_stage_ms(self._h, C.byref(v[0]), C.byref(v[1]), C.byref(v[2]), C.byref(v[3])))
        return dict(prep=v[0].value, graph=v[1].value, clique=v[2].value, rot_trans=v[3].value)

    def stage_log(self, enable: bool):
        """Keep the stage events of every call (no host sync per step); read them with stage_log_read()."""
        self._ck(lib().tzr_ctx_stage_log(self._h, 1 if enable else 0))

    def stage_log_read(self):
        v = (C.c_double * 4)()
        calls = C.c_int32()
        self._ck(lib().tzr_ctx_stage_log_read(self._h, v, C.byref(calls)))
        return dict(prep=v[0], graph=v[1], clique=v[2], rot_trans=v[3]), int(calls.value)

    def last_graph_info(self):
        B, n, has, gen = C.c_int32(), C.c_int32(), C.c_int32(), C.c_uint64()
        self._ck(lib().tzr_last_graph_info(self._h, C.byref(B), C.byref(n), C.byref(has), C.byref(gen)))
        return dict(B=B.value, n=n.value, has_graph=bool(has.value), generation=int(gen.value))

    # -- stages
    def graph_build(self, src, dst, beta):
        s, d = _pts(src), _pts(dst)
        n = s.shape[0]
        W = lib().tzr_words_per_row(n)
        bits = np.zeros((n, W), dtype=np.uint64)
        deg = np.zeros(n, dtype=np.int32)
        ne = C.c_int64()
        self._ck(lib().tzr_graph_build(self._h, _p(s, C.c_double), _p(d, C.c_double), n, beta, _p(bits, C.c_uint64),
                                       _p(deg, C.c_int32), C.byref(ne)))
        return bits, deg, int(ne.value)

    def max_clique(self, bits, n, mode=0, kcore_thr=0.5, time_limit=3600.0):
        bits = np.ascontiguousarray(bits, dtype=np.uint64)
        out = np.zeros(n, dtype=np.int32)
        m = C.c_int32()
        proven = C.c_int32()
        self._ck(lib().tzr_max_clique(self._h, _p(bits, C.c_uint64), n, mode, kcore_thr, time_limit,
                                      _p(out, C.c_int32), C.byref(m), C.byref(proven)))
        return out[:m.value].copy(), bool(proven.value)

    def max_clique_batch(self, bits, mode=0, kcore_thr=0.5, time_limit=3600.0):
        """bits: (B, n, tzr_words_per_row(n)) uint64, one bitset per problem.  Returns (cliques: list of B sorted int32
        arrays, proven: (B,) int32 codes as tzr_solution.clique_proven_optimal, search_flags: (B,) int32)."""
        bits = np.ascontiguousarray(bits, dtype=np.uint64)
        if bits.ndim != 3 or bits.shape[2] != lib().tzr_words_per_row(bits.shape[1]):
            raise ValueError("bits must be (B, n, tzr_words_per_row(n)) uint64")
        B, n = bits.shape[0], bits.shape[1]
        out = np.zeros((B, n), dtype=np.int32)
        sizes = np.zeros(B, dtype=np.int32)
        proven = np.zeros(B, dtype=np.int32)
        flags = np.zeros(B, dtype=np.int32)
        self._ck(lib().tzr_max_clique_batch(self._h, B, n, _p(bits, C.c_uint64), mode, kcore_thr, time_limit,
                                            _p(out, C.c_int32), _p(sizes, C.c_int32), _p(proven, C.c_int32),
                                            _p(flags, C.c_int32)))
        return [out[b, :sizes[b]].copy() for b in range(B)], proven, flags

    def gnc_tls_rotation(self, src, dst, noise_bound, gnc_factor=1.4, max_iterations=100, cost_threshold=1e-6):
        return self.rotation_solve(0, src, dst, noise_bound, gnc_factor, max_iterations, cost_threshold)

    def rotation_solve(self, algorithm, src, dst, noise_bound, gnc_factor=1.4, max_iterations=100,
                       cost_threshold=1e-6):
        """algorithm: 0 GNC_TLS, 1 FGR, 2 QUATRO (ROTATION_ESTIMATION_ALGORITHM, registration.h:382-386)."""
        s, d = _pts(src), _pts(dst)
        m = s.shape[0]
        R = np.zeros(9)
        mask = np.zeros(m, dtype=np.uint8)
        cost = C.c_double()
        it = C.c_int32()
        self._ck(lib().tzr_rotation_solve(self._h, int(algorithm), _p(s, C.c_double), _p(d, C.c_double), m, noise_bound,
                                          gnc_factor, int(max_iterations), cost_threshold, _p(R, C.c_double),
                                          _p(mask, C.c_uint8), C.byref(cost), C.byref(it)))
        return dict(R=R.reshape(3, 3).T.copy(), inliers=mask.astype(bool), cost=cost.value, iterations=it.value)

    def tls_translation(self, src, dst, noise_bound, cbar2=1.0):
        s, d = _pts(src), _pts(dst)
        m = s.shape[0]
        t = np.zeros(3)
        mask = np.zeros(m, dtype=np.uint8)
        self._ck(lib().tzr_tls_translation(self._h, _p(s, C.c_double), _p(d, C.c_double), m, noise_bound, cbar2,
                                           _p(t, C.c_double), _p(mask, C.c_uint8)))
        return t, mask.astype(bool)

    def scalar_tls(self, x, ranges):
        x = np.ascontiguousarray(x, dtype=np.float64)
        r = np.ascontiguousarray(ranges, dtype=np.float64)
        est = C.c_double()
        inl = np.zeros(x.size, dtype=np.uint8)
        self._ck(lib().tzr_scalar_tls(self._h, _p(x, C.c_double), _p(r, C.c_double), x.size, C.byref(est),
                                      _p(inl, C.c_uint8)))
        return est.value, inl.astype(bool)

    # -- downstream of solve(): DRSCertifier (certification.cc)
    @staticmethod
    def _cert_inputs(R, src, dst, theta):
        Rc = np.ascontiguousarray(np.asarray(R, dtype=np.float64).T)      # column-major 3x3
        s = np.ascontiguousarray(np.asarray(src, dtype=np.float64).T)     # (3,N) -> N xyz triples == column-major 3xN
        d = np.ascontiguousarray(np.asarray(dst, dtype=np.float64).T)
        th = np.asarray(theta)
        th = np.where(th, 1.0, -1.0) if th.dtype == np.bool_ else th.astype(np.float64)
        th = np.ascontiguousarray(th.ravel())
        if s.shape[1] != 3 or d.shape != s.shape or th.size != s.shape[0]:
            raise TzrError("certify: src/dst must be (3,N) and theta (N,)")
        return Rc, s, d, th

    @staticmethod
    def certifier_params(**kw) -> "CertifierParams":
        p = CertifierParams()
        lib().tzr_certifier_params_default(C.byref(p))
        for k, v in kw.items():
            if not hasattr(p, k):
                raise AttributeError(k)
            setattr(p, k, v)
        return p

    def certify(self, R, src, dst, theta, **params):
        """DRSCertifier(params).certify(R, src, dst, theta) (certification.cc:22-190); src/dst are (3,N)."""
        p = self.certifier_params(**params)
        Rc, s, d, th = self._cert_inputs(R, src, dst, theta)
        cap = int(max(1, np.ceil(p.max_iterations)))
        traj = np.zeros(cap)
        res = CertificationResult()
        self._ck(lib().tzr_certify(self._h, C.byref(p), _p(Rc, C.c_double), _p(s, C.c_double), _p(d, C.c_double),
                                   _p(th, C.c_double), th.size, C.byref(res), _p(traj, C.c_double), cap))
        return dict(is_optimal=bool(res.is_optimal), best_suboptimality=res.best_suboptimality,
                    suboptimality_traj=traj[:res.n_iterations].copy())

    @staticmethod
    def _cert_batch_inputs(Rs, srcs, dsts, thetas):
        """Validated, contiguous per-problem inputs of certify_batch (no device needed)."""
        Rs, srcs, dsts, thetas = list(Rs), list(srcs), list(dsts), list(thetas)
        B = len(Rs)
        if B == 0 or not (len(srcs) == len(dsts) == len(thetas) == B):
            raise TzrError("certify_batch: four lists of the same non-zero length are required")
        probs = []
        for b in range(B):
            if np.asarray(Rs[b]).shape != (3, 3):
                raise TzrError(f"certify_batch: rotation {b} must be (3,3)")
            Rc, s, d, th = Context._cert_inputs(Rs[b], srcs[b], dsts[b], thetas[b])
            if th.size == 0:
                raise TzrError(f"certify_batch: problem {b} has no measurements")
            probs.append((Rc, s, d, th))
        return probs

    def certify_batch(self, Rs, srcs, dsts, thetas, **params):
        """certify on every problem of the lists in one call (tzr_certify_batch): Rs (3,3), srcs/dsts (3,N_b), thetas
        (N_b,) +-1 or bool.  Returns a list of dicts shaped like certify's."""
        probs = self._cert_batch_inputs(Rs, srcs, dsts, thetas)
        p = self.certifier_params(**params)
        B = len(probs)
        R = np.ascontiguousarray(np.concatenate([pr[0].ravel() for pr in probs]))
        N = np.array([pr[3].size for pr in probs], dtype=np.int32)
        cap = int(max(1, np.ceil(p.max_iterations)))
        trajs = [np.zeros(cap) for _ in range(B)]
        caps = np.full(B, cap, dtype=np.int32)
        res = (CertificationResult * B)()
        dp = C.POINTER(C.c_double)
        arr = lambda xs: (dp * B)(*[_p(x, C.c_double) for x in xs])
        self._ck(lib().tzr_certify_batch(self._h, C.byref(p), B, _p(N, C.c_int32), _p(R, C.c_double),
                                         arr([pr[1] for pr in probs]), arr([pr[2] for pr in probs]),
                                         arr([pr[3] for pr in probs]), res, arr(trajs), _p(caps, C.c_int32)))
        return [dict(is_optimal=bool(r.is_optimal), best_suboptimality=r.best_suboptimality,
                     suboptimality_traj=t[:r.n_iterations].copy()) for r, t in zip(res, trajs)]

    def certifier_initial_matrix(self, R, src, dst, theta, **params):
        p = self.certifier_params(**params)
        Rc, s, d, th = self._cert_inputs(R, src, dst, theta)
        n = 4 * th.size + 4
        M = np.zeros((n, n))
        mu = C.c_double()
        self._ck(lib().tzr_certifier_initial_matrix(self._h, C.byref(p), _p(Rc, C.c_double), _p(s, C.c_double),
                                                    _p(d, C.c_double), _p(th, C.c_double), th.size,
                                                    _p(M, C.c_double), C.byref(mu)))
        return M.T.copy(), mu.value      # column-major buffer -> numpy row-major view of the same matrix

    def certifier_dual_projection(self, W, theta):
        th = np.ascontiguousarray(np.asarray(theta, dtype=np.float64).ravel())
        Wc = np.ascontiguousarray(np.asarray(W, dtype=np.float64).T)
        n = 4 * th.size + 4
        if Wc.shape != (n, n):
            raise TzrError("certifier_dual_projection: W must be (4N+4, 4N+4)")
        out = np.zeros((n, n))
        self._ck(lib().tzr_certifier_dual_projection(self._h, _p(Wc, C.c_double), _p(th, C.c_double), th.size,
                                                     _p(out, C.c_double)))
        return out.T.copy()

    @staticmethod
    def _cert_square(M, what):
        """Column-major copy of a (4N+4, 4N+4) matrix and its N."""
        Mc = np.ascontiguousarray(np.asarray(M, dtype=np.float64).T)
        n = Mc.shape[0]
        if Mc.ndim != 2 or Mc.shape != (n, n) or n < 8 or n % 4:
            raise TzrError(f"{what}: M must be (4N+4, 4N+4) with N >= 1")
        return Mc, (n - 4) // 4

    def certifier_psd_projection(self, M):
        """The nearest-PSD step of tzr_certify on any (4N+4)^2 M: (V+ diag(w+) V+^T of (M + M^T)/2, ascending w)."""
        Mc, N = self._cert_square(M, "certifier_psd_projection")
        out, w = np.zeros_like(Mc), np.zeros(Mc.shape[0])
        self._ck(lib().tzr_certifier_psd_projection(self._h, _p(Mc, C.c_double), N, _p(out, C.c_double),
                                                    _p(w, C.c_double)))
        return out.T.copy(), w

    def certifier_batch_psd_projection(self, Ms):
        """The nearest-PSD step of tzr_certify_batch on every matrix of the list, one call (padded layout, the batch's
        eigensolver route)."""
        ins = [self._cert_square(M, "certifier_batch_psd_projection") for M in Ms]
        if not ins:
            raise TzrError("certifier_batch_psd_projection: no matrices")
        outs = [np.zeros_like(m) for m, _ in ins]
        N = np.array([k for _, k in ins], dtype=np.int32)
        dp = C.POINTER(C.c_double)
        arr = lambda xs: (dp * len(xs))(*[_p(x, C.c_double) for x in xs])
        self._ck(lib().tzr_certifier_batch_psd_projection(self._h, len(ins), _p(N, C.c_int32), arr([m for m, _ in ins]),
                                                          arr(outs)))
        return [o.T.copy() for o in outs]

    def certifier_batch_dual_projection(self, Ws, thetas):
        """The dual projection of tzr_certify_batch on every (W, theta) pair of the lists, one call."""
        ins = [self._cert_square(W, "certifier_batch_dual_projection") for W in Ws]
        ths = [np.ascontiguousarray(np.asarray(t, dtype=np.float64).ravel()) for t in thetas]
        if not ins or len(ths) != len(ins) or any(t.size != k for t, (_, k) in zip(ths, ins)):
            raise TzrError("certifier_batch_dual_projection: one theta of N values per (4N+4)^2 W is required")
        outs = [np.zeros_like(m) for m, _ in ins]
        N = np.array([k for _, k in ins], dtype=np.int32)
        dp = C.POINTER(C.c_double)
        arr = lambda xs: (dp * len(xs))(*[_p(x, C.c_double) for x in xs])
        self._ck(lib().tzr_certifier_batch_dual_projection(self._h, len(ins), _p(N, C.c_int32),
                                                           arr([m for m, _ in ins]), arr(ths), arr(outs)))
        return [o.T.copy() for o in outs]

    # -- upstream of solve(): Matcher::calculateCorrespondences (matcher.cc:21-337)
    def match_correspondences(self, src_pts, dst_pts, src_feat, dst_feat, use_absolute_scale=True,
                              use_crosscheck=True, use_tuple_test=True, tuple_scale=0.0, tuple_seed=0,
                              return_scale=False):
        """Same argument order and defaults as the reference method (matcher.h:39-43); points are (n,3) float32,
        features (n,dim) float32.  Returns an (m,2) int32 array of sorted unique (source, target) index pairs."""
        sp = np.ascontiguousarray(src_pts, dtype=np.float32)
        tp = np.ascontiguousarray(dst_pts, dtype=np.float32)
        sf = np.ascontiguousarray(src_feat, dtype=np.float32)
        tf = np.ascontiguousarray(dst_feat, dtype=np.float32)
        ns, nd = sp.shape[0], tp.shape[0]
        if sp.shape != (ns, 3) or tp.shape != (nd, 3) or sf.ndim != 2 or tf.ndim != 2 or sf.shape[0] != ns or \
                tf.shape[0] != nd or sf.shape[1] != tf.shape[1]:
            raise TzrError("match_correspondences: points must be (n,3) and features (n,dim) with one row per point")
        cap = ns + nd
        pairs = np.zeros((cap, 2), dtype=np.int32)
        cnt = C.c_int64()
        g = C.c_float()
        self._ck(lib().tzr_match_correspondences(
            self._h, _p(sp, C.c_float), ns, _p(tp, C.c_float), nd, _p(sf, C.c_float), _p(tf, C.c_float), sf.shape[1],
            int(bool(use_absolute_scale)), int(bool(use_crosscheck)), int(bool(use_tuple_test)), float(tuple_scale),
            int(tuple_seed), _p(pairs, C.c_int32), cap, C.byref(cnt), C.byref(g)))
        out = pairs[:cnt.value].copy()
        return (out, g.value) if return_scale else out

    def compute_fpfh(self, pts, normal_search_radius=0.03, fpfh_search_radius=0.05, return_normals=False):
        """FPFHEstimation::computeFPFHFeatures (fpfh.h:39-41, same defaults): (n,3) float32 -> (n,33) float32."""
        p = np.ascontiguousarray(pts, dtype=np.float32)
        if p.ndim != 2 or p.shape[1] != 3:
            raise TzrError("compute_fpfh: points must be (n,3)")
        out = np.zeros((p.shape[0], 33), dtype=np.float32)
        nor = np.zeros((p.shape[0], 4), dtype=np.float32)
        self._ck(lib().tzr_compute_fpfh(self._h, _p(p, C.c_float), p.shape[0], float(normal_search_radius),
                                        float(fpfh_search_radius), _p(out, C.c_float), _p(nor, C.c_float)))
        return (out, nor) if return_normals else out

    def compute_fpfh_batch(self, pts_list, normal_search_radius=0.03, fpfh_search_radius=0.05, return_normals=False):
        """compute_fpfh on every (n_b,3) cloud of the list in one call: a list of (n_b,33) descriptors (and a list of
        (n_b,4) normals), each bit-identical to compute_fpfh on that cloud alone.  When a cloud has a point with more
        than 4096 neighbours the TzrError carries `status` (per cloud 0 or the error code) and `result` (the outputs
        of every cloud, written for the others)."""
        pts = [np.ascontiguousarray(p, dtype=np.float32) for p in pts_list]
        if not pts or any(p.ndim != 2 or p.shape[1] != 3 for p in pts):
            raise TzrError("compute_fpfh_batch: a non-empty list of (n,3) clouds is required")
        B = len(pts)
        n = np.array([p.shape[0] for p in pts], dtype=np.int32)
        outs = [np.zeros((p.shape[0], 33), dtype=np.float32) for p in pts]
        nors = [np.zeros((p.shape[0], 4), dtype=np.float32) for p in pts] if return_normals else None
        status = np.zeros(B, dtype=np.int32)
        fp = C.POINTER(C.c_float)
        arr = lambda xs: (fp * B)(*[_p(x, C.c_float) for x in xs])
        rc = lib().tzr_compute_fpfh_batch(self._h, B, _p(n, C.c_int32), arr(pts), float(normal_search_radius),
                                          float(fpfh_search_radius), arr(outs), arr(nors) if nors else None,
                                          _p(status, C.c_int32))
        result = (outs, nors) if return_normals else outs
        try:
            self._ck(rc)
        except TzrError as e:
            e.status, e.result = status, result
            raise
        return result

    def estimate_normals(self, pts, normal_search_radius=0.03):
        """tzr_estimate_normals: compute_fpfh's normals alone, (n,3) float32 -> (n,4) float32 (nx, ny, nz, curvature),
        bit-identical to compute_fpfh(..., return_normals=True)'s normals at the same normal radius."""
        p = _cloud32(pts, "estimate_normals")
        nor = np.zeros((p.shape[0], 4), dtype=np.float32)
        self._ck(lib().tzr_estimate_normals(self._h, _p(p, C.c_float), p.shape[0], float(normal_search_radius),
                                            _p(nor, C.c_float)))
        return nor

    def estimate_normals_batch(self, pts_list, normal_search_radius=0.03):
        """estimate_normals on every (n_b,3) cloud of the list in one call: a list of (n_b,4) normals, each
        bit-identical to estimate_normals on that cloud alone.  When a cloud has a point with more than 4096
        neighbours the TzrError carries `status` (per cloud 0 or the error code) and `result` (every cloud's normals,
        written for the others)."""
        pts = [_cloud32(p, "estimate_normals_batch") for p in pts_list]
        if not pts:
            raise TzrError("estimate_normals_batch: a non-empty list of (n,3) clouds is required")
        B = len(pts)
        n = np.array([p.shape[0] for p in pts], dtype=np.int32)
        nors = [np.zeros((p.shape[0], 4), dtype=np.float32) for p in pts]
        status = np.zeros(B, dtype=np.int32)
        fp = C.POINTER(C.c_float)
        rc = lib().tzr_estimate_normals_batch(self._h, B, _p(n, C.c_int32), (fp * B)(*[_p(p, C.c_float) for p in pts]),
                                              float(normal_search_radius), (fp * B)(*[_p(x, C.c_float) for x in nors]),
                                              _p(status, C.c_int32))
        try:
            self._ck(rc)
        except TzrError as e:
            e.status, e.result = status, nors
            raise
        return nors

    def estimate_color_gradients(self, pts, normals, colors, radius):
        """tzr_estimate_color_gradients: Open3D's colour gradients of one (n,3) float32 cloud with its (n,3) or (n,4)
        normals and (n,3) colours, at `radius`: (n,3) float64."""
        return self.estimate_color_gradients_batch([pts], [normals], [colors], radius, single=True)[0]

    def estimate_color_gradients_batch(self, pts_list, normals, colors, radius, single=False):
        """estimate_color_gradients of every cloud of the list in one call (tzr_estimate_color_gradients_batch): a list
        of (n_b,3) float64 gradients, each bit-identical to estimate_color_gradients on that cloud alone.  single=True
        goes through tzr_estimate_color_gradients (one cloud)."""
        pts = [_cloud32(p, "estimate_color_gradients") for p in pts_list]
        if not pts or len(normals) != len(pts) or len(colors) != len(pts):
            raise TzrError("estimate_color_gradients_batch: one normals and one colours array per cloud are required")
        N = [_normals32(a, p.shape[0], "estimate_color_gradients") for a, p in zip(normals, pts)]
        K = [_colors32(a, p.shape[0], "estimate_color_gradients") for a, p in zip(colors, pts)]
        B = len(pts)
        grads = [np.zeros((p.shape[0], 3), dtype=np.float64) for p in pts]
        fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
        if single:
            assert B == 1
            rc = lib().tzr_estimate_color_gradients(self._h, _p(pts[0], C.c_float), pts[0].shape[0], _p(N[0], C.c_float),
                                                    _p(K[0], C.c_float), float(radius), _p(grads[0], C.c_double))
        else:
            n = np.array([p.shape[0] for p in pts], dtype=np.int32)
            rc = lib().tzr_estimate_color_gradients_batch(
                self._h, B, _p(n, C.c_int32), (fp * B)(*[_p(p, C.c_float) for p in pts]),
                (fp * B)(*[_p(a, C.c_float) for a in N]), (fp * B)(*[_p(a, C.c_float) for a in K]), float(radius),
                (dp * B)(*[_p(g, C.c_double) for g in grads]), None)
        self._ck(rc)
        return grads

    def icp_colored(self, src, dst, dst_normals, src_colors, dst_colors, max_correspondence_distance, init=None,
                    lambda_geometric=0.968, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, kernel=None):
        """tzr_icp_colored: Open3D's coloured ICP of the (ns,3) source onto the (nd,3) target with the target's normals
        and both clouds' (n,3) colours; kernel (see robust_kernel()) may be None.  Returns what icp() returns."""
        res, corr = self.icp_colored_batch([src], [dst], [dst_normals], [src_colors], [dst_colors],
                                           max_correspondence_distance, None if init is None else [init],
                                           lambda_geometric=lambda_geometric, max_iteration=max_iteration,
                                           relative_fitness=relative_fitness, relative_rmse=relative_rmse,
                                           single=True, kernel=kernel)
        return icp_result_dict(res[0]), corr[0]

    def icp_colored_batch(self, srcs, dsts, dst_normals, src_colors, dst_colors, max_correspondence_distance,
                          inits=None, lambda_geometric=0.968, max_iteration=30, relative_fitness=1e-6,
                          relative_rmse=1e-6, single=False, kernel=None):
        """tzr_icp_colored_batch: icp_point_to_plane_batch() with coloured updates and one (n,3) colours array per
        source and per target.  single=True goes through tzr_icp_colored (B must be 1).  Returns what icp_batch()
        returns."""
        S = [_cloud32(a, "icp_colored") for a in srcs]
        D = [_cloud32(a, "icp_colored") for a in dsts]
        B = len(S)
        if B == 0 or len(D) != B or len(dst_normals) != B or len(src_colors) != B or len(dst_colors) != B or \
                (inits is not None and len(inits) != B):
            raise TzrError("icp_colored_batch: one target, normals, colours and seed per source cloud are required")
        N = [_normals32(a, d.shape[0], "icp_colored") for a, d in zip(dst_normals, D)]
        SC = [_colors32(a, x.shape[0], "icp_colored") for a, x in zip(src_colors, S)]
        DC = [_colors32(a, x.shape[0], "icp_colored") for a, x in zip(dst_colors, D)]
        p = icp_params(max_correspondence_distance, max_iteration=int(max_iteration),
                       relative_fitness=float(relative_fitness), relative_rmse=float(relative_rmse))
        init = (Similarity * B)(*[similarity(None if inits is None else x) for x in inits or [None] * B])
        res = (IcpResult * B)()
        corr = [np.zeros((a.shape[0], 2), dtype=np.int32) for a in S]
        kern = robust_kernel(kernel)
        kp = C.byref(kern) if kern is not None else None
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        if single:
            assert B == 1
            rc = lib().tzr_icp_colored(self._h, C.byref(p), _p(S[0], C.c_float), S[0].shape[0], _p(D[0], C.c_float),
                                       D[0].shape[0], _p(N[0], C.c_float), init, res, _p(corr[0], C.c_int32),
                                       _p(SC[0], C.c_float), _p(DC[0], C.c_float), float(lambda_geometric), kp)
        else:
            ns = np.array([a.shape[0] for a in S], dtype=np.int32)
            nd = np.array([a.shape[0] for a in D], dtype=np.int32)
            arr = lambda xs: (fp * B)(*[_p(a, C.c_float) for a in xs])  # noqa: E731
            rc = lib().tzr_icp_colored_batch(self._h, C.byref(p), B, _p(ns, C.c_int32), arr(S), _p(nd, C.c_int32),
                                             arr(D), arr(N), init, res, (i32p * B)(*[_p(c, C.c_int32) for c in corr]),
                                             arr(SC), arr(DC), float(lambda_geometric), kp)
        self._ck(rc)
        out = np.frombuffer(bytes(res), dtype=ICP_RESULT_DTYPE).copy()
        return out, [c[:int(r["n_correspondences"])].copy() for c, r in zip(corr, out)]

    @staticmethod
    def _rows3(a, n, what):
        a = np.ascontiguousarray(a, dtype=np.float32)
        if a.shape != (n, 3):
            raise TzrError(f"{what}: every input must be (n,3)")
        return a

    def fpfh_pair_features(self, p1, n1, p2, n2):
        """pcl::computePairFeatures on n pairs of (point, normal), each (n,3): ((n,3) float32 f1, f2, f3, (n,) bool ok),
        the device function the SPFH kernel runs; rows where ok is False are zero."""
        n = np.asarray(p1).shape[0]
        ins = [self._rows3(a, n, "fpfh_pair_features") for a in (p1, n1, p2, n2)]
        f = np.zeros((n, 3), dtype=np.float32)
        ok = np.zeros(n, dtype=np.int32)
        self._ck(lib().tzr_fpfh_pair_features(self._h, n, *[_p(a, C.c_float) for a in ins], _p(f, C.c_float),
                                              _p(ok, C.c_int32)))
        return f, ok.astype(bool)

    def fpfh_smallest_eigenpair(self, cov):
        """pcl::eigen33's smallest eigenpair of every symmetric (3,3) float32 matrix of an (n,3,3) array, the device
        function the normals kernel runs: ((n,) eigenvalues, (n,3) unit eigenvectors)."""
        c = np.ascontiguousarray(cov, dtype=np.float32)
        if c.ndim != 3 or c.shape[1:] != (3, 3) or c.shape[0] == 0:
            raise TzrError("fpfh_smallest_eigenpair: cov must be (n,3,3) with n >= 1")
        n = c.shape[0]
        ev = np.zeros(n, dtype=np.float32)
        vec = np.zeros((n, 3), dtype=np.float32)
        self._ck(lib().tzr_fpfh_smallest_eigenpair(self._h, n, _p(c, C.c_float), _p(ev, C.c_float),
                                                   _p(vec, C.c_float)))
        return ev, vec

    def match_correspondences_batch(self, src_pts, dst_pts, src_feat, dst_feat, use_absolute_scale=True,
                                    use_crosscheck=True, use_tuple_test=True, tuple_scale=0.0, tuple_seeds=None,
                                    return_scale=False, capacity=None):
        """match_correspondences on B pairs in one call (lists of (n,3) points and (n,dim) features, one dim for all);
        tuple_seeds: B seeds (default 0 each).  Returns a list of (m_b,2) int32 pair arrays (and a list of
        global scales), each bit-identical to match_correspondences on that pair with its seed.  capacity (B row
        counts, default ns + nd) bounds each output; when one is too small the TzrError carries `n_pairs` and
        `result` (the pairs that fit, None for the others)."""
        cast = lambda xs: [np.ascontiguousarray(x, dtype=np.float32) for x in xs]
        sp, tp, sf, tf = cast(src_pts), cast(dst_pts), cast(src_feat), cast(dst_feat)
        B = len(sp)
        if B == 0 or not (len(tp) == len(sf) == len(tf) == B):
            raise TzrError("match_correspondences_batch: four lists of the same non-zero length are required")
        dim = sf[0].shape[1] if sf[0].ndim == 2 else -1
        for a, b, fa, fb in zip(sp, tp, sf, tf):
            if a.ndim != 2 or a.shape[1] != 3 or b.ndim != 2 or b.shape[1] != 3 or fa.shape != (a.shape[0], dim) or \
                    fb.shape != (b.shape[0], dim):
                raise TzrError("match_correspondences_batch: points must be (n,3) and features (n,dim) with one row "
                               "per point and one dim for every pair")
        ns = np.array([a.shape[0] for a in sp], dtype=np.int32)
        nd = np.array([b.shape[0] for b in tp], dtype=np.int32)
        cap = (ns.astype(np.int64) + nd) if capacity is None else np.ascontiguousarray(capacity, dtype=np.int64)
        seeds = np.zeros(B, dtype=np.uint64) if tuple_seeds is None else \
            np.ascontiguousarray([int(s) for s in tuple_seeds], dtype=np.uint64)
        if cap.shape != (B,) or seeds.shape != (B,):
            raise TzrError("match_correspondences_batch: capacity and tuple_seeds need one entry per pair")
        pairs = [np.zeros((max(int(c), 1), 2), dtype=np.int32) for c in cap]
        cnt = np.zeros(B, dtype=np.int64)
        g = np.zeros(B, dtype=np.float32)
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        arr = lambda xs: (fp * B)(*[_p(x, C.c_float) for x in xs])
        rc = lib().tzr_match_correspondences_batch(
            self._h, B, _p(ns, C.c_int32), arr(sp), _p(nd, C.c_int32), arr(tp), arr(sf), arr(tf), dim,
            int(bool(use_absolute_scale)), int(bool(use_crosscheck)), int(bool(use_tuple_test)), float(tuple_scale),
            _p(seeds, C.c_uint64), (i32p * B)(*[_p(p, C.c_int32) for p in pairs]), _p(cap, C.c_int64),
            _p(cnt, C.c_int64), _p(g, C.c_float))
        out = [p[:k].copy() if k <= c else None for p, k, c in zip(pairs, cnt, cap)]
        scales = [float(x) for x in g]
        try:
            self._ck(rc)
        except TzrError as e:
            e.n_pairs, e.result = cnt, out
            raise
        return (out, scales) if return_scale else out

    def feature_nn(self, query, db):
        """Exact 1-NN (flann::L2<float> accumulation order, lowest index among ties) of every query row in db."""
        q = np.ascontiguousarray(query, dtype=np.float32)
        d = np.ascontiguousarray(db, dtype=np.float32)
        if q.ndim != 2 or d.ndim != 2 or q.shape[1] != d.shape[1]:
            raise TzrError("feature_nn: query and db must be (n,dim) with equal dim")
        idx = np.zeros(q.shape[0], dtype=np.int32)
        dist = np.zeros(q.shape[0], dtype=np.float32)
        self._ck(lib().tzr_feature_nn(self._h, _p(q, C.c_float), q.shape[0], _p(d, C.c_float), d.shape[0], q.shape[1],
                                      _p(idx, C.c_int32), _p(dist, C.c_float)))
        return idx, dist

    # -- whole path
    def solve(self, src, dst, params: Params):
        s, d = _pts(src), _pts(dst)
        n = s.shape[0]
        sol = Solution()
        clique = np.zeros(n, dtype=np.int32)
        complete = params.rotation_tim_graph == 1
        rm = np.zeros(n * (n - 1) // 2 if complete else n, dtype=np.uint8)
        tm = np.zeros(n, dtype=np.uint8)
        self._ck(lib().tzr_solve(self._h, C.byref(params), _p(s, C.c_double), _p(d, C.c_double), n, C.byref(sol),
                                 _p(clique, C.c_int32), _p(rm, C.c_uint8), _p(tm, C.c_uint8)))
        m = sol.clique_size
        nrot = m * (m - 1) // 2 if complete else m
        return dict(sol=sol, valid=bool(sol.valid), scale=sol.scale, R=sol.R, t=sol.t, clique=clique[:m].copy(),
                    rot_inliers=rm[:nrot].astype(bool), trans_inliers=tm[:m].astype(bool),
                    gnc_iterations=sol.gnc_iterations, proven=bool(sol.clique_proven_optimal),
                    n_edges=int(sol.n_edges), stage_ms=list(sol.stage_ms))

    def solve_batch(self, srcs, dsts, params: Params):
        """srcs/dsts: lists of (N_b,3) arrays (host). Returns (solutions structured array, list of cliques)."""
        B = len(srcs)
        S = [_pts(a) for a in srcs]
        D = [_pts(a) for a in dsts]
        ns = np.array([a.shape[0] for a in S], dtype=np.int32)
        max_n = int(ns.max())
        dp = C.POINTER(C.c_double)
        sp = (dp * B)(*[_p(a, C.c_double) for a in S])
        dpp = (dp * B)(*[_p(a, C.c_double) for a in D])
        sols = np.zeros(B, dtype=SOLUTION_DTYPE)
        cl = np.zeros((B, max_n), dtype=np.int32)
        self._ck(lib().tzr_solve_batch(self._h, C.byref(params), B, _p(ns, C.c_int32), sp, dpp,
                                       sols.ctypes.data_as(C.POINTER(Solution)), _p(cl, C.c_int32), max_n))
        cliques = [cl[b, :max(0, int(sols[b]["clique_size"]))].copy() for b in range(B)]
        return sols, cliques

    def solve_batch_array(self, src, dst, params: Params, cliques_out=None, sols_out=None):
        """Batch of equally sized problems held in two (B, N, 3) float64 C-contiguous arrays (ideally page-locked,
        e.g. numpy views of torch pinned tensors: the library then DMAs straight from them and overlaps the copy
        of chunk k+1 with the kernels of chunk k).  No per-problem Python work.
        Returns (solutions structured array (B,), cliques (B, N) int32 padded, valid prefix = clique_size)."""
        src = np.asarray(src)
        dst = np.asarray(dst)
        if src.dtype != np.float64 or dst.dtype != np.float64 or src.ndim != 3 or src.shape != dst.shape or \
                src.shape[2] != 3 or not src.flags.c_contiguous or not dst.flags.c_contiguous:
            raise ValueError("src/dst must be C-contiguous float64 arrays of shape (B, N, 3)")
        B, n = src.shape[0], src.shape[1]
        stride = n * 3 * 8
        sp = (src.ctypes.data + np.arange(B, dtype=np.uint64) * np.uint64(stride)).astype(np.uint64)
        dp_ = (dst.ctypes.data + np.arange(B, dtype=np.uint64) * np.uint64(stride)).astype(np.uint64)
        ns = np.full(B, n, dtype=np.int32)
        sols = sols_out if sols_out is not None else np.zeros(B, dtype=SOLUTION_DTYPE)
        cl = cliques_out if cliques_out is not None else np.empty((B, n), dtype=np.int32)
        pp = C.POINTER(C.POINTER(C.c_double))
        self._ck(lib().tzr_solve_batch(self._h, C.byref(params), B, _p(ns, C.c_int32),
                                       C.cast(sp.ctypes.data, pp), C.cast(dp_.ctypes.data, pp),
                                       sols.ctypes.data_as(C.POINTER(Solution)), _p(cl, C.c_int32), n))
        return sols, cl

    def solve_batch_dev(self, params: Params, B: int, n: int, src_ptr: int, dst_ptr: int, sol_ptr: int,
                        clique_ptr: int = 0):
        """Device pointers (e.g. torch tensors' data_ptr()); asynchronous on the context's stream."""
        self._ck(lib().tzr_solve_batch_dev(self._h, C.byref(params), B, n, C.c_void_p(src_ptr), C.c_void_p(dst_ptr),
                                           C.c_void_p(sol_ptr), C.c_void_p(clique_ptr) if clique_ptr else None))

    def solve_batch_ragged_dev(self, params: Params, ns, src_ptr: int, dst_ptr: int, sol_ptr: int, clq_ptr: int = 0):
        """tzr_solve_batch_ragged_dev: ns[b] correspondences per problem, the problems back to back in flat (sum ns, 3)
        float64 device arrays; solutions (B records) and cliques (sum ns int32, -1 past each clique) at device pointers.
        Asynchronous on the context's stream."""
        ns = np.ascontiguousarray(ns, dtype=np.int32)
        self._ck(lib().tzr_solve_batch_ragged_dev(self._h, C.byref(params), int(ns.size), _p(ns, C.c_int32),
                                                  C.c_void_p(src_ptr), C.c_void_p(dst_ptr), C.c_void_p(sol_ptr),
                                                  C.c_void_p(clq_ptr) if clq_ptr else None))

    def last_inliers(self, b: int):
        """tzr_last_inliers: (rotation mask, translation mask) of problem b of the most recent solve on this context,
        as bool arrays (empty for a problem whose solution is not valid)."""
        n_rot, n_trans = C.c_int64(0), C.c_int32(0)
        self._ck(lib().tzr_last_inliers(self._h, int(b), None, None, C.byref(n_rot), C.byref(n_trans)))
        rot = np.zeros(max(1, n_rot.value), dtype=np.uint8)
        trans = np.zeros(max(1, n_trans.value), dtype=np.uint8)
        self._ck(lib().tzr_last_inliers(self._h, int(b), _p(rot, C.c_uint8), _p(trans, C.c_uint8), None, None))
        return rot[:n_rot.value].astype(bool), trans[:n_trans.value].astype(bool)

    @staticmethod
    def _certify_last_problems(problems):
        """certify_last's problem list as contiguous int32 (None: every problem of the retained solve)."""
        if problems is None:
            return None
        pr = np.asarray(problems)
        if pr.ndim != 1 or pr.size == 0 or not np.issubdtype(pr.dtype, np.integer):
            raise TzrError("certify_last: problems must be a non-empty 1-D sequence of integers")
        return np.ascontiguousarray(pr, dtype=np.int32)

    def certify_last(self, problems=None, **params):
        """tzr_certify_last_solve: certify problems of the most recent solve on this context (all of them, in order, by
        default), with their inputs built on the device.  noise_bound is divided by each problem's scale; pass 2x the
        solve's noise_bound to certify what the rotation solver solved.  Returns a list of dicts shaped like
        certify_batch's, plus status (0 certified, else the entry's TZR status)."""
        pr = self._certify_last_problems(problems)
        if pr is None:
            B = C.c_int32(0)
            self._ck(lib().tzr_last_graph_info(self._h, C.byref(B), None, None, None))
            count = max(1, B.value)  # 0: nothing retained, the call below reports it
        else:
            count = int(pr.size)
        p = self.certifier_params(**params)
        cap = int(max(1, np.ceil(p.max_iterations)))
        trajs = [np.zeros(cap) for _ in range(count)]
        caps = np.full(count, cap, dtype=np.int32)
        res = (CertificationResult * count)()
        status = np.zeros(count, dtype=np.int32)
        dp = C.POINTER(C.c_double)
        rc = lib().tzr_certify_last_solve(self._h, C.byref(p), count, None if pr is None else _p(pr, C.c_int32), res,
                                          _p(status, C.c_int32), (dp * count)(*[_p(t, C.c_double) for t in trajs]),
                                          _p(caps, C.c_int32))
        if rc not in (0, TZR_ERR_TOO_LARGE):
            self._ck(rc)
        return [dict(is_optimal=bool(r.is_optimal), best_suboptimality=r.best_suboptimality,
                     suboptimality_traj=t[:r.n_iterations].copy(), status=int(s))
                for r, t, s in zip(res, trajs, status)]

    def register_cloud_pairs(self, clouds, pairs, params: Params, normal_search_radius=0.03, fpfh_search_radius=0.05,
                             use_absolute_scale=True, use_crosscheck=True, use_tuple_test=True, tuple_scale=0.0,
                             tuple_seeds=None):
        """tzr_register_cloud_pairs: FPFH descriptors of every (n,3) float32 cloud, the correspondences of every
        (source cloud, target cloud) index pair, and the robust solve of every pair, chained on the device.
        tuple_seeds: one seed per pair (default 0 each).  Returns (solutions structured array (P,), status (P,) int32,
        problem_index (P,) int32 (-1: not solved), correspondences (list of (m_p,2) int32), cliques (list of sorted
        row indices into the correspondences, empty when not solved), global scales (list of floats)).  The call
        raises only for errors of the whole call; TZR_ERR_TOO_LARGE of some pairs is reported in status."""
        return self._register_pairs(clouds, pairs, params, normal_search_radius, fpfh_search_radius, use_absolute_scale,
                                    use_crosscheck, use_tuple_test, tuple_scale, tuple_seeds, None)

    def register_cloud_pairs_icp(self, clouds, pairs, params: Params, max_correspondence_distance, normal_search_radius=0.03,
                                 fpfh_search_radius=0.05, use_absolute_scale=True, use_crosscheck=True,
                                 use_tuple_test=True, tuple_scale=0.0, tuple_seeds=None, max_iteration=30,
                                 relative_fitness=1e-6, relative_rmse=1e-6, method="point_to_point", epsilon=1e-3,
                                 kernel=None, colors=None, lambda_geometric=0.968):
        """tzr_register_cloud_pairs_icp: register_cloud_pairs, then ICP of every pair with a valid solution on its two
        clouds, seeded with that solution, in the same call.  Returns register_cloud_pairs' six results plus the ICP
        records (structured array (P,) of ICP_RESULT_DTYPE, zeroed for a pair that was not refined).
        method="point_to_plane" runs point-to-plane ICP (tzr_register_cloud_pairs_icp_point_to_plane) with the target
        normals of the call's own FPFH stage; method="generalized" runs generalized ICP
        (tzr_register_cloud_pairs_icp_generalized) with both clouds' normals from that stage and the given epsilon.
        kernel (see robust_kernel(); point-to-plane and generalized only) runs the method with that robust kernel
        (tzr_register_cloud_pairs_icp_robust); None keeps the entries above.  method="colored" runs coloured ICP
        (tzr_register_cloud_pairs_icp_colored) with colors (one (n,3) array per cloud, required for this method and
        refused for the others), lambda_geometric and kernel (None: L2)."""
        if method not in ("point_to_point", "point_to_plane", "generalized", "colored"):
            raise TzrError(f"register_cloud_pairs_icp: unknown method {method!r}")
        if (colors is None) != (method != "colored"):
            raise TzrError("register_cloud_pairs_icp: colors are required by method='colored' and by no other method")
        kernel = robust_kernel(kernel)
        if kernel is not None and method == "point_to_point":
            raise TzrError("register_cloud_pairs_icp: point-to-point ICP takes no robust kernel")
        icp = icp_params(max_correspondence_distance, max_iteration=int(max_iteration),
                         relative_fitness=float(relative_fitness), relative_rmse=float(relative_rmse))
        return self._register_pairs(clouds, pairs, params, normal_search_radius, fpfh_search_radius, use_absolute_scale,
                                    use_crosscheck, use_tuple_test, tuple_scale, tuple_seeds, icp,
                                    plane=method == "point_to_plane",
                                    epsilon=float(epsilon) if method == "generalized" else None, kernel=kernel,
                                    colored=None if colors is None else (colors, float(lambda_geometric)))

    def _register_pairs(self, clouds, pairs, params, normal_search_radius, fpfh_search_radius, use_absolute_scale,
                        use_crosscheck, use_tuple_test, tuple_scale, tuple_seeds, icp, plane=False, epsilon=None,
                        kernel=None, multiway=None, colored=None):
        cl = [np.ascontiguousarray(c, dtype=np.float32) for c in clouds]
        if not cl or any(c.ndim != 2 or c.shape[1] != 3 or c.shape[0] == 0 for c in cl):
            raise TzrError("register_cloud_pairs: a non-empty list of non-empty (n,3) clouds is required")
        pc = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        P = pc.shape[0]
        if P == 0:
            raise TzrError("register_cloud_pairs: at least one pair is required")
        seeds = np.zeros(P, dtype=np.uint64) if tuple_seeds is None else \
            np.ascontiguousarray([int(s) for s in tuple_seeds], dtype=np.uint64)
        if seeds.shape != (P,):
            raise TzrError("register_cloud_pairs: tuple_seeds needs one entry per pair")
        n = np.array([c.shape[0] for c in cl], dtype=np.int32)
        if pc.min() < 0 or pc.max() >= len(cl):
            raise TzrError("register_cloud_pairs: a pair names a cloud that is not in the list")
        if colored is not None:  # (colours per cloud, lambda_geometric): the coloured entries' extra arguments
            cols, lam = colored
            if len(cols) != len(cl):
                raise TzrError("register_cloud_pairs: colors needs one (n,3) array per cloud")
            K = [_colors32(k, c.shape[0], "register_cloud_pairs") for k, c in zip(cols, cl)]
            col_args = ((C.POINTER(C.c_float) * len(cl))(*[_p(k, C.c_float) for k in K]), lam,
                        None if kernel is None else C.byref(kernel))
        fpar = FrontendParams(float(normal_search_radius), float(fpfh_search_radius), int(bool(use_absolute_scale)),
                              int(bool(use_crosscheck)), int(bool(use_tuple_test)), float(tuple_scale))
        cap = [int(n[a]) + int(n[b]) for a, b in pc]
        corr = [np.zeros((c, 2), dtype=np.int32) for c in cap]
        clq = [np.zeros(c, dtype=np.int32) for c in cap]
        sols = np.zeros(P, dtype=SOLUTION_DTYPE)
        status = np.zeros(P, dtype=np.int32)
        index = np.zeros(P, dtype=np.int32)
        cnt = np.zeros(P, dtype=np.int64)
        g = np.zeros(P, dtype=np.float32)
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        args = (self._h, C.byref(fpar), C.byref(params), len(cl), _p(n, C.c_int32),
                (fp * len(cl))(*[_p(c, C.c_float) for c in cl]), P, _p(pc, C.c_int32), _p(seeds, C.c_uint64),
                sols.ctypes.data_as(C.POINTER(Solution)), _p(status, C.c_int32), _p(index, C.c_int32),
                _p(cnt, C.c_int64), (i32p * P)(*[_p(c, C.c_int32) for c in corr]),
                (i32p * P)(*[_p(c, C.c_int32) for c in clq]), _p(g, C.c_float))
        if icp is None:
            rc = lib().tzr_register_cloud_pairs(*args)
        else:
            icp_res = np.zeros(P, dtype=ICP_RESULT_DTYPE)
            out_res = icp_res.ctypes.data_as(C.POINTER(IcpResult))
            if multiway is not None and len(multiway) == 4:  # (uncertain, params, graph offsets, map voxel size)
                rc, mw = self._multiway_batch(args, icp, out_res, n, *multiway,
                                              col_args if colored is not None else None)
            elif multiway is not None:
                unc, pg = multiway
                lp = isinstance(pg, LineProcessParams)
                unc = np.ascontiguousarray(unc, dtype=np.int32)
                if unc.shape != (P,):
                    raise TzrError("register_multiway: uncertain needs one entry per pair")
                info = np.zeros((P, 6, 6))
                icnt = np.zeros(P, dtype=np.int32)
                ew = np.zeros(P)
                em = np.zeros(P, dtype=np.uint8)
                poses = (Similarity * len(cl))()
                summ = LineProcessSummary() if lp else PoseGraphSummary()
                pg_status = C.c_int32(0)
                mw_out = (_p(unc, C.c_int32), C.byref(pg), _p(info, C.c_double), _p(icnt, C.c_int32),
                          _p(ew, C.c_double), _p(em, C.c_uint8), poses, C.byref(summ), C.byref(pg_status))
                if lp:
                    cargs = col_args if colored is not None else (None, 0.0, None)
                    rc = lib().tzr_register_cloud_pairs_multiway_line_process(*args, C.byref(icp), *cargs, out_res,
                                                                              *mw_out)
                elif colored is not None:
                    rc = lib().tzr_register_cloud_pairs_multiway_colored(*args, C.byref(icp), *col_args, out_res,
                                                                         *mw_out)
                else:
                    rc = lib().tzr_register_cloud_pairs_multiway(*args, C.byref(icp), out_res, *mw_out)
                if lp:
                    mw = dict(information=info, counts=icnt, confidence=ew, kept=em.astype(bool), poses=_poses(poses),
                              status=int(pg_status.value), **_line_process_summary(summ))
                else:
                    mw = dict(information=info, counts=icnt, weights=ew, mask=em.astype(bool), poses=_poses(poses),
                              status=int(pg_status.value), iterations=int(summ.iterations),
                              inner_iterations=int(summ.inner_iterations), cost=float(summ.cost))
            elif colored is not None:
                rc = lib().tzr_register_cloud_pairs_icp_colored(*args, C.byref(icp), *col_args, out_res)
            elif kernel is not None:
                rc = lib().tzr_register_cloud_pairs_icp_robust(*args, C.byref(icp), 1 if plane else 2,
                                                               0.0 if epsilon is None else epsilon, C.byref(kernel),
                                                               out_res)
            elif epsilon is not None:
                rc = lib().tzr_register_cloud_pairs_icp_generalized(*args, C.byref(icp), epsilon, out_res)
            else:
                entry = lib().tzr_register_cloud_pairs_icp_point_to_plane if plane else lib().tzr_register_cloud_pairs_icp
                rc = entry(*args, C.byref(icp), out_res)
        if rc not in (0, TZR_ERR_TOO_LARGE):
            self._ck(rc)
        corr = [c[:k].copy() for c, k in zip(corr, cnt)]
        clq = [c[:max(0, int(s["clique_size"]))].copy() if i >= 0 else np.zeros(0, dtype=np.int32)
               for c, s, i in zip(clq, sols, index)]
        out = (sols, status, index, corr, clq, [float(x) for x in g])
        if multiway is not None:
            return out + (icp_res, mw)
        return out if icp is None else out + (icp_res,)

    def _multiway_batch(self, args, icp, out_res, n, unc, pg, off, map_voxel_size, col_args):
        """The many-sequence entries' call over the flat table in args (_register_pairs' arguments) with the graphs at
        graph offsets off; returns (the entry's return, a dict of the per-pair outputs, poses (n_clouds,4,4) and one
        dict per graph: status, the summary's keys, and map / map_colors when map_voxel_size > 0)."""
        P, lp = len(unc), isinstance(pg, LineProcessParams)
        unc = np.ascontiguousarray(unc, dtype=np.int32)
        off = np.ascontiguousarray(off, dtype=np.int32)
        G, vox = len(off) - 1, float(map_voxel_size)
        info, icnt, ew, em = np.zeros((P, 6, 6)), np.zeros(P, dtype=np.int32), np.zeros(P), np.zeros(P, dtype=np.uint8)
        poses = (Similarity * len(n))()
        summ = ((LineProcessSummary if lp else PoseGraphSummary) * max(G, 1))()
        status, mcnt = np.zeros(max(G, 1), dtype=np.int32), np.zeros(max(G, 1), dtype=np.int32)
        tot = [int(n[off[g]:off[g + 1]].sum()) for g in range(G)] if vox > 0 and G >= 1 else []
        maps = [np.zeros((max(t, 1), 3), dtype=np.float32) for t in tot]
        mcols = [np.zeros((max(t, 1), 3), dtype=np.float32) for t in tot] if col_args is not None else []
        fp = C.POINTER(C.c_float)
        entry = lib().tzr_register_cloud_pairs_multiway_line_process_batch if lp else \
            lib().tzr_register_cloud_pairs_multiway_batch
        rc = entry(*args, C.byref(icp), *(col_args if col_args is not None else (None, 0.0, None)), out_res,
                   _p(unc, C.c_int32), C.byref(pg), _p(info, C.c_double), _p(icnt, C.c_int32), _p(ew, C.c_double),
                   _p(em, C.c_uint8), poses, summ, _p(status, C.c_int32), G, _p(off, C.c_int32), vox,
                   (fp * len(maps))(*[_p(m, C.c_float) for m in maps]) if maps else None, _p(mcnt, C.c_int32),
                   (fp * len(mcols))(*[_p(m, C.c_float) for m in mcols]) if mcols else None)
        graphs = []
        for g in range(G):
            d = dict(status=int(status[g]))
            d.update(_line_process_summary(summ[g]) if lp else
                     dict(iterations=int(summ[g].iterations), inner_iterations=int(summ[g].inner_iterations),
                          cost=float(summ[g].cost)))
            if vox > 0:
                d["map"] = maps[g][:mcnt[g]].copy()
                if col_args is not None:
                    d["map_colors"] = mcols[g][:mcnt[g]].copy()
            graphs.append(d)
        mw = dict(information=info, counts=icnt, poses=_poses(poses), graphs=graphs)
        mw.update(dict(confidence=ew, kept=em.astype(bool)) if lp else dict(weights=ew, mask=em.astype(bool)))
        return rc, mw

    def register_cloud_pairs_fgr(self, clouds, pairs, normal_search_radius=0.03, fpfh_search_radius=0.05,
                                 use_absolute_scale=True, use_crosscheck=True, use_tuple_test=True, tuple_scale=0.0,
                                 tuple_seeds=None, fgr=None):
        """tzr_register_cloud_pairs_fgr: register_cloud_pairs' front end (FPFH of every (n,3) float32 cloud, matching of
        every (source cloud, target cloud) pair), then Fast Global Registration of every pair with correspondences on
        its matched rows, with no robust solve.  fgr: an FgrParams (None: fgr_params()).  Returns (status (P,) int32,
        correspondences (list of (m_p,2) int32), global scales (list of floats), FGR records (structured array (P,) of
        ICP_RESULT_DTYPE, zeroed for a pair that was not registered)).  The call raises only for errors of the whole
        call; TZR_ERR_TOO_LARGE of some pairs is reported in status."""
        cl = [np.ascontiguousarray(c, dtype=np.float32) for c in clouds]
        if not cl or any(c.ndim != 2 or c.shape[1] != 3 or c.shape[0] == 0 for c in cl):
            raise TzrError("register_cloud_pairs_fgr: a non-empty list of non-empty (n,3) clouds is required")
        pc = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        P = pc.shape[0]
        if P == 0:
            raise TzrError("register_cloud_pairs_fgr: at least one pair is required")
        if pc.min() < 0 or pc.max() >= len(cl):
            raise TzrError("register_cloud_pairs_fgr: a pair names a cloud that is not in the list")
        seeds = np.zeros(P, dtype=np.uint64) if tuple_seeds is None else \
            np.ascontiguousarray([int(s) for s in tuple_seeds], dtype=np.uint64)
        if seeds.shape != (P,):
            raise TzrError("register_cloud_pairs_fgr: tuple_seeds needs one entry per pair")
        fgr = fgr_params() if fgr is None else fgr
        n = np.array([c.shape[0] for c in cl], dtype=np.int32)
        fpar = FrontendParams(float(normal_search_radius), float(fpfh_search_radius), int(bool(use_absolute_scale)),
                              int(bool(use_crosscheck)), int(bool(use_tuple_test)), float(tuple_scale))
        corr = [np.zeros((int(n[a]) + int(n[b]), 2), dtype=np.int32) for a, b in pc]
        status = np.zeros(P, dtype=np.int32)
        cnt = np.zeros(P, dtype=np.int64)
        g = np.zeros(P, dtype=np.float32)
        res = np.zeros(P, dtype=ICP_RESULT_DTYPE)
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        rc = lib().tzr_register_cloud_pairs_fgr(self._h, C.byref(fpar), C.byref(fgr), len(cl), _p(n, C.c_int32),
                                                (fp * len(cl))(*[_p(c, C.c_float) for c in cl]), P,
                                                _p(pc, C.c_int32), _p(seeds, C.c_uint64), _p(status, C.c_int32),
                                                _p(cnt, C.c_int64), (i32p * P)(*[_p(c, C.c_int32) for c in corr]),
                                                _p(g, C.c_float), res.ctypes.data_as(C.POINTER(IcpResult)))
        if rc not in (0, TZR_ERR_TOO_LARGE):
            self._ck(rc)
        return status, [c[:k].copy() for c, k in zip(corr, cnt)], [float(x) for x in g], res

    def register_cloud_pairs_ransac(self, clouds, pairs, ransac: RansacParams, normal_search_radius=0.03,
                                    fpfh_search_radius=0.05, use_absolute_scale=True, use_crosscheck=True,
                                    use_tuple_test=True, tuple_scale=0.0, tuple_seeds=None, ransac_seeds=None):
        """tzr_register_cloud_pairs_ransac: register_cloud_pairs' front end (FPFH of every (n,3) float32 cloud,
        matching of every (source cloud, target cloud) pair), then RANSAC of every pair with correspondences on its
        matched rows (seed ransac_seeds[p], None: 0; the normal checker reads the FPFH stage's normals), with no robust
        solve.  Returns (status (P,) int32, correspondences (list of (m_p,2) int32), global scales (list of floats),
        RANSAC records (structured array (P,) of ICP_RESULT_DTYPE), infos (structured array (P,) of
        RANSAC_INFO_DTYPE)), both zeroed for a pair that was not registered.  The call raises only for errors of the
        whole call; TZR_ERR_TOO_LARGE of some pairs is reported in status."""
        cl = [np.ascontiguousarray(c, dtype=np.float32) for c in clouds]
        if not cl or any(c.ndim != 2 or c.shape[1] != 3 or c.shape[0] == 0 for c in cl):
            raise TzrError("register_cloud_pairs_ransac: a non-empty list of non-empty (n,3) clouds is required")
        pc = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        P = pc.shape[0]
        if P == 0:
            raise TzrError("register_cloud_pairs_ransac: at least one pair is required")
        if pc.min() < 0 or pc.max() >= len(cl):
            raise TzrError("register_cloud_pairs_ransac: a pair names a cloud that is not in the list")
        seeds = _seeds64(tuple_seeds, P, "register_cloud_pairs_ransac")
        rseeds = _seeds64(ransac_seeds, P, "register_cloud_pairs_ransac")
        n = np.array([c.shape[0] for c in cl], dtype=np.int32)
        fpar = FrontendParams(float(normal_search_radius), float(fpfh_search_radius), int(bool(use_absolute_scale)),
                              int(bool(use_crosscheck)), int(bool(use_tuple_test)), float(tuple_scale))
        corr = [np.zeros((int(n[a]) + int(n[b]), 2), dtype=np.int32) for a, b in pc]
        status = np.zeros(P, dtype=np.int32)
        cnt = np.zeros(P, dtype=np.int64)
        g = np.zeros(P, dtype=np.float32)
        res = np.zeros(P, dtype=ICP_RESULT_DTYPE)
        info = np.zeros(P, dtype=RANSAC_INFO_DTYPE)
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        rc = lib().tzr_register_cloud_pairs_ransac(self._h, C.byref(fpar), C.byref(ransac), len(cl),
                                                   _p(n, C.c_int32), (fp * len(cl))(*[_p(c, C.c_float) for c in cl]),
                                                   P, _p(pc, C.c_int32), _p(seeds, C.c_uint64),
                                                   _p(rseeds, C.c_uint64), _p(status, C.c_int32),
                                                   _p(cnt, C.c_int64), (i32p * P)(*[_p(c, C.c_int32) for c in corr]),
                                                   _p(g, C.c_float), res.ctypes.data_as(C.POINTER(IcpResult)),
                                                   info.ctypes.data_as(C.POINTER(RansacInfo)))
        if rc not in (0, TZR_ERR_TOO_LARGE):
            self._ck(rc)
        return status, [c[:k].copy() for c, k in zip(corr, cnt)], [float(x) for x in g], res, info

    def register_multiway(self, clouds, pairs, params: Params, max_correspondence_distance, uncertain=None,
                          normal_search_radius=0.03, fpfh_search_radius=0.05, use_absolute_scale=True,
                          use_crosscheck=True, use_tuple_test=True, tuple_scale=0.0, tuple_seeds=None, max_iteration=30,
                          relative_fitness=1e-6, relative_rmse=1e-6, pose_graph=None, colors=None,
                          lambda_geometric=0.968, kernel=None, optimizer="gnc_tls", line_process=None):
        """tzr_register_cloud_pairs_multiway: register_cloud_pairs_icp(method="point_to_plane"), the information
        matrix of every refined pair and the GNC-TLS pose graph over the clouds, in one call.  uncertain: one flag per
        pair (None: Open3D's tutorial rule, pair (k, k + 1) certain and every other pair uncertain).  pose_graph: a
        PoseGraphParams (None: the defaults with c = max_correspondence_distance).  Returns register_cloud_pairs_icp's
        seven results plus a dict: information (P,6,6), counts (P,), weights (P,), mask (P,) bool, poses (n_clouds,4,4),
        status (the pose graph's TZR status), iterations, inner_iterations, cost.  colors (one (n,3) array per cloud)
        refines by coloured ICP instead (tzr_register_cloud_pairs_multiway_colored) with lambda_geometric and kernel
        (None: L2); a kernel without colours is refused.  optimizer="line_process" runs Open3D's line process instead of
        GNC-TLS (tzr_register_cloud_pairs_multiway_line_process) with line_process (a LineProcessParams, None: the
        defaults with c = max_correspondence_distance); its dict has confidence (P,) and kept (P,) bool in place of
        weights and mask, and global_optimization()'s summary keys in place of iterations, inner_iterations and cost."""
        if optimizer not in ("gnc_tls", "line_process"):
            raise TzrError(f"register_multiway: unknown optimizer {optimizer!r}")
        if (optimizer == "line_process" and pose_graph is not None) or (optimizer == "gnc_tls" and
                                                                        line_process is not None):
            raise TzrError(f"register_multiway: optimizer={optimizer!r} takes "
                           f"{'line_process' if optimizer == 'line_process' else 'pose_graph'}, not the other's parameters")
        kernel = robust_kernel(kernel)
        if kernel is not None and colors is None:
            raise TzrError("register_multiway: a robust kernel needs colors (coloured ICP)")
        pc = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        if uncertain is None:
            uncertain = [0 if b == a + 1 else 1 for a, b in pc]
        if optimizer == "line_process":
            pg = line_process if line_process is not None else line_process_params(max_correspondence_distance)
        else:
            pg = pose_graph if pose_graph is not None else pose_graph_params(max_correspondence_distance)
        icp = icp_params(max_correspondence_distance, max_iteration=int(max_iteration),
                         relative_fitness=float(relative_fitness), relative_rmse=float(relative_rmse))
        return self._register_pairs(clouds, pc, params, normal_search_radius, fpfh_search_radius, use_absolute_scale,
                                    use_crosscheck, use_tuple_test, tuple_scale, tuple_seeds, icp, plane=True,
                                    kernel=kernel, multiway=(uncertain, pg),
                                    colored=None if colors is None else (colors, float(lambda_geometric)))

    def register_multiway_batch(self, sequences, pairs, params: Params, max_correspondence_distance, uncertain=None,
                                normal_search_radius=0.03, fpfh_search_radius=0.05, use_absolute_scale=True,
                                use_crosscheck=True, use_tuple_test=True, tuple_scale=0.0, tuple_seeds=None,
                                max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, pose_graph=None,
                                colors=None, lambda_geometric=0.968, kernel=None, optimizer="gnc_tls",
                                line_process=None, map_voxel_size=0.0):
        """tzr_register_cloud_pairs_multiway(_line_process)_batch: register_multiway over many scan sequences in one
        call, every sequence's pose graph in the batched pose-graph kernels.  sequences: one list of (n,3) clouds per
        sequence; pairs: one list of local (s, d) pairs per sequence; uncertain, tuple_seeds and colors: None or one
        list per sequence (uncertain None: register_multiway's rule per sequence).  The other arguments as
        register_multiway's.  map_voxel_size > 0 also fuses each solved sequence's clouds into one map (every cloud
        by its pose, concatenated, voxel-downsampled).  Returns one result per sequence, shaped like
        register_multiway's: its pairs' seven registration results (problem_index counted within the sequence) plus
        a dict with its pairs' information, counts, weights and mask (or confidence and kept), its poses, status and
        summary keys, and map / map_colors when a map was asked for (empty for a refused sequence)."""
        flat = multiway_batch_table(sequences, pairs, uncertain, tuple_seeds, colors)
        if optimizer not in ("gnc_tls", "line_process"):
            raise TzrError(f"register_multiway_batch: unknown optimizer {optimizer!r}")
        if (optimizer == "line_process" and pose_graph is not None) or (optimizer == "gnc_tls" and
                                                                        line_process is not None):
            raise TzrError(f"register_multiway_batch: optimizer={optimizer!r} takes "
                           f"{'line_process' if optimizer == 'line_process' else 'pose_graph'}, not the other's parameters")
        kernel = robust_kernel(kernel)
        if kernel is not None and colors is None:
            raise TzrError("register_multiway_batch: a robust kernel needs colors (coloured ICP)")
        if optimizer == "line_process":
            pg = line_process if line_process is not None else line_process_params(max_correspondence_distance)
        else:
            pg = pose_graph if pose_graph is not None else pose_graph_params(max_correspondence_distance)
        icp = icp_params(max_correspondence_distance, max_iteration=int(max_iteration),
                         relative_fitness=float(relative_fitness), relative_rmse=float(relative_rmse))
        out = self._register_pairs(flat["clouds"], flat["pairs"], params, normal_search_radius, fpfh_search_radius,
                                   use_absolute_scale, use_crosscheck, use_tuple_test, tuple_scale, flat["tuple_seeds"],
                                   icp, plane=True, kernel=kernel,
                                   multiway=(flat["uncertain"], pg, flat["offsets"], float(map_voxel_size)),
                                   colored=None if colors is None else (flat["colors"], float(lambda_geometric)))
        return split_multiway_batch(out, flat["pair_offsets"], flat["offsets"])

    def information_matrix(self, src, dst, transform, max_correspondence_distance):
        """tzr_information_matrix: (Lambda (6,6) float64, count) of the (ns,3) source at transform (see similarity())
        against the (nd,3) target."""
        S, D = _cloud32(src, "information_matrix"), _cloud32(dst, "information_matrix")
        info = np.zeros((6, 6))
        cnt = C.c_int32(0)
        tr = similarity(transform)
        self._ck(lib().tzr_information_matrix(self._h, _p(S, C.c_float), S.shape[0], _p(D, C.c_float), D.shape[0],
                                              C.byref(tr), float(max_correspondence_distance), _p(info, C.c_double),
                                              C.byref(cnt)))
        return info, int(cnt.value)

    def information_matrix_batch(self, srcs, dsts, transforms, max_correspondence_distance):
        """tzr_information_matrix_batch over B pairs: (Lambda (B,6,6), counts (B,) int32)."""
        S = [_cloud32(a, "information_matrix_batch") for a in srcs]
        D = [_cloud32(a, "information_matrix_batch") for a in dsts]
        B = len(S)
        if B == 0 or len(D) != B or len(transforms) != B:
            raise TzrError("information_matrix_batch: one target and one transform per source are required")
        ns = np.array([a.shape[0] for a in S], dtype=np.int32)
        nd = np.array([a.shape[0] for a in D], dtype=np.int32)
        fp = C.POINTER(C.c_float)
        tr = (Similarity * B)(*[similarity(x) for x in transforms])
        info = np.zeros((B, 6, 6))
        cnt = np.zeros(B, dtype=np.int32)
        self._ck(lib().tzr_information_matrix_batch(self._h, B, _p(ns, C.c_int32), (fp * B)(*[_p(a, C.c_float) for a in S]),
                                                    _p(nd, C.c_int32), (fp * B)(*[_p(a, C.c_float) for a in D]), tr,
                                                    float(max_correspondence_distance), _p(info, C.c_double),
                                                    _p(cnt, C.c_int32)))
        return info, cnt

    def optimize_pose_graph(self, K, edges, transforms, information, max_correspondence_distance, uncertain=None,
                            initial_poses=None, **params):
        """tzr_pose_graph_optimize: K nodes, edges (E,2) (s, d), transforms (E rigid T_sd: (4,4) matrices or anything
        similarity() takes), information (E,6,6), uncertain (E flags, None: every edge certain), initial_poses (K, None:
        breadth-first from the reference node); params: any PoseGraphParams field.  Returns a dict: poses (K,4,4),
        weights (E,), mask (E,) bool, residuals (E,) r-bar, iterations, inner_iterations, cost."""
        a = _GraphBatch([dict(K=K, edges=edges, transforms=transforms, information=information, uncertain=uncertain,
                              initial_poses=initial_poses)], "optimize_pose_graph")
        pg = pose_graph_params(max_correspondence_distance, **params)
        summ = PoseGraphSummary()
        self._ck(lib().tzr_pose_graph_optimize(self._h, C.byref(pg), *a.one(), C.byref(summ)))
        return _pose_graph_result(a.outs[0], summ)

    def global_optimization(self, K, edges, transforms, information, max_correspondence_distance, uncertain=None,
                            initial_poses=None, **params):
        """tzr_pose_graph_optimize_line_process: Open3D's global_optimization with the Levenberg-Marquardt line process.
        Arguments as optimize_pose_graph's; params: any LineProcessParams field.  Returns a dict: poses (K,4,4),
        confidence (E,), kept (E,) bool, residuals (E,) zeta^T Lambda zeta, and per pass iterations, trials,
        stop_reason (TZR_LP_STOP_*, see LP_STOP) and mu (2-lists), pruned, residual (the final F)."""
        a = _GraphBatch([dict(K=K, edges=edges, transforms=transforms, information=information, uncertain=uncertain,
                              initial_poses=initial_poses)], "global_optimization")
        lp = line_process_params(max_correspondence_distance, **params)
        summ = LineProcessSummary()
        self._ck(lib().tzr_pose_graph_optimize_line_process(self._h, C.byref(lp), *a.one(), C.byref(summ)))
        return _line_process_result(a.outs[0], summ)

    def optimize_pose_graph_batch(self, graphs, max_correspondence_distance, **params):
        """tzr_pose_graph_optimize_batch: many GNC-TLS graphs, one PoseGraphParams (params: any of its fields).  graphs
        as global_optimization_batch's.  Returns one dict per graph as optimize_pose_graph returns, plus status (the
        single entry's return on that graph; a refused graph's outputs are zero).  Raises only on call-level
        refusals."""
        pg = pose_graph_params(max_correspondence_distance, **params)
        a = _GraphBatch(graphs, "optimize_pose_graph_batch")
        summ = (PoseGraphSummary * a.P)()
        self._ck(lib().tzr_pose_graph_optimize_batch(self._h, C.byref(pg), *a.args(), summ, a.status_p))
        return [dict(_pose_graph_result(out, summ[g]), status=int(a.status[g])) for g, out in enumerate(a.outs)]

    def global_optimization_batch(self, graphs, max_correspondence_distance, **params):
        """tzr_pose_graph_optimize_line_process_batch: many graphs, one LineProcessParams (params: any of its fields).
        graphs: dicts with K, edges, transforms, information and optionally uncertain and initial_poses (None or absent:
        the single entry's default).  Returns one dict per graph as global_optimization returns, plus status (the single
        entry's return on that graph; a refused graph's outputs are zero).  Raises only on call-level refusals."""
        lp = line_process_params(max_correspondence_distance, **params)
        a = _GraphBatch(graphs, "global_optimization_batch")
        summ = (LineProcessSummary * a.P)()
        self._ck(lib().tzr_pose_graph_optimize_line_process_batch(self._h, C.byref(lp), *a.args(), summ, a.status_p))
        return [dict(_line_process_result(out, summ[g]), status=int(a.status[g])) for g, out in enumerate(a.outs)]

    def dense_cholesky_batch(self, A, b, x_out=None):
        """tzr_dense_cholesky_batch: the batched pose-graph routes' Cholesky factorisation and solve on given matrices.
        A: G square float64 arrays (only the lower triangle is factored), b: G vectors.  x_out: G contiguous float64
        vectors the solutions are written into (None: NaN-filled ones); a matrix whose factorisation fails leaves its
        vector untouched.  Returns (factors, x, info): factors[g] the whole returned array (L in the lower triangle, the
        strict upper triangle as given), x the x_out vectors, info (G,) int32: 0 or 1 + the failed column."""
        G = len(A)
        if len(b) != G or (x_out is not None and len(x_out) != G):
            raise TzrError("dense_cholesky_batch: one b (and one x_out) per matrix is required")
        mats = [np.asfortranarray(a, dtype=np.float64) for a in A]  # column-major
        ns = np.array([m.shape[0] for m in mats], dtype=np.int32)
        if any(m.ndim != 2 or m.shape[0] != m.shape[1] for m in mats):
            raise TzrError("dense_cholesky_batch: every matrix must be square")
        bs = [np.ascontiguousarray(v, dtype=np.float64).reshape(int(k)) for v, k in zip(b, ns)]
        xs = [np.full(int(k), np.nan) for k in ns] if x_out is None else list(x_out)
        if any(x.dtype != np.float64 or not x.flags.c_contiguous or x.shape != (k,) for x, k in zip(xs, ns)):
            raise TzrError("dense_cholesky_batch: x_out needs one contiguous float64 vector of n entries per matrix")
        out = [np.empty((k, k), order="F") for k in ns]
        info = np.zeros(max(1, G), dtype=np.int32)
        dpp = C.POINTER(C.c_double) * max(1, G)
        self._ck(lib().tzr_dense_cholesky_batch(self._h, G, _p(ns, C.c_int32), dpp(*[_p(m, C.c_double) for m in mats]),
                                                dpp(*[_p(v, C.c_double) for v in bs]),
                                                dpp(*[_p(m, C.c_double) for m in out]),
                                                dpp(*[_p(x, C.c_double) for x in xs]), _p(info, C.c_int32)))
        return out, xs, info[:G]

    def icp(self, src, dst, max_correspondence_distance, init=None, max_iteration=30, relative_fitness=1e-6,
            relative_rmse=1e-6):
        """tzr_icp: point-to-point ICP of the (ns,3) source onto the (nd,3) target (float32), seeded with init (see
        similarity(); None = identity; its scale stays fixed).  Returns (result dict as icp_result_dict, final
        correspondences (m,2) int32 rows (source index, target index) ascending by source)."""
        res, corr = self.icp_batch([src], [dst], max_correspondence_distance, None if init is None else [init],
                                   max_iteration=max_iteration, relative_fitness=relative_fitness,
                                   relative_rmse=relative_rmse, single=True)
        return icp_result_dict(res[0]), corr[0]

    def fgr(self, src, dst, corr, fgr=None):
        """tzr_fgr: Fast Global Registration of the (ns,3) source onto the (nd,3) target (float32) on the (K,2)
        correspondences corr (source index, target index).  fgr: an FgrParams (None: fgr_params()).  Returns (result
        dict as icp_result_dict, the evaluation's correspondences (m,2) int32 ascending by source)."""
        res, ev = self.fgr_batch([src], [dst], [corr], fgr=fgr, single=True)
        return icp_result_dict(res[0]), ev[0]

    def fgr_batch(self, srcs, dsts, corrs, fgr=None, single=False):
        """tzr_fgr_batch over B (source, target, correspondences) problems; corrs: one (K_b,2) integer array per
        problem (K_b = 0 allowed).  Returns (results structured array (B,) of ICP_RESULT_DTYPE, list of B evaluation
        correspondence arrays).  single=True goes through tzr_fgr (B must be 1)."""
        S = [_cloud32(a, "fgr") for a in srcs]
        D = [_cloud32(a, "fgr") for a in dsts]
        B = len(S)
        if B == 0 or len(D) != B or len(corrs) != B:
            raise TzrError("fgr_batch: one target and one correspondence array per source cloud are required")
        K = [corr_rows(c, "fgr_batch") for c in corrs]
        fgr = fgr_params() if fgr is None else fgr
        res = np.zeros(B, dtype=ICP_RESULT_DTYPE)
        out = res.ctypes.data_as(C.POINTER(IcpResult))
        ev = [np.zeros((a.shape[0], 2), dtype=np.int32) for a in S]
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        if single:
            assert B == 1
            rc = lib().tzr_fgr(self._h, C.byref(fgr), _p(S[0], C.c_float), S[0].shape[0], _p(D[0], C.c_float),
                               D[0].shape[0], K[0].shape[0], _p(K[0], C.c_int32), out, _p(ev[0], C.c_int32))
        else:
            ns = np.array([a.shape[0] for a in S], dtype=np.int32)
            nd = np.array([a.shape[0] for a in D], dtype=np.int32)
            nc = np.array([k.shape[0] for k in K], dtype=np.int32)
            rc = lib().tzr_fgr_batch(self._h, C.byref(fgr), B, _p(ns, C.c_int32),
                                     (fp * B)(*[_p(a, C.c_float) for a in S]), _p(nd, C.c_int32),
                                     (fp * B)(*[_p(a, C.c_float) for a in D]), _p(nc, C.c_int32),
                                     (i32p * B)(*[_p(k, C.c_int32) for k in K]), out,
                                     (i32p * B)(*[_p(e, C.c_int32) for e in ev]))
        self._ck(rc)
        return res, [e[:int(r["n_correspondences"])].copy() for e, r in zip(ev, res)]

    def ransac(self, src, dst, corr, ransac: RansacParams, seed=0, src_normals=None, dst_normals=None):
        """tzr_ransac: correspondence RANSAC of the (ns,3) source onto the (nd,3) target (float32) on the (K,2)
        correspondences corr (source index, target index), with a 64-bit seed; the normals ((n,3) or (n,4)) are
        needed by the normal checker only.  Returns (result dict as icp_result_dict, info dict (RANSAC_INFO_DTYPE's
        fields), the evaluation's correspondences (m,2) int32 ascending by source)."""
        res, info, ev = self.ransac_batch([src], [dst], [corr], ransac, seeds=[seed],
                                          src_normals=None if src_normals is None else [src_normals],
                                          dst_normals=None if dst_normals is None else [dst_normals], single=True)
        return icp_result_dict(res[0]), {k: info[0][k].item() for k in RANSAC_INFO_DTYPE.names}, ev[0]

    def ransac_batch(self, srcs, dsts, corrs, ransac: RansacParams, seeds=None, src_normals=None, dst_normals=None,
                     single=False):
        """tzr_ransac_batch over B (source, target, correspondences) problems; corrs: one (K_b,2) integer array per
        problem (K_b = 0 allowed); seeds: B 64-bit seeds (None: 0); src_normals, dst_normals: B arrays each, or None.
        Returns (results structured array (B,) of ICP_RESULT_DTYPE, infos structured array (B,) of RANSAC_INFO_DTYPE,
        list of B evaluation correspondence arrays).  single=True goes through tzr_ransac (B must be 1)."""
        S = [_cloud32(a, "ransac") for a in srcs]
        D = [_cloud32(a, "ransac") for a in dsts]
        B = len(S)
        if B == 0 or len(D) != B or len(corrs) != B:
            raise TzrError("ransac_batch: one target and one correspondence array per source cloud are required")
        K = [corr_rows(c, "ransac_batch") for c in corrs]
        sd = _seeds64(seeds, B, "ransac_batch")
        SN = None if src_normals is None else [_normals32(a, s.shape[0], "ransac") for a, s in zip(src_normals, S)]
        DN = None if dst_normals is None else [_normals32(a, d.shape[0], "ransac") for a, d in zip(dst_normals, D)]
        if (SN is not None and len(SN) != B) or (DN is not None and len(DN) != B):
            raise TzrError("ransac_batch: one normals array per problem is required")
        res = np.zeros(B, dtype=ICP_RESULT_DTYPE)
        info = np.zeros(B, dtype=RANSAC_INFO_DTYPE)
        out = res.ctypes.data_as(C.POINTER(IcpResult))
        iout = info.ctypes.data_as(C.POINTER(RansacInfo))
        ev = [np.zeros((a.shape[0], 2), dtype=np.int32) for a in S]
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        if single:
            assert B == 1
            rc = lib().tzr_ransac(self._h, C.byref(ransac), _p(S[0], C.c_float), S[0].shape[0], _p(D[0], C.c_float),
                                  D[0].shape[0], K[0].shape[0], _p(K[0], C.c_int32), int(sd[0]),
                                  None if SN is None else _p(SN[0], C.c_float),
                                  None if DN is None else _p(DN[0], C.c_float), out, iout, _p(ev[0], C.c_int32))
        else:
            ns = np.array([a.shape[0] for a in S], dtype=np.int32)
            nd = np.array([a.shape[0] for a in D], dtype=np.int32)
            nc = np.array([k.shape[0] for k in K], dtype=np.int32)
            rc = lib().tzr_ransac_batch(self._h, C.byref(ransac), B, _p(ns, C.c_int32),
                                        (fp * B)(*[_p(a, C.c_float) for a in S]), _p(nd, C.c_int32),
                                        (fp * B)(*[_p(a, C.c_float) for a in D]), _p(nc, C.c_int32),
                                        (i32p * B)(*[_p(k, C.c_int32) for k in K]), _p(sd, C.c_uint64),
                                        None if SN is None else (fp * B)(*[_p(a, C.c_float) for a in SN]),
                                        None if DN is None else (fp * B)(*[_p(a, C.c_float) for a in DN]), out, iout,
                                        (i32p * B)(*[_p(e, C.c_int32) for e in ev]))
        self._ck(rc)
        return res, info, [e[:int(r["n_correspondences"])].copy() for e, r in zip(ev, res)]

    def icp_point_to_plane(self, src, dst, dst_normals, max_correspondence_distance, init=None, max_iteration=30,
                           relative_fitness=1e-6, relative_rmse=1e-6, kernel=None):
        """tzr_icp_point_to_plane: icp() with point-to-plane updates; dst_normals: (nd,3) or (nd,4) float32 target
        normals (e.g. estimate_normals(dst)), used as given.  kernel (see robust_kernel()): the robust kernel, through
        tzr_icp_point_to_plane_robust_batch with B = 1.  Returns what icp() returns."""
        res, corr = self.icp_point_to_plane_batch([src], [dst], [dst_normals], max_correspondence_distance,
                                                  None if init is None else [init], max_iteration=max_iteration,
                                                  relative_fitness=relative_fitness, relative_rmse=relative_rmse,
                                                  single=True, kernel=kernel)
        return icp_result_dict(res[0]), corr[0]

    def icp_point_to_plane_batch(self, srcs, dsts, dst_normals, max_correspondence_distance, inits=None,
                                 max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, single=False,
                                 kernel=None):
        """tzr_icp_point_to_plane_batch: icp_batch() with point-to-plane updates and one (nd_b,3) or (nd_b,4) normals
        array per target.  single=True goes through tzr_icp_point_to_plane (B must be 1).  kernel (see
        robust_kernel()): the robust kernel, through tzr_icp_point_to_plane_robust_batch."""
        return self._icp(srcs, dsts, dst_normals, max_correspondence_distance, inits, max_iteration, relative_fitness,
                         relative_rmse, single, kernel=robust_kernel(kernel))

    def icp_generalized(self, src, dst, src_normals, dst_normals, max_correspondence_distance, init=None, epsilon=1e-3,
                        max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, kernel=None):
        """tzr_icp_generalized: icp() with generalized-ICP updates; src_normals / dst_normals: (n,3) or (n,4) float32
        normals of each cloud (e.g. estimate_normals()), used as given; epsilon: the covariances' epsilon (finite,
        > 0).  kernel (see robust_kernel()): the robust kernel, through tzr_icp_generalized_robust_batch with B = 1.
        Returns what icp() returns."""
        res, corr = self.icp_generalized_batch([src], [dst], [src_normals], [dst_normals], max_correspondence_distance,
                                               None if init is None else [init], epsilon=epsilon,
                                               max_iteration=max_iteration, relative_fitness=relative_fitness,
                                               relative_rmse=relative_rmse, single=True, kernel=kernel)
        return icp_result_dict(res[0]), corr[0]

    def icp_generalized_batch(self, srcs, dsts, src_normals, dst_normals, max_correspondence_distance, inits=None,
                              epsilon=1e-3, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6,
                              single=False, kernel=None):
        """tzr_icp_generalized_batch: icp_batch() with generalized-ICP updates and one (n,3) or (n,4) normals array per
        source and per target.  single=True goes through tzr_icp_generalized (B must be 1).  kernel (see
        robust_kernel()): the robust kernel, through tzr_icp_generalized_robust_batch."""
        if len(src_normals) != len(srcs):
            raise TzrError("icp_generalized_batch: one normals array per source cloud is required")
        SN = [_normals32(a, _cloud32(s, "icp").shape[0], "icp_generalized") for a, s in zip(src_normals, srcs)]
        return self._icp(srcs, dsts, dst_normals, max_correspondence_distance, inits, max_iteration, relative_fitness,
                         relative_rmse, single, src_normals=SN, epsilon=float(epsilon), kernel=robust_kernel(kernel))

    def icp_batch(self, srcs, dsts, max_correspondence_distance, inits=None, max_iteration=30, relative_fitness=1e-6,
                  relative_rmse=1e-6, single=False):
        """tzr_icp_batch over B (source, target) cloud pairs; inits: B seeds (None = identity for all).  Returns
        (results structured array (B,) of ICP_RESULT_DTYPE, list of B correspondence arrays).  single=True goes through
        tzr_icp (B must be 1)."""
        return self._icp(srcs, dsts, None, max_correspondence_distance, inits, max_iteration, relative_fitness,
                         relative_rmse, single)

    def _icp(self, srcs, dsts, normals, max_correspondence_distance, inits, max_iteration, relative_fitness,
             relative_rmse, single, src_normals=None, epsilon=None, kernel=None):
        """icp_batch (normals None), icp_point_to_plane_batch and icp_generalized_batch (src_normals: (n,4) float32
        arrays, epsilon given); a RobustKernel goes through the robust batch entries, also for single=True."""
        S = [_cloud32(a, "icp") for a in srcs]
        D = [_cloud32(a, "icp") for a in dsts]
        B = len(S)
        if B == 0 or len(D) != B or (inits is not None and len(inits) != B) or (normals is not None and len(normals) != B):
            raise TzrError("icp_batch: one target, one seed (and one normals array) per source cloud are required")
        N = None if normals is None else [_normals32(a, d.shape[0], "icp_point_to_plane") for a, d in zip(normals, D)]
        p = icp_params(max_correspondence_distance, max_iteration=int(max_iteration),
                       relative_fitness=float(relative_fitness), relative_rmse=float(relative_rmse))
        init = (Similarity * B)(*[similarity(None if inits is None else x) for x in inits or [None] * B])
        res = (IcpResult * B)()
        corr = [np.zeros((a.shape[0], 2), dtype=np.int32) for a in S]
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        if single and kernel is None:
            assert B == 1
            head = (self._h, C.byref(p), _p(S[0], C.c_float), S[0].shape[0], _p(D[0], C.c_float), D[0].shape[0])
            tail = (init, res, _p(corr[0], C.c_int32))
            if src_normals is not None:
                rc = lib().tzr_icp_generalized(self._h, C.byref(p), epsilon, head[2], head[3],
                                               _p(src_normals[0], C.c_float), *head[4:], _p(N[0], C.c_float), *tail)
            else:
                rc = lib().tzr_icp(*head, *tail) if N is None else \
                    lib().tzr_icp_point_to_plane(*head, _p(N[0], C.c_float), *tail)
        else:
            ns = np.array([a.shape[0] for a in S], dtype=np.int32)
            nd = np.array([a.shape[0] for a in D], dtype=np.int32)
            head = (self._h, C.byref(p), B, _p(ns, C.c_int32), (fp * B)(*[_p(a, C.c_float) for a in S]),
                    _p(nd, C.c_int32), (fp * B)(*[_p(a, C.c_float) for a in D]))
            tail = (init, res, (i32p * B)(*[_p(c, C.c_int32) for c in corr]))
            if kernel is not None:
                tail = tail + (C.byref(kernel),)
            if kernel is not None and src_normals is not None:
                rc = lib().tzr_icp_generalized_robust_batch(self._h, C.byref(p), epsilon, B, head[3], head[4],
                                                            (fp * B)(*[_p(a, C.c_float) for a in src_normals]),
                                                            *head[5:], (fp * B)(*[_p(a, C.c_float) for a in N]), *tail)
            elif kernel is not None:
                rc = lib().tzr_icp_point_to_plane_robust_batch(*head, (fp * B)(*[_p(a, C.c_float) for a in N]), *tail)
            elif src_normals is not None:
                rc = lib().tzr_icp_generalized_batch(self._h, C.byref(p), epsilon, B, head[3], head[4],
                                                     (fp * B)(*[_p(a, C.c_float) for a in src_normals]), *head[5:],
                                                     (fp * B)(*[_p(a, C.c_float) for a in N]), *tail)
            else:
                rc = lib().tzr_icp_batch(*head, *tail) if N is None else \
                    lib().tzr_icp_point_to_plane_batch(*head, (fp * B)(*[_p(a, C.c_float) for a in N]), *tail)
        self._ck(rc)
        out = np.frombuffer(bytes(res), dtype=ICP_RESULT_DTYPE).copy()
        return out, [c[:int(r["n_correspondences"])].copy() for c, r in zip(corr, out)]

    def icp_multiscale(self, clouds, pairs, scales, inits=None, method="point_to_plane", colors=None,
                       lambda_geometric=0.968, epsilon=1e-3, kernel=None, information=False):
        """tzr_icp_multiscale_batch: coarse-to-fine ICP of P cloud pairs over S scales in one call.  clouds: (n_c,3)
        float32 arrays; pairs: (P,2) (source cloud, target cloud); scales: S entries for icp_scale() (dicts or tuples);
        inits: P seeds for similarity() (None: identity), e.g. register_cloud_pairs' solutions; method: a name of
        ICP_METHODS or its number; colors: one (n_c,3) array per cloud (read by coloured ICP only, ignored otherwise
        as the library ignores them); inits may be a list, a SOLUTION_DTYPE array or a (P,4,4) array; kernel: see
        robust_kernel().  Returns (results (P,S) ICP_RESULT_DTYPE, n_down (n_clouds,S) int32), and with information
        (Lambda (P,6,6), counts (P,)) after them.  A TzrError for TZR_ERR_TOO_LARGE carries `status` (n_clouds,S) and
        `result` (what the call returns, zeroed where the contract says)."""
        pts = [_cloud32(p, "icp_multiscale") for p in clouds]
        K = len(pts)
        pc = np.ascontiguousarray(pairs, dtype=np.int32)
        if K == 0 or pc.ndim != 2 or pc.shape[1] != 2 or pc.shape[0] == 0:
            raise TzrError("icp_multiscale: a non-empty list of clouds and a (P,2) array of pairs are required")
        P = pc.shape[0]
        if pc.min() < 0 or pc.max() >= K:
            raise TzrError("icp_multiscale: a pair names a cloud outside the list")
        sc = [icp_scale(x) for x in scales]
        S = len(sc)
        if S == 0:
            raise TzrError("icp_multiscale: at least one scale is required")
        m = ICP_METHODS.get(method) if isinstance(method, str) else method
        if m not in ICP_METHODS.values():
            raise TzrError(f"icp_multiscale: unknown method {method!r} (one of {sorted(ICP_METHODS)})")
        if m != ICP_METHODS["colored"]:
            colors = None  # read by coloured ICP only, as the library reads them
        elif colors is None:
            raise TzrError("icp_multiscale: colours are required for coloured ICP")
        if colors is not None and len(colors) != K:
            raise TzrError("icp_multiscale: one colours array per cloud is required")
        if inits is not None and len(inits) != P:
            raise TzrError("icp_multiscale: one seed per pair is required")
        kern = robust_kernel(kernel)
        if kern is not None and m == ICP_METHODS["point_to_point"]:
            raise TzrError("icp_multiscale: point-to-point ICP takes no robust kernel")
        KC = None if colors is None else [_colors32(c, p.shape[0], "icp_multiscale") for c, p in zip(colors, pts)]
        n = np.array([p.shape[0] for p in pts], dtype=np.int32)
        init = (Similarity * P)(*[similarity(x) for x in (inits if inits is not None else [None] * P)])
        res = (IcpResult * (P * S))()
        n_down = np.zeros((K, S), dtype=np.int32)
        status = np.zeros((K, S), dtype=np.int32)
        info = np.zeros((P, 6, 6)) if information else None
        cnt = np.zeros(P, dtype=np.int32) if information else None
        fp = C.POINTER(C.c_float)
        rc = lib().tzr_icp_multiscale_batch(
            self._h, int(m), S, (IcpScale * S)(*sc), K, _p(n, C.c_int32), (fp * K)(*[_p(p, C.c_float) for p in pts]),
            None if KC is None else (fp * K)(*[_p(c, C.c_float) for c in KC]), P, _p(pc, C.c_int32), init,
            float(epsilon), float(lambda_geometric), C.byref(kern) if kern is not None else None, res,
            _p(n_down, C.c_int32), _p(status, C.c_int32), None if info is None else _p(info, C.c_double),
            None if cnt is None else _p(cnt, C.c_int32))
        out = np.frombuffer(bytes(res), dtype=ICP_RESULT_DTYPE).copy().reshape(P, S)
        result = (out, n_down) + ((info, cnt) if information else ())
        try:
            self._ck(rc)
        except TzrError as e:
            e.status, e.result = status, result
            raise
        return result

    def voxel_downsample(self, pts, voxel_size, return_trace=False, colors=None):
        """tzr_voxel_downsample: Open3D's voxel_down_sample of one (n,3) float32 cloud (the definition is
        include/teaser_b200.h's): the (m,3) float32 voxel means ordered by each voxel's first member, and with
        return_trace the (n,) int32 output row of every input point (-1: a non-finite point).  colors ((n,3), through
        tzr_voxel_downsample_colors): the (m,3) float32 colour means are returned after the points."""
        p = _cloud32(pts, "voxel_downsample")
        K = None if colors is None else _colors32(colors, p.shape[0], "voxel_downsample")
        out = np.zeros_like(p)
        cout = None if K is None else np.zeros_like(p)
        trace = np.zeros(p.shape[0], dtype=np.int32)
        m = np.zeros(1, dtype=np.int32)
        args = (self._h, _p(p, C.c_float), p.shape[0], float(voxel_size), _p(out, C.c_float), _p(m, C.c_int32),
                _p(trace, C.c_int32) if return_trace else None)
        if K is None:
            self._ck(lib().tzr_voxel_downsample(*args))
        else:
            self._ck(lib().tzr_voxel_downsample_colors(*args, _p(K, C.c_float), _p(cout, C.c_float)))
        res = [out[:int(m[0])].copy()]
        if K is not None:
            res.append(cout[:int(m[0])].copy())
        if return_trace:
            res.append(trace)
        return res[0] if len(res) == 1 else tuple(res)

    def voxel_downsample_batch(self, pts_list, voxel_size, return_trace=False, colors=None):
        """voxel_downsample of every (n_b,3) cloud of the list in one call (tzr_voxel_downsample_batch): a list of
        (m_b,3) voxel means (and a list of traces), each bit-identical to voxel_downsample on that cloud alone.  colors
        (one (n_b,3) array per cloud, through tzr_voxel_downsample_colors_batch): a list of colour means follows the
        points.  When a cloud's grid is too large the TzrError carries `status` (per cloud 0 or the error code) and
        `result` (the outputs of every cloud, written for the others; empty for the too-large ones)."""
        pts = [_cloud32(p, "voxel_downsample_batch") for p in pts_list]
        if not pts:
            raise TzrError("voxel_downsample_batch: a non-empty list of (n,3) clouds is required")
        B = len(pts)
        if colors is not None and len(colors) != B:
            raise TzrError("voxel_downsample_batch: one colours array per cloud is required")
        K = None if colors is None else [_colors32(c, p.shape[0], "voxel_downsample_batch") for c, p in zip(colors, pts)]
        n = np.array([p.shape[0] for p in pts], dtype=np.int32)
        outs = [np.zeros_like(p) for p in pts]
        couts = None if K is None else [np.zeros_like(p) for p in pts]
        traces = [np.zeros(p.shape[0], dtype=np.int32) for p in pts] if return_trace else None
        m = np.zeros(B, dtype=np.int32)
        status = np.zeros(B, dtype=np.int32)
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        args = (self._h, B, _p(n, C.c_int32), (fp * B)(*[_p(p, C.c_float) for p in pts]), float(voxel_size),
                (fp * B)(*[_p(o, C.c_float) for o in outs]), _p(m, C.c_int32),
                (i32p * B)(*[_p(t, C.c_int32) for t in traces]) if traces else None, _p(status, C.c_int32))
        if K is None:
            rc = lib().tzr_voxel_downsample_batch(*args)
        else:
            rc = lib().tzr_voxel_downsample_colors_batch(*args, (fp * B)(*[_p(c, C.c_float) for c in K]),
                                                         (fp * B)(*[_p(c, C.c_float) for c in couts]))
        outs = [o[:int(k)].copy() for o, k in zip(outs, m)]
        res = [outs]
        if K is not None:
            res.append([o[:int(k)].copy() for o, k in zip(couts, m)])
        if return_trace:
            res.append(traces)
        result = res[0] if len(res) == 1 else tuple(res)
        try:
            self._ck(rc)
        except TzrError as e:
            e.status, e.result = status, result
            raise
        return result

    def last_graph(self, b: int, n: int):
        W = lib().tzr_words_per_row(n)
        bits = np.zeros((n, W), dtype=np.uint64)
        deg = np.zeros(n, dtype=np.int32)
        self._ck(lib().tzr_last_graph(self._h, b, _p(bits, C.c_uint64), _p(deg, C.c_int32)))
        return bits, deg

    def last_filter_consts(self, b: int):
        """Graph filter constants of problem b of the most recent solve: box centres, the Gram tests' constants (float32)
        and which paths the problem takes."""
        cen = np.zeros(6, dtype=np.float64)
        g = np.zeros(7, dtype=np.float32)
        paths = np.zeros(2, dtype=np.int32)
        self._ck(lib().tzr_last_filter_consts(self._h, b, _p(cen, C.c_double), _p(g, C.c_float), _p(paths, C.c_int32)))
        return dict(cs=cen[:3], cd=cen[3:], mhi=g[0], chi=g[1], mlo=g[2], clo=g[3], cu=g[4], cv=g[5], dl=g[6],
                    use_fp64=bool(paths[0]), use_gram=bool(paths[1]))


def rotation_from_solution_record(rec) -> np.ndarray:
    return np.asarray(rec["rotation"]).reshape(3, 3).T.copy()


def solve_batch_multi(src_list, dst_list, params: Params, devices=None):
    """tzr_solve_batch_multi: one host call, the batch sharded over several GPUs inside the library (no torchrun).
    src_list/dst_list: sequences of (N_b,3) float64 arrays.  Returns (solutions structured array, list of cliques)."""
    B = len(src_list)
    srcs = [_pts(a) for a in src_list]
    dsts = [_pts(a) for a in dst_list]
    n = np.array([a.shape[0] for a in srcs], dtype=np.int32)
    max_n = int(n.max())
    sp = (C.POINTER(C.c_double) * B)(*[_p(a, C.c_double) for a in srcs])
    dp_ = (C.POINTER(C.c_double) * B)(*[_p(a, C.c_double) for a in dsts])
    sols = (Solution * B)()
    clq = np.zeros((B, max_n), dtype=np.int32)
    if devices is None:
        dev_p, n_dev = None, 0
    else:
        dev = np.ascontiguousarray(devices, dtype=np.int32)
        dev_p, n_dev = _p(dev, C.c_int32), int(dev.size)
    rc = lib().tzr_solve_batch_multi(dev_p, n_dev, C.byref(params), B, _p(n, C.c_int32), sp, dp_, sols,
                                     _p(clq, C.c_int32), max_n)
    if rc != 0:
        raise TzrError(f"tzr_solve_batch_multi: {lib().tzr_status_string(rc).decode()}")
    out = np.frombuffer(bytes(sols), dtype=SOLUTION_DTYPE).copy()
    return out, [clq[b, :out[b]["clique_size"]].copy() for b in range(B)]
