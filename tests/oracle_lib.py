"""ctypes binding of the CPU oracle (oracle/libteaser_oracle.so). TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB_PATH = os.path.join(ORACLE_DIR, "libteaser_oracle.so")


class Params(C.Structure):
    """Same layout as tzr_params (include/teaser_b200.h) / orc_params (oracle/teaser_oracle.cc)."""
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
        return np.array(self.rotation[:]).reshape(3, 3).T.copy()  # column-major -> numpy

    @property
    def t(self):
        return np.array(self.translation[:])


def default_params(**kw):
    """RobustRegistrationSolver::Params defaults (teaser/include/teaser/registration.h:419-514)."""
    p = Params()
    p.noise_bound = 0.01
    p.cbar2 = 1.0
    p.estimate_scaling = 1
    p.rotation_estimation_algorithm = 0
    p.rotation_gnc_factor = 1.4
    p.rotation_max_iterations = 100
    p.rotation_cost_threshold = 1e-6
    p.rotation_tim_graph = 0
    p.inlier_selection_mode = 0
    p.kcore_heuristic_threshold = 0.5
    p.use_max_clique = 1
    p.max_clique_exact_solution = 1
    p.max_clique_time_limit = 3600.0
    p.max_clique_num_threads = 0
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


_lib = None


def build():
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR])


def lib():
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(ORACLE_DIR, f) for f in ("teaser_oracle.cc", "matcher_oracle.cc", "fpfh_oracle.cc")]
    if not os.path.exists(LIB_PATH) or any(os.path.exists(f) and os.path.getmtime(f) > os.path.getmtime(LIB_PATH)
                                           for f in srcs):
        build()
    L = C.CDLL(LIB_PATH)
    dp = C.POINTER(C.c_double)
    u8p = C.POINTER(C.c_uint8)
    i32p = C.POINTER(C.c_int32)
    i64p = C.POINTER(C.c_int64)
    u64p = C.POINTER(C.c_uint64)
    L.orc_num_threads.restype = C.c_int
    L.orc_set_num_threads.argtypes = [C.c_int]
    L.orc_set_num_threads.restype = None
    L.orc_compute_tims.argtypes = [dp, C.c_int64, dp, i32p]
    L.orc_scale_inliers_selector.argtypes = [dp, dp, C.c_int64, C.c_double, C.c_double, dp, u8p]
    L.orc_tls_scale_solver.argtypes = [dp, dp, C.c_int64, C.c_double, C.c_double, dp, u8p]
    L.orc_scalar_tls.argtypes = [dp, dp, C.c_int64, dp, u8p]
    L.orc_tls_translation.argtypes = [dp, dp, C.c_int64, C.c_double, C.c_double, dp, u8p]
    L.orc_svd_rot.argtypes = [dp, dp, dp, C.c_int64, dp]
    L.orc_svd3.argtypes = [dp, dp, dp, dp]
    L.orc_gnc_tls_rotation.argtypes = [dp, dp, C.c_int64, C.c_uint64, C.c_double, C.c_double, C.c_double, dp, u8p,
                                       dp, dp, C.c_int, dp]
    L.orc_gnc_tls_rotation.restype = C.c_int
    L.orc_fgr_rotation.argtypes = [dp, dp, C.c_int64, C.c_uint64, C.c_double, C.c_double, C.c_double, dp, u8p, dp]
    L.orc_fgr_rotation.restype = C.c_int
    L.orc_quatro_rotation.argtypes = [dp, dp, C.c_int64, C.c_uint64, C.c_double, C.c_double, C.c_double, dp, u8p, dp]
    L.orc_quatro_rotation.restype = C.c_int
    L.orc_max_clique_csr.argtypes = [i64p, i32p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, i32p, i32p]
    L.orc_max_clique_csr.restype = C.c_int
    L.orc_max_clique_bits.argtypes = [u64p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, i32p, i32p]
    L.orc_max_clique_bits.restype = C.c_int
    L.orc_build_graph_bits.argtypes = [dp, dp, C.c_int, C.c_double, C.c_double, u64p, C.c_int, i32p]
    L.orc_build_graph_bits.restype = C.c_int64
    L.orc_solve.argtypes = [C.POINTER(Params), dp, dp, C.c_int, C.POINTER(Solution), i32p, u8p, u8p, u64p, C.c_int]
    L.orc_solve.restype = C.c_int
    fp = C.POINTER(C.c_float)
    L.orc_match_correspondences.argtypes = [fp, C.c_int, fp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_float, C.c_uint64, i32p, C.c_int64, fp]
    L.orc_match_correspondences.restype = C.c_int64
    L.orc_nn1.argtypes = [fp, C.c_int, fp, C.c_int, C.c_int, i32p]
    L.orc_nn1.restype = None
    L.orc_compute_fpfh.argtypes = [fp, C.c_int, C.c_double, C.c_double, C.c_int, fp, fp]
    L.orc_compute_fpfh.restype = None
    L.orc_fpfh_pair_features.argtypes = [C.c_int, fp, fp, fp, fp, fp, i32p]
    L.orc_fpfh_pair_features.restype = None
    L.orc_fpfh_smallest_eigenpair.argtypes = [C.c_int, fp, fp, fp]
    L.orc_fpfh_smallest_eigenpair.restype = None
    L.orc_fpfh_elementary.argtypes = [C.c_int, C.c_int, fp, fp, fp]
    L.orc_fpfh_elementary.restype = None
    _lib = L
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def as_pts(a):
    """(N,3) float64 C-contiguous == column-major 3xN."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    assert a.ndim == 2 and a.shape[1] == 3
    return a


def scalar_tls(X, ranges):
    X = np.ascontiguousarray(X, dtype=np.float64)
    r = np.ascontiguousarray(ranges, dtype=np.float64)
    est = C.c_double()
    inl = np.zeros(X.size, dtype=np.uint8)
    lib().orc_scalar_tls(_dp(X), _dp(r), X.size, C.byref(est), _p(inl, C.c_uint8))
    return est.value, inl.astype(bool)


def compute_tims(v):
    v = as_pts(v)
    n = v.shape[0]
    K = n * (n - 1) // 2
    tims = np.zeros((K, 3))
    mp = np.zeros((K, 2), dtype=np.int32)
    lib().orc_compute_tims(_dp(v), n, _dp(tims), _p(mp, C.c_int32))
    return tims, mp


def scale_inliers_selector(src_tims, dst_tims, nb, cbar2=1.0):
    s, d = as_pts(src_tims), as_pts(dst_tims)
    sc = C.c_double()
    mask = np.zeros(s.shape[0], dtype=np.uint8)
    lib().orc_scale_inliers_selector(_dp(s), _dp(d), s.shape[0], nb, cbar2, C.byref(sc), _p(mask, C.c_uint8))
    return sc.value, mask.astype(bool)


def tls_scale_solver(src_tims, dst_tims, nb, cbar2=1.0):
    s, d = as_pts(src_tims), as_pts(dst_tims)
    sc = C.c_double()
    mask = np.zeros(s.shape[0], dtype=np.uint8)
    lib().orc_tls_scale_solver(_dp(s), _dp(d), s.shape[0], nb, cbar2, C.byref(sc), _p(mask, C.c_uint8))
    return sc.value, mask.astype(bool)


def tls_translation(src, dst, nb, cbar2=1.0):
    s, d = as_pts(src), as_pts(dst)
    t = np.zeros(3)
    mask = np.zeros(s.shape[0], dtype=np.uint8)
    lib().orc_tls_translation(_dp(s), _dp(d), s.shape[0], nb, cbar2, _dp(t), _p(mask, C.c_uint8))
    return t, mask.astype(bool)


def svd3(H):
    Hc = np.asfortranarray(H, dtype=np.float64)
    U = np.zeros((3, 3), order="F")
    V = np.zeros((3, 3), order="F")
    S = np.zeros(3)
    lib().orc_svd3(_dp(Hc), _dp(U), _dp(S), _dp(V))
    return U, S, V


def gnc_tls(src, dst, max_iterations=100, cost_threshold=1e-6, gnc_factor=1.4, noise_bound=0.01, trace=False):
    s, d = as_pts(src), as_pts(dst)
    m = s.shape[0]
    R = np.zeros((3, 3), order="F")
    mask = np.zeros(m, dtype=np.uint8)
    cost = C.c_double()
    tr = np.zeros((int(max_iterations), 4))
    w = np.zeros(m)
    it = lib().orc_gnc_tls_rotation(_dp(s), _dp(d), m, int(max_iterations), cost_threshold, gnc_factor, noise_bound,
                                    _dp(R), _p(mask, C.c_uint8), C.byref(cost), _dp(tr), int(max_iterations), _dp(w))
    out = dict(R=np.array(R), inliers=mask.astype(bool), cost=cost.value, iterations=it, weights=w)
    if trace:
        out["trace"] = tr[:it]
    return out


def fgr(src, dst, max_iterations=100, cost_threshold=0.005, gnc_factor=1.4, noise_bound=0.01):
    s, d = as_pts(src), as_pts(dst)
    m = s.shape[0]
    R = np.zeros((3, 3), order="F")
    mask = np.zeros(m, dtype=np.uint8)
    cost = C.c_double()
    it = lib().orc_fgr_rotation(_dp(s), _dp(d), m, int(max_iterations), cost_threshold, gnc_factor, noise_bound,
                                _dp(R), _p(mask, C.c_uint8), C.byref(cost))
    return dict(R=np.array(R), inliers=mask.astype(bool), cost=cost.value, iterations=it)


def quatro(src, dst, max_iterations=100, cost_threshold=0.005, gnc_factor=1.4, noise_bound=0.01):
    s, d = as_pts(src), as_pts(dst)
    m = s.shape[0]
    R = np.zeros((3, 3), order="F")
    mask = np.zeros(m, dtype=np.uint8)
    cost = C.c_double()
    it = lib().orc_quatro_rotation(_dp(s), _dp(d), m, int(max_iterations), cost_threshold, gnc_factor, noise_bound,
                                   _dp(R), _p(mask, C.c_uint8), C.byref(cost))
    return dict(R=np.array(R), inliers=mask.astype(bool), cost=cost.value, iterations=it)


def max_clique_adj(adj_lists, mode=0, kcore_thr=1.0, time_limit=3600.0, threads=0):
    n = len(adj_lists)
    off = np.zeros(n + 1, dtype=np.int64)
    for i, a in enumerate(adj_lists):
        off[i + 1] = off[i] + len(a)
    edges = np.zeros(max(1, int(off[-1])), dtype=np.int32)
    for i, a in enumerate(adj_lists):
        edges[off[i]:off[i + 1]] = a
    out = np.zeros(max(n, 1), dtype=np.int32)
    info = np.zeros(8, dtype=np.int32)
    m = lib().orc_max_clique_csr(_p(off, C.c_int64), _p(edges, C.c_int32), n, mode, kcore_thr, time_limit, threads,
                                 _p(out, C.c_int32), _p(info, C.c_int32))
    return out[:m].copy(), dict(max_core=int(info[0]), lb=int(info[1]), ub=int(info[2]), exact_ran=int(info[3]),
                                timed_out=int(info[4]), nodes=int(info[5]))


def max_clique_bits(bits, n, mode=0, kcore_thr=1.0, time_limit=3600.0, threads=0):
    bits = np.ascontiguousarray(bits, dtype=np.uint64)
    W = bits.shape[1]
    out = np.zeros(max(n, 1), dtype=np.int32)
    info = np.zeros(8, dtype=np.int32)
    m = lib().orc_max_clique_bits(_p(bits, C.c_uint64), n, W, mode, kcore_thr, time_limit, threads,
                                  _p(out, C.c_int32), _p(info, C.c_int32))
    return np.sort(out[:m]), dict(max_core=int(info[0]), lb=int(info[1]), ub=int(info[2]), exact_ran=int(info[3]),
                                  timed_out=int(info[4]), nodes=int(info[5]))


def build_graph_bits(src, dst, nb, cbar2=1.0):
    s, d = as_pts(src), as_pts(dst)
    n = s.shape[0]
    W = (n + 63) // 64
    bits = np.zeros((n, W), dtype=np.uint64)
    deg = np.zeros(n, dtype=np.int32)
    e = lib().orc_build_graph_bits(_dp(s), _dp(d), n, nb, cbar2, _p(bits, C.c_uint64), W, _p(deg, C.c_int32))
    return bits, deg, int(e)


def solve(src, dst, params, want_adj=False):
    s, d = as_pts(src), as_pts(dst)
    n = s.shape[0]
    sol = Solution()
    clique = np.zeros(n, dtype=np.int32)
    nrot = n * (n - 1) // 2 if params.rotation_tim_graph == 1 else n
    rot_mask = np.zeros(max(nrot, 1), dtype=np.uint8)
    tr_mask = np.zeros(n, dtype=np.uint8)
    W = (n + 63) // 64
    bits = np.zeros((n, W), dtype=np.uint64) if want_adj else None
    lib().orc_solve(C.byref(params), _dp(s), _dp(d), n, C.byref(sol), _p(clique, C.c_int32),
                    _p(rot_mask, C.c_uint8), _p(tr_mask, C.c_uint8),
                    _p(bits, C.c_uint64) if want_adj else None, W)
    m = sol.clique_size
    out = dict(sol=sol, valid=bool(sol.valid), scale=sol.scale, R=sol.R, t=sol.t, clique=clique[:m].copy(),
               trans_inliers=tr_mask[:m].astype(bool), gnc_iterations=sol.gnc_iterations,
               stage_ms=list(sol.stage_ms))
    nr = m if params.rotation_tim_graph == 0 else m * (m - 1) // 2
    out["rot_inliers"] = rot_mask[:nr].astype(bool)
    if want_adj:
        out["adj_bits"] = bits
    return out


def match_correspondences(src_pts, dst_pts, src_feat, dst_feat, use_absolute_scale=True, use_crosscheck=True,
                          use_tuple_test=True, tuple_scale=0.0, tuple_seed=0, return_scale=False):
    """Matcher::calculateCorrespondences restatement (oracle/matcher_oracle.cc)."""
    sp = np.ascontiguousarray(src_pts, dtype=np.float32)
    tp = np.ascontiguousarray(dst_pts, dtype=np.float32)
    sf = np.ascontiguousarray(src_feat, dtype=np.float32)
    tf = np.ascontiguousarray(dst_feat, dtype=np.float32)
    ns, nd = sp.shape[0], tp.shape[0]
    cap = ns + nd
    pairs = np.zeros((cap, 2), dtype=np.int32)
    g = C.c_float()
    cnt = lib().orc_match_correspondences(_p(sp, C.c_float), ns, _p(tp, C.c_float), nd, _p(sf, C.c_float),
                                          _p(tf, C.c_float), sf.shape[1], int(bool(use_absolute_scale)),
                                          int(bool(use_crosscheck)), int(bool(use_tuple_test)), float(tuple_scale),
                                          int(tuple_seed), _p(pairs, C.c_int32), cap, C.byref(g))
    assert cnt >= 0
    out = pairs[:cnt].copy()
    return (out, g.value) if return_scale else out


def nn1(query, db):
    q = np.ascontiguousarray(query, dtype=np.float32)
    d = np.ascontiguousarray(db, dtype=np.float32)
    out = np.zeros(q.shape[0], dtype=np.int32)
    lib().orc_nn1(_p(q, C.c_float), q.shape[0], _p(d, C.c_float), d.shape[0], q.shape[1], _p(out, C.c_int32))
    return out


def fpfh_pair_features(p1, n1, p2, n2):
    """pcl::computePairFeatures restatement on n pairs ((n,3) each): ((n,3) f1 f2 f3, (n,) bool ok)."""
    ins = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 3) for a in (p1, n1, p2, n2)]
    n = ins[0].shape[0]
    f = np.zeros((n, 3), dtype=np.float32)
    ok = np.zeros(n, dtype=np.int32)
    lib().orc_fpfh_pair_features(n, *[_p(a, C.c_float) for a in ins], _p(f, C.c_float), _p(ok, C.c_int32))
    return f, ok.astype(bool)


def fpfh_smallest_eigenpair(cov):
    """pcl::eigen33 restatement on (n,3,3) float32 matrices: ((n,) eigenvalues, (n,3) vectors)."""
    c = np.ascontiguousarray(cov, dtype=np.float32).reshape(-1, 3, 3)
    n = c.shape[0]
    ev = np.zeros(n, dtype=np.float32)
    vec = np.zeros((n, 3), dtype=np.float32)
    lib().orc_fpfh_smallest_eigenpair(n, _p(c, C.c_float), _p(ev, C.c_float), _p(vec, C.c_float))
    return ev, vec


def fpfh_elementary(fn, a, b=None):
    """The FPFH restatement's elementary functions: fn 'atan2' (a = y, b = x), 'acos01', 'sin', 'cos' (of
    det_sincos_0_pi2)."""
    a = np.ascontiguousarray(a, dtype=np.float32).ravel()
    b = np.ascontiguousarray(a if b is None else b, dtype=np.float32).ravel()
    out = np.zeros(a.size, dtype=np.float32)
    code = {"atan2": 0, "acos01": 1, "sin": 2, "cos": 3}[fn]
    lib().orc_fpfh_elementary(code, a.size, _p(a, C.c_float), _p(b, C.c_float), _p(out, C.c_float))
    return out


def compute_fpfh(pts, normal_search_radius=0.03, fpfh_search_radius=0.05, cov_variant=0):
    """FPFHEstimation::computeFPFHFeatures restatement (oracle/fpfh_oracle.cc). Returns (fpfh (n,33), normals (n,4))."""
    p = np.ascontiguousarray(pts, dtype=np.float32)
    out = np.zeros((p.shape[0], 33), dtype=np.float32)
    nor = np.zeros((p.shape[0], 4), dtype=np.float32)
    lib().orc_compute_fpfh(_p(p, C.c_float), p.shape[0], float(normal_search_radius), float(fpfh_search_radius),
                           int(cov_variant), _p(nor, C.c_float), _p(out, C.c_float))
    return out, nor
