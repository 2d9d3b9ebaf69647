"""CPU checks of the robust-kernel C-ABI (tzr_icp_point_to_plane_robust_batch, tzr_icp_generalized_robust_batch,
tzr_register_cloud_pairs_icp_robust): the entry points are exported, declared in the header with the argument lists the
Python binding passes and listed among the symbols capi.lib() checks; tzr_robust_kernel's layout matches the binding;
malformed calls are refused before any device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_icp_point_to_plane_robust_batch": ["ctx", "params", "B", "ns", "src", "nd", "dst", "dst_normals", "init",
                                            "results", "corr", "kernel"],
    "tzr_icp_generalized_robust_batch": ["ctx", "params", "epsilon", "B", "ns", "src", "src_normals", "nd", "dst",
                                         "dst_normals", "init", "results", "corr", "kernel"],
    "tzr_register_cloud_pairs_icp_robust": ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds",
                                            "tuple_seeds", "solutions", "status", "problem_index", "n_corr", "corr",
                                            "cliques", "global_scale", "icp", "method", "epsilon", "kernel",
                                            "icp_results"],
}

fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def header_raw():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return open(os.path.join(ROOT, "include", "teaser_b200.h")).read()


@pytest.fixture(scope="module")
def header(header_raw):
    return re.sub(r"/\*.*?\*/", "", header_raw, flags=re.S)


@pytest.mark.parametrize("name", sorted(ARGS))
def test_symbol_exported_declared_and_bound(header, name):
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, header)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])
    assert "#define TZR_ABI_VERSION 2" in header


def test_batch_entries_extend_the_unweighted_ones(header):
    """Each robust batch entry is its unweighted entry's argument list plus the kernel."""
    def args(name):
        m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, header)
        return [x.strip() for x in " ".join(m.group(1).split()).split(",")]
    assert args("tzr_icp_point_to_plane_robust_batch") == args("tzr_icp_point_to_plane_batch") + [
        "const tzr_robust_kernel* kernel"]
    assert args("tzr_icp_generalized_robust_batch") == args("tzr_icp_generalized_batch") + [
        "const tzr_robust_kernel* kernel"]
    a = args("tzr_register_cloud_pairs_icp")
    assert args("tzr_register_cloud_pairs_icp_robust") == a[:-1] + [
        "int32_t method", "double epsilon", "const tzr_robust_kernel* kernel"] + a[-1:]


def test_kernel_struct_and_type_values(header):
    m = re.search(r"typedef struct tzr_robust_kernel \{(.*?)\} tzr_robust_kernel;", header, flags=re.S)
    assert m
    fields = [f.split()[-1] for f in m.group(1).replace("\n", " ").split(";") if f.strip()]
    assert fields == ["type", "reserved", "k"]
    assert C.sizeof(capi.RobustKernel) == 16
    assert [(f, getattr(capi.RobustKernel, f).offset) for f, _ in capi.RobustKernel._fields_] == [
        ("type", 0), ("reserved", 4), ("k", 8)]
    defined = dict(re.findall(r"#define TZR_LOSS_(\w+) (\d+)", header))
    assert {k.lower(): int(v) for k, v in defined.items()} == capi.LOSS_TYPES


def test_binding_builds_kernels():
    k = capi.robust_kernel(("tukey", 0.05))
    assert (k.type, k.k) == (capi.LOSS_TYPES["tukey"], 0.05)
    assert capi.robust_kernel("L1").type == capi.LOSS_TYPES["l1"]
    assert capi.robust_kernel(None) is None
    same = capi.RobustKernel(2, 0, 1.0)
    assert capi.robust_kernel(same) is same
    with pytest.raises(capi.TzrError):
        capi.robust_kernel(("welsch", 1.0))


def _robust_batch(gicp, ctx, p, kernel, epsilon=1e-3, B=2, ns=4, nd=4, dst_normals="ok"):
    x = np.zeros((max(ns, 1), 3), dtype=np.float32)
    y = np.zeros((max(nd, 1), 3), dtype=np.float32)
    nrm = np.zeros((max(ns, nd, 1), 4), dtype=np.float32)
    Bn = max(B, 1)
    n_s = np.full(Bn, ns, dtype=np.int32)
    n_d = np.full(Bn, nd, dtype=np.int32)
    init = (capi.Similarity * Bn)(*[capi.similarity(None) for _ in range(Bn)])
    res = (capi.IcpResult * Bn)()
    xs = (fp * Bn)(*[x.ctypes.data_as(fp)] * Bn)
    ys = (fp * Bn)(*[y.ctypes.data_as(fp)] * Bn)
    ok = (fp * Bn)(*[nrm.ctypes.data_as(fp)] * Bn)
    dn = None if dst_normals == "null" else ok
    kp = None if kernel is None else C.byref(kernel)
    L = capi.lib()
    if gicp:
        return L.tzr_icp_generalized_robust_batch(ctx, C.byref(p), epsilon, B, n_s.ctypes.data_as(i32p), xs, ok,
                                                  n_d.ctypes.data_as(i32p), ys, dn, init, res, None, kp)
    return L.tzr_icp_point_to_plane_robust_batch(ctx, C.byref(p), B, n_s.ctypes.data_as(i32p), xs,
                                                 n_d.ctypes.data_as(i32p), ys, dn, init, res, None, kp)


K = capi.RobustKernel
CASES = {
    "null_kernel": dict(kernel=None),
    "type_negative": dict(kernel=K(-1, 0, 1.0)),
    "type_unknown": dict(kernel=K(6, 0, 1.0)),
    "huber_k_zero": dict(kernel=K(2, 0, 0.0)),
    "cauchy_k_negative": dict(kernel=K(3, 0, -1.0)),
    "gm_k_nan": dict(kernel=K(4, 0, float("nan"))),
    "tukey_k_inf": dict(kernel=K(5, 0, float("inf"))),
    "null_ctx_l2": dict(kernel=K(0, 0, float("nan"))),
    "null_ctx_l1": dict(kernel=K(1, 0, -1.0)),
    "null_ctx_tukey": dict(kernel=K(5, 0, 0.1)),
    "null_dst_normals": dict(kernel=K(5, 0, 0.1), dst_normals="null"),
    "B_zero": dict(kernel=K(2, 0, 1.0), B=0),
    "ns_zero": dict(kernel=K(2, 0, 1.0), ns=0),
    "r_zero": dict(kernel=K(2, 0, 1.0)),
}


@pytest.mark.parametrize("gicp", [False, True], ids=["point_to_plane", "generalized"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_argument_checks_need_no_device(case, gicp):
    """Malformed calls return TZR_ERR_INVALID_ARG without a device (the context is NULL here, and every argument check
    runs before the device is touched).  The null_ctx cases hold valid kernels, L2 and L1 with a k that is not read."""
    p = capi.icp_params(0.1)
    if case == "r_zero":
        p.max_correspondence_distance = 0.0
    assert _robust_batch(gicp, None, p, **CASES[case]) == capi.TZR_ERR_INVALID_ARG


def test_generalized_robust_batch_checks_epsilon():
    p = capi.icp_params(0.1)
    for eps in (0.0, -1.0, float("nan"), float("inf")):
        assert _robust_batch(True, None, p, K(5, 0, 0.1), epsilon=eps) == capi.TZR_ERR_INVALID_ARG


@pytest.mark.parametrize("method,kernel", [(0, K(5, 0, 0.1)), (3, K(5, 0, 0.1)), (1, None), (2, K(7, 0, 1.0)),
                                           (1, K(2, 0, 0.0))])
def test_chained_entry_refuses_bad_method_and_kernel(method, kernel):
    L = capi.lib()
    icp = capi.icp_params(0.1)
    kp = None if kernel is None else C.byref(kernel)
    assert L.tzr_register_cloud_pairs_icp_robust(None, None, None, 0, None, None, 0, None, None, None, None, None, None,
                                                 None, None, None, C.byref(icp), method, 1e-3, kp, None) == \
        capi.TZR_ERR_INVALID_ARG
    assert L.tzr_register_cloud_pairs_icp_robust(None, None, None, 0, None, None, 0, None, None, None, None, None, None,
                                                 None, None, None, None, 1, 1e-3, C.byref(K(0, 0, 0.0)), None) == \
        capi.TZR_ERR_INVALID_ARG


def test_python_refuses_a_kernel_for_point_to_point():
    ctx = object.__new__(capi.Context)  # no device: the check runs before the library is called
    with pytest.raises(capi.TzrError):
        capi.Context.register_cloud_pairs_icp(ctx, [np.zeros((3, 3))], [(0, 0)], None, 0.1, method="point_to_point",
                                              kernel=("tukey", 0.1))
    with pytest.raises(capi.TzrError):
        capi.Context.register_cloud_pairs_icp(ctx, [np.zeros((3, 3))], [(0, 0)], None, 0.1, method="point_to_plane",
                                              kernel=("welsch", 0.1))


def test_header_states_the_weights(header_raw):
    """The header writes out every weight and the rule for weights that are not finite."""
    for text in ("k / max(e, k)", "1 / (1 + q q)", "k / (t t)", "0 when e > k", "not finite"):
        assert text in header_raw
