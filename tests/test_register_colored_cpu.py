"""CPU checks of coloured ICP inside the chained calls (tzr_register_cloud_pairs_icp_colored,
tzr_register_cloud_pairs_multiway_colored) and of colours from PLY files: the entries are declared with the argument
order the bindings pass, malformed calls are refused before any device work, and PLYReader reads colours."""
import ctypes as C
import importlib
import os
import re
import subprocess

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")

COLOR_ARGS = ["colors", "lambda_geometric", "kernel"]


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)


def _args(header, name):
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, header)
    assert m, f"{name} missing from the header"
    return [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]


@pytest.mark.parametrize("name,base", [("tzr_register_cloud_pairs_icp_colored", "tzr_register_cloud_pairs_icp"),
                                       ("tzr_register_cloud_pairs_multiway_colored",
                                        "tzr_register_cloud_pairs_multiway")])
def test_entries_declared_with_the_colour_arguments_after_icp(header, name, base):
    args, base_args = _args(header, name), _args(header, base)
    at = base_args.index("icp") + 1
    assert args == base_args[:at] + COLOR_ARGS + base_args[at:]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(args)


def _deviceless_context():
    ctx = object.__new__(capi.Context)
    ctx._h = C.c_void_p()  # NULL: any call that reached the library would be refused there, not here
    return ctx


def _clouds():
    rng = np.random.default_rng(0)
    clouds = [rng.standard_normal((20, 3)).astype(np.float32) for _ in range(3)]
    return clouds, [np.full((20, 3), 0.5, dtype=np.float32) for _ in clouds], [(0, 1), (1, 2)]


@pytest.mark.parametrize("case", ["colored_without_colors", "colors_with_point_to_plane", "colors_with_point_to_point",
                                  "colour_count", "colour_rows", "colour_columns"])
def test_chained_python_checks_need_no_device(case):
    ctx = _deviceless_context()
    clouds, cols, pairs = _clouds()
    prm = capi.default_params(noise_bound=0.01)
    kw = dict(method="colored", colors=cols)
    match = "colou?rs"
    if case == "colored_without_colors":
        kw["colors"] = None
    elif case == "colors_with_point_to_plane":
        kw["method"] = "point_to_plane"
    elif case == "colors_with_point_to_point":
        kw["method"] = "point_to_point"
    elif case == "colour_count":
        kw["colors"] = cols[:2]
    elif case == "colour_rows":
        kw["colors"] = [cols[0], cols[1][:19], cols[2]]
    elif case == "colour_columns":
        kw["colors"] = [cols[0], np.zeros((20, 4), dtype=np.float32), cols[2]]
    with pytest.raises(capi.TzrError, match=match):
        ctx.register_cloud_pairs_icp(clouds, pairs, prm, 0.05, **kw)


@pytest.mark.parametrize("case", ["kernel_without_colors", "colour_rows"])
def test_multiway_python_checks_need_no_device(case):
    ctx = _deviceless_context()
    clouds, cols, pairs = _clouds()
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0)
    if case == "kernel_without_colors":
        with pytest.raises(capi.TzrError, match="kernel needs colors"):
            ctx.register_multiway(clouds, pairs, prm, 0.05, kernel=("huber", 0.1))
    else:
        with pytest.raises(capi.TzrError, match="colou?rs"):
            ctx.register_multiway(clouds, pairs, prm, 0.05, colors=[cols[0], cols[1][:3], cols[2]])


def _c_call(name, lam=0.968, kernel=None, drop=None, icp_r=0.05, scaling=0):
    """The entry on three 20-point clouds with a NULL context: every argument check runs before the device is touched."""
    clouds, cols, pairs = _clouds()
    fp = C.POINTER(C.c_float)
    n = np.array([20, 20, 20], dtype=np.int32)
    pc = np.ascontiguousarray(pairs, dtype=np.int32)
    pts = (fp * 3)(*[c.ctypes.data_as(fp) for c in clouds])
    colors = (fp * 3)(*[c.ctypes.data_as(fp) for c in cols])
    if drop == "entry":
        colors[2] = None
    elif drop == "array":
        colors = None
    fpar = capi.FrontendParams(0.1, 0.15, 0, 1, 0, 0.0)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=scaling)
    icp = capi.icp_params(icp_r)
    sols = np.zeros(2, dtype=capi.SOLUTION_DTYPE)
    st, idx, cnt = np.zeros(2, np.int32), np.zeros(2, np.int32), np.zeros(2, np.int64)
    res = np.zeros(2, dtype=capi.ICP_RESULT_DTYPE)
    k = C.byref(kernel) if kernel is not None else None
    args = [None, C.byref(fpar), C.byref(prm), 3, n.ctypes.data_as(C.POINTER(C.c_int32)), pts, 2,
            pc.ctypes.data_as(C.POINTER(C.c_int32)), None, sols.ctypes.data_as(C.POINTER(capi.Solution)),
            st.ctypes.data_as(C.POINTER(C.c_int32)), idx.ctypes.data_as(C.POINTER(C.c_int32)),
            cnt.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None, C.byref(icp), colors, lam, k,
            res.ctypes.data_as(C.POINTER(capi.IcpResult))]
    if name == "tzr_register_cloud_pairs_multiway_colored":
        unc = np.zeros(2, np.int32)
        pg = capi.pose_graph_params(0.05)
        info, icnt, w, m = np.zeros((2, 36)), np.zeros(2, np.int32), np.zeros(2), np.zeros(2, np.uint8)
        poses = (capi.Similarity * 3)()
        pgs = C.c_int32(0)
        args += [unc.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(pg), info.ctypes.data_as(C.POINTER(C.c_double)),
                 icnt.ctypes.data_as(C.POINTER(C.c_int32)), w.ctypes.data_as(C.POINTER(C.c_double)),
                 m.ctypes.data_as(C.POINTER(C.c_uint8)), poses, None, C.byref(pgs)]
    return getattr(capi.lib(), name)(*args)


@pytest.mark.parametrize("name", ["tzr_register_cloud_pairs_icp_colored", "tzr_register_cloud_pairs_multiway_colored"])
@pytest.mark.parametrize("case", ["null_ctx", "lambda_nan", "lambda_inf", "kernel_unknown", "kernel_k_negative",
                                  "null_colors", "null_colors_entry", "r_zero"])
def test_c_argument_checks_need_no_device(name, case):
    kw = {}
    if case == "lambda_nan":
        kw["lam"] = float("nan")
    elif case == "lambda_inf":
        kw["lam"] = float("-inf")
    elif case == "kernel_unknown":
        kw["kernel"] = capi.RobustKernel(9, 0, 1.0)
    elif case == "kernel_k_negative":
        kw["kernel"] = capi.RobustKernel(capi.LOSS_TYPES["cauchy"], 0, -1.0)
    elif case == "null_colors":
        kw["drop"] = "array"
    elif case == "null_colors_entry":
        kw["drop"] = "entry"
    elif case == "r_zero":
        kw["icp_r"] = 0.0
    assert _c_call(name, **kw) == capi.TZR_ERR_INVALID_ARG


def test_ply_colours(tmp_path):
    """PLYReader::read(file, cloud, colors) on files the test writes (tests/cpp/ply_colors_test.cc); host only."""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "ply_colors_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"),
                           os.path.join(ROOT, "tests", "cpp", "ply_colors_test.cc"),
                           os.path.join(HOST, "src", "ply_io.cc"), "-o", exe])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr
