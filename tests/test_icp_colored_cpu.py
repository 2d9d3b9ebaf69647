"""CPU checks of the coloured ICP C-ABI (tzr_estimate_color_gradients(_batch), tzr_icp_colored(_batch)): the entry points
are exported, declared in the header with the argument lists the Python binding passes and listed among the symbols
capi.lib() checks; malformed calls are refused before any device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_estimate_color_gradients": ["ctx", "pts", "n", "normals", "colors", "radius", "grad_out"],
    "tzr_estimate_color_gradients_batch": ["ctx", "B", "n", "pts", "normals", "colors", "radius", "grad_out",
                                           "status"],
    "tzr_icp_colored": ["ctx", "params", "src", "ns", "dst", "nd", "dst_normals", "init", "result", "corr",
                        "src_colors", "dst_colors", "lambda_geometric", "kernel"],
    "tzr_icp_colored_batch": ["ctx", "params", "B", "ns", "src", "nd", "dst", "dst_normals", "init", "results", "corr",
                              "src_colors", "dst_colors", "lambda_geometric", "kernel"],
    "tzr_voxel_downsample_colors": ["ctx", "pts", "n", "voxel_size", "pts_out", "n_out", "voxel_of", "colors",
                                    "colors_out"],
    "tzr_voxel_downsample_colors_batch": ["ctx", "B", "n", "pts", "voxel_size", "pts_out", "n_out", "voxel_of",
                                          "status", "colors", "colors_out"],
}

fp, i32p, dp = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)


@pytest.mark.parametrize("name", sorted(ARGS))
def test_symbol_exported_declared_and_bound(header, name):
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, header)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])


def test_colored_entries_extend_the_point_to_plane_arguments(header):
    plane = re.search(r"int\s+tzr_icp_point_to_plane_batch\s*\(([^)]*)\)", header).group(1)
    col = re.search(r"int\s+tzr_icp_colored_batch\s*\(([^)]*)\)", header).group(1)
    assert " ".join(col.split()).startswith(" ".join(plane.split()) + ",")


def _colored_batch(p, B=2, ns=4, nd=4, lam=0.968, kernel=None, drop=None):
    Bn = max(B, 1)
    x = np.zeros((max(ns, 1), 3), dtype=np.float32)
    y = np.zeros((max(nd, 1), 3), dtype=np.float32)
    nrm = np.zeros((max(nd, 1), 4), dtype=np.float32)
    arrays = {k: (fp * Bn)(*[a.ctypes.data_as(fp)] * Bn)
              for k, a in (("src", x), ("dst", y), ("normals", nrm), ("sc", x), ("dc", y))}
    if drop:
        name, entry = drop
        if entry:
            arrays[name][Bn - 1] = None
        else:
            arrays[name] = None
    n_s, n_d = np.full(Bn, ns, dtype=np.int32), np.full(Bn, nd, dtype=np.int32)
    init = (capi.Similarity * Bn)(*[capi.similarity(None) for _ in range(Bn)])
    res = (capi.IcpResult * Bn)()
    k = C.byref(kernel) if kernel is not None else None
    return capi.lib().tzr_icp_colored_batch(None, C.byref(p), B, n_s.ctypes.data_as(i32p), arrays["src"],
                                            n_d.ctypes.data_as(i32p), arrays["dst"], arrays["normals"], init, res,
                                            None, arrays["sc"], arrays["dc"], lam, k)


@pytest.mark.parametrize("case", ["null_ctx", "lambda_nan", "lambda_inf", "kernel_unknown", "kernel_k_negative",
                                  "kernel_k_nan", "null_normals", "null_src_colors", "null_dst_colors_entry",
                                  "r_zero", "r_nan", "iter_negative", "B_zero", "ns_zero", "nd_zero"])
def test_icp_colored_argument_checks_need_no_device(case):
    """Malformed calls return TZR_ERR_INVALID_ARG without a device (the context is NULL here, and every argument check
    runs before the device is touched)."""
    p = capi.icp_params(0.1)
    kw = {}
    if case == "lambda_nan":
        kw["lam"] = float("nan")
    elif case == "lambda_inf":
        kw["lam"] = float("inf")
    elif case == "kernel_unknown":
        kw["kernel"] = capi.RobustKernel(9, 0, 1.0)
    elif case == "kernel_k_negative":
        kw["kernel"] = capi.RobustKernel(capi.LOSS_TYPES["huber"], 0, -1.0)
    elif case == "kernel_k_nan":
        kw["kernel"] = capi.RobustKernel(capi.LOSS_TYPES["tukey"], 0, float("nan"))
    elif case == "null_normals":
        kw["drop"] = ("normals", False)
    elif case == "null_src_colors":
        kw["drop"] = ("sc", False)
    elif case == "null_dst_colors_entry":
        kw["drop"] = ("dc", True)
    elif case == "r_zero":
        p.max_correspondence_distance = 0.0
    elif case == "r_nan":
        p.max_correspondence_distance = float("nan")
    elif case == "iter_negative":
        p.max_iteration = -1
    elif case == "B_zero":
        kw["B"] = 0
    elif case == "ns_zero":
        kw["ns"] = 0
    elif case == "nd_zero":
        kw["nd"] = 0
    assert _colored_batch(p, **kw) == capi.TZR_ERR_INVALID_ARG
    x = np.zeros((3, 3), dtype=np.float32)
    nrm = np.zeros((3, 4), dtype=np.float32)
    res = capi.IcpResult()
    single_colors = None if case == "null_src_colors" else x.ctypes.data_as(fp)
    k = C.byref(kw["kernel"]) if "kernel" in kw else None
    assert capi.lib().tzr_icp_colored(None, C.byref(p), x.ctypes.data_as(fp), 3, x.ctypes.data_as(fp), 3,
                                      nrm.ctypes.data_as(fp), None, C.byref(res), None, single_colors,
                                      x.ctypes.data_as(fp), kw.get("lam", 0.968), k) == capi.TZR_ERR_INVALID_ARG


@pytest.mark.parametrize("case", ["null_ctx", "radius_zero", "radius_negative", "radius_nan", "radius_inf", "B_zero",
                                  "n_zero", "null_out", "null_out_entry", "null_normals", "null_colors_entry"])
def test_gradient_argument_checks_need_no_device(case):
    x = np.zeros((4, 3), dtype=np.float32)
    nrm = np.zeros((4, 4), dtype=np.float32)
    out = np.zeros((4, 3))
    r, B, n = 0.1, 2, np.array([4, 4], dtype=np.int32)
    outs = (dp * 2)(out.ctypes.data_as(dp), out.ctypes.data_as(dp))
    pts = (fp * 2)(x.ctypes.data_as(fp), x.ctypes.data_as(fp))
    nrms = (fp * 2)(nrm.ctypes.data_as(fp), nrm.ctypes.data_as(fp))
    cols = (fp * 2)(x.ctypes.data_as(fp), x.ctypes.data_as(fp))
    r = {"radius_zero": 0.0, "radius_negative": -1.0, "radius_nan": float("nan"), "radius_inf": float("inf")}.get(case,
                                                                                                                r)
    if case == "B_zero":
        B = 0
    elif case == "n_zero":
        n[1] = 0
    elif case == "null_out":
        outs = None
    elif case == "null_out_entry":
        outs[1] = None
    elif case == "null_normals":
        nrms = None
    elif case == "null_colors_entry":
        cols[1] = None
    L = capi.lib()
    assert L.tzr_estimate_color_gradients_batch(None, B, n.ctypes.data_as(i32p), pts, nrms, cols, r, outs, None) == \
        capi.TZR_ERR_INVALID_ARG
    single_out = None if case in ("null_out", "null_out_entry") else out.ctypes.data_as(dp)
    single_nrm = None if case == "null_normals" else nrm.ctypes.data_as(fp)
    single_n = 0 if case == "n_zero" else 4
    assert L.tzr_estimate_color_gradients(None, x.ctypes.data_as(fp), single_n, single_nrm, x.ctypes.data_as(fp), r,
                                          single_out) == capi.TZR_ERR_INVALID_ARG


def test_python_colour_shapes():
    with pytest.raises(capi.TzrError):
        capi._colors32(np.zeros((4, 4), dtype=np.float32), 4, "t")
    with pytest.raises(capi.TzrError):
        capi._colors32(np.zeros((3, 3), dtype=np.float32), 4, "t")
    c = capi._colors32(np.ones((4, 3)), 4, "t")
    assert c.dtype == np.float32 and c.flags["C_CONTIGUOUS"]


@pytest.mark.parametrize("case", ["null_ctx", "null_colors", "null_colors_entry", "null_colors_out",
                                  "null_colors_out_entry", "voxel_zero", "voxel_nan", "n_zero"])
def test_voxel_colour_argument_checks_need_no_device(case):
    x = np.zeros((4, 3), dtype=np.float32)
    B, n, v = 2, np.array([4, 4], dtype=np.int32), 0.1
    two = lambda: (fp * 2)(x.ctypes.data_as(fp), x.ctypes.data_as(fp))  # noqa: E731
    pts, outs, cols, couts = two(), two(), two(), two()
    m = np.zeros(2, dtype=np.int32)
    if case == "null_colors":
        cols = None
    elif case == "null_colors_entry":
        cols[1] = None
    elif case == "null_colors_out":
        couts = None
    elif case == "null_colors_out_entry":
        couts[1] = None
    elif case == "voxel_zero":
        v = 0.0
    elif case == "voxel_nan":
        v = float("nan")
    elif case == "n_zero":
        n[1] = 0
    L = capi.lib()
    assert L.tzr_voxel_downsample_colors_batch(None, B, n.ctypes.data_as(i32p), pts, v, outs, m.ctypes.data_as(i32p),
                                               None, None, cols, couts) == capi.TZR_ERR_INVALID_ARG
    single_c = None if case in ("null_colors", "null_colors_entry") else x.ctypes.data_as(fp)
    single_co = None if case in ("null_colors_out", "null_colors_out_entry") else x.ctypes.data_as(fp)
    assert L.tzr_voxel_downsample_colors(None, x.ctypes.data_as(fp), 0 if case == "n_zero" else 4, v,
                                         x.ctypes.data_as(fp), m.ctypes.data_as(i32p), None, single_c,
                                         single_co) == capi.TZR_ERR_INVALID_ARG
