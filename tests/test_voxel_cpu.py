"""CPU checks of the voxel downsampling C-ABI (tzr_voxel_downsample, tzr_voxel_downsample_batch): the entry points are
exported, declared in the header with the argument lists the Python binding passes and listed among the symbols
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
    "tzr_voxel_downsample": ["ctx", "pts", "n", "voxel_size", "pts_out", "n_out", "voxel_of"],
    "tzr_voxel_downsample_batch": ["ctx", "B", "n", "pts", "voxel_size", "pts_out", "n_out", "voxel_of", "status"],
}


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
    assert "#define TZR_ABI_VERSION 2" in header
    assert capi.lib().tzr_abi_version() == 2


def call_batch(ctx, B=2, n=4, v=0.1, null=None):
    L = capi.lib()
    x = np.zeros((4, 3), dtype=np.float32)
    out = np.zeros((4, 3), dtype=np.float32)
    fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    nn = np.array([4, n], dtype=np.int32)
    m = np.zeros(2, dtype=np.int32)
    pts = (fp * 2)(x.ctypes.data_as(fp), None if null == "pts_entry" else x.ctypes.data_as(fp))
    outs = (fp * 2)(out.ctypes.data_as(fp), None if null == "pts_out_entry" else out.ctypes.data_as(fp))
    return L.tzr_voxel_downsample_batch(ctx, B, None if null == "n" else nn.ctypes.data_as(i32p),
                                        None if null == "pts" else pts, v, None if null == "pts_out" else outs,
                                        None if null == "n_out" else m.ctypes.data_as(i32p), None, None)


CASES = {
    "null_ctx": {}, "v_zero": dict(v=0.0), "v_negative": dict(v=-0.05), "v_nan": dict(v=float("nan")),
    "v_inf": dict(v=float("inf")), "B_zero": dict(B=0), "B_negative": dict(B=-1), "n_zero": dict(n=0),
    "n_negative": dict(n=-3), "n_null": dict(null="n"), "pts_null": dict(null="pts"),
    "pts_entry_null": dict(null="pts_entry"), "pts_out_null": dict(null="pts_out"),
    "pts_out_entry_null": dict(null="pts_out_entry"), "n_out_null": dict(null="n_out"),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_argument_checks_need_no_device(case):
    """Malformed calls return TZR_ERR_INVALID_ARG without a device (the context is NULL here, and every argument check
    runs before the device is touched)."""
    assert call_batch(None, **CASES[case]) == capi.TZR_ERR_INVALID_ARG
    if case in ("null_ctx", "v_zero", "v_negative", "v_nan", "v_inf", "n_zero"):
        kw = CASES[case]
        x = np.zeros((3, 3), dtype=np.float32)
        fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        m = np.zeros(1, dtype=np.int32)
        assert capi.lib().tzr_voxel_downsample(None, x.ctypes.data_as(fp), kw.get("n", 3), kw.get("v", 0.1),
                                               x.ctypes.data_as(fp), m.ctypes.data_as(i32p), None) == \
            capi.TZR_ERR_INVALID_ARG


def test_python_binding_refuses_malformed_clouds():
    # checked in Python before the library is called: no context or device needed
    ctx = object.__new__(capi.Context)
    with pytest.raises(capi.TzrError):
        capi.Context.voxel_downsample(ctx, np.zeros((4, 2)), 0.1)
    with pytest.raises(capi.TzrError):
        capi.Context.voxel_downsample_batch(ctx, [], 0.1)
    with pytest.raises(capi.TzrError):
        capi.Context.voxel_downsample_batch(ctx, [np.zeros((0, 3))], 0.1)
