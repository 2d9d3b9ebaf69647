"""CPU checks of tzr_register_cloud_pairs' C-ABI: the entry point and its parameter defaults are exported, declared in
the header with the argument list the Python binding passes, listed among the symbols capi.lib() checks, and
tzr_frontend_params has the layout and defaults of the reference's FPFHEstimation::computeFPFHFeatures and
Matcher::calculateCorrespondences."""
import ctypes as C
import importlib
import os
import re

import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds", "tuple_seeds", "solutions", "status",
        "problem_index", "n_corr", "corr", "cliques", "global_scale"]


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)


def test_symbol_exported_declared_and_bound(header):
    m = re.search(r"int\s+tzr_register_cloud_pairs\s*\(([^)]*)\)", header)
    assert m, "tzr_register_cloud_pairs missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS
    for name in ("tzr_register_cloud_pairs", "tzr_frontend_params_default"):
        assert name in capi._SYMBOLS
    assert len(capi.lib().tzr_register_cloud_pairs.argtypes) == len(ARGS)
    assert "#define TZR_ABI_VERSION 2" in header


def test_frontend_params_layout_and_defaults(header):
    m = re.search(r"typedef struct tzr_frontend_params \{(.*?)\} tzr_frontend_params;", header, flags=re.S)
    assert m
    fields = re.findall(r"(double|int32_t|float)\s+(\w+);", m.group(1))
    ctypes_of = {"double": C.c_double, "int32_t": C.c_int32, "float": C.c_float}
    assert [(n, ctypes_of[t]) for t, n in fields] == capi.FrontendParams._fields_
    assert C.sizeof(capi.FrontendParams) == 32
    p = capi.FrontendParams()
    capi.lib().tzr_frontend_params_default(C.byref(p))
    # FPFHEstimation::computeFPFHFeatures(cloud, 0.03, 0.05) and calculateCorrespondences(..., true, true, true, 0)
    assert (p.normal_search_radius, p.fpfh_search_radius) == (0.03, 0.05)
    assert (p.use_absolute_scale, p.use_crosscheck, p.use_tuple_test, p.tuple_scale) == (1, 1, 1, 0.0)


def test_argument_checks_need_no_device():
    """Malformed calls are refused before the device is touched (a NULL context, no clouds, no pairs)."""
    L = capi.lib()
    fp = capi.FrontendParams()
    L.tzr_frontend_params_default(C.byref(fp))
    prm = capi.Params()
    L.tzr_params_default(C.byref(prm))
    assert L.tzr_register_cloud_pairs(None, C.byref(fp), C.byref(prm), 1, None, None, 1, None, None, None, None, None,
                                      None, None, None, None) == capi.TZR_ERR_INVALID_ARG
