"""CPU checks of Fast Global Registration's bindings (tzr_fgr, tzr_fgr_batch, tzr_register_cloud_pairs_fgr): the
entries are declared with the argument order the bindings pass, tzr_fgr_params matches the header and its defaults are
Open3D's, malformed calls are refused before any device work, and ragged correspondences are packed as the library
reads them."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_fgr": ["ctx", "params", "src", "ns", "dst", "nd", "n_corr", "corr", "result", "eval_corr"],
    "tzr_fgr_batch": ["ctx", "params", "B", "ns", "src", "nd", "dst", "n_corr", "corr", "results", "eval_corr"],
    "tzr_register_cloud_pairs_fgr": ["ctx", "fparams", "fgr", "n_clouds", "n", "pts", "P", "pair_clouds", "tuple_seeds",
                                     "status", "n_corr", "corr", "global_scale", "results"],
}


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)


@pytest.mark.parametrize("name", sorted(ARGS))
def test_declared_in_the_order_the_bindings_pass(header, name):
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, header)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])


def test_argument_types(header):
    L = capi.lib()
    i32p = C.POINTER(C.c_int32)
    assert L.tzr_fgr.argtypes[1] is C.POINTER(capi.FgrParams) and L.tzr_fgr.argtypes[6] is C.c_int
    assert L.tzr_fgr.argtypes[8] is C.POINTER(capi.IcpResult)
    at = L.tzr_fgr_batch.argtypes
    assert at[7] is i32p and at[8] is C.POINTER(i32p) and at[9] is C.POINTER(capi.IcpResult)
    at = L.tzr_register_cloud_pairs_fgr.argtypes
    assert at[1] is C.POINTER(capi.FrontendParams) and at[2] is C.POINTER(capi.FgrParams)
    assert at[10] is C.POINTER(C.c_int64) and at[13] is C.POINTER(capi.IcpResult)


def test_params_struct_and_defaults(header):
    m = re.search(r"typedef struct tzr_fgr_params \{(.*?)\} tzr_fgr_params;", header, flags=re.S)
    names = re.findall(r"(\w+)\s*;", m.group(1))
    assert names == [f[0] for f in capi.FgrParams._fields_]
    assert C.sizeof(capi.FgrParams) == 32
    assert [getattr(capi.FgrParams, f).offset for f in names] == [0, 8, 12, 16, 24, 28]
    p = capi.fgr_params()
    assert (p.division_factor, p.use_absolute_scale, p.decrease_mu, p.maximum_correspondence_distance,
            p.iteration_number, p.reserved) == (1.4, 0, 1, 0.025, 64, 0)
    assert capi.fgr_params(iteration_number=3).iteration_number == 3
    with pytest.raises(AttributeError):
        capi.fgr_params(iterations=3)


def test_library_refuses_without_a_context():
    L = capi.lib()
    p = capi.fgr_params()
    res = capi.IcpResult()
    x = np.zeros((4, 3), dtype=np.float32)
    fp = x.ctypes.data_as(C.POINTER(C.c_float))
    assert L.tzr_fgr(None, C.byref(p), fp, 4, fp, 4, 0, None, C.byref(res), None) == capi.TZR_ERR_INVALID_ARG
    assert L.tzr_register_cloud_pairs_fgr(None, None, C.byref(p), 1, None, None, 1, None, None, None, None, None, None,
                                          None) == capi.TZR_ERR_INVALID_ARG


def test_corr_rows_packing():
    assert capi.corr_rows([]).shape == (0, 2) and capi.corr_rows([]).dtype == np.int32
    assert capi.corr_rows(np.zeros((0, 2), dtype=np.int64)).shape == (0, 2)
    a = capi.corr_rows([(0, 1), (2, 3)])
    assert a.dtype == np.int32 and a.flags.c_contiguous and a.tolist() == [[0, 1], [2, 3]]
    b = np.arange(12, dtype=np.int64).reshape(6, 2)[::2]  # a strided int64 view
    assert not b.flags.c_contiguous and capi.corr_rows(b).tolist() == b.tolist()
    for bad in ([0, 1, 2], np.zeros((3, 3), dtype=np.int32), np.zeros((2, 2)), [[0, 2 ** 31]]):
        with pytest.raises(capi.TzrError, match="fgr"):
            capi.corr_rows(bad)


def _deviceless_context():
    ctx = object.__new__(capi.Context)
    ctx._h = C.c_void_p()
    return ctx


class _Recorder:
    """Stands in for the library: records tzr_fgr_batch's packed arguments and returns TZR_OK."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name != "tzr_fgr_batch":
            return getattr(self.real, name)

        def call(h, prm, B, ns, src, nd, dst, nc, corr, res, ev):
            rows = [np.ctypeslib.as_array(corr[b], shape=(nc[b], 2)).copy() if nc[b] else None for b in range(B)]
            self.calls.append(dict(B=B, ns=[ns[b] for b in range(B)], nd=[nd[b] for b in range(B)],
                                   nc=[nc[b] for b in range(B)], rows=rows, it=prm._obj.iteration_number))
            return 0
        return call


def test_ragged_correspondences_are_packed_per_problem(monkeypatch):
    rec = _Recorder(capi.lib())
    monkeypatch.setattr(capi, "lib", lambda: rec)
    ctx = _deviceless_context()
    rng = np.random.default_rng(0)
    S = [rng.standard_normal((n, 3)) for n in (5, 7, 3)]
    D = [rng.standard_normal((n, 3)) for n in (6, 2, 9)]
    K = [np.array([[0, 1], [4, 5]], dtype=np.int64), [], [(2, 8)]]
    ctx.fgr_batch(S, D, K, fgr=capi.fgr_params(iteration_number=5))
    c = rec.calls[0]
    assert c["B"] == 3 and c["ns"] == [5, 7, 3] and c["nd"] == [6, 2, 9] and c["nc"] == [2, 0, 1] and c["it"] == 5
    assert c["rows"][0].tolist() == [[0, 1], [4, 5]] and c["rows"][1] is None and c["rows"][2].tolist() == [[2, 8]]


@pytest.mark.parametrize("case", ["no_problems", "count_mismatch", "bad_rows", "empty_cloud", "cloud_shape"])
def test_python_checks_need_no_device(case):
    ctx = _deviceless_context()
    x = np.zeros((4, 3), dtype=np.float32)
    kw = dict(srcs=[x], dsts=[x], corrs=[[(0, 0)]])
    if case == "no_problems":
        kw = dict(srcs=[], dsts=[], corrs=[])
    elif case == "count_mismatch":
        kw["corrs"] = []
    elif case == "bad_rows":
        kw["corrs"] = [[0, 1, 2]]
    elif case == "empty_cloud":
        kw["srcs"] = [np.zeros((0, 3), dtype=np.float32)]
    elif case == "cloud_shape":
        kw["dsts"] = [np.zeros((4, 2), dtype=np.float32)]
    with pytest.raises(capi.TzrError):
        ctx.fgr_batch(**kw)


@pytest.mark.parametrize("case", ["no_clouds", "pair_index", "seed_count"])
def test_chained_python_checks_need_no_device(case):
    ctx = _deviceless_context()
    clouds = [np.zeros((5, 3), dtype=np.float32)] * 2
    kw = dict(clouds=clouds, pairs=[(0, 1)])
    if case == "no_clouds":
        kw["clouds"] = []
    elif case == "pair_index":
        kw["pairs"] = [(0, 2)]
    elif case == "seed_count":
        kw["tuple_seeds"] = [1, 2]
    with pytest.raises(capi.TzrError, match="register_cloud_pairs_fgr"):
        ctx.register_cloud_pairs_fgr(**kw)
