"""CPU checks of correspondence RANSAC's bindings (tzr_ransac, tzr_ransac_batch, tzr_register_cloud_pairs_ransac): the
entries are declared with the argument order the bindings pass, tzr_ransac_params and tzr_ransac_info match the header
and the defaults are Open3D's, malformed calls are refused before any device work, and ragged correspondences, seeds and
normals are packed as the library reads them."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = {
    "tzr_ransac": ["ctx", "params", "src", "ns", "dst", "nd", "n_corr", "corr", "seed", "src_normals", "dst_normals",
                   "result", "info", "eval_corr"],
    "tzr_ransac_batch": ["ctx", "params", "B", "ns", "src", "nd", "dst", "n_corr", "corr", "seeds", "src_normals",
                         "dst_normals", "results", "info", "eval_corr"],
    "tzr_register_cloud_pairs_ransac": ["ctx", "fparams", "ransac", "n_clouds", "n", "pts", "P", "pair_clouds",
                                        "tuple_seeds", "ransac_seeds", "status", "n_corr", "corr", "global_scale",
                                        "results", "info"],
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
    i32p, fpp = C.POINTER(C.c_int32), C.POINTER(C.POINTER(C.c_float))
    at = L.tzr_ransac.argtypes
    assert at[1] is C.POINTER(capi.RansacParams) and at[8] is C.c_uint64 and at[12] is C.POINTER(capi.RansacInfo)
    at = L.tzr_ransac_batch.argtypes
    assert at[8] is C.POINTER(i32p) and at[9] is C.POINTER(C.c_uint64) and at[10] is fpp and at[11] is fpp
    assert at[12] is C.POINTER(capi.IcpResult) and at[13] is C.POINTER(capi.RansacInfo)
    at = L.tzr_register_cloud_pairs_ransac.argtypes
    assert at[2] is C.POINTER(capi.RansacParams) and at[8] is C.POINTER(C.c_uint64) and at[9] is C.POINTER(C.c_uint64)
    assert at[14] is C.POINTER(capi.IcpResult) and at[15] is C.POINTER(capi.RansacInfo)


def _fields(header, name):
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), header, flags=re.S)
    return re.findall(r"(\w+)\s*;", m.group(1))


def test_structs_and_defaults(header):
    names = _fields(header, "tzr_ransac_params")
    assert names == [f[0] for f in capi.RansacParams._fields_]
    assert [getattr(capi.RansacParams, f).offset for f in names] == [0, 8, 12, 16, 24, 28, 32, 40, 48, 52, 56]
    names = _fields(header, "tzr_ransac_info")
    assert names == [f[0] for f in capi.RansacInfo._fields_] == list(capi.RANSAC_INFO_DTYPE.names)
    assert [getattr(capi.RansacInfo, f).offset for f in names] == [0, 4, 8, 12, 16, 20, 24]
    p = capi.RansacParams()
    capi.lib().tzr_ransac_params_default(C.byref(p))
    assert (p.max_correspondence_distance, p.ransac_n, p.max_iteration, p.confidence) == (0.0, 3, 100000, 0.999)
    assert (p.check_edge_length, p.check_distance, p.check_normal) == (0, 0, 0)
    assert p.edge_length_similarity == 0.9 and p.normal_angle_threshold == 0.52359877559829882
    q = capi.ransac_params(0.05, ransac_n=4, check_edge_length=1)
    assert (q.max_correspondence_distance, q.ransac_n, q.check_edge_length) == (0.05, 4, 1)
    with pytest.raises(AttributeError):
        capi.ransac_params(0.05, iterations=3)


def test_library_refuses_without_a_context():
    L = capi.lib()
    p = capi.ransac_params(0.05)
    res, info = capi.IcpResult(), capi.RansacInfo()
    x = np.zeros((4, 3), dtype=np.float32)
    fp = x.ctypes.data_as(C.POINTER(C.c_float))
    assert L.tzr_ransac(None, C.byref(p), fp, 4, fp, 4, 0, None, 0, None, None, C.byref(res), C.byref(info),
                        None) == capi.TZR_ERR_INVALID_ARG
    assert L.tzr_register_cloud_pairs_ransac(None, None, C.byref(p), 1, None, None, 1, None, None, None, None, None,
                                             None, None, None, None) == capi.TZR_ERR_INVALID_ARG


def _deviceless_context():
    ctx = object.__new__(capi.Context)
    ctx._h = C.c_void_p()
    return ctx


class _Recorder:
    """Stands in for the library: records tzr_ransac_batch's packed arguments and returns TZR_OK."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name != "tzr_ransac_batch":
            return getattr(self.real, name)

        def call(h, prm, B, ns, src, nd, dst, nc, corr, seeds, sn, dn, res, info, ev):
            rows = [np.ctypeslib.as_array(corr[b], shape=(nc[b], 2)).copy() if nc[b] else None for b in range(B)]
            nrm = None if not sn else [np.ctypeslib.as_array(sn[b], shape=(ns[b], 4)).copy() for b in range(B)]
            self.calls.append(dict(B=B, ns=[ns[b] for b in range(B)], nd=[nd[b] for b in range(B)],
                                   nc=[nc[b] for b in range(B)], rows=rows, seeds=[seeds[b] for b in range(B)],
                                   nrm=nrm, dn=bool(dn), n=prm._obj.ransac_n))
            return 0
        return call


def test_ragged_rows_seeds_and_normals_are_packed_per_problem(monkeypatch):
    rec = _Recorder(capi.lib())
    monkeypatch.setattr(capi, "lib", lambda: rec)
    ctx = _deviceless_context()
    rng = np.random.default_rng(0)
    S = [rng.standard_normal((n, 3)) for n in (5, 7, 3)]
    D = [rng.standard_normal((n, 3)) for n in (6, 2, 9)]
    K = [np.array([[0, 1], [4, 5]], dtype=np.int64), [], [(2, 8)]]
    ctx.ransac_batch(S, D, K, capi.ransac_params(0.1, ransac_n=4), seeds=[1, 2 ** 64 - 1, -1])
    c = rec.calls[0]
    assert c["B"] == 3 and c["ns"] == [5, 7, 3] and c["nd"] == [6, 2, 9] and c["nc"] == [2, 0, 1] and c["n"] == 4
    assert c["rows"][0].tolist() == [[0, 1], [4, 5]] and c["rows"][1] is None and c["rows"][2].tolist() == [[2, 8]]
    assert c["seeds"] == [1, 2 ** 64 - 1, 2 ** 64 - 1] and c["nrm"] is None and not c["dn"]
    SN = [rng.standard_normal((n, 3)) for n in (5, 7, 3)]
    ctx.ransac_batch(S, D, K, capi.ransac_params(0.1), src_normals=SN, dst_normals=[np.ones((n, 4)) for n in (6, 2, 9)])
    c = rec.calls[1]
    assert c["seeds"] == [0, 0, 0] and c["dn"]
    for a, b in zip(c["nrm"], SN):
        assert np.array_equal(a[:, :3], b.astype(np.float32)) and not a[:, 3].any()


@pytest.mark.parametrize("case", ["no_problems", "count_mismatch", "bad_rows", "empty_cloud", "seed_count",
                                  "normal_rows"])
def test_python_checks_need_no_device(case):
    ctx = _deviceless_context()
    x = np.zeros((4, 3), dtype=np.float32)
    kw = dict(srcs=[x], dsts=[x], corrs=[[(0, 0)]], ransac=capi.ransac_params(0.1))
    if case == "no_problems":
        kw.update(srcs=[], dsts=[], corrs=[])
    elif case == "count_mismatch":
        kw["corrs"] = []
    elif case == "bad_rows":
        kw["corrs"] = [[0, 1, 2]]
    elif case == "empty_cloud":
        kw["srcs"] = [np.zeros((0, 3), dtype=np.float32)]
    elif case == "seed_count":
        kw["seeds"] = [1, 2]
    elif case == "normal_rows":
        kw["src_normals"] = [np.zeros((3, 3))]
    with pytest.raises(capi.TzrError):
        ctx.ransac_batch(**kw)


@pytest.mark.parametrize("case", ["no_clouds", "pair_index", "seed_count", "ransac_seed_count"])
def test_chained_python_checks_need_no_device(case):
    ctx = _deviceless_context()
    clouds = [np.zeros((5, 3), dtype=np.float32)] * 2
    kw = dict(clouds=clouds, pairs=[(0, 1)], ransac=capi.ransac_params(0.1))
    if case == "no_clouds":
        kw["clouds"] = []
    elif case == "pair_index":
        kw["pairs"] = [(0, 2)]
    elif case == "seed_count":
        kw["tuple_seeds"] = [1, 2]
    elif case == "ransac_seed_count":
        kw["ransac_seeds"] = [1, 2]
    with pytest.raises(capi.TzrError, match="register_cloud_pairs_ransac"):
        ctx.register_cloud_pairs_ransac(**kw)
