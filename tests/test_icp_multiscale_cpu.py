"""CPU checks of multi-scale ICP (tzr_icp_multiscale_batch): the entry is declared with the argument order the bindings
pass, the structs and method numbers match the header, scales parse as documented, and malformed calls are refused by
the bindings before any device work."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARGS = ["ctx", "method", "S", "scales", "n_clouds", "n", "pts", "colors", "P", "pair_clouds", "init", "epsilon",
        "lambda_geometric", "kernel", "results", "n_down", "status", "information", "info_counts"]


@pytest.fixture(scope="module")
def header_text():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return open(os.path.join(ROOT, "include", "teaser_b200.h")).read()


@pytest.fixture(scope="module")
def header(header_text):
    return re.sub(r"/\*.*?\*/", "", header_text, flags=re.S)


def test_declared_in_the_order_the_bindings_pass(header):
    m = re.search(r"int\s+tzr_icp_multiscale_batch\s*\(([^)]*)\)", header)
    assert m, "tzr_icp_multiscale_batch missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS
    assert "tzr_icp_multiscale_batch" in capi._SYMBOLS
    at = capi.lib().tzr_icp_multiscale_batch.argtypes
    assert len(at) == len(ARGS)
    assert at[3] is C.POINTER(capi.IcpScale) and at[10] is C.POINTER(capi.Similarity)
    assert at[13] is C.POINTER(capi.RobustKernel) and at[14] is C.POINTER(capi.IcpResult)
    assert at[11] is C.c_double and at[12] is C.c_double


def test_struct_and_methods_match_the_header(header):
    m = re.search(r"typedef struct tzr_icp_scale \{(.*?)\} tzr_icp_scale;", header, flags=re.S)
    names = re.findall(r"(\w+)\s*[,;]", m.group(1))
    assert names == [f[0] for f in capi.IcpScale._fields_]
    assert C.sizeof(capi.IcpScale) == 48
    for name, v in capi.ICP_METHODS.items():
        assert re.search(r"#define TZR_ICP_%s\s+%d\b" % (name.upper(), v), header), name


def test_scales_parse():
    a = capi.icp_scale(dict(voxel_size=0.05, max_correspondence_distance=0.07, max_iteration=50))
    assert (a.voxel_size, a.max_correspondence_distance, a.normal_search_radius, a.relative_fitness, a.relative_rmse,
            a.max_iteration) == (0.05, 0.07, 0.1, 1e-6, 1e-6, 50)
    b = capi.icp_scale((0.025, 0.035, 30, 0.06, 1e-5, 1e-4))
    assert (b.normal_search_radius, b.relative_fitness, b.relative_rmse, b.max_iteration) == (0.06, 1e-5, 1e-4, 30)
    c = capi.icp_scale((0.0, 0.01, 14))
    assert c.voxel_size == 0.0 and c.normal_search_radius == 0.0  # a dense scale names its own normal radius
    assert capi.icp_scale(a) is a
    # the library checks the values, the bindings only the shape
    assert capi.icp_scale(dict(voxel_size=-1, max_correspondence_distance=0, max_iteration=-3)).max_iteration == -3


@pytest.mark.parametrize("bad", [dict(voxel_size=0.05, max_iteration=3), dict(voxel_size=0.05, max_correspondence_distance=1,
                                                                              max_iteration=3, radius=1),
                                 (0.05, 0.07), (0.05, 0.07, 3, 0.1, 1e-6, 1e-6, 0)])
def test_malformed_scales_refused(bad):
    with pytest.raises(capi.TzrError, match="icp_scale"):
        capi.icp_scale(bad)


def _deviceless_context():
    ctx = object.__new__(capi.Context)
    ctx._h = C.c_void_p()  # NULL: any call that reached the library would be refused there, not here
    return ctx


def _scene():
    rng = np.random.default_rng(0)
    clouds = [rng.standard_normal((20, 3)).astype(np.float32) for _ in range(3)]
    return clouds, [np.full((20, 3), 0.5, dtype=np.float32) for _ in clouds], [(0, 1), (2, 1)]


SCALES = [(0.1, 0.2, 5), (0.05, 0.1, 3)]


@pytest.mark.parametrize("case,match", [
    ("no_clouds", "clouds"), ("pairs_shape", r"\(P,2\)"), ("pair_index", "outside"), ("no_scales", "scale"),
    ("method_name", "unknown method"), ("method_number", "unknown method"), ("colored_without_colors", "colou?rs"),
("colour_count", "colou?rs"), ("colour_rows", "colou?rs"),
    ("seed_count", "seed"), ("kernel_point_to_point", "kernel"), ("kernel_name", "kernel"), ("empty_cloud", "non-empty")])
def test_python_checks_need_no_device(case, match):
    ctx = _deviceless_context()
    clouds, cols, pairs = _scene()
    kw = dict(clouds=clouds, pairs=pairs, scales=SCALES, method="point_to_plane")
    if case == "no_clouds":
        kw["clouds"] = []
    elif case == "pairs_shape":
        kw["pairs"] = [0, 1]
    elif case == "pair_index":
        kw["pairs"] = [(0, 3)]
    elif case == "no_scales":
        kw["scales"] = []
    elif case == "method_name":
        kw["method"] = "point_to_line"
    elif case == "method_number":
        kw["method"] = 4
    elif case == "colored_without_colors":
        kw["method"] = "colored"
    elif case == "colour_count":
        kw.update(method="colored", colors=cols[:2])
    elif case == "colour_rows":
        kw.update(method="colored", colors=[cols[0], cols[1][:19], cols[2]])
    elif case == "seed_count":
        kw["inits"] = [None]
    elif case == "kernel_point_to_point":
        kw.update(method="point_to_point", kernel=("huber", 0.1))
    elif case == "kernel_name":
        kw["kernel"] = "welsch"
    elif case == "empty_cloud":
        kw["clouds"] = [clouds[0], np.zeros((0, 3), np.float32), clouds[2]]
    with pytest.raises(capi.TzrError, match=match):
        ctx.icp_multiscale(**kw)


def test_null_context_is_refused_by_the_library():
    clouds, _, pairs = _scene()
    fp = C.POINTER(C.c_float)
    n = np.array([20, 20, 20], dtype=np.int32)
    pc = np.ascontiguousarray(pairs, dtype=np.int32)
    sc = (capi.IcpScale * 2)(*[capi.icp_scale(s) for s in SCALES])
    init = (capi.Similarity * 2)(capi.similarity(None), capi.similarity(None))
    res = (capi.IcpResult * 4)()
    rc = capi.lib().tzr_icp_multiscale_batch(None, 1, 2, sc, 3, n.ctypes.data_as(C.POINTER(C.c_int32)),
                                             (fp * 3)(*[c.ctypes.data_as(fp) for c in clouds]), None, 2,
                                             pc.ctypes.data_as(C.POINTER(C.c_int32)), init, 1e-3, 0.968, None, res,
                                             None, None, None, None)
    assert rc == capi.TZR_ERR_INVALID_ARG


def test_header_states_the_contract(header_text):
    i = header_text.index("refining registrations coarse to fine")
    block = header_text[i:header_text.index("tzr_icp_multiscale_batch(", i)]
    for phrase in ["The chain it equals", "tzr_information_matrix_batch", "INT_MAX", "4096 neighbours",
                   "carries its pose", "Launches, per scale", "a retained solve stays retained"]:
        assert phrase in block, phrase


class _Recorder:
    """Stands in for the library: records the arguments of tzr_icp_multiscale_batch and returns TZR_OK."""

    def __init__(self):
        self.args = None

    def tzr_icp_multiscale_batch(self, *args):
        self.args = args
        return 0


def _seeds_reaching_the_library(monkeypatch, inits, **kw):
    rec = _Recorder()
    monkeypatch.setattr(capi, "lib", lambda: rec)
    clouds, cols, pairs = _scene()
    _deviceless_context().icp_multiscale(clouds, pairs, SCALES, inits, **kw)
    init = rec.args[10]
    return rec.args, [(s.scale, list(s.rotation), list(s.translation)) for s in init]


def _solutions():
    sols = np.zeros(2, dtype=capi.SOLUTION_DTYPE)
    R = [np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]]), np.eye(3)]
    for k in range(2):
        sols[k]["valid"] = 1
        sols[k]["scale"] = 1.0 + 0.5 * k
        sols[k]["rotation"] = R[k].T.reshape(-1)  # column-major
        sols[k]["translation"] = [k, 2.0, -1.0]
    return sols, R


def test_solution_array_seeds_the_call(monkeypatch):
    sols, R = _solutions()
    _, got = _seeds_reaching_the_library(monkeypatch, sols)
    for k in range(2):
        assert got[k] == (1.0 + 0.5 * k, list(R[k].T.reshape(-1)), [k, 2.0, -1.0])


def test_matrix_array_seeds_the_call(monkeypatch):
    sols, R = _solutions()
    mats = np.stack([np.eye(4)] * 2)
    for k in range(2):
        mats[k, :3, :3] = R[k]
        mats[k, :3, 3] = [k, 2.0, -1.0]
    _, got = _seeds_reaching_the_library(monkeypatch, mats)
    for k in range(2):
        assert got[k] == (1.0, list(R[k].T.reshape(-1)), [k, 2.0, -1.0])


def test_colours_are_passed_for_coloured_icp_only(monkeypatch):
    _, cols, _ = _scene()
    args, _ = _seeds_reaching_the_library(monkeypatch, None, method="point_to_plane", colors=cols)
    assert args[7] is None
    args, _ = _seeds_reaching_the_library(monkeypatch, None, method="colored", colors=cols)
    assert args[7] is not None
