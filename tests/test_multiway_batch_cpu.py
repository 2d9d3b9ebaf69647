"""CPU checks of many-sequence multiway registration (tzr_register_cloud_pairs_multiway(_line_process)_batch):
exported, declared with their argument names and bound in capi; call-level refusals without a context (no crash,
nothing written); the binding's flattening and splitting on a fake; the host transform-and-concatenate reference of the fused
map against a float64 numpy restatement.  The refusals with a real context are checked in
test_gpu_multiway_batch.py."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from multiway_map_reference import transform_concat

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEAD = ["ctx", "fparams", "params", "n_clouds", "n", "pts", "P", "pair_clouds", "tuple_seeds", "solutions", "status",
        "problem_index", "n_corr", "corr", "cliques", "global_scale", "icp", "colors", "lambda_geometric", "kernel",
        "icp_results", "uncertain"]
TAIL = ["G", "graph_offsets", "map_voxel_size", "map_points", "map_counts", "map_colors"]
ARGS = {
    "tzr_register_cloud_pairs_multiway_batch": HEAD + ["pg", "information", "info_counts", "edge_weights", "edge_mask",
                                                       "poses", "pg_summaries", "pg_status"] + TAIL,
    "tzr_register_cloud_pairs_multiway_line_process_batch": HEAD + ["lp", "information", "info_counts",
                                                                    "edge_confidence", "edge_kept", "poses",
                                                                    "lp_summaries", "lp_status"] + TAIL,
}


@pytest.fixture(scope="module")
def header():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    return open(os.path.join(ROOT, "include", "teaser_b200.h")).read()


@pytest.mark.parametrize("name", sorted(ARGS))
def test_symbols_exported_declared_and_bound(header, name):
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, code)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ARGS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(ARGS[name])
    assert callable(capi.Context.register_multiway_batch)


def table(offsets=(0, 2, 4), pairs=((0, 1), (2, 3)), G=None, map_voxel_size=0.0):
    """The arguments of a call over four 8-point clouds (kept alive in the returned dict) and its outputs, every output
    filled with 0x5a so that a write shows"""
    n_clouds = offsets[-1] if len(offsets) else 4
    rng = np.random.default_rng(0)
    k = dict(n=np.full(n_clouds, 8, dtype=np.int32),
             clouds=[rng.normal(size=(8, 3)).astype(np.float32) for _ in range(n_clouds)],
             pc=np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2),
             off=np.ascontiguousarray(offsets, dtype=np.int32))
    P = k["pc"].shape[0]
    G = len(offsets) - 1 if G is None else G

    def fill(shape, dt):
        return np.frombuffer(b"\x5a" * (int(np.prod(shape)) * np.dtype(dt).itemsize), dtype=dt).reshape(shape).copy()

    k.update(status=fill(P, np.int32), n_corr=fill(P, np.int64), unc=np.zeros(P, dtype=np.int32),
             info=fill((P, 36), np.float64), icnt=fill(P, np.int32), w=fill(P, np.float64), m=fill(P, np.uint8),
             pg_status=fill(max(G, 1), np.int32), counts=fill(max(G, 1), np.int32),
             maps=[fill((32, 3), np.float32) for _ in range(max(G, 1))])
    k["watch"] = [k[x] for x in ("status", "n_corr", "info", "icnt", "w", "m", "pg_status", "counts")] + k["maps"]
    k["before"] = [a.tobytes() for a in k["watch"]]
    k["vox"] = map_voxel_size
    return k


def call(ctx, k, G, lp=False, colors=None):
    """One of the two entries on table(k); returns its return code and whether any output was written"""
    f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    P = k["pc"].shape[0]
    n_clouds = len(k["clouds"])
    fp = capi.FrontendParams(0.1, 0.15, 0, 1, 0, 0.0)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0)
    icp = capi.icp_params(0.05)
    sols = np.zeros(P, dtype=capi.SOLUTION_DTYPE)
    icp_res = np.zeros(P, dtype=capi.ICP_RESULT_DTYPE)
    poses = (capi.Similarity * n_clouds)()
    maps = None if k["maps"] is None else (f32p * len(k["maps"]))(*[m.ctypes.data_as(f32p) for m in k["maps"]])
    cols = None if colors is None else (f32p * n_clouds)(*[c.ctypes.data_as(f32p) for c in colors])
    opt = capi.line_process_params(0.05) if lp else capi.pose_graph_params(0.05)
    summ = ((capi.LineProcessSummary if lp else capi.PoseGraphSummary) * max(G, 1))()
    entry = getattr(capi.lib(), "tzr_register_cloud_pairs_multiway_line_process_batch" if lp else
                    "tzr_register_cloud_pairs_multiway_batch")
    rc = entry(ctx, C.byref(fp), C.byref(prm), n_clouds, k["n"].ctypes.data_as(i32p),
               (f32p * n_clouds)(*[c.ctypes.data_as(f32p) for c in k["clouds"]]), P, k["pc"].ctypes.data_as(i32p),
               None, sols.ctypes.data_as(C.POINTER(capi.Solution)), k["status"].ctypes.data_as(i32p), None,
               k["n_corr"].ctypes.data_as(C.POINTER(C.c_int64)), None, None, None, C.byref(icp), cols, 0.968, None,
               icp_res.ctypes.data_as(C.POINTER(capi.IcpResult)), k["unc"].ctypes.data_as(i32p), C.byref(opt),
               k["info"].ctypes.data_as(C.POINTER(C.c_double)), k["icnt"].ctypes.data_as(i32p),
               k["w"].ctypes.data_as(C.POINTER(C.c_double)), k["m"].ctypes.data_as(C.POINTER(C.c_uint8)), poses, summ,
               k["pg_status"].ctypes.data_as(i32p), G, k["off"].ctypes.data_as(i32p) if k["off"].size else None,
               k["vox"], maps, k["counts"].ctypes.data_as(i32p), None)
    written = [a.tobytes() for a in k["watch"]] != k["before"] or any(bytes(poses)) or sols.tobytes().strip(b"\0") \
        or icp_res.tobytes().strip(b"\0")
    return rc, bool(written)


# (offsets, pairs, G): every call-level refusal of the partition; test_gpu_multiway_batch.py runs them with a context
REFUSALS = {
    "G < 1": ((0, 4), ((0, 1),), 0),
    "off[0] != 0": ((1, 2, 4), ((1, 2),), None),
    "decreasing offsets": ((0, 3, 2, 4), ((0, 1),), None),
    "off[G] != n_clouds": ((0, 2, 3), ((0, 1),), None),
    "pair across graphs": ((0, 2, 4), ((0, 1), (1, 2)), None),
}


@pytest.mark.parametrize("lp", [False, True])
@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusals_without_a_context_write_nothing(case, lp):
    """Each refused partition with a NULL context: refused, no crash and no output written.  A NULL context is refused
    on its own, so this does not show which check refused the call; test_gpu_multiway_batch.py's
    test_call_level_refusals does, with a context and tzr_last_error."""
    offsets, pairs, G = REFUSALS[case]
    k = table(offsets, pairs, G)
    k["clouds"] += [k["clouds"][0]] * (4 - len(k["clouds"]))  # four clouds whatever off[G] says
    k["n"] = np.full(4, 8, dtype=np.int32)
    assert call(None, k, len(offsets) - 1 if G is None else G, lp=lp) == (capi.TZR_ERR_INVALID_ARG, False)


@pytest.mark.parametrize("lp", [False, True])
def test_null_context_refused(lp):
    k = table()
    assert call(None, k, 2, lp=lp) == (capi.TZR_ERR_INVALID_ARG, False)


# ---- the binding's flattening and splitting, on a fake ----------------------------------------------------------------
def test_flat_table():
    seqs = [[np.zeros((3, 3), np.float32)] * 3, [np.ones((2, 3), np.float32)] * 2, [np.zeros((1, 3), np.float32)]]
    pairs = [[(0, 1), (1, 2), (2, 0)], [(0, 1)], []]
    t = capi.multiway_batch_table(seqs, pairs, tuple_seeds=[[1, 2, 3], [4], []])
    assert t["offsets"].tolist() == [0, 3, 5, 6] and t["pair_offsets"] == [0, 3, 4, 4]
    assert t["pairs"].tolist() == [[0, 1], [1, 2], [2, 0], [3, 4]]
    assert t["uncertain"].tolist() == [0, 0, 1, 0]  # register_multiway's rule per sequence: (k, k + 1) certain
    assert t["tuple_seeds"] == [1, 2, 3, 4] and len(t["clouds"]) == 6 and t["colors"] is None
    t = capi.multiway_batch_table(seqs[:2], pairs[:2], uncertain=[[1, 1, 0], None])
    assert t["uncertain"].tolist() == [1, 1, 0, 0]
    for bad in (dict(pairs=pairs[:2]), dict(uncertain=[[0]] * 3), dict(pairs=[[(0, 3)], [], []]),
                dict(tuple_seeds=[[1], [2], []])):
        kw = dict(pairs=pairs, uncertain=None, tuple_seeds=None)
        kw.update(bad)
        with pytest.raises(capi.TzrError):
            capi.multiway_batch_table(seqs, kw["pairs"], kw["uncertain"], kw["tuple_seeds"])


def _deviceless_context():
    ctx = object.__new__(capi.Context)
    ctx._h = C.c_void_p()
    return ctx


@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_flattening_and_splitting_on_a_fake(monkeypatch, optimizer):
    """register_multiway_batch on a fake _register_pairs: the flat table it is given, and the per-sequence split of
    outputs that carry their own index"""
    seqs = [[np.full((4, 3), s * 10 + c, np.float32) for c in range(k)] for s, k in enumerate([3, 2, 4])]
    pairs = [[(0, 1), (1, 2)], [(1, 0)], [(0, 1), (2, 3), (3, 0)]]
    seen = {}

    def fake(self, clouds, pc, params, *a, multiway=None, colored=None, **kw):
        seen.update(clouds=clouds, pairs=np.asarray(pc), multiway=multiway, seeds=a[6], plane=kw["plane"])
        P, K = len(pc), len(clouds)
        sols = np.zeros(P, dtype=capi.SOLUTION_DTYPE)
        sols["clique_size"] = np.arange(P)
        index = np.array([-1, 0, 1, 2, -1, 3], dtype=np.int32)
        mw = dict(information=np.arange(P * 36.).reshape(P, 6, 6), counts=np.arange(P, dtype=np.int32),
                  poses=np.arange(K * 16.).reshape(K, 4, 4),
                  graphs=[dict(status=g, iterations=g + 1, map=np.full((g + 1, 3), g, np.float32)) for g in range(3)])
        mw.update(weights=np.arange(P) / 10, mask=np.arange(P) % 2 == 0)
        icp = np.zeros(P, dtype=capi.ICP_RESULT_DTYPE)
        icp["iterations"] = np.arange(P)
        return (sols, np.arange(P, dtype=np.int32), index, [np.full((p, 2), p, np.int32) for p in range(P)],
                [np.arange(p) for p in range(P)], [float(p) for p in range(P)], icp, mw)

    monkeypatch.setattr(capi.Context, "_register_pairs", fake)
    kw = dict(optimizer=optimizer, map_voxel_size=0.02)
    res = _deviceless_context().register_multiway_batch(seqs, pairs, None, 0.05, tuple_seeds=[[5, 6], [7], [8, 9, 1]],
                                                        **kw)
    assert [float(c[0, 0]) for c in seen["clouds"]] == [0, 1, 2, 10, 11, 20, 21, 22, 23]
    assert seen["pairs"].tolist() == [[0, 1], [1, 2], [4, 3], [5, 6], [7, 8], [8, 5]]
    unc, pg, off, vox = seen["multiway"]
    assert unc.tolist() == [0, 0, 1, 0, 0, 1] and off.tolist() == [0, 3, 5, 9] and vox == 0.02
    assert isinstance(pg, capi.LineProcessParams if optimizer == "line_process" else capi.PoseGraphParams)
    assert seen["seeds"] == [5, 6, 7, 8, 9, 1] and seen["plane"]
    assert len(res) == 3
    for s, (lo, hi) in enumerate([(0, 2), (2, 3), (3, 6)]):
        sols, status, index, corr, clq, gs, icp, d = res[s]
        assert sols["clique_size"].tolist() == list(range(lo, hi)) and status.tolist() == list(range(lo, hi))
        assert [int(c[0, 0]) if len(c) else 0 for c in corr] == list(range(lo, hi)) and gs == [float(p) for p in
                                                                                                 range(lo, hi)]
        assert [len(c) for c in clq] == list(range(lo, hi)) and icp["iterations"].tolist() == list(range(lo, hi))
        assert d["counts"].tolist() == list(range(lo, hi)) and d["information"].shape == (hi - lo, 6, 6)
        assert np.array_equal(d["weights"], np.arange(lo, hi) / 10)
        assert d["poses"][:, 0, 0].tolist() == [16. * c for c in range(*[(0, 3), (3, 5), (5, 9)][s])]
        assert d["status"] == s and d["iterations"] == s + 1 and d["map"].shape == (s + 1, 3)
    # problem indices counted within each sequence
    assert [r[2].tolist() for r in res] == [[-1, 0], [0], [0, -1, 1]]


def test_binding_checks_need_no_device():
    ctx = _deviceless_context()
    seqs = [[np.zeros((3, 3), np.float32)] * 2]
    with pytest.raises(capi.TzrError, match="optimizer"):
        ctx.register_multiway_batch(seqs, [[(0, 1)]], None, 0.05, optimizer="lm")
    with pytest.raises(capi.TzrError, match="kernel"):
        ctx.register_multiway_batch(seqs, [[(0, 1)]], None, 0.05, kernel="huber")
    with pytest.raises(capi.TzrError, match="per sequence"):
        ctx.register_multiway_batch(seqs, [[(0, 1)], []], None, 0.05)


# ---- the fused map's host reference ------------------------------------------------------------------------------------
def test_transform_concat_against_float64_restatement():
    rng = np.random.default_rng(3)
    clouds = [(rng.normal(size=(n, 3)) * 3).astype(np.float32) for n in (50, 1, 300)]
    poses = []
    for _ in clouds:
        T = np.eye(4)
        T[:3, :3] = Rotation.from_rotvec(rng.normal(size=3)).as_matrix()
        T[:3, 3] = rng.normal(size=3)
        poses.append(T)
    got = transform_concat(clouds, poses)
    want = np.concatenate([c.astype(np.float64) @ T[:3, :3].T + T[:3, 3] for c, T in zip(clouds, poses)])
    assert got.dtype == np.float32 and got.shape == (351, 3)
    # the same float64 values up to their summation order, so at most one float32 rounding apart
    assert np.all(np.abs(got.astype(np.float64) - want) <= np.spacing(np.abs(want).astype(np.float32)))
    assert np.mean(got == want.astype(np.float32)) > 0.99
    # the operation order, exactly: one point by hand
    T, p = poses[2], clouds[2][7].astype(np.float64)
    assert got[51 + 7, 1] == np.float32(((T[1, 0] * p[0] + T[1, 1] * p[1]) + T[1, 2] * p[2]) + T[1, 3])
    assert transform_concat([], []).shape == (0, 3)
