"""GPU tests of the certifier batch (`pytest -m gpu`): tzr_certify_batch against the reference's fixtures (1e-7, as in
certification-test.cc:29), against tzr_certify on each problem alone and against oracle/certifier_oracle.py."""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import certifier_oracle as co  # noqa: E402
import certifier_fixtures as cf  # noqa: E402

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu
TOL = 1e-7
LOOP_EIG = 2097152  # debug flag: one cusolverDnDsyevd per active problem instead of cusolverDnXsyevBatched
FIXTURES = cf.cases("small") + cf.cases("large")
NB = FIXTURES[0]["params"]["noise_bound"]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _fixture_problem(c):
    """(R, v1, v2, theta) of a fixture under the batch's common noise bound NB.  The problem is homogeneous: scaling
    v1, v2 and the noise bound by s scales M_init, every iterate and mu by s^2, so the gap trajectory is unchanged."""
    s = NB / c["params"]["noise_bound"]
    return c["R_est"], s * c["v1"], s * c["v2"], c["theta_est"]


def _instance(N, seed, wrong_rotation=False, outliers=0.1):
    """Random100Points-style instance (certification-test.cc:529-644): exact rotation with far outliers converges on
    the first iteration; a wrong rotation never reaches the sub-optimality threshold."""
    rng = np.random.default_rng(seed)
    v1 = rng.uniform(-1, 1, size=(3, N))
    R = synth.random_rotation(rng)
    v2 = R @ v1
    theta = np.ones(N)
    k0 = int(N * (1 - outliers))
    v2[:, k0:] = rng.uniform(-1, 1, size=(3, N - k0)) * 5 + 5
    theta[k0:] = -1
    if wrong_rotation:
        R = synth.random_rotation(rng)
    return R, v1, v2, theta


def _batch(ctx, probs, **kw):
    return ctx.certify_batch([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs],
                             [p[3] for p in probs], **kw)


def _close(a, b, tol):
    return len(a) == len(b) and (len(a) == 0 or np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()))


@pytest.mark.parametrize("order", ["forward", "reversed"])
def test_all_fixtures_in_one_batch(ctx, order):
    cases = FIXTURES if order == "forward" else FIXTURES[::-1]
    probs = [_fixture_problem(c) for c in cases]
    out = _batch(ctx, probs, noise_bound=NB, cbar2=1.0, max_iterations=1000)
    for c, p, r in zip(cases, probs, out):
        want = c["suboptimality_traj"]
        assert len(r["suboptimality_traj"]) == len(want), c["name"]
        assert np.abs(r["suboptimality_traj"] - want).max() < TOL, c["name"]
        assert abs(r["best_suboptimality"] - want.min()) < TOL
        one = ctx.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"], noise_bound=c["params"]["noise_bound"],
                          cbar2=1.0, max_iterations=c["params"].get("max_iterations", 200))
        assert r["is_optimal"] == one["is_optimal"], c["name"]
        assert len(r["suboptimality_traj"]) == len(one["suboptimality_traj"]), c["name"]


def _mixed_problems():
    return [_instance(1, 0), _instance(40, 1, wrong_rotation=True), _instance(250, 2), _instance(12, 3),
            _instance(30, 4, wrong_rotation=True), _instance(5, 5)]


@pytest.mark.parametrize("flags", [0, LOOP_EIG], ids=["default_route", "loop_route"])
def test_mixed_random_batch_matches_oracle_and_single_call(ctx, flags):
    probs = _mixed_problems()
    kw = dict(noise_bound=0.01, cbar2=1.0, max_iterations=25)
    ctx.set_flags(flags)
    try:
        out = _batch(ctx, probs, **kw)
    finally:
        ctx.set_flags(0)
    lens = [len(r["suboptimality_traj"]) for r in out]
    assert min(lens) == 1 and max(lens) == 25  # a problem done on iteration 1 beside ones that run to the cap
    for p, r in zip(probs, out):
        o = co.certify(*p, 0.01, 1.0, max_iterations=25)
        one = ctx.certify(*p, **kw)
        assert _close(r["suboptimality_traj"], o["suboptimality_traj"], 1e-6)
        assert _close(r["suboptimality_traj"], one["suboptimality_traj"], 1e-6)
        assert r["is_optimal"] == one["is_optimal"] == o["is_optimal"]


def test_single_problem_batch_equals_certify(ctx):
    """tzr_certify is tzr_certify_batch with B = 1: the same results, bit for bit."""
    cases = [((c["R_est"], c["v1"], c["v2"], c["theta_est"]), dict(noise_bound=c["params"]["noise_bound"], cbar2=1.0))
             for c in FIXTURES[:4]]
    cases += [(p, dict(noise_bound=0.01, cbar2=1.0, max_iterations=25)) for p in _mixed_problems()]
    for args, kw in cases:
        (r,) = ctx.certify_batch(*[[a] for a in args], **kw)
        one = ctx.certify(*args, **kw)
        assert r["is_optimal"] == one["is_optimal"]
        assert np.array_equal(r["suboptimality_traj"], one["suboptimality_traj"])
        assert r["best_suboptimality"] == one["best_suboptimality"]


def test_eigen_routes_agree(ctx):
    """Nine problems: the batched call over all of them, then over the eight still active after iteration 9 (compact
    batch), then the Dsyevd loop once fewer than eight remain; against the Dsyevd loop throughout."""
    probs = [_fixture_problem(c) for c in FIXTURES[:4]] + [_instance(60, 9, wrong_rotation=True)] + \
        [_instance(20 + 5 * b, 70 + b, wrong_rotation=True) for b in range(4)]
    kw = dict(noise_bound=NB, cbar2=1.0, max_iterations=40)
    a = _batch(ctx, probs, **kw)
    ctx.set_flags(LOOP_EIG)
    try:
        b = _batch(ctx, probs, **kw)
    finally:
        ctx.set_flags(0)
    for x, y in zip(a, b):
        assert x["is_optimal"] == y["is_optimal"]
        assert _close(x["suboptimality_traj"], y["suboptimality_traj"], 1e-7)


def _raw_batch(ctx, probs, params, traj_caps, null_traj=()):
    """tzr_certify_batch through ctypes with caller-chosen trajectory capacities and NULL entries."""
    B = len(probs)
    ins = [capi.Context._cert_inputs(*p) for p in probs]
    R = np.ascontiguousarray(np.concatenate([i[0].ravel() for i in ins]))
    N = np.array([i[3].size for i in ins], dtype=np.int32)
    trajs = [np.full(max(1, k), -7.0) for k in traj_caps]
    caps = np.array(traj_caps, dtype=np.int32)
    res = (capi.CertificationResult * B)()
    for r in res:
        r.is_optimal, r.n_iterations, r.best_suboptimality = -5, -5, -5.0
    dp = C.POINTER(C.c_double)
    arr = lambda xs: (dp * B)(*[C.cast(None, dp) if x is None else capi._p(x, C.c_double) for x in xs])
    rc = capi.lib().tzr_certify_batch(ctx._h, C.byref(params), B, capi._p(N, C.c_int32), capi._p(R, C.c_double),
                                      arr([i[1] for i in ins]), arr([i[2] for i in ins]), arr([i[3] for i in ins]),
                                      res, arr([None if b in null_traj else t for b, t in enumerate(trajs)]),
                                      capi._p(caps, C.c_int32))
    return rc, res, trajs


def test_short_capacity_and_null_trajectories(ctx):
    probs = [_instance(20, 11, wrong_rotation=True), _instance(8, 12), _instance(16, 13, wrong_rotation=True)]
    p = ctx.certifier_params(noise_bound=0.01, cbar2=1.0, max_iterations=12)
    rc, res, trajs = _raw_batch(ctx, probs, p, [5, 12, 12], null_traj=(2,))
    assert rc == 0
    full = _batch(ctx, probs, noise_bound=0.01, cbar2=1.0, max_iterations=12)
    for b in range(3):
        assert res[b].n_iterations == len(full[b]["suboptimality_traj"])
        assert bool(res[b].is_optimal) == full[b]["is_optimal"]
    assert res[0].n_iterations == 12
    assert np.array_equal(trajs[0], full[0]["suboptimality_traj"][:5])  # capacity 5 < 12 iterations
    k = res[1].n_iterations
    assert np.array_equal(trajs[1][:k], full[1]["suboptimality_traj"]) and np.all(trajs[1][k:] == -7.0)
    # traj itself NULL
    B = len(probs)
    ins = [capi.Context._cert_inputs(*q) for q in probs]
    R = np.ascontiguousarray(np.concatenate([i[0].ravel() for i in ins]))
    N = np.array([i[3].size for i in ins], dtype=np.int32)
    out = (capi.CertificationResult * B)()
    dp = C.POINTER(C.c_double)
    arr = lambda xs: (dp * B)(*[capi._p(x, C.c_double) for x in xs])
    assert capi.lib().tzr_certify_batch(ctx._h, C.byref(p), B, capi._p(N, C.c_int32), capi._p(R, C.c_double),
                                        arr([i[1] for i in ins]), arr([i[2] for i in ins]), arr([i[3] for i in ins]),
                                        out, None, None) == 0
    assert [o.n_iterations for o in out] == [r.n_iterations for r in res]


def test_launch_count_does_not_grow_with_batch(ctx):
    """At a fixed iteration count (sub_optimality < 0: no problem stops early) the batched-eigen route launches the
    same kernels and eigensolver calls for B = 8 and B = 12: per iteration 13 kernels and one cusolverDnXsyevBatched
    call per eigen step, plus the update.  Under flag 2097152 every problem costs one cusolverDnDsyevd per step, so a
    silent fall-back to the loop would show in the count.  (Fewer than 8 active problems take the loop route.)"""
    prob = _instance(24, 21)
    p = ctx.certifier_params(noise_bound=0.01, cbar2=1.0, max_iterations=6, sub_optimality=-1.0)
    counts = {}
    for flags in (0, LOOP_EIG):
        ctx.set_flags(flags)
        try:
            for B in (8, 12):
                before = ctx.kernel_launches()
                rc, res, _ = _raw_batch(ctx, [prob] * B, p, [6] * B)
                assert rc == 0 and all(r.n_iterations == 6 for r in res)
                counts[flags, B] = ctx.kernel_launches() - before
        finally:
            ctx.set_flags(0)
    assert counts[0, 8] == counts[0, 12] == 3 + 6 * (13 + 2) + 5
    for B in (8, 12):
        assert counts[LOOP_EIG, B] == 3 + 6 * (13 + 2 * B) + 5


def test_finished_problems_leave_the_eigensolver(ctx):
    """Six problems done on iteration 1 beside ten that run to the cap: from iteration 2 on, the ten active ones are
    gathered into a compact batch (gather + XsyevBatched + scatter per eigen step), so the eigensolver never sees the
    finished ones; results as on the loop route."""
    done = (0, 3, 5)
    probs = [_instance(8 + 3 * b, 60 + b, wrong_rotation=b % 8 not in done) for b in range(16)]
    p = ctx.certifier_params(noise_bound=0.01, cbar2=1.0, max_iterations=8)
    before = ctx.kernel_launches()
    rc, res, trajs = _raw_batch(ctx, probs, p, [8] * 16)
    launches = ctx.kernel_launches() - before
    assert rc == 0 and [r.n_iterations for r in res] == [1 if b % 8 in done else 8 for b in range(16)]
    # iteration 1: 13 + 2 in place, update; iterations 2-8: 13 + 2 * 3 (gather, call, scatter), updates but the last
    assert launches == 3 + (13 + 2 + 1) + 7 * (13 + 6) + 6
    ctx.set_flags(LOOP_EIG)
    try:
        rc2, res2, trajs2 = _raw_batch(ctx, probs, p, [8] * 16)
    finally:
        ctx.set_flags(0)
    assert rc2 == 0
    for r, r2, t, t2 in zip(res, res2, trajs, trajs2):
        assert r.n_iterations == r2.n_iterations and r.is_optimal == r2.is_optimal
        k = r.n_iterations
        assert _close(t[:k], t2[:k], 1e-7)


def test_trajectories_without_capacities_rejected(ctx):
    probs = [_instance(6, 51), _instance(7, 52)]
    ins = [capi.Context._cert_inputs(*q) for q in probs]
    R = np.ascontiguousarray(np.concatenate([i[0].ravel() for i in ins]))
    N = np.array([i[3].size for i in ins], dtype=np.int32)
    out = (capi.CertificationResult * 2)()
    trajs = [np.zeros(200), np.zeros(200)]
    dp = C.POINTER(C.c_double)
    arr = lambda xs: (dp * 2)(*[capi._p(x, C.c_double) for x in xs])
    p = ctx.certifier_params()
    assert capi.lib().tzr_certify_batch(ctx._h, C.byref(p), 2, capi._p(N, C.c_int32), capi._p(R, C.c_double),
                                        arr([i[1] for i in ins]), arr([i[2] for i in ins]), arr([i[3] for i in ins]),
                                        out, arr(trajs), None) == -1  # TZR_ERR_INVALID_ARG


def test_too_large_problem_writes_no_result(ctx):
    big = _instance(8192, 31)  # 4N + 4 = 32772 > 32768
    probs = [_instance(10, 32), big, _instance(12, 33)]
    p = ctx.certifier_params(noise_bound=0.01, cbar2=1.0)
    rc, res, trajs = _raw_batch(ctx, probs, p, [200, 200, 200])
    assert rc == -6  # TZR_ERR_TOO_LARGE
    assert all(r.n_iterations == -5 and r.is_optimal == -5 for r in res)
    assert all(np.all(t == -7.0) for t in trajs)


def test_pybind_certify_batch_matches_fixtures():
    """teaserpp_python.DRSCertifier.certify_batch through the C++ façade's certifyBatch (bool and +-1 overloads)."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tpp
    cases = cf.cases("small")
    p = tpp.DRSCertifier.Params()
    p.noise_bound = cases[0]["params"]["noise_bound"]
    p.cbar2 = 1.0
    cert = tpp.DRSCertifier(p)
    args = [[c[k] for c in cases] for k in ("R_est", "v1", "v2")]
    r = cert.certify_batch(*args, [c["theta_est"] for c in cases])
    r2 = cert.certify_batch(*args, [c["theta_est"] > 0 for c in cases])
    for c, x, y in zip(cases, r, r2):
        assert np.abs(np.asarray(x.suboptimality_traj) - c["suboptimality_traj"]).max() < TOL
        assert x.is_optimal and abs(x.best_suboptimality - c["suboptimality_traj"].min()) < TOL
        assert np.array_equal(np.asarray(y.suboptimality_traj), np.asarray(x.suboptimality_traj))
