"""The unknown-scale stage's regenerating route (run on an H100: `pytest -m gpu`).

Above 8192 points, or at any n above 256 with a forced chunk capacity, the stage regenerates every TIM's ratio and range
from the points and sweeps the sorted end points in chunks (DESIGN.md §3.4).  That must not change anything: forced
small chunks (many chunks, tie groups split across them, partial tiles carried from chunk to chunk) give the records,
cliques and graphs of the default route, the radix sort of all 2K end points at once over stored ratios and ranges,
bit for bit, and the scale tzr_scalar_tls gives on its large path.  At 50000 and 65536 points, where the one-shot sort does not fit, default
parameters solve within a bounded scratch.
"""
import importlib
import math
import os
import subprocess
import sys

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

FLAG_LARGE = 262144     # tzr_scalar_tls through the radix-sort path at every size
SCRATCH_BOUND = 4 << 30  # the stage's scratch at any n <= 65536 (DESIGN.md §3.4: at most 3.5 GiB)
MAX_N = 65536


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0, max_n=MAX_N)
    yield c
    c.close()


@pytest.fixture()
def chunk(ctx):
    yield ctx.set_scale_chunk
    ctx.set_scale_chunk(0)
    ctx.set_flags(0)


def params(nb, **kw):
    return capi.default_params(noise_bound=nb, cbar2=1.0, **kw)


def lattice(n, rng):
    """Points on an integer lattice and an exact scaled, permuted-free copy: every TIM length repeats many times,
    so the sorted end points hold huge groups of equal keys."""
    side = int(math.ceil(n ** (1 / 3))) + 1
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    src = g[rng.choice(len(g), size=n, replace=False)]
    dst = src * 2.0
    out = rng.random(n) < 0.3
    dst[out] = g[rng.choice(len(g), size=int(out.sum()))] * 2.0
    return src, dst, 0.01


def duplicated(n, rng):
    pr = synth.make_problem(n, 0.5, int(rng.integers(1 << 30)), "ball", sigma=0.01,
                            noise_bound=synth.NOISE_BOUND_SIGMA_001)
    src, dst = pr["src"].copy(), pr["dst"] * 1.3
    k = n // 10
    src[-k:] = src[:k]          # repeated source points: d1 = 0, excluded measurements between kept ones
    dst[-2 * k:-k] = dst[:k]    # repeated target points: ratio 0
    return src, dst, pr["noise_bound"] * 1.3


def ball(n, rng, s=1.7):
    pr = synth.make_problem(n, 0.8, int(rng.integers(1 << 30)), "ball", sigma=0.01,
                            noise_bound=synth.NOISE_BOUND_SIGMA_001)
    return pr["src"], pr["dst"] * s, pr["noise_bound"] * s


CASES = {"lattice": lattice, "duplicated": duplicated, "ball": ball}


def _solve(ctx, src, dst, nb):
    out = ctx.solve(src, dst, params(nb))
    bits, deg = ctx.last_graph(0, src.shape[0])
    return out, bits, deg, ctx.last_scale_chunks()


def _same(a, b):
    off = capi.Solution.stage_ms.offset
    assert bytes(a[0]["sol"])[:off] == bytes(b[0]["sol"])[:off]  # every field but stage_ms, the scale's bits included
    assert np.array_equal(a[0]["clique"], b[0]["clique"])
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def _tims(src, dst, beta):
    """Each TIM's ratio and range in the stage's packed order, with its IEEE operation sequence."""
    i, j = np.triu_indices(src.shape[0], 1)

    def norm(p):
        d = p[j] - p[i]
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])

    d1, d2 = norm(src), norm(dst)
    with np.errstate(divide="ignore", invalid="ignore"):
        return d2 / d1, beta * (1.0 / d1)


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("n", [257, 300, 2000, 5000])
def test_chunks_match_default(ctx, chunk, n, case):
    src, dst, nb = CASES[case](n, np.random.default_rng(n + len(case)))
    ref = _solve(ctx, src, dst, nb)
    assert ref[3] == 1
    M = n * (n - 1)
    for k in sorted({2048, 3000, M // 5 + 1, M // 2 + 2048}):
        if M // k > 400:
            continue
        chunk(k)
        got = _solve(ctx, src, dst, nb)
        assert got[3] == -(-M // k) and got[3] > 1, (k, got[3])
        _same(ref, got)
    if n <= 2000:  # the one-shot radix sort over stored ratios and ranges
        x, r = _tims(src, dst, 2.0 * nb)
        ctx.set_flags(FLAG_LARGE)
        est, _ = ctx.scalar_tls(x, r)
        assert np.float64(est).tobytes() == np.float64(ref[0]["scale"]).tobytes()


def test_tie_groups_split_at_300(ctx, chunk):
    src, dst, nb = lattice(300, np.random.default_rng(3))
    x, r = _tims(src, dst, 2.0 * nb)
    kept = np.isfinite(x) & np.isfinite(r)
    q = np.arange(2 * len(x))
    keys = np.where(np.repeat(kept, 2), np.stack([x - r, x + r], 1).reshape(-1), np.inf)
    srt = keys[np.lexsort((q, keys))]
    cuts = np.arange(2048, len(srt), 2048)
    assert np.any(srt[cuts - 1] == srt[cuts])  # some chunk boundary falls inside a group of equal keys
    ref = _solve(ctx, src, dst, nb)
    chunk(2048)
    got = _solve(ctx, src, dst, nb)
    assert got[3] == -(-300 * 299 // 2048)
    _same(ref, got)


def _batch_same(ctx, chunk, srcs, dsts, nb):
    sols, cls = ctx.solve_batch(srcs, dsts, params(nb))
    chunk(3000)
    sols2, cls2 = ctx.solve_batch(srcs, dsts, params(nb))
    assert ctx.last_scale_chunks() > 1
    chunk(0)
    off = capi.Solution.stage_ms.offset
    for b in range(len(srcs)):
        assert sols[b].tobytes()[:off] == sols2[b].tobytes()[:off], b
        assert np.array_equal(cls[b], cls2[b]), b
        one, _ = ctx.solve_batch([srcs[b]], [dsts[b]], params(nb))  # the problem alone
        assert one[0]["scale"].tobytes() == sols[b]["scale"].tobytes(), b


def test_ragged_batch(ctx, chunk):
    rng = np.random.default_rng(11)
    probs = [CASES[sorted(CASES)[b % 3]](m, rng) for b, m in enumerate([300, 257, 1500, 700, 300, 2100])]
    _batch_same(ctx, chunk, [p[0] for p in probs], [p[1] for p in probs], max(p[2] for p in probs))


def test_uniform_batch(ctx, chunk):
    rng = np.random.default_rng(12)
    probs = [ball(700, rng, s=1.2 + 0.2 * b) for b in range(4)]
    _batch_same(ctx, chunk, [p[0] for p in probs], [p[1] for p in probs], max(p[2] for p in probs))


@pytest.mark.parametrize("n", [50000, 65536])
def test_default_params_large_n(ctx, n):
    torch = pytest.importorskip("torch")
    pr = synth.make_problem(n, 0.80, 45 + n, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    s = 1.7
    p = capi.default_params(noise_bound=pr["noise_bound"] * s)
    fresh = capi.Context(0, max_n=MAX_N)
    try:
        fixed = capi.default_params(noise_bound=pr["noise_bound"] * s, estimate_scaling=0)
        torch.cuda.synchronize()
        free0, _ = torch.cuda.mem_get_info()
        fresh.solve(pr["src"], pr["dst"] * s, fixed)
        free1, _ = torch.cuda.mem_get_info()
        out = fresh.solve(pr["src"], pr["dst"] * s, p)
        free2, _ = torch.cuda.mem_get_info()
        assert free1 - free2 <= SCRATCH_BOUND, (free0 - free1, free1 - free2)
        assert fresh.last_scale_chunks() > 1
    finally:
        fresh.close()
    assert out["valid"] and abs(out["scale"] - s) < 0.02 * s
    again = ctx.solve(pr["src"], pr["dst"] * s, p)
    assert np.float64(again["scale"]).tobytes() == np.float64(out["scale"]).tobytes()
    assert np.array_equal(again["clique"], out["clique"])


def test_teaserpp_python_50000_default_params():
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tp
    pr = synth.make_problem(50000, 0.80, 46, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    s = 1.7
    p = tp.RobustRegistrationSolver.Params()
    assert p.estimate_scaling
    p.noise_bound = pr["noise_bound"] * s
    solver = tp.RobustRegistrationSolver(p)
    sol = solver.solve(pr["src"].T, (pr["dst"] * s).T)
    assert sol.valid and abs(sol.scale - s) < 0.02 * s
    assert synth.angular_error(np.asarray(sol.rotation), pr["R"]) < 0.02
