"""The batched pose-graph routes' dense Cholesky on the device (run on an H100: `pytest -m gpu`), through
tzr_dense_cholesky_batch: exact systems (tests/dense_cholesky_reference.py) at every panel shape bit for bit, with the
strict upper triangle untouched; the failure column of every failure variant, with the finished panels and x_out
checked; mixed sizes in one call (panel stride n_max) against each matrix alone; rounded inputs against the
backward-error bounds; one launch per call and none for a refusal."""
import ctypes as C
import importlib

import numpy as np
import pytest

import dense_cholesky_reference as dc
import line_process_reference as lp
import pose_graph_reference as pg
from line_process_fragments import fragment
from test_gpu_line_process import R_CORR

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def cap_n():
    import torch
    return 6 * dc.batch_cap(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


def with_sentinels(A):
    """A's lower triangle with a distinct quiet NaN in every strict-upper entry (the device must not touch them)."""
    n = A.shape[0]
    M = np.tril(A)
    iu = np.triu_indices(n, 1)
    M[iu] = (np.uint64(0x7FF8000000000001) + np.arange(len(iu[0]), dtype=np.uint64)).view(np.float64)
    return M


def upper_bits(M):
    return np.ascontiguousarray(M)[np.triu_indices(M.shape[0], 1)].view(np.uint64)


def lower(M):
    return np.tril(M)


# ---- exact systems at every panel shape ------------------------------------------------------------------------------
def exact_batch(ns, seed):
    out = []
    for n in ns:
        rng = np.random.default_rng(seed + 7 * n)
        out.append(dc.exact_system(rng, n, density=0.5 if n < 64 else 0.2))
    return out


def check_exact(ctx, systems):
    As = [with_sentinels(A) for A, _, _, _ in systems]
    fac, xs, info = ctx.dense_cholesky_batch(As, [b for _, b, _, _ in systems])
    for (A, b, L, x), M, F, xh, i in zip(systems, As, fac, xs, info):
        n = len(b)
        assert i == 0, n
        assert lower(F).tobytes() == L.tobytes(), n
        assert xh.tobytes() == x.tobytes(), n
        assert upper_bits(F).tobytes() == upper_bits(M).tobytes(), n


def test_every_panel_shape_exact(ctx):
    ns = list(range(131)) + [191, 192, 193, 255, 256, 257, 383, 384, 385, 762, 768, cap_n()]
    systems = exact_batch(ns, 1)
    check_exact(ctx, systems)                        # panel stride: the cap
    check_exact(ctx, [s for s in systems if len(s[1]) <= 130])  # panel stride 130
    for s in systems[::13]:                           # alone: panel stride n
        check_exact(ctx, [s])


# ---- the failure column ------------------------------------------------------------------------------------------------
def failure_columns(n):
    last = ((n - 1) // dc.NB) * dc.NB
    return sorted({j for j in (0, 1, 30, 31, 32, 33, 63, 64, 65, last, n - 1) if j < n})


@pytest.mark.parametrize("which", ["33", "96", "190", "768", "cap"])
def test_failure_column(ctx, which):
    n = cap_n() if which == "cap" else int(which)
    A, b, L, x = dc.exact_system(np.random.default_rng(50 + n), n, density=0.2)
    cases, As, bs, xo = [], [], [], []
    for variant in dc.VARIANTS:
        for j in failure_columns(n):
            if variant == "nan_below" and j == 0:
                continue
            Af, want = dc.failure(A, L, variant, j)
            cases.append((variant, j, want))
            As.append(with_sentinels(Af))
            bs.append(b)
            xo.append(np.full(n, -3.5))
    # one matrix that succeeds in the same call
    As.append(with_sentinels(A))
    bs.append(b)
    xo.append(np.full(n, -3.5))
    fac, xs, info = ctx.dense_cholesky_batch(As, bs, x_out=xo)
    for (variant, j, want), M, F, xh, i in zip(cases, As, fac, xs, info):
        assert i == want, (variant, j)
        c = (j // dc.NB) * dc.NB
        fin = dc.finished_columns(L, variant, j)
        got = lower(F)[:, :c]
        assert np.array_equal(got, fin, equal_nan=True), (variant, j)
        if variant in ("zero", "negative"):
            assert got.tobytes() == fin.tobytes(), (variant, j)
        assert xh.tobytes() == np.full(n, -3.5).tobytes(), (variant, j)  # untouched
        assert upper_bits(F).tobytes() == upper_bits(M).tobytes(), (variant, j)
    assert info[-1] == 0 and lower(fac[-1]).tobytes() == L.tobytes() and xs[-1].tobytes() == x.tobytes()


# ---- mixed sizes in one call -------------------------------------------------------------------------------------------
def rounded(n, seed):
    rng = np.random.default_rng(seed)
    A = dc.spd(rng, n, 10.0 ** rng.uniform(0, 8))
    return with_sentinels(A), rng.standard_normal(n)


def same(a, b):
    (Fa, xa), (Fb, xb) = a, b
    return Fa.tobytes() == Fb.tobytes() and xa.tobytes() == xb.tobytes()


def test_mixed_strides(ctx):
    ns = [6, 31, 32, 33, 64, 190, 768]
    mats = [rounded(n, 300 + n) for n in ns]
    alone = []
    for A, b in mats:
        F, x, info = ctx.dense_cholesky_batch([A], [b])
        assert info[0] == 0
        alone.append((F[0], x[0]))
    rng = np.random.default_rng(4)
    for order in (list(range(len(ns))), list(range(len(ns)))[::-1], list(rng.permutation(len(ns))),
                  [5, 0, 6, 1, 4, 2, 3]):
        F, x, info = ctx.dense_cholesky_batch([mats[k][0] for k in order], [mats[k][1] for k in order])
        assert not info.any()
        for j, k in enumerate(order):
            assert same((F[j], x[j]), alone[k]), (order, ns[k])
    for (A, b), (F, x) in zip(mats, alone):
        assert dc.factor_violation(np.tril(A) + np.tril(A, -1).T, lower(F)) <= 1.0


def test_256_mixed_sizes(ctx):
    rng = np.random.default_rng(6)
    ns = [int(n) for n in rng.choice([1, 5, 6, 31, 32, 33, 63, 64, 65, 96, 127, 128, 190, 200, 384, 600], size=256)]
    systems = exact_batch(ns, 77)
    sys_ = [(with_sentinels(A), b) for A, b, _, _ in systems]
    F, x, info = ctx.dense_cholesky_batch([A for A, _ in sys_], [b for _, b in sys_])
    assert not info.any()
    rev = ctx.dense_cholesky_batch([A for A, _ in sys_[::-1]], [b for _, b in sys_[::-1]])
    for j, ((A, b, L, xx), (M, _)) in enumerate(zip(systems, sys_)):
        assert lower(F[j]).tobytes() == L.tobytes() and x[j].tobytes() == xx.tobytes(), ns[j]
        assert upper_bits(F[j]).tobytes() == upper_bits(M).tobytes()
        assert same((F[j], x[j]), (rev[0][255 - j], rev[1][255 - j]))
    for j in range(0, 256, 17):
        one = ctx.dense_cholesky_batch([sys_[j][0]], [sys_[j][1]])
        assert same((F[j], x[j]), (one[0][0], one[1][0]))


# ---- rounded inputs ----------------------------------------------------------------------------------------------------
def check_bounds(A, b, F, xh, forward=True):
    Lh = lower(F)
    assert dc.factor_violation(A, Lh) <= 1.0
    assert dc.solve_violation(A, b, Lh, xh) <= 1.0
    if forward:
        fb = dc.forward_bound(A, Lh)
        assert fb is not None
        assert dc.forward_error(xh, dc.longdouble_solve(A, b)) <= fb


@pytest.mark.parametrize("n,kappa", [(33, 1.0), (64, 1e12), (96, 1e12), (190, 1e3), (257, 1e6), (190, 1e9),
                                     (768, 1e6)])
def test_random_spd_within_the_bounds(ctx, n, kappa):
    rng = np.random.default_rng(n + int(np.log10(kappa)))
    A = dc.spd(rng, n, kappa)
    b = rng.standard_normal(n)
    F, x, info = ctx.dense_cholesky_batch([with_sentinels(A)], [b])
    assert info[0] == 0
    check_bounds(A, b, F[0], x[0])


@pytest.mark.parametrize("n,rank", [(64, 40), (190, 150), (768, 700)])
def test_nearly_singular_within_the_bounds(ctx, n, rank):
    rng = np.random.default_rng(n + rank)
    A = dc.nearly_singular(rng, n, rank)
    b = rng.standard_normal(n)
    F, x, info = ctx.dense_cholesky_batch([A], [b])
    assert info[0] == 0
    check_bounds(A, b, F[0], x[0], forward=n <= 190)


def first_damped_system(K, seed):
    """H + 1e-5 max diag(H) I and b of the line process's first trial on a fragment of K nodes, assembled by the numpy
    restatement (gauge-singular H, damped as the device damps it)."""
    gt, edges, T, L, unc = fragment(seed, K, n_wrong=2)
    edges = np.asarray(edges)
    E = len(edges)
    live = [True] * E
    start = pg.bfs(K, edges, T, live, np.asarray(unc).astype(bool), 0)
    mu = lp._mu(L, range(E), R_CORR, 1.0)
    terms = lp._terms(start, edges, T, L)
    conf = [lp.confidence(mu, terms[e][2]) if unc[e] else 1.0 for e in range(E)]
    H, b = lp.linear_system(K, edges, live, conf, terms)
    return H + 1e-5 * float(np.max(np.diag(H))) * np.eye(6 * K), b


@pytest.mark.parametrize("K", [100, 128])
def test_line_process_systems_within_the_bounds(ctx, K):
    A, b = first_damped_system(K, 400 + K)
    F, x, info = ctx.dense_cholesky_batch([with_sentinels(A)], [b])
    assert info[0] == 0
    check_bounds(A, b, F[0], x[0], forward=False)


# ---- launches ------------------------------------------------------------------------------------------------------------
def test_one_launch_per_call(ctx):
    for G in (1, 256):
        systems = exact_batch([(7 * g) % 97 for g in range(G)], 9)
        l0 = ctx.kernel_launches()
        _, _, info = ctx.dense_cholesky_batch([s[0] for s in systems], [s[1] for s in systems])
        assert ctx.kernel_launches() - l0 == 1 and not info.any()


def raw_call(ctx, ns, drop=None, drop_entry=False):
    """tzr_dense_cholesky_batch with identity matrices of sizes ns (a negative size gets a 1 x 1 buffer); drop names one
    array argument passed as NULL, drop_entry makes the last matrix's A entry NULL.  Returns (rc, info, A_out, x_out)."""
    dp = C.POINTER(C.c_double)
    G = len(ns)
    m = [max(n, 1) for n in ns]
    A = [np.eye(k) for k in m]
    b = [np.ones(k) for k in m]
    Ao = [np.full((k, k), 5.0) for k in m]
    xo = [np.full(k, 5.0) for k in m]
    info = np.full(max(G, 1), 9, dtype=np.int32)
    nn = np.array(ns if G else [0], dtype=np.int32)

    def ptrs(arrs, name):
        if drop == name:
            return None
        p = (dp * max(G, 1))(*[a.ctypes.data_as(dp) for a in arrs])
        if drop_entry and name == "A":
            p[G - 1] = dp()
        return p
    args = [ctx._h, G, None if drop == "n" else nn.ctypes.data_as(C.POINTER(C.c_int32)), ptrs(A, "A"), ptrs(b, "b"),
            ptrs(Ao, "A_out"), ptrs(xo, "x_out"), None if drop == "info" else info.ctypes.data_as(C.POINTER(C.c_int32))]
    rc = capi.lib().tzr_dense_cholesky_batch(*args)
    return rc, info, Ao, xo


def test_refusals_launch_nothing_and_write_nothing(ctx):
    big = cap_n() + 1
    cases = [([], None, False, capi.TZR_ERR_INVALID_ARG), ([4, -1], None, False, capi.TZR_ERR_INVALID_ARG),
             ([4, 3], None, True, capi.TZR_ERR_INVALID_ARG), ([4, big], None, False, capi.TZR_ERR_TOO_LARGE)]
    cases += [([4, 3], d, False, capi.TZR_ERR_INVALID_ARG) for d in ("n", "A", "b", "A_out", "x_out", "info")]
    for ns, drop, entry, want in cases:
        l0 = ctx.kernel_launches()
        rc, info, Ao, xo = raw_call(ctx, ns, drop, entry)
        assert rc == want, (ns, drop, entry)
        assert ctx.kernel_launches() == l0, (ns, drop, entry)
        assert (info == 9).all() and all((a == 5.0).all() for a in Ao) and all((v == 5.0).all() for v in xo)
    # the largest size is accepted, and the same call with every argument given succeeds
    assert raw_call(ctx, [4, big - 1])[0] == capi.TZR_OK
    rc, info, Ao, xo = raw_call(ctx, [4, 3])
    assert rc == capi.TZR_OK and not info.any() and np.array_equal(xo[0], np.ones(4))
