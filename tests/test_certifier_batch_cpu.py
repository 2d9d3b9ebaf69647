"""CPU checks of the certifier batch (tzr_certify_batch, DESIGN.md 3.9).

The batch pads every problem's symmetric matrix to the batch's largest size with c * I (c > 0) in the pad block, c the
largest power of two not above the largest |entry| of the problem's starting matrix (pad_value below), and
decomposes the padded matrices together.  These tests check, with numpy and oracle/certifier_oracle.py, that the two
quantities the certifier takes from a decomposition do not change under that padding: the positive-part projection
V+ L+ V+^T restricted to the real block, and the sub-optimality gap of certification.cc:192-231.  They also check the
Python argument validation that needs no device, and that the entry point is exported, declared and bound."""
import importlib
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import certifier_oracle as co  # noqa: E402
import certifier_fixtures as cf  # noqa: E402

capi = importlib.import_module("teaser-plusplus_b200.capi")
HEADER = os.path.join(ROOT, "include", "teaser_b200.h")
def pad_value(A):
    """cert_pad in csrc/certify.cu: the largest power of two not above max |A|, 1 for a zero matrix."""
    m = np.abs(A).max()
    return float(np.ldexp(1.0, np.frexp(m)[1] - 1)) if m > 0 else 1.0


def _pad(A, nmax, c=None):
    c = pad_value(A) if c is None else c
    n = A.shape[0]
    P = np.zeros((nmax, nmax))
    P[:n, :n] = A
    P[np.arange(n, nmax), np.arange(n, nmax)] = c
    return P


def _psd_part(A):
    """V+ diag(w+) V+^T over the positive eigenpairs, as the device computes it (linalg.h:84-99 on a symmetric A)."""
    w, V = np.linalg.eigh(A)
    pos = w > 0
    return (V[:, pos] * w[pos]) @ V[:, pos].T


def _gap(A, mu, N):
    """The gap rule of certification.cc:192-231 on the smallest eigenvalue of a symmetric A."""
    mn = np.linalg.eigvalsh(A)[0]
    return 0.0 if mn > 0 else (-mn * (N + 1)) / mu


def _random_sym(rng, n, spectrum):
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    return (Q * spectrum) @ Q.T


def _fixture_matrices():
    out = []
    for c in cf.cases("small"):
        N = c["v1"].shape[1]
        r = co.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"], c["params"]["noise_bound"],
                       c["params"]["cbar2"], max_iterations=1, return_intermediates=True)
        for M in (c["W_1st_iter"], r["M_init"], r["M_affine"]):
            out.append((c["name"], (M + M.T) / 2, r["mu"], N))
    return out


FIXTURES = _fixture_matrices()


@pytest.mark.parametrize("k", range(len(FIXTURES)), ids=[f"{f[0]}-{i % 3}" for i, f in enumerate(FIXTURES)])
@pytest.mark.parametrize("extra", [4, 40, 200])
def test_padded_projection_and_gap_on_fixture_matrices(k, extra):
    _, A, mu, N = FIXTURES[k]
    n = A.shape[0]
    P = _pad(A, n + extra)
    want = _psd_part(A)
    got = _psd_part(P)
    scale = max(1.0, np.abs(want).max())
    assert np.abs(got[:n, :n] - want).max() < 1e-12 * scale
    assert np.abs(got[n:, :n]).max() < 1e-12 * scale  # the pad eigenvectors add nothing outside the pad block
    g0, g1 = _gap(A, mu, N), _gap(P, mu, N)
    assert abs(g0 - g1) <= 1e-12 * max(1.0, abs(g0))


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("kind", ["mixed", "all_positive", "c_in_middle", "c_below_all", "c_above_all", "zero_min"])
def test_padded_projection_and_gap_on_random_spectra(seed, kind):
    rng = np.random.default_rng(seed)
    n = 4 * int(rng.integers(1, 30)) + 4
    if kind == "mixed":
        spec = rng.uniform(-3, 3, n)
    elif kind == "all_positive":
        spec = rng.uniform(0.1, 5, n)
    elif kind == "c_in_middle":         # eigenvalues on both sides of c, negative ones too
        spec = np.concatenate([rng.uniform(-2, -0.1, n // 3), rng.uniform(0.2, 0.9, n // 3),
                               rng.uniform(1.1, 4, n - 2 * (n // 3))])
    elif kind == "c_below_all":
        spec = rng.uniform(1.5, 6, n)
    elif kind == "c_above_all":
        spec = rng.uniform(-0.5, 0.5, n)
    else:                               # smallest eigenvalue exactly representable as 0 is the "> 0 fails" case
        spec = np.concatenate([[0.0], rng.uniform(0.5, 2, n - 1)])
    A = _random_sym(rng, n, spec)
    A = (A + A.T) / 2
    mu, N = float(rng.uniform(0.1, 10)), (n - 4) // 4
    for extra in (4, 64):
        P = _pad(A, n + extra)
        want = _psd_part(A)
        assert np.abs(_psd_part(P)[:n, :n] - want).max() < 1e-12 * max(1.0, np.abs(want).max())
        g0, g1 = _gap(A, mu, N), _gap(P, mu, N)
        if kind in ("all_positive", "c_below_all"):
            assert g0 == 0.0 and g1 == 0.0
        assert abs(g0 - g1) <= 1e-12 * max(1.0, abs(g0))


def test_pad_value_positive_keeps_nonpositive_minimum():
    """The smallest eigenvalue is unchanged whenever it is <= 0, for any c > 0; when it is > 0 the gap is 0 either
    way."""
    rng = np.random.default_rng(7)
    for c in (1e-6, 0.5, 1.0, 30.0, None):
        A = _random_sym(rng, 24, rng.uniform(-1, 2, 24))
        A = (A + A.T) / 2
        w0 = np.linalg.eigvalsh(A)[0]
        w1 = np.linalg.eigvalsh(_pad(A, 40, c))[0]
        if w0 <= 0:
            assert abs(w0 - w1) < 1e-12
        assert _gap(A, 2.0, 5) == pytest.approx(_gap(_pad(A, 40, c), 2.0, 5), abs=1e-12)


# ---- argument validation of Context.certify_batch (no device) -------------------------------------------------------
def _problem(N, seed=0):
    rng = np.random.default_rng(seed)
    return np.eye(3), rng.uniform(-1, 1, (3, N)), rng.uniform(-1, 1, (3, N)), np.ones(N)


def test_batch_inputs_accept_ragged_problems_and_bool_theta():
    a, b = _problem(3), _problem(7, 1)
    probs = capi.Context._cert_batch_inputs([a[0], b[0]], [a[1], b[1]], [a[2], b[2]], [a[3] > 0, b[3]])
    assert [p[3].size for p in probs] == [3, 7]
    assert probs[0][3].dtype == np.float64 and np.all(probs[0][3] == 1.0)
    assert probs[1][1].shape == (7, 3) and probs[1][1].flags.c_contiguous


@pytest.mark.parametrize("case", ["empty", "lengths", "rotation", "src_shape", "dst_width", "theta_len", "no_meas"])
def test_batch_inputs_reject(case):
    R, s, d, t = _problem(4)
    Rs, ss, ds, ts = [R, R], [s, s], [d, d], [t, t]
    if case == "empty":
        Rs, ss, ds, ts = [], [], [], []
    elif case == "lengths":
        ts = [t]
    elif case == "rotation":
        Rs = [R, np.eye(4)]
    elif case == "src_shape":
        ss = [s, s.T]
    elif case == "dst_width":
        ds = [d, d[:, :3]]
    elif case == "theta_len":
        ts = [t, t[:3]]
    else:
        ss, ds, ts = [s, s[:, :0]], [d, d[:, :0]], [t, t[:0]]
    with pytest.raises(capi.TzrError):
        capi.Context._cert_batch_inputs(Rs, ss, ds, ts)


def test_entry_point_exported_declared_bound_and_flag_documented():
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    raw = open(HEADER).read()
    hdr = re.sub(r"/\*.*?\*/", "", raw, flags=re.S)
    m = re.search(r"int\s+tzr_certify_batch\s*\(([^)]*)\)", hdr)
    assert m, "tzr_certify_batch missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == ["ctx", "params", "B", "N", "R_colmajor9xB", "src_3xN", "dst_3xN", "theta", "results", "traj",
                    "traj_capacity"]
    assert "tzr_certify_batch" in capi._SYMBOLS
    assert len(capi.lib().tzr_certify_batch.argtypes) == len(args)
    assert "bit 21 (2097152)" in raw


@pytest.mark.parametrize("k", [-1074, -1060, -40, -1, 0, 1, 40, 1000])
def test_pad_value_follows_the_scale_exactly(k):
    """The pad is a power of two in (max|A| / 2, max|A|], so scaling A by 2^k scales it by 2^k: the padded matrix
    scales exactly and its norm is the real block's."""
    A = np.array([[0.75, -3.0], [-3.0, 1.5]])
    c = pad_value(np.ldexp(A, k))
    assert c == np.ldexp(pad_value(A), k) == np.ldexp(2.0, k)
    assert c <= np.abs(np.ldexp(A, k)).max() < 2 * c
    assert pad_value(np.zeros((4, 4))) == 1.0
