"""tests/rotation_reference.py against exact arithmetic and against the CPU oracle (no GPU needed).

The replica's svd_rot / yaw_rot must reach the exact Procrustes maximiser (Horn's quaternion matrix at 60 digits) on
every H family the device is tested with, including the ones where the maximiser is not unique; its GNC-TLS, FGR and
Quatro loops must agree with the oracle's up to summation order.  The power-of-two normalisation of H makes the
rotation exactly scale-invariant: R(H 2^k) == R(H) bit for bit wherever H 2^k is exact, and the unscaled algorithm
(normalise=False) is shown to fail there, so these cases test the normalisation and nothing else.
"""
import math

import numpy as np
import pytest

import oracle_lib as orc
import rotation_reference as ref

H3 = ref.h_families()
H2 = ref.h2_families()
SWEEP_EXACT = (-1000, -960, -600, 600, 1000, 1015)
SWEEP_ROUNDED = (-1060, -1070)


@pytest.mark.parametrize("name", list(H3))
def test_svd_rot_reaches_exact_maximiser(name):
    H = H3[name]
    R = ref.svd_rot(H)
    ok, detail = ref.within_exact(R, H)
    assert ok, (name, detail)
    assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-14 and abs(np.linalg.det(R) - 1.0) <= 1e-14


def test_svd_rot_zero_is_identity():
    assert np.array_equal(ref.svd_rot(np.zeros((3, 3))), np.eye(3))
    assert np.array_equal(ref.yaw_rot(np.zeros((3, 3))), np.eye(3))


@pytest.mark.parametrize("name", list(H2))
def test_yaw_rot_reaches_exact_maximiser(name):
    H = H2[name]
    R = ref.yaw_rot(H)
    ok, detail = ref.within_exact(R, H, planar=True)
    assert ok, (name, detail)
    assert np.array_equal(R[2], [0.0, 0.0, 1.0]) and np.array_equal(R[:, 2], [0.0, 0.0, 1.0])


def test_yaw_rot_extremes_need_the_normalisation():
    """Without it the squares of the closed form underflow (1e-160: inexact, 1e-170: identity) or overflow (1e160)."""
    for name in ("yaw_1e-160", "yaw_1e-170", "yaw_1e+160"):
        H = H2[name]
        assert not np.array_equal(ref.yaw_rot(H, normalise=False), ref.yaw_rot(H2["yaw_plain"])), name
        assert np.array_equal(ref.yaw_rot(H), ref.yaw_rot(H2["yaw_plain"])), name


def test_scale_sweep_is_bitwise_invariant():
    H = ref.scale_sweep_h()
    R0, Y0 = ref.svd_rot(H), ref.yaw_rot(H)
    for k in SWEEP_EXACT:
        Hk = np.ldexp(H, k)
        assert np.array_equal(np.ldexp(Hk, -k), H), k  # H 2^k is exact
        assert np.array_equal(ref.svd_rot(Hk), R0), k
        assert np.array_equal(ref.yaw_rot(Hk), Y0), k
    # the unscaled algorithm loses the rotation in the subnormal range (the Jacobi threshold stops every rotation)
    # and every extreme yaw (the squares leave the double range)
    assert not np.array_equal(ref.svd_rot(np.ldexp(H, -1000), normalise=False), R0)
    for k in SWEEP_EXACT:
        assert not np.array_equal(ref.yaw_rot(np.ldexp(H, k), normalise=False), Y0), k


@pytest.mark.parametrize("k", SWEEP_ROUNDED)
def test_scale_sweep_subnormal_rounding_within_exact(k):
    """H 2^k rounds into the subnormal range: another matrix, held to the exact reference of that matrix."""
    Hk = np.ldexp(ref.scale_sweep_h(), k)
    ok, detail = ref.within_exact(ref.svd_rot(Hk), Hk)
    assert ok, detail
    ok, detail = ref.within_exact(ref.yaw_rot(Hk), Hk, planar=True)
    assert ok, detail


def test_block_sum_replays_the_thread_order():
    """Thread 0 adds 1 + 2^-53 (-> 1), thread 1 holds 2^-53, the butterfly adds 1 + 2^-53 (-> 1): the device's order
    gives 1 where the exact sum is 1 + 2^-52."""
    v = np.zeros(256)
    v[0], v[128], v[1] = 1.0, 2.0 ** -53, 2.0 ** -53
    t = ref.plain_tims(np.zeros((256, 3)), np.zeros((256, 3)))
    assert t.block_sum(v) == 1.0 and math.fsum(v) == 1.0 + 2.0 ** -52
    assert np.array_equal(t.block_sum(np.stack([v, 2 * v], 1)), [1.0, 2.0])


# ------------------------------------------------------------------------------------------------ loops vs oracle
def _mask_ok(mask, omask, w, thr):
    diff = mask != omask
    return not diff.any() or bool(np.all(np.abs(w[diff] - thr) <= 1e-9))


LOOP_M = (3, 33, 129, 257, 1000)


@pytest.mark.parametrize("outliers", [0.0, 0.3, 0.8])
@pytest.mark.parametrize("m", LOOP_M)
def test_gnc_tls_matches_oracle(m, outliers):
    x, y, _ = ref.tim_problem(m, outliers, 1000 + m)
    t = ref.plain_tims(x, y)
    nb = 0.01
    g = ref.gnc_tls(t, nb, 1.4, 100, 1e-6)
    o = orc.gnc_tls(x, y, 100, 1e-6, 1.4, nb)
    assert np.abs(g["R"] - o["R"]).max() <= 1e-9
    assert abs(g["iterations"] - o["iterations"]) <= 1
    assert _mask_ok(g["inliers"], o["inliers"], g["weights"], 0.5)


@pytest.mark.parametrize("outliers", [0.0, 0.3, 0.8])
@pytest.mark.parametrize("m", LOOP_M)
def test_quatro_matches_oracle(m, outliers):
    x, y, _ = ref.tim_problem(m, outliers, 2000 + m, planar=True)
    t = ref.plain_tims(x, y)
    nb = 0.01
    g = ref.quatro(t, nb, 1.4, 100, 1e-6)
    o = orc.quatro(x, y, 100, 1e-6, 1.4, nb)
    assert np.abs(g["R"] - o["R"]).max() <= 1e-9
    assert abs(g["iterations"] - o["iterations"]) <= 1
    assert _mask_ok(g["inliers"], o["inliers"], g["weights"], 0.4)


@pytest.mark.parametrize("outliers", [0.0, 0.3, 0.8])
@pytest.mark.parametrize("m", LOOP_M)
def test_fgr_matches_oracle(m, outliers):
    x, y, _ = ref.tim_problem(m, outliers, 3000 + m)
    t = ref.plain_tims(x, y)
    nb = 0.05
    g = ref.fgr(t, nb, 1.4, 100, 0.005)
    o = orc.fgr(x, y, 100, 0.005, 1.4, nb)
    assert np.abs(g["R"] - o["R"]).max() <= 1e-9
    assert abs(g["iterations"] - o["iterations"]) <= 1
    assert _mask_ok(g["inliers"], o["inliers"], g["weights"], 0.0)


def test_gnc_edges_match_oracle():
    x, y, _ = ref.tim_problem(50, 0.0, 7, noise=0.0)
    t = ref.plain_tims(x, y)
    g = ref.gnc_tls(t, 0.01)  # noise-free: mu <= 0 at iteration 0
    o = orc.gnc_tls(x, y, 100, 1e-6, 1.4, 0.01)
    assert g["iterations"] == o["iterations"] == 1 and g["cost"] == o["cost"] == np.inf
    assert g["inliers"].all() and o["inliers"].all()
    g = ref.gnc_tls(t, 0.01, max_iterations=0)
    o = orc.gnc_tls(x, y, 0, 1e-6, 1.4, 0.01)
    assert g["iterations"] == o["iterations"] == 0 and np.array_equal(g["R"], np.eye(3)) and g["cost"] == np.inf
    assert g["inliers"].all() and o["inliers"].all()


def test_scale_extremes_match_oracle():
    """The oracle applies the same normalisation: equal rotations at H scaled to 2^-1000 and 2^1000."""
    x, y, _ = ref.tim_problem(40, 0.0, 11)
    for k in (-500, 500):
        xs, ys = np.ldexp(x, k), np.ldexp(y, k)  # H ~ 2^(2k)
        o = orc.gnc_tls(xs, ys, 1, 1e-6, 1.4, 1.0)
        g = ref.gnc_tls(ref.plain_tims(xs, ys), 1.0, max_iterations=1)
        assert np.abs(g["R"] - o["R"]).max() <= 1e-12, k
        assert np.abs(g["R"] - ref.gnc_tls(ref.plain_tims(x, y), 1.0, max_iterations=1)["R"]).max() <= 1e-12, k
