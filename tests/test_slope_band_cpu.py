"""CPU check of the single-slope Gram test's band (scripts/slope_band_check.py, DESIGN.md §3.1): the kernel's FP32
sequence and the full proven error bound (modes pp/pm/mp/mm) give no wrong decision on any fixture, the benchmark
geometries leave fewer than 1e-3 of the pairs undecided, a perturbation a few percent beyond the bound does give wrong
decisions where the band is tight, so the check can fail, and each constant meets its derived inequality with less than
2 % to spare."""
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
slope = importlib.import_module("slope_band_check")
gbc = importlib.import_module("gram_band_check")

FIXTURES = slope.fixtures(small=True)
MODES = ("kernel", "pp", "pm", "mp", "mm")


@pytest.mark.parametrize("label", [f[0] for f in FIXTURES])
def test_no_wrong_decision(label):
    _, src, dst, nb = next(f for f in FIXTURES if f[0] == label)
    for mode in MODES:
        wrong, und, _, err = slope.check(src, dst, nb, mode, label, verbose=False)
        assert wrong == 0, (label, mode)
        if mode == "kernel":
            assert err <= 28.0, (label, err)  # the errors that occur stay inside the bound prep_kernel uses
        if label in slope.BENCH:
            assert und < 1e-3, (label, mode, und)


def test_benchmark_geometries_take_the_gram_test():
    for label, src, dst, nb in FIXTURES:
        if label in slope.BENCH:
            assert slope.consts(src, dst, 2 * nb)["use_gram"], label


def test_lattice_ties_are_undecided():
    """Every exact FP64 tie must land in the band: the kernel alone could not settle it."""
    src, dst, nb = gbc.lattice(permute_seed=1)
    c = slope.consts(src, dst, 2 * nb)
    assert c["cv"] - c["cu"] == 0.25
    _, und, _, _ = slope.check(src, dst, nb, "kernel", verbose=False)
    assert und * len(src) * (len(src) - 1) / 2 >= 3630


def test_beyond_the_bound_gives_wrong_decisions():
    """Where the band is tight (corner_ties: ties across the box diagonal, |T| near sqrt(A_s), at the guard edge), the
    full bound gives no wrong decision, norms moved by 1.05 times the bound do, and so does an edge-side constant c_u
    5 % below its derived value: the check can fail, and it would see a moderately wrong derivation."""
    src, dst, nb = slope.corner_ties(1.0)
    assert sum(slope.check(src, dst, nb, m, verbose=False)[0] for m in MODES) == 0
    assert sum(slope.check(src, dst, nb, m, verbose=False, mult=1.05)[0] for m in MODES[1:]) > 0
    assert sum(slope.check(src, dst, nb, m, verbose=False, cu_scale=0.95)[0] for m in MODES[1:]) > 0


@pytest.mark.parametrize("label", ["C2", "C5", "g1.0/0.6", "dmin0", "lat0/+0e+00", "corner1.0"])
def test_constants_meet_their_inequalities_tightly(label):
    """Each constant against the inequality it is derived from (DESIGN.md §3.1), as the kernel receives it (rounded to
    float): c_u covers the edge side, K = |dl|(1 - u) - c_u - E_u the non-edge side, and each is within 2 % of its bound,
    so a constant that is off by more than that fails here even where no fixture has pairs at the tight spot."""
    _, src, dst, nb = next(f for f in FIXTURES if f[0] == label)
    c = slope.consts(src, dst, 2 * nb)
    u, As, Eu = slope.u, c["As"], c["Eu"]
    E1 = Eu + c["Ev"]
    assert c["cv"] - c["cu"] == 0.25

    def edge_rhs(cu):
        return Eu + 5.0 * u * (As + Eu) + 2.0 * (1.0 + 2.0 * u) * E1 * np.sqrt(As + Eu) + E1 * E1

    def non_edge_lhs(K):
        return K * (1.0 - 2.0 * u) - 2.0 * u * As - 2.0 * E1 * np.sqrt(As + K)

    assert c["cu"] >= edge_rhs(c["cu"]) > 0.98 * c["cu"]
    K = -c["dl"] * (1.0 - u) - c["cu"] - Eu
    assert non_edge_lhs(K) > 0.0625 >= non_edge_lhs(0.98 * K)
