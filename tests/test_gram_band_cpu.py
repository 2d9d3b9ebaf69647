"""CPU check of the Gram-form pair test of the default graph kernel (DESIGN.md §3.1; constants as in prep_kernel,
graph_build.cu): the kernel's FP32 operation sequence is emulated in numpy, and every DECIDED pair must agree with the
exact FP64 predicate of the reference (registration.cc:427-443), both for the emulated Gram norms and for norms moved by
the full proven error bound.  The GPU counterpart is debug flag 2 (every decided pair re-checked on the device)."""
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
synth = importlib.import_module("teaser-plusplus_b200.synth")
band = importlib.import_module("gram_band_check")


@pytest.mark.parametrize("cfg,n", [("C2", 900), ("C2cube", 600), ("C3", 900), ("C5", 800)])
@pytest.mark.parametrize("mode", ["kernel", "pp", "pm", "mp", "mm"])
def test_gram_decided_pairs_agree_with_the_exact_predicate(cfg, n, mode):
    pr = synth.config_problem(cfg, 21, n=n)
    wrong, undecided, use_gram, err = band.check(pr["src"], pr["dst"], pr["noise_bound"], mode, cfg, verbose=False)
    assert use_gram  # every benchmark geometry but C1 passes the conditioning guard
    assert wrong == 0
    assert undecided < 1e-3  # the exact re-check is the exception
    if mode == "kernel":
        assert err <= 24.0  # the proven bound on |a' - a| (DESIGN.md §3.1), in units of u R^2


def test_gram_duplicates_and_large_noise_bounds_never_decide_wrongly():
    """Zero-length TIMs (s = a + b <= beta^2, where the sign of the polynomial says nothing) and noise bounds up to half
    the extent (beyond the conditioning guard): never a wrong decision, only more undecided pairs."""
    src, dst, nb = band.duplicates(n=500)
    for mode in ("kernel", "pp", "pm", "mp", "mm"):
        assert band.check(src, dst, nb, mode, "dups", verbose=False)[0] == 0
    pr = synth.config_problem("C2", 3, n=400)
    for nb in (0.05, 0.2, 0.5):
        for mode in ("kernel", "pm", "mp"):
            wrong, _, use_gram, _ = band.check(pr["src"], pr["dst"], nb, mode, "big", verbose=False)
            assert wrong == 0
    assert not use_gram  # beta = 1.0 on a unit ball: prep_kernel keeps this problem on the interval test


def test_gram_guard_rejects_far_outliers():
    """C1-like: outliers moved several extents away with a tiny noise bound make the band wide against beta, so the
    problem keeps the interval test."""
    pr = synth.config_problem("C2", 4, n=300)
    dst = pr["dst"].copy()
    dst[::7] += 8.0
    assert not band.consts(pr["src"], dst, 2 * 1e-3)["use_gram"]
    assert band.consts(pr["src"], pr["dst"], 2 * pr["noise_bound"])["use_gram"]


MODES = ("kernel", "pp", "pm", "mp", "mm")


def _no_wrong_decision(src, dst, nb, label):
    for mode in MODES:
        wrong, undecided, use_gram, err = band.check(src, dst, nb, mode, label, verbose=False)
        assert wrong == 0, (label, mode)
        # kernel: the proven bound on |a' - a|; bound modes: the norms were moved by at most e_a = 28 u R^2
        assert err <= (24.0 if mode == "kernel" else 28.0 + 1e-9), (label, mode, err)
    return undecided


@pytest.mark.parametrize("factor", [1.0, 1.02, 1.2, 2.0])
@pytest.mark.parametrize("rho", [0.3, 0.6, 1.0])
def test_gram_guard_edge_never_decides_wrongly(factor, rho):
    """beta a small multiple of beta*, the first beta the conditioning guard admits: the band is as wide against beta as
    the guard allows, and the pairs at distance rho sit on the threshold (about 2 % of all pairs are undecided)."""
    src, dst, nb = band.guard_edge(factor, rho)
    assert band.consts(src, dst, 2 * nb)["use_gram"]
    assert _no_wrong_decision(src, dst, nb, f"edge{factor}/{rho}") < 0.05


def test_gram_band_check_detects_a_band_5_percent_too_narrow():
    """The check can fail: at the guard edge, norms moved 5 % beyond the bound give wrong decisions (the first appear
    at about 1 % beyond it; DESIGN.md §3.1), so the zero above is a statement about the band, not about the fixture."""
    src, dst, nb = band.guard_edge(1.0, 0.6)
    assert sum(band.check(src, dst, nb, m, verbose=False, mult=1.0)[0] for m in MODES[1:]) == 0
    assert sum(band.check(src, dst, nb, m, verbose=False, mult=1.05)[0] for m in MODES[1:]) > 0


@pytest.mark.parametrize("rho", [0.3, 0.6, 1.0])
def test_gram_guard_routing_at_beta_star(rho):
    """beta* passes the guard, one ulp below it fails (the device makes the same choice: test_gpu_graph_boundary.py)."""
    src = band._cube(1200, 5)
    b = band.guard_beta(src, rho)
    below = np.nextafter(b, 0.0)
    assert band.consts(src, band._stretched(src, b, rho), b)["use_gram"]
    assert not band.consts(src, band._stretched(src, below, rho), below)["use_gram"]


@pytest.mark.parametrize("beyond", [False, True])
def test_gram_dmin_edge(beyond):
    """8 beta = D_min exactly passes the guard; one ulp of beta more fails it.  Either way no wrong decision."""
    src, dst, nb = band.dmin_edge(beyond)
    assert band.consts(src, dst, 2 * nb)["use_gram"] == (not beyond)
    _no_wrong_decision(src, dst, nb, f"dmin{int(beyond)}")


@pytest.mark.parametrize("offset,scale,edges", [(0.0, 1.0, 3630), (1024.0, 1.0, 3630), (0.0, 1.0 + 2.0 ** -50, 363),
                                                (0.0, 1.0 - 2.0 ** -50, 3630)])
def test_gram_lattice_exact_ties(offset, scale, edges):
    """11^3 lattice, dst = 2 src, beta = h: the 3630 lattice-neighbour pairs are exact FP64 ties, hence edges; a 2^-50
    stretch moves them a few ulp across the threshold (only 363 stay edges) or inside it.  The Gram test must leave every
    tie undecided."""
    src, dst, nb = band.lattice(offset, scale, permute_seed=1)
    assert band.edge_count(src, dst, nb) == edges
    assert band.consts(src, dst, 2 * nb)["use_gram"]
    assert _no_wrong_decision(src, dst, nb, "lattice") < 0.01
