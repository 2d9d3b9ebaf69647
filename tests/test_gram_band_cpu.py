"""CPU check of the Gram-form pair test of the default graph kernel (DESIGN.md §3.1; constants as in prep_kernel,
graph_build.cu): the kernel's FP32 operation sequence is emulated in numpy, and every DECIDED pair must agree with the
exact FP64 predicate of the reference (registration.cc:427-443), both for the emulated Gram norms and for norms moved by
the full proven error bound.  The GPU counterpart is debug flag 2 (every decided pair re-checked on the device)."""
import importlib
import os
import sys

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
