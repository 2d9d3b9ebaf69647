"""CPU check of the Gram-form pair test of graph_strip2_kernel (DESIGN.md §3.1; constants as in prep_kernel,
graph_build.cu).  The kernel's FP32 operations are emulated in numpy in their order:

    N = fl(|q|^2) of the centred float copy q,  a = fma(z_j, -2 z_i, fma(y_j, -2 y_i, fma(x_j, -2 x_i, N_i + N_j))),
    t = a - b, s = a + b,  d_hi = fma(t, t, fma(s, mhi, chi)),  d_lo = fma(t, t, fma(s, mlo, clo))

(an FMA is emulated as one FP64 operation rounded to FP32: the product of two floats is exact in FP64, so only the
rare double rounding of the sum can differ from the hardware, by one ulp).  sign(d_hi) = 1 decides an edge,
sign(d_lo) = 0 a non-edge; every decided pair must agree with the reference's FP64 predicate.  Mode "kernel" is the
emulation itself; modes "pp", "pm", "mp", "mm" replace the Gram norms by the exact squared norms moved by the full proven
error bound (+-ea, +-eb), so the band is checked against the bound and not only against the errors that happen to occur.
The moved norm is a float; where rounding f32(a +- ea) would carry it beyond the bound it is stepped one float back
toward a, so the check never perturbs by more than the bound (times `mult`, which a test sets above 1 to show that the
check can fail).

Fixtures beyond the benchmark geometries, where a wrong band would show:
  guard_edge   unit-cube source, dst = (1 + beta/rho) src + offset: pairs at distance rho sit on the threshold, and beta is
               a multiple of beta*, the smallest beta that passes the conditioning guard (64 E <= 0.75 D_min beta)
  dmin_edge    beta = D_min / 8 exactly (guard passes) or one ulp above (guard fails)
  lattice      11^3 integer lattice scaled by h = 2^-4, dst = 2 src, beta = h: every pair of lattice neighbours is an
               exact FP64 tie (|d1 - d2| = h = beta), so an edge
usage: python scripts/gram_band_check.py"""
import importlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
synth = importlib.import_module("teaser-plusplus_b200.synth")
u = 2.0 ** -24
UP, DN = 1.0 + 2.0 ** -20, 1.0 - 2.0 ** -20


def f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def fma(a, b, c):
    return f32(a * b + c)


def consts(src, dst, beta):
    """prep_kernel's centres, float copies, norms and Gram-test constants (fixed scale)."""
    mn_s, mx_s, mn_d, mx_d = src.min(0), src.max(0), dst.min(0), dst.max(0)
    cs, cd = 0.5 * (mn_s + mx_s), 0.5 * (mn_d + mx_d)
    Ds2, Dd2 = float(((mx_s - mn_s) ** 2).sum()), float(((mx_d - mn_d) ** 2).sum())
    b2 = beta * beta
    b4 = b2 * b2
    lam = 0.75 * beta * np.sqrt(0.5 * (Ds2 + Dd2))
    Dmin = np.sqrt(min(Ds2, Dd2))
    E = 7.0 * u * (Ds2 + Dd2)
    k, S = E / lam, Ds2 + Dd2 + E
    C = E * lam + E * E + 2.0 * b2 * E
    c = dict(mhi=f32(-2.0 * b2 * (1.0 - 4.0 * u) / (1.0 + k) * DN),
             chi=f32(((b4 + C) / (1.0 + k) + 8.0 * u * b2 * S) * UP),
             mlo=f32(-2.0 * b2 * (1.0 + 4.0 * u) / (1.0 - k) * UP),
             clo=f32(-(C + 9.0 * u * b2 * S) / (1.0 - k) * UP * UP))
    c["use_gram"] = bool(Ds2 > 0 and Dd2 > 0 and Ds2 < 1e8 and Dd2 < 1e8 and b4 > 1e-30 and 8.0 * beta <= Dmin and
                         64.0 * E <= 0.75 * Dmin * beta)
    c["ea"], c["eb"] = 7.0 * u * Ds2, 7.0 * u * Dd2  # 28 u R^2 with R^2 = D^2 / 4
    qs, qd = f32(src - cs), f32(dst - cd)
    c["qs"], c["qd"] = qs, qd
    c["Ns"], c["Nd"] = f32((qs * qs).sum(1)), f32((qd * qd).sum(1))
    return c


def gram(q, N, i, j):
    a = f32(N[i] + N[j])
    for k in range(3):
        a = fma(q[j, k], -2.0 * q[i, k], a)
    return a


def tim_norm(p, i, j):  # the reference's FP64 sequence: (dx^2 + dy^2) + dz^2
    d = p[j] - p[i]
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def moved(x, e, sign):
    """The float nearest to x + sign * e that lies within e of x (x, e >= 0 FP64 arrays / scalars)."""
    y = f32(x + sign * e)
    over = np.abs(y - x) > e
    if np.any(over):  # f32 rounded beyond the bound: one float back toward x
        back = np.nextafter(y.astype(np.float32), np.float32(-np.inf if sign > 0 else np.inf)).astype(np.float64)
        y = np.where(over, back, y)
    assert np.all(np.abs(y - x) <= e), "perturbed norm beyond the bound"
    return y


def check(src, dst, noise_bound, mode="kernel", label="", verbose=True, mult=1.0):
    """Returns (wrong decisions, undecided fraction, use_gram, largest |a' - a| / (u R^2)).  In the bound modes the norms
    are moved by mult * (ea, eb)."""
    beta = 2.0 * noise_bound
    c = consts(src, dst, beta)
    i, j = np.triu_indices(len(src), 1)
    d1, d2 = tim_norm(src, i, j), tim_norm(dst, i, j)
    exact = np.abs(d1 - d2) <= beta
    a_true = ((src[j] - src[i]) ** 2).sum(1)
    b_true = ((dst[j] - dst[i]) ** 2).sum(1)
    if mode == "kernel":
        a, b = gram(c["qs"], c["Ns"], i, j), gram(c["qd"], c["Nd"], i, j)
    else:
        a = moved(a_true, mult * c["ea"], 1.0 if mode[0] == "p" else -1.0)
        b = moved(b_true, mult * c["eb"], 1.0 if mode[1] == "p" else -1.0)
    err = max(np.abs(a - a_true).max() / (c["ea"] / 28.0), np.abs(b - b_true).max() / (c["eb"] / 28.0))
    t, s = f32(a - b), f32(a + b)
    dh = fma(t, t, fma(s, c["mhi"], c["chi"]))
    dl = fma(t, t, fma(s, c["mlo"], c["clo"]))
    sure_edge, sure_non = np.signbit(dh), ~np.signbit(dl)
    wrong = int((sure_edge & ~exact).sum() + (sure_non & exact).sum())
    und = float((~sure_edge & ~sure_non).mean())
    if verbose:
        print(f"{label:8s} {mode:6s} use_gram={c['use_gram']!s:5s} pairs={len(i)} edges={int(exact.sum())} "
              f"undecided={und:.2e} wrong={wrong} max|a'-a|={err:.1f} u R^2")
    return wrong, und, c["use_gram"], err


def duplicates(cfg="C2cube", seed=8, n=700):
    pr = synth.config_problem(cfg, seed, n=n)
    src, dst = pr["src"].copy(), pr["dst"].copy()
    for k in range(0, 60, 3):
        src[k + 1] = src[k]
    for k in range(100, 160, 3):
        dst[k + 1] = dst[k]
        src[k + 1] = src[k] + 1e-9
    return src, dst, pr["noise_bound"]


GUARD_OFFSET = np.array([1000.0, -2000.0, 500.0])


def _cube(n, seed):
    return np.random.default_rng(seed).uniform(size=(n, 3))


def _stretched(src, beta, rho):
    return (1.0 + beta / rho) * src + GUARD_OFFSET


def guard_beta(src, rho):
    """beta*: the smallest beta (to one ulp) for which consts() passes the conditioning guard on (src, _stretched(src,
    beta, rho)); the binding condition is 64 E <= 0.75 D_min beta."""
    def ok(beta):
        return consts(src, _stretched(src, beta, rho), beta)["use_gram"]
    lo, hi = 1e-7, 1e-2
    assert not ok(lo) and ok(hi)
    while np.nextafter(lo, hi) < hi:
        mid = 0.5 * (lo + hi)
        if mid <= lo or mid >= hi:
            break
        lo, hi = (lo, mid) if ok(mid) else (mid, hi)
    return hi


def guard_edge(factor, rho, n=1200, seed=5):
    """(src, dst, noise_bound) with beta = factor * beta* (factor 1.0: the first beta the guard admits)."""
    src = _cube(n, seed)
    beta = factor * guard_beta(src, rho)
    return src, _stretched(src, beta, rho), 0.5 * beta


def dmin_edge(beyond, rho=1.0, n=600, seed=6):
    """beta = D_min / 8 (8 beta = D_min exactly: the guard passes) or one ulp above (it fails).  dst is stretched, so
    D_min is the source diagonal and does not move with beta."""
    src = _cube(n, seed)
    mn, mx = src.min(0), src.max(0)
    beta = np.sqrt(float(((mx - mn) ** 2).sum())) / 8.0
    if beyond:
        beta = np.nextafter(beta, np.inf)
    return src, _stretched(src, beta, rho), 0.5 * beta


def lattice(offset=0.0, scale=1.0, permute_seed=None, k=11):
    """k^3 integer lattice scaled by h = 2^-4, dst = (2 src) * scale + offset, beta = h (noise bound h / 2).  With
    scale = 1 and a power-of-two offset all arithmetic is exact and the 3 k^2 (k - 1) lattice-neighbour pairs are exact
    ties; scale = 1 +- 2^-50 moves them a few ulp above or below the threshold."""
    h = 2.0 ** -4
    g = np.arange(k, dtype=np.float64)
    src = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) * h
    if permute_seed is not None:
        src = src[np.random.default_rng(permute_seed).permutation(len(src))]
    dst = 2.0 * src * scale + offset
    return np.ascontiguousarray(src), np.ascontiguousarray(dst), 0.5 * h


def edge_count(src, dst, noise_bound):
    i, j = np.triu_indices(len(src), 1)
    return int((np.abs(tim_norm(src, i, j) - tim_norm(dst, i, j)) <= 2.0 * noise_bound).sum())


def main():
    total = 0
    modes = ("kernel", "pp", "pm", "mp", "mm")
    for cfg, n in [("C2", 1500), ("C2cube", 1100), ("C3", 2000), ("C4", 640), ("C5", 1700)]:
        pr = synth.config_problem(cfg, 21, n=n)
        for mode in modes:
            total += check(pr["src"], pr["dst"], pr["noise_bound"], mode, cfg)[0]
    src, dst, nb = duplicates()
    for mode in modes:
        total += check(src, dst, nb, mode, "dups")[0]
    pr = synth.config_problem("C2", 3, n=600)
    for nb in (0.05, 0.2, 0.5):
        for mode in modes:
            total += check(pr["src"], pr["dst"], nb, mode, f"nb{nb}")[0]
    for factor in (1.0, 1.02, 1.2, 2.0):
        for rho in (0.3, 0.6, 1.0):
            src, dst, nb = guard_edge(factor, rho)
            for mode in modes:
                total += check(src, dst, nb, mode, f"g{factor}/{rho}")[0]
    for beyond in (False, True):
        src, dst, nb = dmin_edge(beyond)
        for mode in modes:
            total += check(src, dst, nb, mode, f"dmin{int(beyond)}")[0]
    for off, sc in ((0.0, 1.0), (1024.0, 1.0), (0.0, 1.0 + 2.0 ** -50), (0.0, 1.0 - 2.0 ** -50)):
        src, dst, nb = lattice(off, sc, permute_seed=1)
        for mode in modes:
            total += check(src, dst, nb, mode, "lattice")[0]
    print("TOTAL WRONG", total)


if __name__ == "__main__":
    main()
