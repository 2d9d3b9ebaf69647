"""CPU check of the single-slope form of the Gram pair test of graph_strip2_kernel (DESIGN.md §3.1; constants as in
prep_kernel, graph_build.cu).  Lengths are in units of 2 beta (sig = 1 / (2 beta)), where the test is

    f = (A - B + 1/4)^2 - A:   f <= 0 => edge,  f > 1/16 => not an edge      (A, B the squared TIM norms in these units)

and the kernel's FP32 operations are emulated in numpy in their order:

    q = fl((p - c) sig), N = fl(|q|^2)                     (prep_kernel, FP64 then one rounding)
    u = fma(z_j, 2 z_i, fma(y_j, 2 y_i, fma(x_j, 2 x_i, fl(c_u - N_i) - N_j)))     (= c_u - A'),  v likewise with c_v
    T = v - u,  dh = fma(T, T, u),  dl = dh + dl_c

(an FMA is one FP64 operation rounded to FP32, as in scripts/gram_band_check.py).  sign(dh) = 1 decides an edge,
sign(dl) = 0 a non-edge; every decided pair must agree with the reference's FP64 predicate.  Mode "kernel" is the
emulation; modes "pp", "pm", "mp", "mm" replace u and v by c_u - A and c_v - B moved by the full proven bound (+-Eu,
+-Ev, times `mult`), so that the band is checked against the bound and not only against the errors that happen to occur.
The fixtures are gram_band_check's, plus a far offset of both clouds and corner_ties(), where the band is tight.
usage: python scripts/slope_band_check.py"""
import importlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
gbc = importlib.import_module("gram_band_check")
synth = gbc.synth
f32, fma, moved, u = gbc.f32, gbc.fma, gbc.moved, gbc.u


def f32_up(x):
    """The smallest float >= x (__double2float_ru)."""
    y = np.float32(x)
    if float(y) < x:
        y = np.nextafter(y, np.float32(np.inf))
    return float(y)


def consts(src, dst, beta, cu_scale=1.0, k_scale=1.0):
    """prep_kernel's single-slope constants and operands (fixed scale), and the guard of gram_band_check.consts().
    cu_scale, k_scale (tests only) shrink the edge-side constant c_u and the non-edge margin K before rounding."""
    c = {"use_gram": gbc.consts(src, dst, beta)["use_gram"]}
    mn_s, mx_s, mn_d, mx_d = src.min(0), src.max(0), dst.min(0), dst.max(0)
    cs, cd = 0.5 * (mn_s + mx_s), 0.5 * (mn_d + mx_d)
    Ds2, Dd2 = float(((mx_s - mn_s) ** 2).sum()), float(((mx_d - mn_d) ** 2).sum())
    sig = 0.5 / beta
    As, Ad = sig * sig * Ds2, sig * sig * Dd2

    def eu(cc):
        return u * (7.0 * As + 6.0 * cc)

    def ev(cc):
        return u * (7.0 * Ad + 6.0 * (cc + 0.25))

    cu = 0.0
    for _ in range(8):
        Eu = eu(cu)
        E1 = Eu + ev(cu)
        cu = Eu + 5.0 * u * (As + Eu) + 2.0 * (1.0 + 2.0 * u) * E1 * np.sqrt(As + Eu) + E1 * E1
    cv = f32_up(f32_up(cu_scale * cu * (1.0 + 2.0 ** -16)) + 0.25)
    cu = cv - 0.25
    Eu, Ev = eu(cu), ev(cu)
    E1 = Eu + Ev
    K = 0.0
    for _ in range(8):
        K = (0.0625 + 2.0 * u * As + 2.0 * E1 * np.sqrt(As + K)) / (1.0 - 2.0 * u)
    K *= (1.0 + 2.0 ** -16) * k_scale
    c.update(sig=sig, As=As, cu=cu, cv=cv, dl=-f32_up((K + cu + Eu) / (1.0 - u)), Eu=Eu, Ev=Ev)
    c["qs"], c["qd"] = f32((src - cs) * sig), f32((dst - cd) * sig)
    c["Ns"], c["Nd"] = f32((c["qs"] ** 2).sum(1)), f32((c["qd"] ** 2).sum(1))
    return c


def chain(q, N, cc, i, j):
    """fl(c - N_i) - N_j + sum_k (2 q_ik) q_jk in the kernel's order."""
    x = f32(f32(cc - N[i]) - N[j])
    for k in range(3):
        x = fma(q[j, k], 2.0 * q[i, k], x)
    return x


def check(src, dst, noise_bound, mode="kernel", label="", verbose=True, mult=1.0, cu_scale=1.0, k_scale=1.0):
    """Returns (wrong decisions, undecided fraction, use_gram, largest |u - (c_u - A)| / (u R^2))."""
    beta = 2.0 * noise_bound
    c = consts(src, dst, beta, cu_scale, k_scale)
    i, j = np.triu_indices(len(src), 1)
    d1, d2 = gbc.tim_norm(src, i, j), gbc.tim_norm(dst, i, j)
    exact = np.abs(d1 - d2) <= beta
    s2 = c["sig"] ** 2
    A = ((src[j] - src[i]) ** 2).sum(1) * s2
    B = ((dst[j] - dst[i]) ** 2).sum(1) * s2
    if mode == "kernel":
        uu, vv = chain(c["qs"], c["Ns"], c["cu"], i, j), chain(c["qd"], c["Nd"], c["cv"], i, j)
    else:
        uu = moved(c["cu"] - A, mult * c["Eu"], 1.0 if mode[0] == "p" else -1.0)
        vv = moved(c["cv"] - B, mult * c["Ev"], 1.0 if mode[1] == "p" else -1.0)
    err = np.abs(uu - (c["cu"] - A)).max() / (u * c["As"] / 4.0)
    T = f32(vv - uu)
    dh = fma(T, T, uu)
    dl = f32(dh + c["dl"])
    sure_edge, sure_non = np.signbit(dh), ~np.signbit(dl)
    wrong = int((sure_edge & ~exact).sum() + (sure_non & exact).sum())
    und = float((~sure_edge & ~sure_non).mean())
    if verbose:
        print(f"{label:10s} {mode:6s} use_gram={c['use_gram']!s:5s} pairs={len(i)} edges={int(exact.sum())} "
              f"undecided={und:.2e} wrong={wrong} max|u-(c_u-A)|={err:.1f} u R^2")
    return wrong, und, c["use_gram"], err


FAR = np.array([3.0e4, -5.0e4, 1.0e5])


def corner_ties(factor=1.0, n=1200, seed=5, eps=0.02):
    """Where the band is tight: two clusters in opposite corners of the unit cube, dst = (1 + beta/rho) src + offset with
    rho = 0.98 sqrt(3), so the ties are pairs across the diagonal, with |T| close to sqrt(A_s), the value the band is
    derived for; beta = factor * beta* (the guard edge)."""
    p = np.random.default_rng(seed).uniform(size=(n, 3)) * eps
    p[n // 2:] += 1.0 - eps
    p[0], p[-1] = 0.0, 1.0
    rho = 0.98 * np.sqrt(3.0)
    beta = factor * gbc.guard_beta(p, rho)
    return p, gbc._stretched(p, beta, rho), 0.5 * beta


def fixtures(small=False):
    """(label, src, dst, noise bound): the benchmark geometries, duplicates, noise bounds up to D/4, the guard edge, the
    8 beta = D_min edge, the exact-tie lattices and a far offset.  small: the sizes of the GPU tests."""
    out = []
    k = 2 if small else 1
    for cfg, n in [("C2", 1500), ("C2cube", 1100), ("C3", 2000), ("C4", 640), ("C5", 1700)]:
        pr = synth.config_problem(cfg, 21, n=n // k)
        out.append((cfg, pr["src"], pr["dst"], pr["noise_bound"]))
    out.append(("dups",) + gbc.duplicates())
    pr = synth.config_problem("C2", 3, n=600)
    D = float(np.sqrt(((pr["src"].max(0) - pr["src"].min(0)) ** 2).sum()))
    for nb in (0.05, 0.2, 0.5, D / 4):
        out.append((f"nb{nb:.3g}", pr["src"], pr["dst"], nb))
    for factor in (1.0, 1.02, 1.2, 2.0):
        for rho in (0.3, 0.6, 0.65, 0.7, 1.0):
            out.append((f"g{factor}/{rho}",) + gbc.guard_edge(factor, rho, n=1200 // k))
    for beyond in (False, True):
        out.append((f"dmin{int(beyond)}",) + gbc.dmin_edge(beyond))
    for off, sc in ((0.0, 1.0), (1024.0, 1.0), (0.0, 1.0 + 2.0 ** -50), (0.0, 1.0 - 2.0 ** -50)):
        out.append((f"lat{off:g}/{sc - 1.0:+.0e}",) + gbc.lattice(off, sc, permute_seed=1))
    pr = synth.config_problem("C2", 5, n=1500 // k)
    out.append(("C2far", pr["src"] + FAR, pr["dst"] - FAR, pr["noise_bound"]))
    for factor in (1.0, 1.02):
        out.append((f"corner{factor}",) + corner_ties(factor, n=1200 // k))
    return out


BENCH = ("C2", "C2cube", "C3", "C4", "C5", "C2far")


def main():
    total = 0
    for label, src, dst, nb in fixtures():
        for mode in ("kernel", "pp", "pm", "mp", "mm"):
            total += check(src, dst, nb, mode, label)[0]
    print("TOTAL WRONG", total)


if __name__ == "__main__":
    main()
