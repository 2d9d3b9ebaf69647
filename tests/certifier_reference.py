"""Exact references for the certifier's building blocks (csrc/certify.cu, DESIGN.md 3.9), and the tolerance rules the
GPU tests hold them to.

Dense symmetric matrices with an exactly known spectrum and positive part.  Q is orthogonal and dyadic:

    Q = P . diag(H_1 / 2^k1, H_2 / 2^k2, ...) . (I - 2 v1 v1^T / m) . (I - 2 v2 v2^T / m)

with P a row permutation, H_i Sylvester-Hadamard blocks of sizes 4^ki (H H^T = 4^k I), and v1, v2 vectors of m = 2^j
entries of +-1 on random coordinates (v^T v = m, so each factor is a Householder reflection).  Every entry of Q is an
integer multiple of 2^-a, and with dyadic eigenvalues lambda, M = Q diag(lambda) Q^T is dyadic too.  Whether FP64 holds
it exactly is a bit count, checked by `exactness` below: 2^a Q and 2^e lambda are integer, and every partial sum of
sum_k (2^a Q_ik)(2^e lambda_k)(2^a Q_jk) is bounded by 2^(2a+e) max|lambda| (the rows of 2^a Q have norm 2^a, and
Cauchy-Schwarz), so when that bound is below 2^53 every product and every partial sum of any summation order is an
integer that FP64 represents, and the FP64 product is M itself.  The same argument, with lambda = 1, makes Q Q^T == I
exact.  The positive part P+(M) = Q diag(max(lambda, 0)) Q^T is exact by the same bound.

Scaling M by 2^s is exact (no over- or underflow at the scales used), so the positive part of 2^s M is 2^s P+(M)."""
import numpy as np

EPS = np.finfo(np.float64).eps

# ---- tolerance rules ---------------------------------------------------------------------------------------------
# Nearest-PSD step.  P+ (the Frobenius-nearest PSD matrix) is 1-Lipschitz in the Frobenius norm, because it is the
# projection onto a closed convex set.  A backward-stable symmetric eigensolver returns the exact decomposition of
# M + E with ||E||_F <= c1 n eps ||M||_F, and forming V+ diag(w+) V+^T in FP64 from those (orthogonal to c2 n eps)
# vectors adds at most c3 n eps ||M||_F.  So ||M_psd - P+(M)||_F <= C n eps ||M||_F.  The eigenvalues satisfy Weyl's
# bound |w_i - lambda_i| <= ||E||_2 <= C n eps ||M||_2.  C = 4 is what these constants come to with room; the CPU test
# shows LAPACK (certifier_oracle.nearest_psd) meets it on every exact matrix, so C is set by the mathematics and not
# by the device.
C_PSD = 4.0


def psd_bound(M):
    """Frobenius bound on ||M_psd - P+(M)||_F for an n x n M."""
    n = M.shape[0]
    return C_PSD * n * EPS * np.linalg.norm(M)


def eig_bound(lam):
    """Bound on max |w_i - lambda_i| (ascending), ||M||_2 = max |lambda|."""
    return C_PSD * lam.size * EPS * np.abs(lam).max()


# Dual projection.  It is linear in W: every entry of W_dual is a sum of at most 2N+6 terms, each a product of W
# entries with +-1 thetas and the constants x + 2y, y of the closed-form inverse map (or 1/2, or 1/(N+1) for the
# diagonal mean), and the sums Rs, Cs, the block-row sums and the mean each run over at most N+1 terms.  Summed in any
# order, each entry is within C N eps max|W| of the exact value, the same for the numpy restatement, so two FP64
# evaluations differ by at most 2 C (N + 1) eps max|W|.  The restatement's (N+1)-term sums of N+1-term sums give C = 8.
C_DUAL = 8.0


def dual_bound(W, N):
    return 2 * C_DUAL * (N + 1) * EPS * np.abs(W).max()


# ---- exact dyadic matrices -----------------------------------------------------------------------------------------
def _hadamard(k):
    H = np.ones((1, 1))
    for _ in range(2 * k):
        H = np.block([[H, H], [H, -H]])
    return H


def _blocks(n):
    """n as a sum of powers of 4 (largest first, at most 1024)."""
    out, r = [], n
    while r:
        k = min(5, int(np.floor(np.log(r) / np.log(4) + 1e-12)))
        out.append(k)
        r -= 4 ** k
    return out


def orthogonal(n, seed, reflections=2):
    """The dyadic orthogonal Q described above, and a (its entries are integer multiples of 2^-a)."""
    rng = np.random.default_rng(seed)
    Hb = np.zeros((n, n))
    o = 0
    a = 0
    for k in _blocks(n):
        s = 4 ** k
        Hb[o:o + s, o:o + s] = _hadamard(k) / 2.0 ** k
        o += s
        a = max(a, k)
    m = 2 ** int(min(6, np.floor(np.log2(n))))
    Q = Hb
    for _ in range(reflections):
        v = np.zeros(n)
        v[rng.choice(n, m, replace=False)] = rng.choice([-1.0, 1.0], m)
        Q = Q - np.outer(Q @ v, v) * (2.0 / m)
        a += int(np.log2(m)) - 1
    return Q[rng.permutation(n)], a


def _exponent(x):
    """Smallest e >= 0 with 2^e x integral (x dyadic), or None."""
    for e in range(0, 1100):
        y = np.ldexp(x, e)
        if np.all(np.floor(y) == y):
            return e
    return None


def exactness(Q, lam):
    """True when Q diag(lam) Q^T, Q Q^T and the positive part are provably exact in FP64 (module docstring)."""
    a = _exponent(Q)
    e = _exponent(lam)
    if a is None or e is None:
        return False
    Qi = np.ldexp(Q, a)
    if not np.array_equal(Qi @ Qi.T, np.ldexp(np.eye(Q.shape[0]), 2 * a)):   # 2^(2a) bound: exact integer test
        return False
    top = max(1.0, float(np.abs(lam).max()))
    return 2 * a + e + np.log2(top) < 52


def spectrum(n, kind, seed=0):
    """Ascending dyadic eigenvalues of the named kind."""
    rng = np.random.default_rng(seed)
    if kind == "all_positive":
        lam = rng.integers(1, 64, n) / 8.0
    elif kind == "all_negative":
        lam = -rng.integers(1, 64, n) / 8.0
    elif kind == "zeros":            # exact zeros between negative and positive ones
        z = max(1, n // 8)
        lam = np.concatenate([-rng.integers(1, 64, (n - z) // 2) / 4.0, np.zeros(z),
                              rng.integers(1, 64, n - z - (n - z) // 2) / 4.0])
    elif kind == "repeated":         # three values, each many times
        lam = rng.choice([-3.0, 0.5, 2.0], n)
    elif kind == "wide":             # powers of two over 2^-20 .. 2^20, both signs
        lam = np.ldexp(rng.choice([-1.0, 1.0], n), rng.integers(-20, 21, n))
    elif kind.startswith("first_pos_"):   # first positive eigenvalue at index p (n - 1 for "last")
        t = kind[len("first_pos_"):]
        p = n - 1 if t == "last" else int(t)
        lam = np.concatenate([-rng.integers(1, 64, p) / 8.0, rng.integers(1, 64, n - p) / 8.0])
    else:
        raise ValueError(kind)
    return np.sort(lam)


def first_positive_kinds(n):
    """First positive index at 0, n-1 and either side of the 16-wide k slabs (== 0, 1, 15 mod 16) that fit n."""
    ps = {0, n - 1}
    for base in (16, 48, n // 2 // 16 * 16):
        for d in (-1, 0, 1):
            if 0 < base + d < n:
                ps.add(base + d)
    return ["first_pos_last" if p == n - 1 else f"first_pos_{p}" for p in sorted(ps)]


def exact_matrix(n, kind, seed=0):
    """(M, P+(M), lambda) exact in FP64.  The wide spectrum uses the Hadamard blocks alone (a <= 5), which leaves the
    bits for 2^+-20; every other kind gets both reflections."""
    lam = spectrum(n, kind, seed)
    Q, _ = orthogonal(n, seed + 1000 * n, reflections=0 if kind == "wide" else 2)
    M = (Q * lam) @ Q.T
    P = (Q * np.maximum(lam, 0)) @ Q.T
    return M, P, lam, Q


PSD_SIZES = (8, 64, 68, 128, 132, 1024, 1028)   # 64-tile edges and one past them (n = 4N + 4)
BASE_KINDS = ("all_positive", "all_negative", "zeros", "repeated", "wide")
SCALES = (-40, -20, 20, 40)                    # exact 2^s scalings of the batch tests


def psd_cases():
    """Every (n, kind) the PSD-step tests decompose."""
    return [(n, k) for n in PSD_SIZES for k in BASE_KINDS + tuple(first_positive_kinds(n))]


def psd_part(A):
    """V+ diag(w+) V+^T over the positive eigenpairs of sym(A), LAPACK."""
    B = (A + A.T) / 2
    w, V = np.linalg.eigh(B)
    pos = w > 0
    return (V[:, pos] * w[pos]) @ V[:, pos].T
