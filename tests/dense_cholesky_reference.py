"""References for the batched pose-graph routes' dense Cholesky (tzr_dense_cholesky_batch, DESIGN.md §3.23).

- Exact systems: L lower triangular with power-of-two diagonals 2^e (e in -3 ... 3) and off-diagonal entries that are
  small multiples of 1/8; A = L L^T and b = A x with small integer x.  Every entry of L is a multiple of 2^-3, so every
  product L_ik L_jk is a multiple of 2^-6; every value a right-looking (or any other) Cholesky or substitution forms is
  a partial sum of such products, or of L_ik x_k, bounded by (|L| |L|^T)_ij or (|L| |L|^T |x|)_i, and exact while
  that bound stays below 2^47 (checked).  Every pivot is L_jj^2 = 4^e, so its square root and every division by it are
  exact too: any correct order of operations returns L and x bit for bit, and a missing division, square root or
  update changes them.
- Failure variants of an exact system, each with the info a correct factorisation reports (1 + the first column whose
  pivot is not > 0).
- Backward-error bounds for rounded inputs (Higham, Accuracy and Stability of Numerical Algorithms, Thms 10.3, 10.4):
  |fl(L^ L^T) - A| <= (gamma_{n+1} + gamma_n + u) |L^| |L^T| for the factor and |b - A x^| <= (gamma_{3n+1} + gamma_n + u)
  |L^| |L^T| |x^| for the solve (gamma_n + u covers forming the residual in float64), and x^ against a long-double
  solve within the normwise bound kappa eta / (1 - kappa eta)."""
import numpy as np

U = 2.0 ** -53
NB = 32        # the device's panel width
EXACT_LIMIT = 2.0 ** 47  # values that are multiples of 2^-6 are exact below this


def gamma(k):
    return k * U / (1.0 - k * U)


# ---- exact systems -----------------------------------------------------------------------------------------------------
def exact_factor(rng, n, density=0.3, off_max=2.0):
    """L (n x n, lower): diagonal 2^e with e uniform in -3 ... 3 (never all 1), off-diagonal entries at the given density,
    multiples of 1/8 in [-off_max, off_max]."""
    e = rng.integers(-3, 4, size=n)
    if n and not (e != 0).any():
        e[0] = 1
    L = np.zeros((n, n))
    steps = int(off_max * 8)
    off = rng.integers(-steps, steps + 1, size=(n, n)) / 8.0
    mask = np.tril(rng.random((n, n)) < density, -1)
    L[mask] = off[mask]
    L[np.arange(n), np.arange(n)] = np.ldexp(1.0, e)
    return L


def exact_bounds(L, x):
    """(max of |L| |L|^T, max of |L| |L|^T |x|): bounds of every partial sum the factorisation and the solve form."""
    aL = np.abs(L)
    P = aL @ aL.T
    return float(P.max(initial=0.0)), float((P @ np.abs(x)).max(initial=0.0))


def exact_system(rng, n, density=0.3, off_max=2.0, x_max=4):
    """(A, b, L, x): A = L L^T and b = A x, both exact, with L from exact_factor and integer x in [-x_max, x_max]."""
    L = exact_factor(rng, n, density, off_max)
    x = rng.integers(-x_max, x_max + 1, size=n).astype(np.float64)
    fb, sb = exact_bounds(L, x)
    assert 2.0 * fb < EXACT_LIMIT and 2.0 * sb < EXACT_LIMIT, (fb, sb)
    A = L @ L.T
    b = A @ x
    # the products above are exact: check them against a sum in exact integer arithmetic (entries scaled by 2^3)
    Li = (L * 8).astype(np.int64)
    assert np.array_equal((Li @ Li.T).astype(np.float64) / 64.0, A)
    assert np.array_equal(((Li @ Li.T) @ x.astype(np.int64)).astype(np.float64) / 64.0, b)
    return A, b, L, x


def right_looking(A, nb=NB):
    """The device's schedule in float64: panels of nb columns, the diagonal tile column by column, the rows below by
    forward substitution, then the trailing lower triangle.  Returns (L, info) with info as the device reports it."""
    A = np.tril(np.array(A, dtype=np.float64))
    n = A.shape[0]
    for j0 in range(0, n, nb):
        p = min(j0 + nb, n)
        for k in range(j0, p):
            piv = A[k, k]
            if not piv > 0:
                return A, k + 1
            lkk = np.sqrt(piv)
            A[k + 1:p, k] = A[k + 1:p, k] / lkk
            A[k, k] = lkk
            for c in range(k + 1, p):
                A[c:p, c] = A[c:p, c] - A[c:p, k] * A[c, k]
        for k in range(j0, p):
            s = A[p:, k]
            for q in range(j0, k):
                s = s - A[p:, q] * A[k, q]
            A[p:, k] = s / A[k, k]
        L21 = A[p:, j0:p]
        A[p:, p:] = A[p:, p:] - np.tril(L21 @ L21.T)
    return A, 0


def substitute(L, b):
    """x = (L L^T)^-1 b by row-wise forward and backward substitution in float64."""
    n = len(b)
    y = np.array(b, dtype=np.float64)
    for i in range(n):
        y[i] = (y[i] - L[i, :i] @ y[:i]) / L[i, i]
    x = y.copy()
    for i in range(n - 1, -1, -1):
        x[i] = (x[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
    return x


# ---- failure variants --------------------------------------------------------------------------------------------------
VARIANTS = ("zero", "negative", "nan_diag", "nan_below")


def failure(A, L, variant, j):
    """A copy of the exact A = L L^T that fails at column j (variant "nan_below": the NaN at (j, j // 2), so j >= 1).
    Returns (A', info)."""
    A = A.copy()
    if variant == "zero":       # the pivot is exactly 0
        A[j, j] = A[j, j] - L[j, j] * L[j, j]
    elif variant == "negative":  # the pivot is exactly -1/4
        A[j, j] = A[j, j] - (L[j, j] * L[j, j] + 0.25)
    elif variant == "nan_diag":
        A[j, j] = np.nan
    elif variant == "nan_below":  # column j // 2 is factored with a NaN in row j, whose pivot is the first NaN one
        A[j, j // 2] = A[j // 2, j] = np.nan
    else:
        raise ValueError(variant)
    return A, j + 1


def finished_columns(L, variant, j):
    """The columns a factorisation that fails at column j has finished (every panel before j's) as a correct one leaves
    them: L's, with a NaN in row j from column j // 2 on for "nan_below"."""
    c = (j // NB) * NB
    want = L[:, :c].copy()
    if variant == "nan_below":
        want[j, j // 2:c] = np.nan
    return want


# ---- backward-error bounds -----------------------------------------------------------------------------------------------
def factor_violation(A, Lh):
    """max over the lower triangle of |fl(L^ L^T) - A| / ((gamma_{n+1} + gamma_n + u) |L^| |L^T|): <= 1 when the
    factor meets its bound."""
    n = A.shape[0]
    Lh = np.tril(Lh)
    R = np.abs(Lh @ Lh.T - A)
    B = (gamma(n + 1) + gamma(n) + U) * (np.abs(Lh) @ np.abs(Lh).T)
    lo = np.tril(np.ones((n, n), dtype=bool))
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(R[lo] == 0, 0.0, R[lo] / B[lo])
    return float(q.max(initial=0.0))


def solve_violation(A, b, Lh, xh):
    """max of |b - A x^| / ((gamma_{3n+1} + gamma_n + u) |L^| |L^T| |x^|): <= 1 when the solve meets its bound."""
    n = A.shape[0]
    aL = np.abs(np.tril(Lh))
    R = np.abs(b - A @ xh)
    B = (gamma(3 * n + 1) + gamma(n) + U) * (aL @ (aL.T @ np.abs(xh)))
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(R == 0, 0.0, R / B)
    return float(q.max(initial=0.0))


def longdouble_solve(A, b):
    """A^-1 b by a right-looking Cholesky and two substitutions in np.longdouble."""
    A = np.array(A, dtype=np.longdouble)
    n = A.shape[0]
    for k in range(n):
        A[k, k] = np.sqrt(A[k, k])
        A[k + 1:, k] = A[k + 1:, k] / A[k, k]
        A[k + 1:, k + 1:] -= np.outer(A[k + 1:, k], A[k + 1:, k])
    y = np.array(b, dtype=np.longdouble)
    for i in range(n):
        y[i] = (y[i] - A[i, :i] @ y[:i]) / A[i, i]
    for i in range(n - 1, -1, -1):
        y[i] = (y[i] - A[i + 1:, i] @ y[i + 1:]) / A[i, i]
    return y


def forward_bound(A, Lh):
    """kappa_2(A) eta / (1 - kappa_2(A) eta) with eta = gamma_{3n+1} || |L^| |L^T| ||_2 / ||A||_2: the relative 2-norm
    error a solve meeting its backward bound can have (None when kappa eta >= 1 and the bound says nothing)."""
    n = A.shape[0]
    w = np.linalg.eigvalsh(A)
    kappa = w[-1] / w[0] if w[0] > 0 else np.inf
    aL = np.abs(np.tril(Lh))
    eta = gamma(3 * n + 1) * np.linalg.norm(aL @ aL.T, 2) / np.linalg.norm(A, 2)
    ke = kappa * eta
    return None if not ke < 1 else ke / (1 - ke)


def forward_error(xh, x_ld):
    """||x^ - x|| / ||x|| against the long-double solution."""
    d = np.asarray(xh, dtype=np.longdouble) - x_ld
    return float(np.sqrt(np.sum(d * d)) / np.sqrt(np.sum(x_ld * x_ld)))


# ---- rounded inputs ------------------------------------------------------------------------------------------------------
def spd(rng, n, kappa):
    """A random SPD matrix with eigenvalues log-spaced from 1 down to 1 / kappa (a random orthogonal basis)."""
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.logspace(0, -np.log10(kappa), n) if n > 1 else np.ones(n)
    A = (Q * lam) @ Q.T
    return (A + A.T) / 2


def nearly_singular(rng, n, rank):
    """A rank-deficient PSD matrix plus 1e-5 max diag times I, as the line process damps its gauge-singular H."""
    B = rng.standard_normal((n, rank))
    A = B @ B.T
    return A + 1e-5 * float(np.max(np.diag(A))) * np.eye(n)


# ---- the batched routes' size limit --------------------------------------------------------------------------------------
def batch_smem(n_max):
    """line_process_batch_smem: the batch kernels' dynamic shared memory with panel stride n_max (the panel, the
    diagonal tile, the right-hand side, the reduction slots, the backward sweep's sums)."""
    return 8 * ((NB + 1) * n_max + NB * 33 + 256 + NB)


def batch_cap(optin):
    """The largest K whose line-process batch kernel (6 K rows) fits optin bytes of shared memory: the batched routes'
    cap, and 6 x it the largest n of tzr_dense_cholesky_batch."""
    K = 1024
    while K > 2 and batch_smem(6 * K) > optin:
        K -= 1
    return K
