"""Numpy float64 restatement of the generalized ICP of include/teaser_b200.h (tzr_icp_generalized, DESIGN.md §3.14).

Everything but the system is point-to-plane ICP's (tests/icp_plane_reference.py): the transform, the search, the
evaluation, the loop, the 6 x 6 solve and the Euler update are reused from there.  The system follows the header's
formulas (the covariances C(v), M = s^2 C(R m) + C(n), its adjugate inverse A, then J^T A J and J^T A d), with the
sums in numpy's order, so R and t agree with the device to rounding, not bit for bit.
"""
from __future__ import annotations

import numpy as np

import icp_plane_reference as plane
from icp_plane_reference import evaluate, margins, transform  # noqa: F401  (re-exported for the tests)


def _len2(v):
    return (v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]


def covariance(v, epsilon):
    """C(v) = I - (k v_a) v_b with k = (1 - epsilon) / ((v0 v0 + v1 v1) + v2 v2), per row of v: (n, 3, 3)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        k = (1.0 - epsilon) / _len2(v)
    kv = k[:, None] * v
    return np.eye(3)[None] - kv[:, :, None] * v[:, None, :]


def inverse_adjugate(M):
    """A = M^-1 by the symmetric adjugate of the header (upper triangle used), and det."""
    M00, M01, M02, M11, M12, M22 = M[:, 0, 0], M[:, 0, 1], M[:, 0, 2], M[:, 1, 1], M[:, 1, 2], M[:, 2, 2]
    c00, c01, c02 = M11 * M22 - M12 * M12, M02 * M12 - M01 * M22, M01 * M12 - M02 * M11
    c11, c12, c22 = M00 * M22 - M02 * M02, M01 * M02 - M00 * M12, M00 * M11 - M01 * M01
    det = (M00 * c00 + M01 * c01) + M02 * c02
    C = np.stack([np.stack([c00, c01, c02], 1), np.stack([c01, c11, c12], 1), np.stack([c02, c12, c22], 1)], 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return C / det[:, None, None], det


def jacobian(u):
    """J = [e_k x u (k = 0..2), I] per row of u: (n, 3, 6)."""
    J = np.zeros((u.shape[0], 3, 6))
    for k in range(3):
        e = np.zeros(3)
        e[k] = 1.0
        J[:, :, k] = np.cross(e, u)
        J[:, k, 3 + k] = 1.0
    return J


def system(ev, y, src_normals, dst_normals, R, s, epsilon, centre):
    """(A, g) = (sum J^T A J, sum J^T A d) over the correspondences of an evaluation whose normals are finite and of
    non-zero length and whose det is finite and > 0; R: the current rotation, s the scale."""
    m = ev["idx"] >= 0
    P = ev["p"][m]
    Q = np.asarray(y, dtype=np.float32).astype(np.float64)[ev["idx"][m]]
    Ms = np.asarray(src_normals, dtype=np.float32)[:, :3].astype(np.float64)[np.nonzero(m)[0]]
    Nt = np.asarray(dst_normals, dtype=np.float32)[:, :3].astype(np.float64)[ev["idx"][m]]
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.isfinite(Ms).all(axis=1) & np.isfinite(Nt).all(axis=1) & (_len2(Ms) > 0) & (_len2(Nt) > 0)
    P, Q, Ms, Nt = P[ok], Q[ok], Ms[ok], Nt[ok]
    R = np.asarray(R, dtype=np.float64)
    Mr = np.stack([(R[r, 0] * Ms[:, 0] + R[r, 1] * Ms[:, 1]) + R[r, 2] * Ms[:, 2] for r in range(3)], axis=1)
    s2 = float(s) * float(s)
    M = s2 * covariance(Mr, epsilon) + covariance(Nt, epsilon)
    A, det = inverse_adjugate(M)
    keep = (det > 0) & np.isfinite(det)
    A, P, Q = A[keep], P[keep], Q[keep]
    J = jacobian(P - np.asarray(centre, dtype=np.float64))
    d = P - Q
    return np.einsum("nki,nkl,nlj->ij", J, A, J), np.einsum("nki,nkl,nl->i", J, A, d)


class Update:
    """The update of tzr_icp_generalized as an icp_plane_reference.icp update_fn.  The system needs the current
    rotation, which an evaluation does not carry, so this follows it: R <- R_u R after every step, as the loop
    composes."""

    def __init__(self, src_normals, s, R, epsilon):
        self.src_normals, self.s, self.epsilon = src_normals, float(s), float(epsilon)
        self.R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64).copy()

    def __call__(self, ev, y, dst_normals):
        m = ev["idx"] >= 0
        if not m.any():
            Ru, tu = np.eye(3), np.zeros(3)
        else:
            c = ev["p"][m].mean(axis=0)
            A, g = system(ev, y, self.src_normals, dst_normals, self.R, self.s, self.epsilon, c)
            x = plane.solve6(A, g)
            if np.isfinite(x).all():
                Ru = plane.euler(*x[:3])
                tu = (c + x[3:]) - Ru @ c
            else:
                Ru, tu = np.eye(3), np.zeros(3)
        self.R = Ru @ self.R
        return Ru, tu


def icp(x, y, src_normals, dst_normals, r, s=1.0, R=None, t=None, epsilon=1e-3, **kw):
    """The loop of tzr_icp_generalized.  Returns what icp_reference.icp returns."""
    return plane.icp(x, y, dst_normals, r, s=s, R=R, t=t, update_fn=Update(src_normals, s, R, epsilon), **kw)
