"""Test infrastructure: QuadraticErrorSolver::solve (fidget-mesh/src/qef.rs:67-118) restated in float64.

The device and tests/mesh_collapse_oracle.py solve the QEF with the same float32 Jacobi eigen-solve, so their bit
for bit agreement says nothing about whether that solve is right.  This module is the independent answer: given a QEF
exactly as the reference accumulates it (float32 A^T A, A^T b, b^T b and mass point), it solves what qef.rs specifies
with LAPACK's symmetric eigen-solver in float64 and reports what a test needs to judge a float32 solve against it.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

CUTOFF = 1e-3          # EIGENVALUE_CUTOFF_RELATIVE (qef.rs:96)
ERR_FLOOR = float(np.float32(1e-6))   # the error is clamped to >= 1e-6f (qef.rs:112-115)


@dataclass
class Solution:
    pos: np.ndarray        # float64 vertex
    err: float             # clamped error term at pos
    quad: float            # pos^T A^T A pos
    lin: float             # 2 pos^T A^T b
    btb: float
    magnitude: float       # |pos|^T |A^T A| |pos| + 2 |pos|^T |A^T b| + b^T b: what the error term's rounding scales with
    rank: int
    ratios: np.ndarray     # |w_k| / |w_0| for the eigenvalues sorted by |w| descending
    kept: np.ndarray       # eigenvectors (columns) of the kept directions
    dropped: np.ndarray    # eigenvectors (columns) of the dropped directions
    center: np.ndarray     # the mass point

    @property
    def ambiguous(self) -> bool:
        """Some eigenvalue ratio lies within 1 % of the cutoff: float32 rounding may decide the rank either way."""
        return bool((np.abs(self.ratios[1:] / CUTOFF - 1.0) < 0.01).any())

    @property
    def min_kept_ratio(self) -> float:
        return float(self.ratios[self.rank - 1]) if self.rank else 0.0


def error_at(ata, atb, btb, pos):
    """pos^T A^T A pos - 2 pos^T A^T b + b^T b in float64: (clamped error, quad, lin)."""
    a = np.asarray(ata, dtype=np.float64)
    p = np.asarray(pos, dtype=np.float64)
    quad = float(p @ a @ p)
    lin = float(2.0 * p @ np.asarray(atb, dtype=np.float64))
    err = quad - lin + float(btb)
    return (err if err > ERR_FLOOR else ERR_FLOOR), quad, lin


def solve(ata, atb, btb, mp) -> Solution:
    """QuadraticErrorSolver::solve in float64 on the float32 accumulators."""
    a = np.asarray(ata, dtype=np.float64).reshape(3, 3)
    atb = np.asarray(atb, dtype=np.float64)
    mp = np.asarray(mp, dtype=np.float64)
    center = mp[:3] / mp[3]
    b = atb - a @ center
    w, v = np.linalg.eigh(a)
    order = np.argsort(-np.abs(w), kind="stable")
    w, v = w[order], v[:, order]
    aw = np.abs(w)
    ratios = aw / aw[0] if aw[0] > 0 else np.zeros(3)
    cutoff = aw[0] * CUTOFF
    rank = next((k for k in range(3) if aw[k] < cutoff), 3)
    eps = aw[rank] if rank < 3 else 0.0
    keep = aw > eps                   # svd.solve: singular values <= eps are dropped
    sol = np.zeros(3)
    for k in range(3):
        if keep[k]:
            sol += v[:, k] * (v[:, k] @ b / w[k])
    pos = sol + center
    if np.isnan(pos).any():
        pos = center.copy()
    err, quad, lin = error_at(a, atb, btb, pos)
    ap = np.abs(pos)
    magnitude = float(ap @ np.abs(a) @ ap + 2.0 * ap @ np.abs(atb) + float(btb))
    return Solution(pos=pos, err=err, quad=quad, lin=lin, btb=float(btb), magnitude=magnitude, rank=rank, ratios=ratios,
                    kept=v[:, keep], dropped=v[:, ~keep], center=center)


def solve_qef(q) -> Solution:
    """solve() on a mesh_collapse_oracle.Qef"""
    return solve(q.ata, q.atb, q.btb, q.mp)


EPS32 = float(np.finfo(np.float32).eps)
POS_C = 1024           # measured: 260 (tests/test_qef_f64.py)
DROP_C = 256           # measured: 36
ERR_C = 8              # measured: 0.8


def position_bound(s: Solution) -> float:
    """Allowed |pos32 - pos64| (max norm, world units) for a QEF that is not rank-ambiguous.  A float32 solve is
    accurate to a few ulps of the centre, plus the solved offset's ulps times the condition number of the kept
    eigenvalues, 1 / (smallest kept ratio)."""
    return POS_C * EPS32 * (np.abs(s.center).max() + np.abs(s.pos - s.center).max() / s.min_kept_ratio)


def check_vertex(pos32, s: Solution, err32=None):
    """Failures of a float32 vertex (and optionally its error term) against the float64 solution s, which must not be
    rank-ambiguous: position within position_bound, no component along a dropped eigenvector beyond rounding of
    the centre and the offset, error term within rounding of the magnitude of its terms."""
    out = []
    p = np.asarray(pos32, dtype=np.float64)
    dev = float(np.abs(p - s.pos).max())
    if not dev <= position_bound(s):
        out.append(f"|pos32 - pos64| = {dev:.3g} > {position_bound(s):.3g} (ratios {s.ratios})")
    off = p - s.center
    if s.dropped.shape[1]:
        drop = float(np.abs(s.dropped.T @ off).max())
        if not drop <= DROP_C * EPS32 * (np.abs(s.center).max() + np.abs(off).max()):
            out.append(f"component {drop:.3g} along a dropped direction (ratios {s.ratios})")
    if err32 is not None:
        diff = abs(float(err32) - s.err)
        if not diff <= ERR_C * EPS32 * s.magnitude:
            out.append(f"err32 {float(err32):.9g} vs err64 {s.err:.9g}")
    return out
