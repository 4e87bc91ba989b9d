"""Constraint sketches for the large-problem solver tests: a W x H grid of 2D points joined by distance constraints
sqrt((xi - xj)^2 + (yi - yj)^2) - L along the grid's edges and one diagonal per cell (a triangulated, rigid sheet), the
bottom row fixed, the start at the rest positions plus seeded noise.  n_free = 2 W (H - 1).  Builders take a
``Context`` (the product's or the oracle's) and return ``solver_cases.Case``, free variables first."""
from __future__ import annotations

import numpy as np

from solver_cases import Case

DIAG = float(np.float32(np.sqrt(2.0)))


def sketch_edges(w, h):
    """(a, b, rest length) over point indices j * w + i; edges between two bottom-row (fixed) points are left out"""
    edges = []
    for j in range(h):
        for i in range(w):
            p = j * w + i
            if i + 1 < w and j > 0:
                edges.append((p, p + 1, 1.0))
            if j + 1 < h:
                edges.append((p, p + w, 1.0))
                if i + 1 < w:
                    edges.append((p, p + w + 1, DIAG))
    return edges


def sketch(ctx, w, h, seed=0, noise=0.1):
    """The W x H sketch with its start; returns (Case, edges).  Parameters: x, y of rows 1 .. H-1 (free), then x, y of
    row 0 (fixed)."""
    xs, ys, xk, yk = [], [], [], []
    for _ in range(w * h):
        (x, kx), (y, ky) = ctx.var(), ctx.var()
        xs.append(x)
        ys.append(y)
        xk.append(kx)
        yk.append(ky)
    roots = []
    for a, b, length in sketch_edges(w, h):
        dx, dy = ctx.sub(xs[a], xs[b]), ctx.sub(ys[a], ys[b])
        roots.append(ctx.sub(ctx.sqrt(ctx.add(ctx.square(dx), ctx.square(dy))), length))
    free = [k for p in range(w, w * h) for k in (xk[p], yk[p])]
    fixed = [k for p in range(w) for k in (xk[p], yk[p])]
    rest = np.array([[p % w, p // w] for p in range(w * h)], dtype=np.float32)
    rng = np.random.default_rng([w, h, seed])
    moved = rest[w:] + rng.uniform(-noise, noise, rest[w:].shape).astype(np.float32)
    start = [float(v) for v in moved.reshape(-1)] + [float(v) for v in rest[:w].reshape(-1)]
    return Case(roots, free, fixed, start), sketch_edges(w, h)


def sketch_starts(case, count, seed, noise=0.1):
    """`count` start rows: the case's start with fresh noise on the free entries"""
    rows = np.tile(np.array(case.start, dtype=np.float32), (count, 1))
    n = len(case.free)
    rng = np.random.default_rng([count, seed, n])
    rows[1:, :n] += rng.uniform(-noise, noise, (count - 1, n)).astype(np.float32)
    return rows


def sketch_residuals(w, h, edges, row):
    """float64 constraint values of one solved row (free entries first, as the Case orders them)"""
    row = np.asarray(row, dtype=np.float64)
    n = 2 * w * (h - 1)
    pts = np.concatenate([row[n:].reshape(w, 2), row[:n].reshape(-1, 2)])
    a = np.array([e[0] for e in edges])
    b = np.array([e[1] for e in edges])
    length = np.array([e[2] for e in edges], dtype=np.float64)
    return np.hypot(*(pts[a] - pts[b]).T) - length
