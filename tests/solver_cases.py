"""Constraint systems for the solver tests: restatements of fidget-solver's own test cases (fidget-solver/src/lib.rs)
and seeded families for batch comparisons.  Every builder takes a ``Context`` (the product's or the oracle's; both
share the host front end) and returns ``Case``: constraint roots plus the free / fixed variable keys ("x", "y", "z"
or ``Context.var()`` ids) and the starting values in that order.  Constants are passed as Python floats."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


@dataclass
class Case:
    roots: list
    free: list
    fixed: list = field(default_factory=list)
    start: list = field(default_factory=list)   # free values, then fixed values


def slot_keys(tape_data):
    return [kind if kind in "xyz" else vid for kind, vid in tape_data.vars()]


def slot_map(tape_data, keys):
    index = {k: i for i, k in enumerate(keys)}
    return np.array([index.get(k, -1) for k in slot_keys(tape_data)], dtype=np.int32)


def _f(v):
    return float(np.float32(v))


def _vars(ctx, n):
    nodes, keys = [], []
    for _ in range(n):
        node, vid = ctx.var()
        nodes.append(node)
        keys.append(vid)
    return nodes, keys


# ---- the reference's cases -------------------------------------------------------------------------------------
def basic_solver(ctx):
    return Case([ctx.add(ctx.x(), ctx.y())], ["x"], ["y"], [0.0, -1.0])


def four_vars_at_once(ctx):
    vs, keys = _vars(ctx, 4)
    root = vs[0]
    for v in vs[1:]:
        root = ctx.add(root, v)
    return Case([root], keys, [], [float(i) for i in range(4)])


def four_vars_independent(ctx):
    vs, keys = _vars(ctx, 4)
    return Case([ctx.sub(v, float(i)) for i, v in enumerate(vs)], keys, [], [2.0 * i for i in range(4)])


def xy_nonlinear(ctx):
    x, y = ctx.x(), ctx.y()
    a = ctx.sub(ctx.mul(ctx.add(ctx.mul(x, 2.0), ctx.mul(y, 3.0)), ctx.sub(x, y)), 2.0)
    b = ctx.sub(ctx.add(ctx.mul(x, 3.0), y), 5.0)
    return Case([a, b], ["x", "y"], [], [0.0, 0.0])


def one_var_no_solution(ctx):
    x = ctx.x()
    return Case([ctx.sub(x, 1.0), ctx.sub(x, 2.0)], ["x"], [], [0.0])


def banana(ctx, start=(0.0, 0.0)):
    x, y = ctx.x(), ctx.y()
    return Case([ctx.sub(1.0, x), ctx.mul(100.0, ctx.sub(y, ctx.square(x)))], ["x", "y"], [], list(start))


def circle(ctx, start=(0.0, 0.0)):
    x, y = ctx.x(), ctx.y()
    return Case([ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y)))], ["x", "y"], [], list(start))


def linear(ctx, n, rng):
    """one_linear: n random equations sum_c mat[r][c] v_c = sol[r] built like the reference's trees, start 0."""
    values = rng.random(n, dtype=np.float32)
    mat = rng.random((n, n), dtype=np.float32)
    sol = (mat.astype(np.float64) @ values.astype(np.float64)).astype(np.float32)
    vs, keys = _vars(ctx, n)
    roots = []
    for row in range(n):
        out = ctx.constant(_f(-sol[row]))
        for col in range(n):
            out = ctx.add(out, ctx.mul(_f(mat[row, col]), vs[col]))
        roots.append(out)
    return Case(roots, keys, [], [0.0] * n), (mat, sol)


def linear_ok(check, x):
    mat, sol = check
    got = mat.astype(np.float64) @ np.asarray(x, dtype=np.float64)
    return float(np.sum((sol - got) ** 2)) < 1e-3 and bool(np.all(np.abs(sol - got) <= 1e-2))


def quadratic(ctx, n, rng):
    """one_quadratic: n equations over [v, v_i v_j] with random coefficients, start 0.5."""
    values = rng.random(n, dtype=np.float32)
    m = n * n + n
    col = np.zeros(m, dtype=np.float32)
    col[:n] = values
    for i in range(n):
        for j in range(n):
            col[i * n + j + n] = values[i] * values[j]
    mat = rng.random((n, m), dtype=np.float32)
    sol = (mat.astype(np.float64) @ col.astype(np.float64)).astype(np.float32)
    vs, keys = _vars(ctx, n)
    roots = []
    for row in range(n):
        out = ctx.constant(_f(-sol[row]))
        for c in range(n):
            out = ctx.add(out, ctx.mul(_f(mat[row, c]), vs[c]))
        for i in range(n):
            for j in range(n):
                out = ctx.add(out, ctx.mul(ctx.mul(_f(mat[row, i * n + j + n]), vs[i]), vs[j]))
        roots.append(out)
    return Case(roots, keys, [], [0.5] * n), (mat, sol, n)


def quadratic_ok(check, x):
    mat, sol, n = check
    x = np.asarray(x, dtype=np.float64)
    col = np.concatenate([x, np.outer(x, x).reshape(-1)])
    got = mat.astype(np.float64) @ col
    return float(np.sum((sol - got) ** 2)) < 1e-3 and bool(np.all(np.abs(sol - got) <= 1e-2))


# ---- families for batch comparisons ----------------------------------------------------------------------------
def rosenbrock_chain(ctx, n):
    """1 - v_i and 10 (v_{i+1} - v_i^2): a banana valley in n variables (n >= 2)."""
    vs, keys = _vars(ctx, n)
    roots = [ctx.sub(1.0, v) for v in vs]
    roots += [ctx.mul(10.0, ctx.sub(vs[i + 1], ctx.square(vs[i]))) for i in range(n - 1)]
    return Case(roots, keys, [], [0.0] * n)


def sphere(ctx, n, radius=0.75):
    """sqrt(sum v_i^2) - radius: one constraint, a whole sphere of solutions."""
    vs, keys = _vars(ctx, n)
    s = ctx.square(vs[0])
    for v in vs[1:]:
        s = ctx.add(s, ctx.square(v))
    return Case([ctx.sub(ctx.sqrt(s), radius)], keys, [], [0.5] * n)


def transcendental(ctx):
    x, y = ctx.x(), ctx.y()
    return Case([ctx.sub(ctx.sin(x), 0.5), ctx.sub(ctx.exp(ctx.mul(x, y)), 2.0)], ["x", "y"], [], [0.1, 0.2])
