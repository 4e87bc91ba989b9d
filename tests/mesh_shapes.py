"""Test infrastructure: seeded random CSG shapes for the mesher, drawn to reach the corners of Octree::build and the
dual walks that smooth shapes miss.  Only IEEE-exact opcodes (add, sub, mul, sqrt, square, abs, min, max, neg) are
used, so the device sampler's leaves are bit for bit the oracle's and every comparison can be exact.

  sphere / box / rounded box   at random centres, combined by union, difference and intersection
  thin slab                    thinner than one cell at the meshing depth, as a cut or a sheet, axis-aligned or
                               diagonal through grid points: leaves with two to four vertex groups
  grid-plane faces             box faces and slab planes on dyadic grid planes: samples that are exactly 0
  boundary crossers            centres near or beyond the faces of [-1, 1]^3: sign changes on the domain boundary
  cone                         its axis on a grid line: d sqrt at 0 is 0/0, a NaN gradient on that edge (a forced vertex)
  empty / full                 no surface at all
"""
from __future__ import annotations

import numpy as np


def _f(v):
    return float(np.float32(v))


def random_shape(ctx, rng, depth):
    """(root node, kind) of a random shape for meshing at ``depth``."""
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    axes = (x, y, z)
    cell = 2.0 / 2 ** depth

    def grid(lo, hi):                     # a grid plane of the meshing depth in [lo, hi]
        k = rng.integers(int(np.ceil((lo + 1) / cell)), int(np.floor((hi + 1) / cell)) + 1)
        return _f(-1 + k * cell)

    def centre():
        r = rng.random()
        if r < 0.25:
            return [grid(-0.75, 0.75) for _ in range(3)]
        if r < 0.45:                      # near or beyond a face of the domain
            c = [_f(rng.uniform(-0.6, 0.6)) for _ in range(3)]
            a = rng.integers(0, 3)
            c[a] = _f(rng.choice([-1, 1]) * rng.uniform(0.85, 1.15))
            return c
        return [_f(rng.uniform(-0.7, 0.7)) for _ in range(3)]

    def rel(c):
        return [ctx.sub(a, v) for a, v in zip(axes, c)]

    def sphere():
        p = rel(centre())
        return ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(p[0]), ctx.square(p[1])), ctx.square(p[2]))),
                       _f(rng.uniform(0.1, 0.6)))

    def box():
        if rng.random() < 0.5:            # faces on grid planes
            b = []
            for a in axes:
                lo = grid(-0.9, 0.4)
                hi = grid(lo + cell, min(lo + 0.8, 1.0))
                b.append(ctx.max(ctx.sub(lo, a), ctx.sub(a, hi)))
        else:
            c, h = centre(), [_f(rng.uniform(0.05, 0.45)) for _ in range(3)]
            b = [ctx.sub(ctx.abs(p), hk) for p, hk in zip(rel(c), h)]
        return ctx.max(ctx.max(b[0], b[1]), b[2])

    def rounded_box():
        c, h, r = centre(), [_f(rng.uniform(0.05, 0.35)) for _ in range(3)], _f(rng.uniform(0.02, 0.2))
        q = [ctx.max(ctx.sub(ctx.abs(p), hk), 0.0) for p, hk in zip(rel(c), h)]
        return ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(q[0]), ctx.square(q[1])), ctx.square(q[2]))), r)

    def slab():
        w = _f(cell * rng.uniform(0.05, 0.3))
        a, b = rng.choice(3, size=2, replace=False)
        if rng.random() < 0.5:            # axis-aligned, at a grid plane or between two
            off = grid(-0.75, 0.75) if rng.random() < 0.5 else _f(rng.uniform(-0.75, 0.75))
            s = ctx.sub(axes[a], off)
        else:                             # diagonal through grid points: catches opposite corners of a face
            s = ctx.add(ctx.sub(axes[a], axes[b]), grid(-0.5, 0.5) + 1.0)
        return ctx.sub(ctx.abs(s), w)

    def cone():
        a = rng.integers(0, 3)
        u, v = axes[(a + 1) % 3], axes[(a + 2) % 3]
        cu, cv, tip = grid(-0.6, 0.6), grid(-0.6, 0.6), _f(rng.uniform(-0.3, 0.6))
        rad = ctx.sqrt(ctx.add(ctx.square(ctx.sub(u, cu)), ctx.square(ctx.sub(v, cv))))
        return ctx.add(rad, ctx.mul(ctx.sub(axes[a], tip), _f(rng.uniform(0.4, 1.5))))

    r = rng.random()
    if r < 0.04:
        return ctx.add(ctx.square(x), 0.5), "empty"
    if r < 0.08:
        return ctx.sub(ctx.square(x), 2.0), "full"
    prims = [sphere, box, rounded_box, slab, cone]
    n = int(rng.integers(1, 6))
    kinds = [int(rng.choice(5, p=[0.25, 0.2, 0.15, 0.25, 0.15])) for _ in range(n)]
    shape = prims[kinds[0]]()
    if kinds[0] == 3:                     # a slab alone is a sheet; make it a cut through something
        shape = ctx.max(box(), ctx.neg(shape))
    for k in kinds[1:]:
        p = prims[k]()
        op = rng.random()
        if op < 0.5 or k == 3 and op < 0.7:
            shape = ctx.min(shape, p)               # union
        elif op < 0.85:
            shape = ctx.max(shape, ctx.neg(p))      # difference
        else:
            shape = ctx.max(shape, p)               # intersection
    return shape, "+".join("sbrlc"[k] for k in kinds)


def tape_pair(orc, fb, seed, depth):
    """(device tape data, oracle tape, kind) of seed's shape; ``fb`` may be None on a machine without a GPU."""
    out = []
    for Ctx in ((fb.Context,) if fb else ()) + (orc.Context,):
        ctx = Ctx()
        root, kind = random_shape(ctx, np.random.default_rng(seed), depth)
        out.append(ctx.tape(root))
    dev = out[0] if fb else None
    return dev, orc.Tape.from_data(out[-1]), kind


FUZZ_SEEDS = range(48)        # tests/test_gpu_mesh_fuzz.py


def fuzz_depth(seed):
    """Meshing depth of a fuzz seed: mostly 2-5, where the oracle is fast, with one in six at 6 or 7."""
    return int(np.random.default_rng(10_000 + seed).choice([2, 3, 4, 4, 5, 5, 6, 5, 3, 4, 5, 7]))
