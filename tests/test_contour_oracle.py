"""The 2D contour oracle (tests/contour_oracle.py, which fc_contour_build matches bit for bit) on shapes with known
answers, its float32 QEF solve against a float64 solve, and fb.contours_svg.  CPU only."""
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import contour_oracle as co
import mesh_shapes
from conftest import model_text

CUTOFF = 1e-3
EPS32 = float(np.finfo(np.float32).eps)
# |p32 - p64| <= POS_C * eps32 * (|centre| + |p64 - centre| + 1) / (smallest kept |w| / largest |w|); the largest
# normalised deviation test_qef2_matches_float64 measured on its corpus is noted in DESIGN.md section 10
POS_C = 4.0


def _disc(orc, r, cx=0.0, cy=0.0):
    ctx = orc.Context()
    x, y = ctx.x(), ctx.y()
    return orc.Tape.from_data(ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.square(ctx.sub(x, cx)), ctx.square(ctx.sub(y, cy)))), r)))


def _box(ctx, x, y, x0, x1, y0, y1):
    return ctx.max(ctx.max(ctx.sub(x, x1), ctx.sub(x0, x)), ctx.max(ctx.sub(y, y1), ctx.sub(y0, y)))


def _area(v):
    p = np.asarray(v, dtype=np.float64)
    return 0.5 * np.sum(p[:, 0] * np.roll(p[:, 1], -1) - np.roll(p[:, 0], -1) * p[:, 1])


@pytest.mark.parametrize("depth", [6, 7, 8, 9, 10])
def test_disc_is_one_counter_clockwise_loop(orc, depth):
    r = 0.6
    c = co.contour(_disc(orc, r), depth)
    assert c.closed.tolist() == [True] and c.n_open == 0
    h = 2.0 / (1 << depth)
    # a vertex is where the tangents at two neighbouring intersections meet: outside the circle by about h^2 / (8 r)
    dev = np.abs(np.hypot(c.vertices[:, 0].astype(np.float64), c.vertices[:, 1]) - r)
    assert dev.max() < h * h / (4 * r) + 1e-6
    if depth == 10:
        assert dev.max() < 1e-5
    area = _area(c.vertices)
    assert area > 0                                            # counter-clockwise, y up
    assert abs(area - np.pi * r * r) < 2 * np.pi * r * h * h / (4 * r) + 1e-6


def test_square_keeps_its_corners(orc):
    ctx = orc.Context()
    x, y = ctx.x(), ctx.y()
    t = orc.Tape.from_data(ctx.tape(_box(ctx, x, y, -0.45, 0.45, -0.45, 0.45)))
    depth = 6
    c = co.contour(t, depth)
    assert c.closed.tolist() == [True] and _area(c.vertices) > 0
    h = 2.0 / (1 << depth)
    for corner in [(-0.45, -0.45), (0.45, -0.45), (0.45, 0.45), (-0.45, 0.45)]:
        d = np.hypot(c.vertices[:, 0] - corner[0], c.vertices[:, 1] - corner[1]).min()
        assert d < h / 1000, (corner, d)      # Hermite data: the corner itself, to the edge search's resolution
    # every other vertex lies on a side
    side = np.minimum(np.abs(np.abs(c.vertices[:, 0]) - 0.45), np.abs(np.abs(c.vertices[:, 1]) - 0.45))
    assert side.max() < h / 1000


def test_diagonal_touching_squares_give_two_loops(orc):
    ctx = orc.Context()
    x, y = ctx.x(), ctx.y()
    shape = ctx.min(_box(ctx, x, y, -0.5, 0.01, -0.5, 0.01), _box(ctx, x, y, 0.01, 0.5, 0.01, 0.5))
    c = co.contour(orc.Tape.from_data(ctx.tape(shape)), 6)
    assert c.closed.tolist() == [True, True]
    for k in range(2):
        assert _area(c.vertices[c.offsets[k]:c.offsets[k + 1]]) > 0
    # the cell holding the touching point has two vertices, one in each loop
    cell = [tuple(v[:2]) for v in c.cells]
    shared = {p for p in cell if cell.count(p) == 2}
    assert len(shared) == 1


def test_hole_winds_the_other_way(orc):
    ctx = orc.Context()
    x, y = ctx.x(), ctx.y()
    ring = ctx.max(ctx.sub(ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y))), 0.7),
                   ctx.sub(0.3, ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y)))))
    c = co.contour(orc.Tape.from_data(ctx.tape(ring)), 7)
    assert c.closed.tolist() == [True, True]
    areas = sorted(_area(c.vertices[c.offsets[k]:c.offsets[k + 1]]) for k in range(2))
    assert areas[0] < 0 < areas[1]


def solve2_f64(q):
    """QuadraticErrorSolver::solve in the plane, float64 (LAPACK's eigh) on the float32 accumulators:
    (vertex, eigenvalue ratios |w_k| / |w_0| sorted descending, rank)."""
    a = np.array([[q.ata[0], q.ata[1]], [q.ata[1], q.ata[2]]], dtype=np.float64)
    mp = np.array(q.mp, dtype=np.float64)
    center = mp[:2] / mp[2]
    b = np.array(q.atb, dtype=np.float64) - a @ center
    w, v = np.linalg.eigh(a)
    order = np.argsort(-np.abs(w), kind="stable")
    w, v = w[order], v[:, order]
    ratios = np.abs(w) / np.abs(w[0]) if w[0] != 0 else np.zeros(2)
    rank = next((k for k in range(2) if abs(w[k]) < abs(w[0]) * CUTOFF), 2)
    sol = np.zeros(2)
    for k in range(rank):
        sol += (v[:, k] @ b) / w[k] * v[:, k]
    return sol + center, ratios, rank, center


def _corpus(orc):
    for name, z in (("quarter", 0.0), ("hi", 0.0), ("bear", 0.0), ("gyroid-sphere", 0.0), ("tanglecube", 0.3)):
        yield name, orc.Tape.from_vm(model_text(name + ".vm")), 7, z
    for seed in range(12):
        _, t, kind = mesh_shapes.tape_pair(orc, None, seed, 6)
        yield f"csg{seed}:{kind}", t, 6, float(np.random.default_rng(20_000 + seed).uniform(-0.6, 0.6))


def test_qef2_matches_float64(orc):
    worst, n = 0.0, 0
    for name, t, depth, z in _corpus(orc):
        for q in co.contour(t, depth, z=z).qefs:
            p64, ratios, rank, center = solve2_f64(q)
            if rank == 0 or (np.abs(ratios[1:] / CUTOFF - 1.0) < 0.01).any():
                continue          # float32 rounding may decide the rank either way
            p32 = q.vertex().astype(np.float64)
            scale = EPS32 * (np.abs(center).max() + np.abs(p64 - center).max() + 1.0) / ratios[rank - 1]
            dev = np.abs(p32 - p64).max() / scale
            worst = max(worst, dev)
            n += 1
            assert dev < POS_C, (name, p32, p64, dev)
    assert n > 1000
    print(f"qef2: {n} solves, largest normalised deviation {worst:.2f}")


def test_svg_has_one_path_per_polyline(orc):
    import fidget_b200 as fb
    c = co.contour(orc.Tape.from_vm(model_text("hi.vm")), 7)
    svg = fb.contours_svg(c.vertices, c.offsets, c.closed)
    root = ET.fromstring(svg)
    paths = root.findall("{http://www.w3.org/2000/svg}path")
    assert len(paths) == len(c.closed) > 1
    for p, cl in zip(paths, c.closed):
        assert p.get("fill-rule") == "nonzero"
        assert p.get("d").endswith("Z") == bool(cl)
    # y is flipped for SVG's y-down frame
    first = paths[0].get("d").split()[0][1:].split(",")
    assert float(first[0]) == float(c.vertices[0, 0]) and float(first[1]) == -float(c.vertices[0, 1])
