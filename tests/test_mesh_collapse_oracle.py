"""Pins of the collapse oracle (tests/mesh_collapse_oracle.py: Octree::build with cell collapse + walk_dual) by the
reference's own tests (fidget-mesh/src/octree.rs:1143-1685, qef.rs:126-168), with their assertions.  CPU only."""
import numpy as np
import pytest

import mesh_collapse_oracle as mco
import mesh_shapes
from conftest import model_text
from oracle import mesh as om

f32 = np.float32


def _tape(orc, build):
    ctx = orc.Context()
    return orc.Tape.from_data(ctx.tape(build(ctx)))


def sphere(ctx, center, r):
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    sq = [ctx.square(ctx.sub(a, float(c))) for a, c in zip((x, y, z), center)]
    return ctx.sub(ctx.sqrt(ctx.add(ctx.add(sq[0], sq[1]), sq[2])), float(r))


def cube(ctx, bx, by, bz):
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    b = [ctx.max(ctx.sub(float(lo), a), ctx.sub(a, float(hi))) for a, (lo, hi) in zip((x, y, z), (bx, by, bz))]
    return ctx.max(ctx.max(b[0], b[1]), b[2])


def _build(orc, build, depth):
    t = _tape(orc, build)
    return mco.build(orc, t, depth, sign_at=lambda p: t.point_eval(np.array(p, dtype=f32))[0] < 0)


def test_qef_rank2():
    q = mco.Qef()
    q.add_intersection([-0.5, -0.75, -0.75], [0.24, 0.12, 0.0, 0.0])
    q.add_intersection([-0.75, -1.0, -0.6], [0.0, 0.0, 0.31, 0.0])
    q.add_intersection([-0.50, -1.0, -0.6], [0.0, 0.0, 0.31, 0.0])
    _, err = q.solve()
    assert err == f32(1e-6)


def test_qef_near_planar_solver():
    q = mco.Qef()
    q.add_intersection([-0.5, -0.25, 0.4999981], [-0.66666776, -0.33333388, 0.66666526, -1.2516975e-6])
    q.add_intersection([-0.5, -0.25, 0.50], [-0.6666667, -0.33333334, 0.6666667, 0.0])
    q.add_intersection([-0.5, -0.25, 0.50], [-0.6666667, -0.33333334, 0.6666667, 0.0])
    pos, err = q.solve()
    assert err == f32(1e-6)
    assert np.linalg.norm(pos - np.array([-0.5, -0.25, 0.5])) < 1e-3


def test_mesh_basic(orc):
    # depth 0: the sampler leaves nothing; the root is Empty and the mesh is empty
    o = _build(orc, lambda c: sphere(c, (0, 0, 0), 0.2), 0)
    assert o.root["kind"] == "E" and o.n_octree_verts() == 0
    v, t, _ = o.walk_dual()
    assert len(v) == 0 and len(t) == 0
    # depth 1: eight leaves with one vertex and three intersections each
    o = _build(orc, lambda c: sphere(c, (0, 0, 0), 0.2), 1)
    assert o.root["kind"] == "B"
    assert o.n_octree_verts() == 6 * 4 + 8
    for c in range(8):
        cell = o.cells[(1, c & 1, (c >> 1) & 1, (c >> 2) & 1)]
        assert cell["kind"] == "L" and bin(cell["mask"]).count("1") == 1 and len(cell["verts"]) == 4
    v, t, _ = o.walk_dual()
    assert len(v) > 1 and len(t) > 0


def test_collapsible(orc):
    o = _build(orc, lambda c: sphere(c, (0, 0, 0), 0.1), 1)
    kids = [(1, c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)]
    assert o.collapsible(kids) is None
    for depth in (1, 4):
        o = _build(orc, lambda c: sphere(c, (-1, -1, -1), 0.1), depth)
        assert o.root["kind"] == "L", depth
    o = _build(orc, lambda c: sphere(c, (-1, 0, 1), 0.1), 1)
    assert o.collapsible(kids) is None
    o = _build(orc, lambda c: c.min(sphere(c, (-1, -1, -1), 0.1), sphere(c, (1, 1, 1), 0.1)), 1)
    assert o.collapsible(kids) is None


def test_empty_collapse(orc):
    o = _build(orc, lambda c: sphere(c, (0.1, 0.1, 0.1), 0.05), 1)
    assert o.root["kind"] == "E"


def test_qef_merging():
    grad = np.array([1, 0, 0, 0], dtype=f32)
    pos = np.array([0, 0, 0], dtype=f32)
    hermites = []
    for _ in range(8):
        h = mco.Hermite()
        h.inter = [(pos, grad)] * 12
        hermites.append(h)
    for i in range(12):   # only one of the two sub-edges per edge holds an intersection
        t = 1 << (i // 4)
        u = mco.nxt(t)
        v = mco.nxt(u)
        start = (u if i & 1 else 0) | (v if i & 2 else 0)
        hermites[start | t].inter[i] = None
    merged = mco.Hermite.merge(hermites)
    for i in merged.inter:
        assert np.array_equal(i[0], pos) and np.array_equal(i[1], grad)
    for f in merged.face:
        assert f.mp[3] == 4.0
    assert merged.center.mp[3] == 6.0


def _edge_sum(v):
    return int(v[0] != 0) + int(v[1] != 0) + int(v[2] != 0)


def test_sphere_verts(orc):
    v, _, _ = _build(orc, lambda c: sphere(c, (0, 0, 0), 0.2), 1).walk_dual()
    edges = 0
    for p in v:
        s = _edge_sum(p)
        assert s in (1, 3)
        if s == 1:
            assert abs(np.linalg.norm(p) - 0.2) < 2.0 / 65535
            edges += 1
        else:
            assert np.linalg.norm(np.abs(p) - 0.2) < 2.0 / 65535
    assert edges == 6


def test_cube_verts(orc):
    bounds = ((-0.1, 0.6), (-0.2, 0.75), (-0.3, 0.4))
    v, _, _ = _build(orc, lambda c: cube(c, *bounds), 1).walk_dual()
    eps = 2.0 / 65535
    assert len(v)
    for p in v:
        s = _edge_sum(p)
        assert s in (1, 3)
        on = [abs(p[a] - b[0]) < eps or abs(p[a] - b[1]) < eps for a, b in enumerate(bounds)]
        if s == 1:
            assert any(on[a] and p[a] != 0 for a in range(3))
        else:
            assert all(on)


@pytest.mark.parametrize("mask", range(256))
def test_mesh_manifold(orc, mask):
    def build(ctx):
        shapes = [sphere(ctx, (0.5 * (j & 1), 0.5 * ((j >> 1) & 1), 0.5 * ((j >> 2) & 1)), 0.1)
                  for j in range(8) if (mask >> j) & 1]
        if not shapes:
            return None
        s = shapes.pop()
        for q in shapes:
            s = ctx.min(s, q)
        return s
    if mask == 0:
        return
    v, t, _ = _build(orc, build, 2).walk_dual()
    if mask != 255:
        assert len(v) and len(t)
    assert mco.check_for_vertex_dupes(v)
    assert mco.check_for_edge_matching(t)


def test_sphere_manifold(orc):
    v, t, _ = _build(orc, lambda c: sphere(c, (0, 0, 0), 0.85), 5).walk_dual()
    assert mco.check_for_vertex_dupes(v)
    assert mco.check_for_edge_matching(t)


def test_colonnade_manifold(orc):
    v, t, _ = mco.build(orc, orc.Tape.from_vm(model_text("colonnade.vm")), 5).walk_dual()
    assert mco.check_for_edge_matching(t)


def test_colonnade_bounds(orc):
    v, _, _ = mco.build(orc, orc.Tape.from_vm(model_text("colonnade.vm")), 8).walk_dual()
    assert len(v)
    assert (v[:, 0] < 1).all() and (v[:, 0] > -1).all() and (v[:, 1] < 1).all() and (v[:, 1] > -1).all()
    assert (v[:, 2] < 1).all() and (v[:, 2] > -0.5).all()


def test_bear_bounds(orc):
    v, _, _ = mco.build(orc, orc.Tape.from_vm(model_text("bear.vm")), 5).walk_dual()
    assert len(v)
    assert (v[:, :2] < 1).all() and (v[:, :2] > -0.75).all()
    assert (v[:, 2] < 0.75).all() and (v[:, 2] > -0.75).all()


def test_qef_near_planar(orc):
    v, _, _ = _build(orc, lambda c: sphere(c, (0, 0, 0), 0.75), 4).walk_dual()
    n = np.linalg.norm(v, axis=1)
    assert len(n) and (n > 0.7).all() and (n < 0.8).all()


def test_fuzz_reaches_the_edge_cases(orc):
    """The GPU mesh fuzz corpus (tests/test_gpu_mesh_fuzz.py) reaches what it is drawn for: leaves with several
    vertex groups, NaN gradients (forced vertices), sign changes on the domain boundary, and shapes without a surface."""
    multi = nan = boundary = empty = 0
    for seed in mesh_shapes.FUZZ_SEEDS:
        depth = mesh_shapes.fuzz_depth(seed)
        _, o, _ = mesh_shapes.tape_pair(orc, None, seed, depth)
        leaves, _ = orc.octree_sample(o, depth)
        empty += len(leaves) == 0
        for l in leaves:
            multi += om.corner_groups(int(l["mask"]))[1] > 1
            present = [e for e in range(12) if (int(l["present"]) >> e) & 1]
            nan += bool(np.isnan(l["grad"][present]).any())
            boundary += bool({int(l["ix"]), int(l["iy"]), int(l["iz"])} & {0, 2 ** depth - 1})
    assert multi >= 100 and nan >= 8 and boundary >= 100 and empty >= 3, (multi, nan, boundary, empty)


@pytest.mark.parametrize("seed,open_edges", [(5, 25), (43, 13)])
def test_open_edges_skip_segments_smaller_leaves_own(orc, seed, open_edges):
    """Regression: a sign-changing boundary edge of a coarse final leaf whose neighbour at its depth is a Branch
    reachable from the root belongs to the smaller leaves there, not to the coarse leaf.  The oracle used to take such
    a Branch for an Empty cell and counted the edge; the counts here are fc_mesh_build's on an H100."""
    depth = mesh_shapes.fuzz_depth(seed)
    _, tape, _ = mesh_shapes.tape_pair(orc, None, seed, depth)
    assert mco.build(orc, tape, depth).open_edges() == open_edges
