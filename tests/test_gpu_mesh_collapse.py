"""fc_mesh_build with FC_FLAG_MESH_COLLAPSE (cell collapse + the adaptive dual walk on the device) against the numpy
restatement of Octree::build / walk_dual (tests/mesh_collapse_oracle.py) on the oracle's sampler output, and the
reference's own mesh properties (fidget-mesh/src/octree.rs tests) run through ``fb.mesh(..., collapse=True)``."""
import numpy as np
import pytest

import fidget_b200 as fb
import mesh_collapse_oracle as mco
import mesh_compare
from conftest import model_text

pytestmark = pytest.mark.gpu


def _sphere(ctx, center, r):
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    sq = [ctx.square(ctx.sub(a, float(c))) for a, c in zip((x, y, z), center)]
    return ctx.sub(ctx.sqrt(ctx.add(ctx.add(sq[0], sq[1]), sq[2])), float(r))


def _cube(ctx, bx, by, bz):
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    b = [ctx.max(ctx.sub(float(lo), a), ctx.sub(a, float(hi))) for a, (lo, hi) in zip((x, y, z), (bx, by, bz))]
    return ctx.max(ctx.max(b[0], b[1]), b[2])


def _pair(orc, cuda, build):
    """(device shape, oracle tape) of the expression build(ctx)"""
    gc, oc = fb.Context(), orc.Context()
    return fb.CudaShape(cuda, gc.tape(build(gc))), orc.Tape.from_data(oc.tape(build(oc)))


def _compare_exact(cuda, g, o_tape, orc, depth):
    """final leaves, cell vertices (bit for bit), vertices, triangles and open_edges against the oracle, and every final
    leaf's vertex against the float64 QEF solve (tests/mesh_compare.py)"""
    leaves, _ = orc.octree_sample(o_tape, depth)
    verts, tris, info, octree, _ = mesh_compare.compare_collapse(cuda, g, leaves, depth)
    return verts, tris, info, octree


@pytest.mark.parametrize("r", [0.2, 0.6, 0.85])
@pytest.mark.parametrize("depth", [1, 2, 3, 4, 5])
def test_sphere_matches_oracle(orc, cuda, r, depth):
    g, o = _pair(orc, cuda, lambda c: _sphere(c, (0, 0, 0), r))
    _compare_exact(cuda, g, o, orc, depth)


@pytest.mark.parametrize("depth", [1, 3, 4])
def test_off_centre_cube_matches_oracle(orc, cuda, depth):
    """test_cube_verts' cube (octree.rs:1235-1276)"""
    g, o = _pair(orc, cuda, lambda c: _cube(c, (-0.1, 0.6), (-0.2, 0.75), (-0.3, 0.4)))
    verts, tris, info, _ = _compare_exact(cuda, g, o, orc, depth)
    if depth == 1:
        eps = 2.0 / 65535
        for v in verts:
            nz = (v != 0).sum()
            assert nz in (1, 3)
            on = [np.isclose(v[a], b, atol=eps).any() for a, b in enumerate(((-0.1, 0.6), (-0.2, 0.75), (-0.3, 0.4)))]
            assert any(on) if nz == 1 else all(on)


@pytest.mark.parametrize("depth", [1, 4])
def test_corner_sphere_collapses_to_the_root(orc, cuda, depth):
    """test_collapsible (octree.rs:1400-1453): a sphere at a corner of the domain leaves a single leaf"""
    g, o = _pair(orc, cuda, lambda c: _sphere(c, (-1, -1, -1), 0.1))
    _compare_exact(cuda, g, o, orc, depth)
    cells = fb.mesh_cells(cuda)
    assert len(cells) == 1 and cells["depth"][0] == 0


def _check_manifold(verts, tris, info):
    assert mco.check_for_vertex_dupes(verts)
    assert mco.check_for_edge_matching(tris)
    assert info["open_edges"] == 0


def test_mesh_manifold_all_masks(cuda):
    """test_mesh_manifold_single_thread (octree.rs:1345-1391): 0-8 spheres at the corners of [0, 0.5]^3, depth 2"""
    for mask in range(1, 256):
        def build(ctx):
            shapes = [_sphere(ctx, (0.5 * (j & 1), 0.5 * ((j >> 1) & 1), 0.5 * ((j >> 2) & 1)), 0.1)
                      for j in range(8) if (mask >> j) & 1]
            s = shapes.pop()
            for q in shapes:
                s = ctx.min(s, q)
            return s
        ctx = fb.Context()
        verts, tris, info = fb.mesh(fb.CudaShape(cuda, ctx.tape(build(ctx))), 2, collapse=True)
        assert len(verts) and len(tris), mask
        assert mco.check_for_vertex_dupes(verts), mask
        assert mco.check_for_edge_matching(tris), mask


def test_sphere_manifold(cuda):
    ctx = fb.Context()
    _check_manifold(*fb.mesh(fb.CudaShape(cuda, ctx.tape(_sphere(ctx, (0, 0, 0), 0.85))), 5, collapse=True))


def test_colonnade_manifold(cuda):
    """test_colonnade_manifold (octree.rs:1476-1499): edges pair up (the model has duplicate vertices)"""
    verts, tris, info = fb.mesh(fb.CudaShape.from_vm(cuda, model_text("colonnade.vm")), 5, collapse=True)
    assert len(tris) and mco.check_for_edge_matching(tris)


def test_colonnade_bounds(cuda):
    verts, tris, info = fb.mesh(fb.CudaShape.from_vm(cuda, model_text("colonnade.vm")), 8, collapse=True)
    assert len(verts)
    assert (verts[:, 0] < 1).all() and (verts[:, 0] > -1).all() and (verts[:, 1] < 1).all() and (verts[:, 1] > -1).all()
    assert (verts[:, 2] < 1).all() and (verts[:, 2] > -0.5).all()


def test_bear_bounds(cuda):
    verts, tris, info = fb.mesh(fb.CudaShape.from_vm(cuda, model_text("bear.vm")), 5, collapse=True)
    assert len(verts)
    assert (verts[:, :2] < 1).all() and (verts[:, :2] > -0.75).all()
    assert (verts[:, 2] < 0.75).all() and (verts[:, 2] > -0.75).all()


def test_qef_near_planar(cuda):
    ctx = fb.Context()
    verts, _, _ = fb.mesh(fb.CudaShape(cuda, ctx.tape(_sphere(ctx, (0, 0, 0), 0.75))), 4, collapse=True)
    n = np.linalg.norm(verts, axis=1)
    assert len(n) and (n > 0.7).all() and (n < 0.8).all()


def test_mesh_vars(cuda):
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    v, _ = ctx.var()
    g = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), v)))
    for r in (0.5, 0.75):
        verts, _, _ = fb.mesh(g, 4, var_values=(r,), collapse=True)
        n = np.linalg.norm(verts, axis=1)
        assert len(n) and (n > r - 0.05).all() and (n < r + 0.05).all()


@pytest.mark.parametrize("name,depth", [("colonnade.vm", 6), ("bear.vm", 6), ("gyroid-sphere.vm", 6), ("colonnade.vm", 7)])
def test_model_leaves_match_oracle(orc, cuda, name, depth):
    """On the device sampler's own leaves the oracle's collapse and walk must give the device's mesh exactly: final
    leaves, cell vertices, vertices, triangles and open_edges.  The models' gradients (bear's, say) are not bit for bit
    the oracle sampler's, and a last-bit change of the Hermite data flips collapse decisions that sit at the 2x error
    threshold, so the agreement with the all-oracle pipeline is only printed."""
    text = model_text(name)
    g = fb.CudaShape.from_vm(cuda, text)
    verts, tris, info, octree, rep = mesh_compare.compare_collapse(cuda, g, fb.octree_sample(g, depth), depth)
    dev = {tuple(int(v) for v in c) for c in octree.final_leaves()}
    full = {tuple(int(v) for v in c) for c in mco.build(orc, orc.Tape.from_vm(text), depth).final_leaves()}
    print(f"{name} depth {depth}: {len(dev)} final leaves, {info['n_triangles']} triangles; {rep}; "
          f"{len(dev & full)} of {len(full)} leaves of the oracle's own sampler match")
    assert mco.check_for_edge_matching(tris) or info["open_edges"] > 0


def test_collapse_reduces_triangles(orc, cuda):
    g, o = _pair(orc, cuda, lambda c: _sphere(c, (0, 0, 0), 0.85))
    _, uni, _ = fb.mesh(g, 6)
    verts, tris, info = fb.mesh(g, 6, collapse=True)
    _, o_tris, _ = mco.build(orc, o, 6).walk_dual()
    assert len(tris) < len(uni)
    assert abs(len(tris) - len(o_tris)) <= 0.01 * len(o_tris)
    _check_manifold(verts, tris, info)


def test_collapsed_mesh_stl(cuda):
    ctx = fb.Context()
    verts, tris, info, stl = fb.mesh(fb.CudaShape(cuda, ctx.tape(_sphere(ctx, (0, 0, 0), 0.6))), 5, stl=True, collapse=True)
    assert len(stl) == 84 + 50 * len(tris) and int.from_bytes(stl[80:84], "little") == len(tris)
    rec = np.frombuffer(stl, dtype=np.uint8, offset=84).reshape(-1, 50)
    body = np.ascontiguousarray(rec[:, :48]).view(np.float32).reshape(-1, 4, 3)
    assert np.array_equal(body[:, 1:], verts[tris.astype(np.int64)])
    a, b, c = body[:, 1], body[:, 2], body[:, 3]
    assert np.allclose(body[:, 0], np.cross(b - a, c - a), atol=1e-6)
    assert not rec[:, 48:].any()


def test_uniform_build_lists_no_cells(cuda):
    ctx = fb.Context()
    fb.mesh(fb.CudaShape(cuda, ctx.tape(_sphere(ctx, (0, 0, 0), 0.6))), 3)
    assert len(fb.mesh_cells(cuda)) == 0
