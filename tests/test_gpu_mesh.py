"""fc_mesh_build (QEF vertices + dual walk + STL on the device) against the numpy oracle of the same steps
(oracle/mesh.py) on the oracle's sampler output, plus the reference's own mesh properties
(fidget-mesh/src/octree.rs test_sphere_manifold, test_cube_verts, test_colonnade_manifold)."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import fidget_b200 as fb
import mesh_compare
from conftest import model_text
from oracle import mesh as om

pytestmark = pytest.mark.gpu


def _sphere(Ctx, r=0.6):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    return ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), r))


def _cube(Ctx, h=0.4):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    return ctx.tape(ctx.max(ctx.max(ctx.sub(ctx.abs(x), h), ctx.sub(ctx.abs(y), h)), ctx.sub(ctx.abs(z), h)))


def _canon(tris):
    """rotation-normalised index triples (orientation preserved) as a sorted array"""
    t = np.asarray(tris, dtype=np.int64)
    k = np.argmin(t, axis=1)
    rolled = np.stack([np.roll(row, -s) for row, s in zip(t, k)]) if len(t) else t
    return rolled[np.lexsort((rolled[:, 2], rolled[:, 1], rolled[:, 0]))]


def _manifold(tris):
    e = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]).astype(np.int64)
    keys = e[:, 0] * (1 << 32) + e[:, 1]
    rev = e[:, 1] * (1 << 32) + e[:, 0]
    return len(np.unique(keys)) == len(keys) and np.array_equal(np.sort(keys), np.sort(rev))


@pytest.mark.parametrize("shape_fn,depth", [(_sphere, 4), (_sphere, 5), (_cube, 4)])
def test_mesh_matches_numpy_oracle(orc, cuda, shape_fn, depth):
    g = fb.CudaShape(cuda, shape_fn(fb.Context))
    o = orc.Tape.from_data(shape_fn(orc.Context))
    verts, tris, info, stl = fb.mesh(g, depth, stl=True)
    leaves, _ = orc.octree_sample(o, depth)
    o_verts, o_tris, o_open = om.build(leaves)
    assert info["n_leaves"] == len(leaves) and info["open_edges"] == o_open == 0
    assert len(tris) == len(o_tris) and len(tris) % 4 == 0
    # oracle vertices (cell vertices + the intersection vertices its triangles use), matched by position
    pos = {}
    o_idx = []
    for tri in o_tris:
        o_idx.append([pos.setdefault(p.tobytes(), len(pos)) for p in tri])
    o_pos = np.array([np.frombuffer(k, dtype=np.float32) for k in pos])
    assert len(o_pos) == len(verts)
    cell = 2.0 / 2 ** depth
    d, nn = cKDTree(o_pos).query(verts)
    assert d.max() < 2e-3 * cell, d.max()            # Jacobi in f32 (device) vs SVD in f64 (numpy): not bit for bit
    assert len(np.unique(nn)) == len(verts)
    assert np.array_equal(_canon(nn[tris.astype(np.int64)]), _canon(o_idx))
    assert _manifold(tris)
    # STL: framing, and every record is (normal, a, b, c) of the indexed mesh
    assert len(stl) == 84 + 50 * len(tris) and int.from_bytes(stl[80:84], "little") == len(tris)
    rec = np.frombuffer(stl, dtype=np.uint8, offset=84).reshape(-1, 50)
    body = np.ascontiguousarray(rec[:, :48]).view(np.float32).reshape(-1, 4, 3)
    assert np.array_equal(body[:, 1:], verts[tris.astype(np.int64)])
    a, b, c = body[:, 1], body[:, 2], body[:, 3]
    assert np.allclose(body[:, 0], np.cross(b - a, c - a), atol=1e-6)
    assert not rec[:, 48:].any()
    # exactly the oracle's walk with the device's float32 solve, and every cell vertex within the float64 bound
    print(mesh_compare.compare_uniform(g, leaves, depth))


@pytest.mark.parametrize("name,depth", [("colonnade.vm", 6), ("bear.vm", 6), ("gyroid-sphere.vm", 6), ("colonnade.vm", 7)])
def test_model_mesh_matches_oracle(cuda, name, depth):
    """On the device sampler's leaves: vertices, triangles and open_edges exactly as oracle/mesh.py's walk with the
    device's float32 vertex solve, and every cell vertex within the float64 bound of its QEF's solution."""
    g = fb.CudaShape.from_vm(cuda, model_text(name))
    print(f"{name} depth {depth}: {mesh_compare.compare_uniform(g, fb.octree_sample(g, depth), depth)}")


def test_cube_mesh_has_sharp_corners(cuda):
    """test_cube_verts (octree.rs:1235-1276): the QEF puts vertices on the cube's corners and edges."""
    verts, tris, info = fb.mesh(fb.CudaShape(cuda, _cube(fb.Context, 0.4)), 4)
    a = np.abs(verts)
    assert np.all(a.max(axis=1) <= 0.4 + 1e-3)
    on_face = np.isclose(a, 0.4, atol=2e-3).sum(axis=1)
    assert (on_face == 3).sum() == 8                    # the eight corners, exactly once each
    assert (on_face >= 2).sum() > 8                     # edges carry vertices too
    assert _manifold(tris)


@pytest.mark.parametrize("name,depth", [("colonnade.vm", 6), ("gyroid-sphere.vm", 6), ("bear.vm", 6)])
def test_model_meshes_are_manifold_where_closed(cuda, name, depth):
    """test_colonnade_manifold (octree.rs:1476-1499) in spirit: away from the [-1,1]^3 boundary every directed edge
    has its opposite; triangles never repeat; the signed volume is positive (outward orientation)."""
    g = fb.CudaShape.from_vm(cuda, model_text(name))
    verts, tris, info = fb.mesh(g, depth)
    assert info["n_triangles"] == len(tris) > 1000 and info["n_vertices"] == len(verts)
    assert tris.max() < len(verts)
    e = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]).astype(np.int64)
    keys, rev = e[:, 0] * (1 << 32) + e[:, 1], e[:, 1] * (1 << 32) + e[:, 0]
    assert len(np.unique(keys)) == len(keys)
    unmatched = ~np.isin(keys, rev)
    # unmatched edges may only occur next to boundary cells (fc_mesh_info.open_edges of them)
    assert unmatched.sum() <= 8 * info["open_edges"] + 0
    v = verts.astype(np.float64)
    vol = np.einsum("ij,ij->i", v[tris[:, 0]], np.cross(v[tris[:, 1]], v[tris[:, 2]])).sum() / 6
    assert vol > 0
    assert info["mesh_ms"] > 0 and info["sampler_ms"] > 0
