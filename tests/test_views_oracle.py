"""The CPU oracle under the catalogue of views (tests/views.py) against the float64 projective reference, so that what
the device is compared with is itself pinned for general matrices: rotated, sheared, mirrored, perspective (mild, and
strong enough that the homogeneous term changes sign or vanishes inside the volume), degenerate and non-finite.

  renders      heightmaps inside the float64 bracket, normals within views.NORMAL_TOLERANCE of the float64 gradient of
               f(T(p)) with respect to the voxel, 2D signs and shaded values within the band;
  transform    the oracle's transform_f32 against model_points64, exactly undivided where w == 0;
  octree       corner masks equal the float64 signs at the transformed cell corners;
  mesh         the mesh oracles return model-space vertices (Octree::build's last step, fidget-mesh/src/octree.rs:58-65).

The interval transform is not exposed by the oracle's C face; its soundness is covered through the renders: a tile
filled on an unsound interval puts depths outside the bracket, or flips the sign of a pixel."""
import ctypes as C

import numpy as np
import pytest

import mesh_collapse_oracle as mco
import views as V
from oracle import mesh as om

SIZE3, TILES3 = 48, (16, 8)
SIZE2, TILES2 = 64, (32, 8)
LOOSE = {"strong": 0.5, "degenerate": 1.0}    # share of columns / pixels that may carry a sample within the error band:
# next to a w = 0 plane the model points are far away and badly conditioned; a degenerate view may put every sample on
# one model point, which may lie on the surface (the signs outside the band are checked all the same)
FINITE3 = V.names3("affine", "persp", "strong", "degenerate")
FINITE2 = V.names2("affine", "persp", "strong", "degenerate")

_TAPES = {}


def _tape(orc, shape):
    if shape not in _TAPES:
        _TAPES[shape] = orc.Tape.from_data(V.SHAPES[shape].tape(orc.Context))
    return _TAPES[shape]


@pytest.mark.parametrize("shape", ["sphere", "box", "colonnade.vm", "bear.vm"])
@pytest.mark.parametrize("view", FINITE3)
def test_render3d_lies_in_the_float64_bracket(orc, view, shape):
    kind = V.VIEWS3[view][1]
    n = 64 if view == "persp_w0_plane" else SIZE3    # a power of two: w is then exactly 0 on the plane z = n / 2
    mat = orc.voxel_mat(n, n, n, V.view3(view))
    img, _ = orc.render3d(_tape(orc, shape), n, n, n, mat=mat, tile_sizes=TILES3, var_values=V.SHAPES[shape].var_values)
    vals, band = V.field64(shape, mat, n, n, n)
    # persp_w0_plane: the voxels either side of the w = 0 plane sit 32 times further out than the cube, where the
    # band is wide; most columns hold one, so only the bracket itself is asserted there
    tight = V.check_heightmap(img["depth"], vals, band, max_loose=1.0 if view == "persp_w0_plane" else LOOSE.get(kind, 0.05))
    if shape == "sphere" and view == "scale_1e-6":      # the camera inside the solid: saturated, normals [0, 0, 1]
        assert (img["depth"] == n).all() and (img["normal"] == np.float32([0, 0, 1])).all()
    if shape == "sphere" and view == "out_of_view":
        assert not img["depth"].any()
    # normals: not under zero_last_row (Transformable for Grad always divides, there by a zero w); under the other
    # strong views most of what shows is saturated, so no minimum number of checkable columns is asked for
    if kind in ("affine", "persp", "strong") and view != "zero_last_row" and V.SHAPES[shape].ieee:
        V.check_normals(img, shape, mat, tight, n, min_checked=0 if kind == "strong" else 20)


@pytest.mark.parametrize("shape", ["hi.vm", "colonnade.vm", "sphere"])
@pytest.mark.parametrize("view", FINITE2)
def test_render2d_agrees_with_float64(orc, view, shape):
    n = SIZE2
    mat = orc.pixel_mat(n, n, V.view2(view))
    for z, perfect in ((0.0, False), (0.25, True)):
        img, _ = orc.render2d(_tape(orc, shape), n, n, mat=mat, z=z, pixel_perfect=perfect, tile_sizes=TILES2)
        vals, band = V.field64(shape, mat, n, n, z=z)
        V.check_image2d(img, vals, band, max_loose=LOOSE.get(V.VIEWS2[view][1], 0.05))


@pytest.mark.parametrize("view", V.names3("nonfinite"))
def test_render3d_returns_under_a_non_finite_matrix(orc, view):
    """A NaN or an infinity in the matrix is an input a viewer can produce: the render returns, and a NaN model
    coordinate makes a voxel outside, so nothing the interval proofs filled may hold an inside depth there."""
    n = 64
    mat = orc.voxel_mat(n, n, n, V.view3(view))
    img, st = orc.render3d(_tape(orc, "sphere"), n, n, n, mat=mat, tile_sizes=(32, 8))
    vals, _ = V.field64("sphere", mat, n, n, n)
    with np.errstate(invalid="ignore"):
        inside = vals < 0
    top = np.where(inside.any(axis=0), n - np.argmax(inside[::-1], axis=0), 0)
    assert np.array_equal(np.minimum(img["depth"], n), top)


@pytest.mark.parametrize("view", V.names2("nonfinite"))
def test_render2d_returns_under_a_non_finite_matrix(orc, view):
    n = 64
    mat = orc.pixel_mat(n, n, V.view2(view))
    img, _ = orc.render2d(_tape(orc, "hi.vm"), n, n, mat=mat, tile_sizes=(32, 8))
    vals, _ = V.field64("hi.vm", mat, n, n)
    with np.errstate(invalid="ignore"):
        assert np.array_equal(orc.pixel_inside(img), vals < 0)


def test_zero_last_row_renders_like_a_unit_last_row(orc):
    """transform_point divides only by a non-zero w, so a last row of zeros shows the depths and distances (0, 0, 0, 1)
    shows, bit for bit; the interval transform divides by [0, 0], so no tile of it can be proven either way (and the
    gradient transform by 0, so the normals are not finite)."""
    n = 64
    t = _tape(orc, "colonnade.vm")
    zero = V.view3("zero_last_row")
    a, sa = orc.render3d(t, n, n, n, mat=orc.voxel_mat(n, n, n, zero), tile_sizes=(32, 8))
    b, sb = orc.render3d(t, n, n, n, mat=orc.voxel_mat(n, n, n, V.with_unit_last_row(zero)), tile_sizes=(32, 8))
    assert np.array_equal(a["depth"], b["depth"]) and a["depth"].any()
    assert not any(sa["filled_inside"]) and not any(sa["filled_outside"])
    assert any(sb["filled_outside"])
    t = _tape(orc, "hi.vm")
    zero = V.view2("zero_last_row")
    a, sa = orc.render2d(t, n, n, mat=orc.pixel_mat(n, n, zero), tile_sizes=(32, 8))
    b, sb = orc.render2d(t, n, n, mat=orc.pixel_mat(n, n, V.with_unit_last_row(zero)), tile_sizes=(32, 8))
    assert not any(sa["filled_inside"]) and not any(sa["filled_outside"]) and not V.is_fill(a).any()
    assert np.array_equal(orc.pixel_inside(a), orc.pixel_inside(b))
    shaded = ~V.is_fill(b)
    assert np.array_equal(a.view(np.uint32)[shaded], b.view(np.uint32)[shaded]) and V.is_fill(b).any()


def _transform_f32(orc, mat, pts):
    m = np.ascontiguousarray(mat, dtype=np.float32).reshape(16)
    fp = C.POINTER(C.c_float)
    out = np.zeros((len(pts), 3), dtype=np.float32)
    tmp = np.zeros(3, dtype=np.float32)
    for i, (x, y, z) in enumerate(pts):
        orc.lib().orc_transform_f32(m.ctypes.data_as(fp), float(x), float(y), float(z), tmp.ctypes.data_as(fp))
        out[i] = tmp
    return out


@pytest.mark.parametrize("view", FINITE3)
def test_transform_f32_agrees_with_float64(orc, view):
    """Within the first-order rounding bound of the largest term (views.transform_error64: 4 u of the terms' magnitudes
    through the quotient), and exactly the undivided rows where w == 0."""
    n = 64
    mat = orc.voxel_mat(n, n, n, V.view3(view))
    rng = np.random.default_rng(3)
    pts = rng.integers(0, n, (2000, 3)).astype(np.float64)
    pts[:200, 2] = n // 2                                # the plane on which persp_w0_plane has w == 0
    got = _transform_f32(orc, mat, pts).astype(np.float64)
    want = V.model_points64(mat, *pts.T)
    err = V.transform_error64(mat, *pts.T)
    with np.errstate(invalid="ignore"):
        assert (np.abs(got - want) <= err + 1e-45).all(), np.argwhere(~(np.abs(got - want) <= err + 1e-45))[0]
    m64 = np.asarray(mat, dtype=np.float64)
    w = pts @ m64[3, :3] + m64[3, 3]
    if view in ("persp_w0_plane", "zero_last_row"):
        assert (w == 0).sum() >= 200
    rows = (pts @ m64[:3, :3].T + m64[:3, 3]).astype(np.float32)   # exact in f64, rounded once: within 4 u of f32's sum
    assert np.allclose(got[w == 0], rows[w == 0], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("shape", ["sphere", "colonnade.vm"])
@pytest.mark.parametrize("view", V.names3("affine", "persp"))
def test_octree_corner_masks_equal_float64_signs(orc, view, shape):
    """OctreeBuilder::leaf under world_to_model (octree.rs:590-640): a depth-D cell is a surface leaf iff the field seen
    through the view changes sign over its 8 corners; bit i of the mask is corner i inside.  Cells with a corner within
    the float32 error band of the surface may go either way."""
    depth = 4
    wm = V.view3(view)
    leaves, _ = orc.octree_sample(_tape(orc, shape), depth, wm)
    n = 1 << depth
    g = np.arange(n + 1) * (2.0 / n) - 1.0
    zz, yy, xx = np.meshgrid(g, g, g, indexing="ij")
    pts = V.model_points64(wm, xx.ravel(), yy.ravel(), zz.ravel())
    vals, err = V.eval64(shape, pts)
    terr = np.linalg.norm(V.transform_error64(wm, xx.ravel(), yy.ravel(), zz.ravel()), axis=-1)
    vals = vals.reshape(n + 1, n + 1, n + 1)
    band = (err + V.slope64(vals, pts.reshape(n + 1, n + 1, n + 1, 3)) * terr).reshape(vals.shape)
    inside, sure = vals < 0, np.abs(vals) > band
    mask = np.zeros((n, n, n), dtype=np.uint16)
    known = np.ones((n, n, n), dtype=bool)
    for i in range(8):
        dx, dy, dz = i & 1, (i >> 1) & 1, (i >> 2) & 1
        mask |= inside[dz:dz + n, dy:dy + n, dx:dx + n].astype(np.uint16) << i
        known &= sure[dz:dz + n, dy:dy + n, dx:dx + n]
    got = {(int(l["ix"]), int(l["iy"]), int(l["iz"])): int(l["mask"]) for l in leaves}
    checked = 0
    for z, y, x in zip(*np.nonzero(known)):
        m = int(mask[z, y, x])
        assert got.get((int(x), int(y), int(z)), m if m in (0, 255) else None) == m, (view, x, y, z)
        checked += m not in (0, 255)
    assert checked > 30 and known.mean() > 0.8       # colonnade's flat faces pass through cell corners


def _mesh_view():
    """translate . scale . rotate: the sphere's centre lands off the origin of the world cube, at another size"""
    m = V._translate(0.1, -0.05, 0.15) @ V._diag(0.8, 0.8, 0.8) @ V._rot((1, 2, 3), 50)
    return m.astype(np.float32)


@pytest.mark.parametrize("collapse", [False, True])
def test_mesh_oracles_return_model_space_vertices(orc, collapse):
    """Octree::build samples the field seen through world_to_model and maps the vertices back through it: a sphere of
    radius 0.6 meshed through any similarity view has its vertices at radius 0.6 in model space, within a fraction of
    a (model-space) cell, and nowhere near that in the world cube the octree was built in."""
    depth, wm = 5, _mesh_view()
    leaves, _ = orc.octree_sample(_tape(orc, "sphere"), depth, wm)
    if collapse:
        octree = mco.Octree(leaves, depth)
        verts, tris, _ = octree.walk_dual(wm)
        world, _, _ = octree.walk_dual()
    else:
        verts, tris, _, _ = om.build_indexed(leaves, world_to_model=wm)
        world, _, _, _ = om.build_indexed(leaves)
    assert len(tris) > 500 and len(verts) == len(world)
    cell = 0.8 * 2.0 / (1 << depth)
    r = np.linalg.norm(verts.astype(np.float64), axis=1)
    assert np.abs(r - 0.6).max() < 0.25 * cell, np.abs(r - 0.6).max()
    assert np.abs(np.linalg.norm(world.astype(np.float64), axis=1) - 0.6).max() > 2 * cell
    # f32 transform_point, nalgebra's order, against float64
    want = V.model_points64(wm, *world.astype(np.float64).T)
    assert np.abs(verts - want).max() < 1e-6
    assert np.array_equal(om.to_model(world, np.eye(4, dtype=np.float32)), world)    # the identity is left alone


def test_to_model_divides_only_by_a_non_zero_w():
    m = V.view3("persp_w0_plane")
    p = np.array([[0.25, -0.5, 0.0], [0.25, -0.5, 0.5], [0.3, 0.1, -0.25]], dtype=np.float32)
    got = om.to_model(p, m)
    assert np.array_equal(got[0], p[0])                                  # w == 0: undivided
    assert np.array_equal(got[1], (p[1] / np.float32(0.5)).astype(np.float32))
    assert np.array_equal(got[2], (p[2] / np.float32(-0.25)).astype(np.float32))
