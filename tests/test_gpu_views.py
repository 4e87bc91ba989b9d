"""The renderers, the frame and scene batches, the octree sampler and the mesher under the catalogue of views
(tests/views.py): rotated, sheared, mirrored, perspective -- mild, and strong enough that the homogeneous term changes
sign or vanishes inside the volume -- degenerate and non-finite.  Every result is compared with the CPU oracle (which
tests/test_views_oracle.py pins against float64 for the same views), bit for bit on IEEE models; renders are also held
directly against the float64 projective reference, so that an error the oracle and the kernels share still shows."""
import numpy as np
import pytest

import fidget_b200 as fb
import mesh_compare
import views as V
from conftest import same_f32
from scene_merge import fold

pytestmark = pytest.mark.gpu

CENSUS = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")
ALL3, ALL2 = V.names3(), V.names2()
_PAIRS, _ORC3 = {}, {}


def _pair(orc, cuda, shape):
    """(oracle tape, device shape) of views.SHAPES[shape], built once"""
    if shape not in _PAIRS:
        s = V.SHAPES[shape]
        _PAIRS[shape] = (orc.Tape.from_data(s.tape(orc.Context)), fb.CudaShape(cuda, s.tape(fb.Context)))
    return _PAIRS[shape]


def _size3(view, n):
    return 64 if V.VIEWS3[view][1] == "nonfinite" else n


def _oracle3(orc, cuda, shape, view, w, h, d, tiles=(128, 64, 32, 16, 8)):
    key = (shape, view, w, h, d, tiles)
    if key not in _ORC3:
        mat = orc.voxel_mat(w, h, d, V.view3(view))
        _ORC3[key] = orc.render3d(_pair(orc, cuda, shape)[0], w, h, d, mat=mat, tile_sizes=tiles, threads=8,
                                  var_values=V.SHAPES[shape].var_values)
    return _ORC3[key]


def _same3(got, want, where):
    bad = got["depth"] != want["depth"]
    if bad.any():
        y, x = np.argwhere(bad)[0]
        raise AssertionError(f"{where}: {int(bad.sum())} depths differ; first at x={x} y={y}: {got['depth'][y, x]} vs "
                             f"{want['depth'][y, x]}")
    assert same_f32(got["normal"], want["normal"]), f"{where}: normals differ"


def _same_census(got, want, where):
    for k in CENSUS:
        assert got[k] == want[k], (where, k, got[k], want[k])
    assert got["pixels"] == want["pixels"], where


# ---- fc_render3d -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["colonnade.vm", "tanglecube.vm", "sphere_var"])
@pytest.mark.parametrize("view", ALL3)
def test_render3d_equals_the_oracle(orc, cuda, view, shape):
    """Device ladder, the reference's full ladder and the exact census, bit for bit; the device ladder's shortcut (a
    sub-region never contradicts its parent's choices) must hold when a tile's interval is NaN, as it is wherever w
    touches zero."""
    n = _size3(view, 128)
    _, g = _pair(orc, cuda, shape)
    want, want_st = _oracle3(orc, cuda, shape, view, n, n, n)
    kw = dict(world_to_model=V.view3(view), var_values=V.SHAPES[shape].var_values)
    _same3(fb.render3d(g, fb.RenderConfig3D(n, n, n, **kw)), want, "device ladder")
    _same3(fb.render3d(g, fb.RenderConfig3D(n, n, n, full_ladder=True, **kw)), want, "full ladder")
    if n == 128:
        got, st = fb.render3d(g, fb.RenderConfig3D(n, n, n, exact_census=True, **kw), stats=True)
        _same3(got, want, "exact census")
        _same_census(st, want_st, view)


@pytest.mark.parametrize("view", V.names3("affine", "persp", "strong"))
def test_render3d_ragged_volume_and_custom_tiles(orc, cuda, view):
    _, g = _pair(orc, cuda, "colonnade.vm")
    w, h, d = 200, 136, 72
    want, _ = _oracle3(orc, cuda, "colonnade.vm", view, w, h, d)
    _same3(fb.render3d(g, fb.RenderConfig3D(w, h, d, world_to_model=V.view3(view))), want, "ragged")
    want, _ = _oracle3(orc, cuda, "colonnade.vm", view, 128, 128, 128, tiles=(64, 16, 4))
    _same3(fb.render3d(g, fb.RenderConfig3D(128, 128, 128, world_to_model=V.view3(view), tile_sizes=(64, 16, 4))), want,
           "custom tiles")


def test_render3d_prospero_under_the_bench_camera(orc, cuda):
    n = 256
    o, g = _pair(orc, cuda, "prospero.vm")
    want, _ = orc.render3d(o, n, n, n, mat=orc.voxel_mat(n, n, n, V.view3("bench_camera")), threads=8)
    _same3(fb.render3d(g, fb.RenderConfig3D(n, n, n, world_to_model=V.view3("bench_camera"))), want, "prospero")


def test_render3d_bear_within_libm_tolerance(orc, cuda):
    """bear.vm uses exp / ln / sin / cos, where libdevice and glibc differ by ulps: the tolerances of
    test_gpu_parity.test_render3d_bear_within_tolerance, under the benchmark camera."""
    n = 128
    _, g = _pair(orc, cuda, "bear.vm")
    want, _ = _oracle3(orc, cuda, "bear.vm", "bench_camera", n, n, n)
    got = fb.render3d(g, fb.RenderConfig3D(n, n, n, world_to_model=V.view3("bench_camera")))
    same = got["depth"] == want["depth"]
    assert same.mean() > 0.9995, f"{(~same).sum()} depth mismatches"
    n_ok = np.isclose(got["normal"], want["normal"], rtol=1e-4, atol=1e-4, equal_nan=True).all(axis=-1)
    assert (n_ok | ~same).mean() > 0.999


def test_zero_last_row_renders_like_a_unit_last_row(orc, cuda):
    """f32 skips the division by a zero w, the interval path divides by [0, 0]: the same depths and distances as with
    the last row (0, .., 0, 1), and no tile filled at any level."""
    n = 128
    _, g = _pair(orc, cuda, "colonnade.vm")
    zero = V.view3("zero_last_row")
    a, sa = fb.render3d(g, fb.RenderConfig3D(n, n, n, world_to_model=zero, full_ladder=True), stats=True)
    b, sb = fb.render3d(g, fb.RenderConfig3D(n, n, n, world_to_model=V.with_unit_last_row(zero), full_ladder=True), stats=True)
    assert np.array_equal(a["depth"], b["depth"]) and a["depth"].any()
    assert not any(sa["filled_inside"]) and not any(sa["filled_outside"]) and any(sb["filled_outside"])
    _, g = _pair(orc, cuda, "hi.vm")
    zero = V.view2("zero_last_row")
    a, sa = fb.render2d(g, fb.RenderConfig2D(n, n, world_to_model=zero), stats=True)
    b, sb = fb.render2d(g, fb.RenderConfig2D(n, n, world_to_model=V.with_unit_last_row(zero)), stats=True)
    assert not any(sa["filled_inside"]) and not any(sa["filled_outside"]) and not V.is_fill(a).any()
    assert np.array_equal(fb.pixel_inside(a), fb.pixel_inside(b)) and V.is_fill(b).any()
    shaded = ~V.is_fill(b)
    assert np.array_equal(a.view(np.uint32)[shaded], b.view(np.uint32)[shaded])


def test_degenerate_views_show_nothing_or_everything(orc, cuda):
    n = 128
    _, g = _pair(orc, cuda, "sphere")
    img, st = fb.render3d(g, fb.RenderConfig3D(n, n, n, world_to_model=V.view3("out_of_view")), stats=True)
    assert not img["depth"].any() and st["filled_outside"][0] == st["evaluated"][0] > 0
    img = fb.render3d(g, fb.RenderConfig3D(n, n, n, world_to_model=V.view3("scale_1e-6")))
    assert (img["depth"] == n).all() and (img["normal"] == np.float32([0, 0, 1])).all()


# ---- fc_render2d -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["hi.vm", "colonnade.vm"])
@pytest.mark.parametrize("view", ALL2)
def test_render2d_equals_the_oracle(orc, cuda, view, shape):
    n = 64 if V.VIEWS2[view][1] == "nonfinite" else 256
    o, g = _pair(orc, cuda, shape)
    wm = V.view2(view)
    mat = orc.pixel_mat(n, n, wm)
    for kw in ({}, {"tile_sizes": (64, 16, 4)}, {"pixel_perfect": True}, {"z": 0.25}, {"fused_tail": True}):
        okw = {k: v for k, v in kw.items() if k != "fused_tail"}
        want, want_st = orc.render2d(o, n, n, mat=mat, threads=8, **okw)
        got, st = fb.render2d(g, fb.RenderConfig2D(n, n, world_to_model=wm, **kw), stats=True)
        bad = got.view(np.uint32) != want.view(np.uint32)
        assert not bad.any(), (kw, int(bad.sum()), np.argwhere(bad)[0])
        if "fused_tail" not in kw:
            _same_census(st, want_st, (view, kw))


# ---- frames and scenes -----------------------------------------------------------------------------------------------
def _dolly(n_frames):
    """rotation_k x perspective_k: a turntable whose perspective grows from mild into the range where w changes sign"""
    return np.stack([V._f32(V._rot((0, 1, 0), 20.0 + 25.0 * k) @ V._eye(m32=0.3 + 0.35 * k)) for k in range(n_frames)])


def test_render3d_frames_turntable_with_a_dolly(orc, cuda, monkeypatch):
    n, views = 128, _dolly(5)
    o, g = _pair(orc, cuda, "colonnade.vm")
    cfg = fb.RenderConfig3D(n, n, n, exact_census=True)
    got, st = fb.render3d_frames(g, cfg, world_to_model=views, stats=True)
    total = None
    for k, wm in enumerate(views):
        want, want_st = orc.render3d(o, n, n, n, mat=orc.voxel_mat(n, n, n, wm), threads=8)
        _same3(got[k], want, f"frame {k}")
        total = want_st if total is None else {key: ([a + b for a, b in zip(total[key], want_st[key])]
                                                     if key != "pixels" else total[key] + want_st[key]) for key in total}
    _same_census(st, total, "summed census")
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", "2")
    again, st2 = fb.render3d_frames(g, cfg, world_to_model=views, stats=True)
    assert got.tobytes() == again.tobytes()
    _same_census(st2, total, "summed census, two frames per pass")


def test_render2d_frames_turntable_with_a_dolly(orc, cuda, monkeypatch):
    n = 256
    o, g = _pair(orc, cuda, "hi.vm")
    views = np.stack([V._f32(np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
                             @ V._eye(3, m21=0.3 + 0.4 * k)) for k, a in enumerate(np.linspace(0.2, 2.0, 5))])
    cfg = fb.RenderConfig2D(n, n)
    got, st = fb.render2d_frames(g, cfg, world_to_model=views, stats=True)
    pixels = 0
    for k, wm in enumerate(views):
        want, want_st = orc.render2d(o, n, n, mat=orc.pixel_mat(n, n, wm), threads=8)
        assert np.array_equal(got[k].view(np.uint32), want.view(np.uint32)), f"frame {k}"
        pixels += want_st["pixels"]
    assert st["pixels"] == pixels
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", "2")
    assert got.tobytes() == fb.render2d_frames(g, cfg, world_to_model=views).tobytes()


def test_scene_of_four_views_equals_the_fold_of_oracle_renders(orc, cuda):
    """Four placements of one shape, rotated and in perspective, overlapping on screen: culling behind a shape seen
    in perspective must not remove what the fold of the four separate renders keeps."""
    n = 128
    o, g = _pair(orc, cuda, "colonnade.vm")
    names = ["bench_camera", "rot_persp", "mirror_x", "persp_strong"]
    views = np.stack([V.view3(v) for v in names])
    got, index = fb.render3d_scene([g] * 4, fb.RenderConfig3D(n, n, n), world_to_model=views)
    want, want_index = fold([_oracle3(orc, cuda, "colonnade.vm", v, n, n, n)[0] for v in names])
    _same3(got, want, "scene")
    assert np.array_equal(index, want_index) and len(np.unique(want_index)) >= 3


# ---- octree and mesh -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("view,depth", [("rot_axis_123_50", 5), ("mirror_x", 5), ("shear", 5), ("persp_z", 5),
                                        ("bench_camera", 5), ("persp_strong", 4)])
def test_octree_sample_equals_the_oracle(orc, cuda, view, depth):
    o, g = _pair(orc, cuda, "colonnade.vm")
    wm = V.view3(view)
    want, want_st = orc.octree_sample(o, depth, wm)
    got, st = fb.octree_sample(g, depth, world_to_model=wm, stats=True)
    assert len(got) == len(want) > 0
    for k in ("ix", "iy", "iz", "mask", "n_edges", "present"):
        assert np.array_equal(got[k], want[k]), k
    present = ((want["present"][:, None] >> np.arange(12)[None, :]) & 1).astype(bool)
    assert same_f32(got["pos"][present], want["pos"][present])
    assert same_f32(got["grad"][present], want["grad"][present])
    for k in ("evaluated", "full", "empty", "ambiguous"):
        assert st[k][:depth + 1] == want_st[k][:depth + 1], k


def _mesh_view():
    return (V._translate(0.1, -0.05, 0.15) @ V._diag(0.8, 0.8, 0.8) @ V._rot((1, 2, 3), 50)).astype(np.float32)


@pytest.mark.parametrize("collapse", [False, True])
def test_mesh_vertices_are_in_model_space(orc, cuda, collapse):
    """Octree::build maps every vertex back through world_to_model (fidget-mesh/src/octree.rs:58-65): a sphere of
    radius 0.6 meshed through a similarity view has its vertices at radius 0.6, in fc_mesh_read and in the STL; and the
    whole mesh equals the oracles' (mesh_compare), bit for bit."""
    depth, wm = 5, _mesh_view()
    o, g = _pair(orc, cuda, "sphere")
    leaves, _ = orc.octree_sample(o, depth, wm)
    if collapse:
        print(mesh_compare.compare_collapse(cuda, g, leaves, depth, world_to_model=wm)[4])
    else:
        print(mesh_compare.compare_uniform(g, leaves, depth, world_to_model=wm))
    verts, tris, info, stl = fb.mesh(g, depth, world_to_model=wm, collapse=collapse, stl=True)
    cell = 0.8 * 2.0 / (1 << depth)
    assert len(tris) > 100
    r = np.linalg.norm(verts.astype(np.float64), axis=1)
    assert np.abs(r - 0.6).max() < (1.0 if collapse else 0.25) * cell, np.abs(r - 0.6).max()
    body = np.ascontiguousarray(np.frombuffer(stl, dtype=np.uint8, offset=84).reshape(-1, 50)[:, :48]).view(np.float32)
    assert np.array_equal(body.reshape(-1, 4, 3)[:, 1:], verts[tris.astype(np.int64)])
    # an identity matrix is left alone, as the reference leaves it
    plain = fb.mesh(g, depth)[0]
    same = fb.mesh(g, depth, world_to_model=np.eye(4, dtype=np.float32))[0]
    assert sorted(map(bytes, plain.view(np.uint32))) == sorted(map(bytes, same.view(np.uint32)))


@pytest.mark.parametrize("view", ["rot_axis_123_50", "persp_z"])
def test_mesh_of_a_model_under_a_view_equals_the_oracles(orc, cuda, view):
    o, g = _pair(orc, cuda, "colonnade.vm")
    wm = V.view3(view)
    leaves, _ = orc.octree_sample(o, 5, wm)
    print(mesh_compare.compare_uniform(g, leaves, 5, world_to_model=wm))
    print(mesh_compare.compare_collapse(cuda, g, leaves, 5, world_to_model=wm)[4])


# ---- the device against float64, without the oracle in between -------------------------------------------------------
@pytest.mark.parametrize("shape", ["sphere", "box", "colonnade.vm"])
@pytest.mark.parametrize("view", ["bench_camera", "persp_strong", "mirror_x"])
def test_device_renders_agree_with_float64(cuda, orc, view, shape):
    n = 96
    _, g = _pair(orc, cuda, shape)
    kind = V.VIEWS3[view][1]
    # tiles that divide the volume: under a root tile that hangs over it the reference also renders the voxels beyond the
    # image depth, and a column that is hit only there saturates (test_gpu_parity covers that against the oracle)
    cfg = fb.RenderConfig3D(n, n, n, world_to_model=V.view3(view), tile_sizes=(32, 8))
    img = fb.render3d(g, cfg)
    vals, band = V.field64(shape, cfg.matrix(), n, n, n)
    tight = V.check_heightmap(img["depth"], vals, band, max_loose=0.5 if kind == "strong" else 0.05)
    V.check_normals(img, shape, cfg.matrix(), tight, n, min_checked=0 if kind == "strong" else 20)
    name2 = {"bench_camera": "rot_persp", "persp_strong": "persp_strong", "mirror_x": "mirror_x"}[view]
    cfg2 = fb.RenderConfig2D(n, n, world_to_model=V.view2(name2))
    vals, band = V.field64(shape, cfg2.matrix(), n, n)
    V.check_image2d(fb.render2d(g, cfg2), vals, band, max_loose=0.5 if kind == "strong" else 0.05)
