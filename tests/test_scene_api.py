"""The host side of fb.render3d_scene, without a GPU: the numpy fold that stands for the per-shape merge, the placement
table (each entry what frame_table_3d gives for that placement, the rest broadcast from the config), the length and
`out` / `index_out` checks made before the library is called, and the ctypes signature against the header."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib
from scene_merge import clamp_image, fold

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _img(depths, normals=None):
    d = np.asarray(depths, dtype=np.uint32)
    img = np.zeros(d.shape, dtype=fb.GEOMETRY_PIXEL)
    img["depth"] = d
    if normals is not None:
        img["normal"] = np.asarray(normals, dtype=np.float32)
    return img


# ---- the fold helper against hand-derived cases -----------------------------------------------------------------------
def test_fold_greatest_depth_then_lowest_index():
    a = _img([[5, 0, 7, 3]], [[[1, 0, 0]] * 4])
    b = _img([[6, 0, 7, 2]], [[[0, 1, 0]] * 4])
    c = _img([[6, 0, 9, 3]], [[[0, 0, 1]] * 4])
    img, index = fold([a, b, c])
    assert img["depth"].tolist() == [[6, 0, 9, 3]]
    assert index.tolist() == [[1, 0, 2, 0]]          # 6: b before c; empty: 0; 3: a before c
    assert img["normal"][0, 0].tolist() == [0, 1, 0] and img["normal"][0, 3].tolist() == [1, 0, 0]
    assert img["normal"][0, 2].tolist() == [0, 0, 1]


def test_fold_of_one_image_is_that_image():
    a = _img([[4, 0], [1, 2]], np.random.default_rng(0).normal(size=(2, 2, 3)))
    img, index = fold([a])
    assert np.array_equal(img.view(np.uint32), a.view(np.uint32)) and not index.any()


def test_clamp_tie_lower_index_wins():
    """raw D - 1 and raw D tie at D after the clamp: the lower index wins, in both orders; without the clamp raw D wins"""
    D = 64
    lo = _img([[D - 1]], [[[0.25, 0.5, 0.75]]])
    hi = _img([[D]], [[[0.5, 0.25, 0.75]]])
    for images, want in (([lo, hi], 0), ([hi, lo], 0)):
        img, index = fold([clamp_image(i, D) for i in images])
        assert index.tolist() == [[want]] and img["depth"].tolist() == [[D]]
        assert img["normal"][0, 0].tolist() == [0, 0, 1]
    img, index = fold([lo, hi])                       # clamp=False
    assert index.tolist() == [[1]] and img["depth"].tolist() == [[D]] and img["normal"][0, 0].tolist() == [0.5, 0.25, 0.75]
    img, index = fold([hi, lo])
    assert index.tolist() == [[0]]


def test_clamp_image_only_touches_the_zone():
    D = 10
    img = clamp_image(_img([[0, 8, 9, 11]], [[[1, 2, 3]] * 4]), D)
    assert img["depth"].tolist() == [[0, 8, 10, 10]]
    assert img["normal"][0, 1].tolist() == [1, 2, 3] and img["normal"][0, 2].tolist() == [0, 0, 1]


# ---- the placement table ----------------------------------------------------------------------------------------------
def _same(a, b):
    assert bytes(a) == bytes(b)


def test_each_placement_is_frame_table_3d_of_its_values():
    rng = np.random.default_rng(5)
    cfg = fb.RenderConfig3D(200, 136, 72, var_values=(0.0, 0.0, 0.0, 0.25))
    n = 5
    vv = rng.uniform(-2, 2, (n, 4)).astype(np.float32)
    wm = rng.uniform(-1, 1, (n, 4, 4)).astype(np.float32)
    table = fb.scene_table(cfg, n, var_values=vv, world_to_model=wm)
    assert len(table) == n
    for k in range(n):
        _same(table[k], fb.frame_table_3d(cfg, var_values=vv[k:k + 1], world_to_model=wm[k:k + 1])[0])
    mats = rng.uniform(-3, 3, (n, 4, 4)).astype(np.float32)
    table = fb.scene_table(cfg, n, mats=mats)
    for k in range(n):
        _same(table[k], fb.frame_table_3d(cfg, mats=mats[k:k + 1])[0])


def test_broadcast_from_cfg():
    wm = np.diag([2.0, 0.5, 1.0, 1.0]).astype(np.float32)
    cfg = fb.RenderConfig3D(64, 64, 64, world_to_model=wm, var_values=(0.0, 0.0, 0.0, 1.5))
    one = fb.frame_table_3d(cfg)[0]
    table = fb.scene_table(cfg, 3)                    # nothing per placement: cfg's view and vars for all three
    assert len(table) == 3
    for k in range(3):
        _same(table[k], one)
    views = np.stack([np.eye(4, dtype=np.float32)] * 3)
    table = fb.scene_table(cfg, 3, world_to_model=views)   # the vars come from cfg
    for k in range(3):
        _same(table[k], fb.frame_table_3d(cfg, world_to_model=views[k:k + 1])[0])
        assert list(table[k].var_values[:4]) == [0.0, 0.0, 0.0, 1.5]


@pytest.mark.parametrize("kw", [
    dict(world_to_model=np.zeros((2, 4, 4))),
    dict(mats=np.zeros((4, 4, 4))),
    dict(var_values=np.zeros((2, 4))),
    dict(var_values=np.zeros((3, 4)), mats=np.zeros((2, 4, 4))),
    dict(mats=np.zeros((3, 4, 4)), world_to_model=np.zeros((3, 4, 4))),
])
def test_mismatched_lengths_raise(kw):
    with pytest.raises(ValueError):
        fb.scene_table(fb.RenderConfig3D(64, 64, 64), 3, **kw)


# ---- out / index_out checks before the library is called -------------------------------------------------------------
class _Lib:
    def __init__(self):
        self.called = []

    def fc_render3d_scene(self, *a):
        self.called.append(a)
        return 0


class _Cuda:
    _h = None

    def _cancellable(self, token, fn, asynchronous=False):
        return fn()


def _shapes(n, lib):
    class Shape:
        _lib, cuda, _h = lib, _Cuda(), None
    return [Shape() for _ in range(n)]


def test_out_and_index_checks():
    lib = _Lib()
    cfg = fb.RenderConfig3D(16, 8, 8)
    shapes = _shapes(3, lib)
    bad = [dict(out=np.zeros((8, 15), fb.GEOMETRY_PIXEL)),
           dict(out=np.zeros((8, 32), fb.GEOMETRY_PIXEL)[:, ::2]),
           dict(index_out=np.zeros((8, 15), np.uint16)),
           dict(index_out=np.zeros((8, 32), np.uint16)[:, ::2])]
    for kw in bad:
        with pytest.raises(ValueError):
            fb.render3d_scene(shapes, cfg, **kw)
    with pytest.raises(ValueError):
        fb.render3d_scene(shapes, cfg, world_to_model=np.zeros((2, 4, 4)))
    with pytest.raises(ValueError):
        fb.render3d_scene([], cfg)
    assert not lib.called
    out, index = np.zeros((8, 16), fb.GEOMETRY_PIXEL), np.zeros((8, 16), np.uint16)
    got = fb.render3d_scene(shapes, cfg, out=out, index_out=index)
    assert got[0] is out and got[1] is index
    assert len(lib.called) == 1 and lib.called[0][3] == 3
    img, idx = fb.render3d_scene(shapes, cfg)
    assert img.shape == (8, 16) and img.dtype == fb.GEOMETRY_PIXEL and idx.shape == (8, 16) and idx.dtype == np.uint16


def test_shapes_of_two_contexts_are_refused():
    lib = _Lib()
    shapes = _shapes(2, lib) + _shapes(1, lib)     # (each _shapes call makes its own context)
    with pytest.raises(ValueError):
        fb.render3d_scene(shapes, fb.RenderConfig3D(16, 8, 8))
    assert not lib.called


def test_signature_matches_header():
    text = open(os.path.join(ROOT, "include", "fidget_cuda.h")).read()
    m = re.search(r"int32_t fc_render3d_scene\((.*?)\);", text, re.S)
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")]
    types = [p.rsplit(" ", 1)[0].replace(" *", "*").strip() for p in params]
    assert types == ["fc_ctx*", "const fc_tape* const*", "const fc_frame3d*", "uint32_t", "const fc_render3d_cfg*",
                     "fc_geometry_pixel*", "uint16_t*", "fc_render_stats*"]
    res, args = _lib.CUDA_API["fc_render3d_scene"]
    assert res is C.c_int32
    assert args == [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(_lib.FcFrame3d), C.c_uint32,
                    C.POINTER(_lib.FcRender3dCfg), C.c_void_p, C.c_void_p, C.POINTER(_lib.FcRenderStats)]
    assert _lib.FC_SCENE_MAX_SHAPES >= 1024
