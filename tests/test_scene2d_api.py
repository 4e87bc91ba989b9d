"""The host side of fb.render2d_scene, without a GPU: the numpy fold that stands for the viewer's draw list, the
draw_rgb colour conversion, the placement and colour tables, the `out` / `index_out` checks made before the library is
called, the ctypes signature against the header, and the fold of the CPU oracle's per-shape renders against shapes
evaluated at every pixel in numpy."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib
from scene2d_fold import NONE, bitmap_1bit, fold, fold_inside, mask_u8, rgba

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILL_IN = np.array([0x7FC00000 | (0xF6 << 9) | 1], dtype=np.uint32).view(np.float32)[0]    # inside fill
FILL_OUT = np.array([0x7FC00000 | (0xF6 << 9)], dtype=np.uint32).view(np.float32)[0]      # outside fill


# ---- the fold helper against hand-made images --------------------------------------------------------------------------
def test_fold_topmost_wins_and_none_elsewhere():
    a = np.array([[-1.0, 1.0, FILL_IN, np.nan, 2.0]], dtype=np.float32)
    b = np.array([[-0.5, FILL_OUT, FILL_IN, -3.0, 1.0]], dtype=np.float32)
    c = np.array([[0.5, -2.0, 3.0, 4.0, 1.0]], dtype=np.float32)
    index = fold([a, b, c])
    assert index.tolist() == [[1, 2, 1, 1, NONE]]      # NaN distance is outside; fills by their inside bit
    assert fold([a]).tolist() == [[0, NONE, 0, NONE, NONE]]


def test_rgba_mask_and_bitmap_of_an_index():
    index = np.array([[0, 2, NONE, 1, NONE, NONE, NONE, NONE, 0]], dtype=np.uint16)
    colors = np.array([[10, 20, 30], [40, 50, 60], [70, 80, 90]], dtype=np.uint8)
    img = rgba(index, colors)
    assert img[0, 0].tolist() == [10, 20, 30, 255] and img[0, 1].tolist() == [70, 80, 90, 255]
    assert img[0, 2].tolist() == [0, 0, 0, 0] and img[0, 3].tolist() == [40, 50, 60, 255]
    assert rgba(index)[0, 3].tolist() == [255, 255, 255, 255]          # draw(): white
    assert mask_u8(index).tolist() == [[255, 255, 0, 255, 0, 0, 0, 0, 255]]
    assert bitmap_1bit(index).tolist() == [[0b00001011, 0b00000001]]
    assert fold_inside([np.zeros((2, 3), bool)]).tolist() == [[NONE] * 3] * 2


# ---- draw_rgb's colour conversion --------------------------------------------------------------------------------------
def test_colors_convert_as_draw_rgb():
    got = fb.scene_colors([[0.5, -1.0, 2.0], [np.nan, 1.0, 0.0], [0.999, 0.1, 1.0000001]], 3)
    assert got.dtype == np.uint8
    assert got.tolist() == [[127, 0, 255], [0, 255, 0], [254, 25, 255]]
    raw = np.array([[1, 2, 3]], dtype=np.uint8)
    assert fb.scene_colors(raw, 1).tolist() == [[1, 2, 3]]            # uint8 is taken as is
    for bad in (np.zeros((2, 3)), np.zeros((3, 4)), np.zeros(3)):
        with pytest.raises(ValueError):
            fb.scene_colors(bad, 3)


# ---- the placement table -----------------------------------------------------------------------------------------------
def _same(a, b):
    assert bytes(a) == bytes(b)


def test_each_placement_is_frame_table_of_its_values():
    rng = np.random.default_rng(3)
    cfg = fb.RenderConfig2D(200, 136, z=0.25, var_values=(0.0, 0.0, 0.0, 0.5))
    n = 4
    z = rng.uniform(-1, 1, n).astype(np.float32)
    vv = rng.uniform(-2, 2, (n, 4)).astype(np.float32)
    wm = rng.uniform(-1, 1, (n, 3, 3)).astype(np.float32)
    table = fb.scene_table_2d(cfg, n, z=z, var_values=vv, world_to_model=wm)
    assert len(table) == n
    for k in range(n):
        _same(table[k], fb.frame_table(cfg, z=z[k:k + 1], var_values=vv[k:k + 1], world_to_model=wm[k:k + 1])[0])
    mats = rng.uniform(-3, 3, (n, 4, 4)).astype(np.float32)
    table = fb.scene_table_2d(cfg, n, mats=mats)
    for k in range(n):
        _same(table[k], fb.frame_table(cfg, mats=mats[k:k + 1])[0])
        assert table[k].z == np.float32(0.25)


def test_broadcast_from_cfg():
    cfg = fb.RenderConfig2D(64, 48, z=-0.5, world_to_model=np.diag([2.0, 0.5, 1.0]), var_values=(0.0, 0.0, 0.0, 1.5))
    one = fb.frame_table(cfg)[0]
    table = fb.scene_table_2d(cfg, 3)
    assert len(table) == 3
    for k in range(3):
        _same(table[k], one)


@pytest.mark.parametrize("kw", [
    dict(z=np.zeros(2)),
    dict(mats=np.zeros((4, 4, 4))),
    dict(var_values=np.zeros((2, 4))),
    dict(world_to_model=np.zeros((3, 3, 3)), z=np.zeros(2)),
    dict(mats=np.zeros((3, 4, 4)), world_to_model=np.zeros((3, 3, 3))),
])
def test_mismatched_lengths_raise(kw):
    with pytest.raises(ValueError):
        fb.scene_table_2d(fb.RenderConfig2D(64, 64), 3, **kw)


# ---- out / index_out checks before the library is called --------------------------------------------------------------
class _Lib:
    def __init__(self):
        self.called = []

    def fc_render2d_scene(self, *a):
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
    cfg = fb.RenderConfig2D(16, 8, out_format="rgba8")
    shapes = _shapes(3, lib)
    bad = [dict(out=np.zeros((8, 15, 4), np.uint8)),
           dict(out=np.zeros((8, 32, 4), np.uint8)[:, ::2]),
           dict(index_out=np.zeros((8, 15), np.uint16)),
           dict(index_out=np.zeros((8, 32), np.uint16)[:, ::2]),
           dict(colors=np.zeros((2, 3))),
           dict(z=np.zeros(2))]
    for kw in bad:
        with pytest.raises(ValueError):
            fb.render2d_scene(shapes, cfg, **kw)
    with pytest.raises(ValueError):
        fb.render2d_scene([], cfg)
    assert not lib.called
    out, index = np.zeros((8, 16, 4), np.uint8), np.zeros((8, 16), np.uint16)
    got = fb.render2d_scene(shapes, cfg, out=out, index_out=index, colors=np.ones((3, 3)))
    assert got[0] is out and got[1] is index
    assert len(lib.called) == 1 and lib.called[0][3] == 3 and lib.called[0][5] is not None
    img, idx = fb.render2d_scene(shapes, cfg)
    assert img.shape == (8, 16, 4) and img.dtype == np.uint8 and idx.shape == (8, 16) and idx.dtype == np.uint16
    assert lib.called[-1][5] is None                                   # no colours: the library paints white
    for fmt, shape in (("mask_u8", (8, 16)), ("bitmap_1bit", (8, 2))):
        img, _ = fb.render2d_scene(shapes, fb.RenderConfig2D(16, 8, out_format=fmt))
        assert img.shape == shape and img.dtype == np.uint8


def test_shapes_of_two_contexts_are_refused():
    lib = _Lib()
    shapes = _shapes(2, lib) + _shapes(1, lib)     # (each _shapes call makes its own context)
    with pytest.raises(ValueError):
        fb.render2d_scene(shapes, fb.RenderConfig2D(16, 8, out_format="rgba8"))
    assert not lib.called


def test_signature_matches_header():
    text = open(os.path.join(ROOT, "include", "fidget_cuda.h")).read()
    m = re.search(r"int32_t fc_render2d_scene\((.*?)\);", text, re.S)
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")]
    types = [p.rsplit(" ", 1)[0].replace(" *", "*").strip() for p in params]
    assert types == ["fc_ctx*", "const fc_tape* const*", "const fc_frame2d*", "uint32_t", "const fc_render2d_cfg*",
                     "const uint8_t*", "void*", "uint16_t*", "fc_render_stats*"]
    res, args = _lib.CUDA_API["fc_render2d_scene"]
    assert res is C.c_int32
    assert args == [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(_lib.FcFrame2d), C.c_uint32,
                    C.POINTER(_lib.FcRender2dCfg), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(_lib.FcRenderStats)]
    assert re.search(r"#define FC_SCENE2D_NONE 0xFFFFu", text) and _lib.FC_SCENE2D_NONE == fb.FC_SCENE2D_NONE == NONE


# ---- the fold of the oracle's renders against numpy ---------------------------------------------------------------------
def _scene():
    """(tape, distance in float64 of world x, y) for two half-planes under three circles, each peeking out"""
    out = []
    g = fb.Context()
    out.append((g.tape(g.sub(g.x(), 0.6)), lambda X, Y: X - 0.6))                   # x < 0.6
    g = fb.Context()
    out.append((g.tape(g.mul(g.add(g.y(), 0.7), -1.0)), lambda X, Y: -(Y + 0.7)))   # y > -0.7
    for cx, cy, r in ((-0.3, 0.2, 0.5), (0.25, 0.1, 0.4), (0.0, -0.35, 0.3)):
        g = fb.Context()
        x, y = g.sub(g.x(), cx), g.sub(g.y(), cy)
        out.append((g.tape(g.sub(g.sqrt(g.add(g.square(x), g.square(y))), r)),
                    lambda X, Y, cx=cx, cy=cy, r=r: np.sqrt((X - cx) ** 2 + (Y - cy) ** 2) - r))
    return out


def test_oracle_fold_matches_numpy(orc):
    w, h = 160, 120
    mat = fb.pixel_mat(w, h).astype(np.float64)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    X = mat[0, 0] * xs + mat[0, 1] * ys + mat[0, 3]
    Y = mat[1, 0] * xs + mat[1, 1] * ys + mat[1, 3]
    scene = _scene()
    images = [orc.render2d(orc.Tape.from_data(td), w, h)[0] for td, _ in scene]
    dists = [f(X, Y) for _, f in scene]
    index = fold(images)
    want = fold_inside([d < 0 for d in dists])
    clear = np.all([np.abs(d) > 1e-3 for d in dists], axis=0)         # (pixels on an edge may round either way)
    assert clear.mean() > 0.9
    assert np.array_equal(index[clear], want[clear])
    assert set(np.unique(index[clear]).tolist()) == {0, 1, 2, 3, 4, NONE}
