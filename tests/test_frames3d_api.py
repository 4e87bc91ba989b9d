"""The host side of fb.render3d_frames, without a GPU: the fc_frame3d table frame_table_3d builds holds, bit for bit,
the mat / var_values render3d would put into fc_render3d_cfg for each frame, broadcasts what is not given per frame
from the config, and rejects per-frame arguments whose lengths disagree; its ctypes layout is the header's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg_of(cfg):
    return fb.shape._render3d_cfg(cfg, False)


def _same_frame(frame, c):
    assert bytes(frame.mat) == bytes(c.mat)
    assert frame.n_var_values == c.n_var_values
    assert bytes(frame.var_values) == bytes(c.var_values)


def test_per_frame_values_equal_render3d_cfg():
    rng = np.random.default_rng(7)
    base = fb.RenderConfig3D(200, 136, 72, var_values=(0.0, 0.0, 0.0, 0.25))
    n = 6
    vv = rng.uniform(-2, 2, (n, 4)).astype(np.float32)
    wm = rng.uniform(-1, 1, (n, 4, 4)).astype(np.float32)
    table = fb.frame_table_3d(base, var_values=vv, world_to_model=wm)
    assert len(table) == n
    for k in range(n):
        single = fb.RenderConfig3D(200, 136, 72, var_values=tuple(vv[k]), world_to_model=wm[k])
        _same_frame(table[k], _cfg_of(single))
        assert bytes(table[k].mat) == fb.voxel_mat(200, 136, 72, wm[k]).astype(np.float32).tobytes()


def test_explicit_matrices_pass_through():
    mats = np.random.default_rng(2).uniform(-3, 3, (4, 4, 4)).astype(np.float32)
    cfg = fb.RenderConfig3D(100, 50, 80)
    table = fb.frame_table_3d(cfg, mats=mats)
    for k in range(4):
        _same_frame(table[k], _cfg_of(fb.RenderConfig3D(100, 50, 80, mat=mats[k])))


def test_broadcast_from_cfg():
    wm = np.diag([2.0, 0.5, 1.0, 1.0]).astype(np.float32)
    cfg = fb.RenderConfig3D(256, 128, 64, world_to_model=wm, var_values=(0.0, 0.0, 0.0, 1.5))
    radii = [[0.0, 0.0, 0.0, r] for r in (0.25, 0.5, 1.0)]
    table = fb.frame_table_3d(cfg, var_values=radii)                    # the view comes from cfg
    assert len(table) == 3
    for k, vv in enumerate(radii):
        _same_frame(table[k], _cfg_of(fb.RenderConfig3D(256, 128, 64, world_to_model=wm, var_values=tuple(vv))))
    views = np.stack([np.eye(4, dtype=np.float32)] * 2)
    table = fb.frame_table_3d(cfg, world_to_model=views)                # the vars come from cfg
    for k in range(2):
        _same_frame(table[k], _cfg_of(fb.RenderConfig3D(256, 128, 64, world_to_model=views[k], var_values=cfg.var_values)))
    one = fb.frame_table_3d(cfg)                                        # nothing per frame: one frame, the config itself
    assert len(one) == 1
    _same_frame(one[0], _cfg_of(cfg))
    assert len(fb.frame_table_3d(cfg, mats=np.zeros((0, 4, 4)))) == 0


@pytest.mark.parametrize("kw", [
    dict(var_values=np.zeros((3, 4)), world_to_model=np.zeros((2, 4, 4))),
    dict(var_values=np.zeros((1, 4)), mats=np.zeros((2, 4, 4))),
    dict(mats=np.zeros((2, 4, 4)), world_to_model=np.zeros((2, 4, 4))),
    dict(world_to_model=np.zeros((2, 3, 3))),
    dict(mats=np.zeros((4, 4))),
    dict(var_values=np.zeros((2, 17))),
])
def test_mismatched_arguments_raise(kw):
    with pytest.raises(ValueError):
        fb.frame_table_3d(fb.RenderConfig3D(64, 64, 64), **kw)


def test_frame_struct_layout_matches_header(tmp_path):
    assert C.sizeof(_lib.FcFrame3d) == 64 + 4 + 64
    src = tmp_path / "frame.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fidget_cuda.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu\\n", sizeof(fc_frame3d), offsetof(fc_frame3d, n_var_values),\n'
                   '         offsetof(fc_frame3d, var_values));\n  return 0;\n}\n')
    exe = tmp_path / "frame"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(_lib.FcFrame3d), _lib.FcFrame3d.n_var_values.offset, _lib.FcFrame3d.var_values.offset]


def test_out_size_check(monkeypatch):
    """render3d_frames refuses an `out` that is too small or not contiguous before it calls the library"""
    called = []

    class Lib:
        def fc_render3d_frames(self, *a):
            called.append(a)
            return 0

    class Cuda:
        _h = None

        def _cancellable(self, token, fn, asynchronous=False):
            return fn()

    class Shape:
        _lib, cuda, _h = Lib(), Cuda(), None

    cfg = fb.RenderConfig3D(16, 8, 8)
    views = np.stack([np.eye(4, dtype=np.float32)] * 3)
    with pytest.raises(ValueError):
        fb.render3d_frames(Shape(), cfg, world_to_model=views, out=np.zeros((2, 8, 16), fb.GEOMETRY_PIXEL))
    with pytest.raises(ValueError):
        fb.render3d_frames(Shape(), cfg, world_to_model=views, out=np.zeros((3, 8, 32), fb.GEOMETRY_PIXEL)[:, :, ::2])
    assert not called
    out = np.zeros((3, 8, 16), fb.GEOMETRY_PIXEL)
    assert fb.render3d_frames(Shape(), cfg, world_to_model=views, out=out) is out
    assert len(called) == 1 and called[0][4] == 3
