"""The host side of fb.render2d_frames, without a GPU: the fc_frame2d table frame_table builds holds, bit for bit,
the mat / z / var_values render2d would put into fc_render2d_cfg for each frame, broadcasts what is not given per
frame from the config, and rejects per-frame arguments whose lengths disagree; its ctypes layout is the header's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg_of(cfg):
    return fb.shape._render2d_cfg(cfg, False)


def _same_frame(frame, c):
    assert bytes(frame.mat) == bytes(c.mat)
    assert np.float32(frame.z).tobytes() == np.float32(c.z).tobytes()
    assert frame.n_var_values == c.n_var_values
    assert bytes(frame.var_values) == bytes(c.var_values)


def test_per_frame_values_equal_render2d_cfg():
    rng = np.random.default_rng(5)
    base = fb.RenderConfig2D(640, 360, var_values=(0.0, 0.0, 0.0, 0.25))
    n = 7
    zs = rng.uniform(-1, 1, n).astype(np.float32)
    vv = rng.uniform(-2, 2, (n, 4)).astype(np.float32)
    wm = rng.uniform(-1, 1, (n, 3, 3)).astype(np.float32)
    table = fb.frame_table(base, z=zs, var_values=vv, world_to_model=wm)
    assert len(table) == n
    for k in range(n):
        single = fb.RenderConfig2D(640, 360, z=float(zs[k]), var_values=tuple(vv[k]), world_to_model=wm[k])
        _same_frame(table[k], _cfg_of(single))


def test_explicit_matrices_pass_through():
    mats = np.random.default_rng(1).uniform(-3, 3, (4, 4, 4)).astype(np.float32)
    cfg = fb.RenderConfig2D(100, 50)
    table = fb.frame_table(cfg, mats=mats)
    for k in range(4):
        _same_frame(table[k], _cfg_of(fb.RenderConfig2D(100, 50, mat=mats[k])))


def test_broadcast_from_cfg():
    cfg = fb.RenderConfig2D(256, 128, z=0.375, world_to_model=np.diag([2.0, 0.5, 1.0]).astype(np.float32),
                            var_values=(0.0, 0.0, 0.0, 1.5))
    table = fb.frame_table(cfg, z=[0.0, 0.5, -0.5])
    assert len(table) == 3
    for k, z in enumerate((0.0, 0.5, -0.5)):
        single = fb.RenderConfig2D(256, 128, z=z, world_to_model=cfg.world_to_model, var_values=cfg.var_values)
        _same_frame(table[k], _cfg_of(single))
    one = fb.frame_table(cfg)                      # nothing per frame: one frame, the config itself
    assert len(one) == 1
    _same_frame(one[0], _cfg_of(cfg))
    empty = fb.frame_table(cfg, z=np.zeros(0))
    assert len(empty) == 0


@pytest.mark.parametrize("kw", [
    dict(z=[0.0, 1.0], var_values=np.zeros((3, 4))),
    dict(z=[0.0, 1.0, 2.0], world_to_model=np.zeros((2, 3, 3))),
    dict(mats=np.zeros((2, 4, 4)), z=[0.0]),
    dict(mats=np.zeros((2, 4, 4)), world_to_model=np.zeros((2, 3, 3))),
    dict(world_to_model=np.zeros((2, 4, 4))),
    dict(var_values=np.zeros((2, 17))),
])
def test_mismatched_arguments_raise(kw):
    with pytest.raises(ValueError):
        fb.frame_table(fb.RenderConfig2D(64, 64), **kw)


def test_frame_struct_layout_matches_header(tmp_path):
    assert C.sizeof(_lib.FcFrame2d) == 64 + 4 + 4 + 64
    src = tmp_path / "frame.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fidget_cuda.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(fc_frame2d), offsetof(fc_frame2d, z),\n'
                   '         offsetof(fc_frame2d, n_var_values), offsetof(fc_frame2d, var_values));\n  return 0;\n}\n')
    exe = tmp_path / "frame"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(_lib.FcFrame2d), _lib.FcFrame2d.z.offset, _lib.FcFrame2d.n_var_values.offset,
                   _lib.FcFrame2d.var_values.offset]


def test_out_size_check():
    from fidget_b200.shape import _check_out
    _check_out(np.zeros((3, 4, 5), np.float32), 3 * 4 * 5 * 4)
    with pytest.raises(ValueError):
        _check_out(np.zeros((2, 4, 5), np.float32), 3 * 4 * 5 * 4)
    with pytest.raises(ValueError):
        _check_out(np.zeros((3, 4, 10), np.float32)[:, :, ::2], 3 * 4 * 5 * 4)
