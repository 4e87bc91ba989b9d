"""fc_render2d_scene / fb.render2d_scene: a 2D draw list rendered in one call.

The index and the image must be, bit for bit, the fold of the per-shape fb.render2d images (tests/scene2d_fold.py: the
last shape inside a pixel wins): for overlapping mixed models, many placements of one tape, per-placement ShapeVars and
Z, a ragged image, tile sizes and pixel_perfect, and against the oracle's renders.  Culling must be real (a fewer tiles
evaluated under a covering shape) and safe (shapes peeking out of partly covered tiles, outside fills, equal inside
sets); the stats do not depend on the launch grid; passes, outputs, refusals and cancellation behave as
fc_render2d_frames's do."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import fidget_b200 as fb
from conftest import model_text
from fidget_b200 import _lib
from scene2d_fold import NONE, bitmap_1bit, fold, mask_u8, rgba

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CENSUS = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")
_SHAPES = {}


def _shape(cuda, name):
    key = (id(cuda), name)
    if key not in _SHAPES:
        _SHAPES[key] = (cuda, fb.CudaShape.from_vm(cuda, model_text(name)))
    return _SHAPES[key][1]


def _place(scale, tx, ty):
    """world -> model of a shape scaled by `scale` and centred at (tx, ty)"""
    s = 1.0 / scale
    return np.array([[s, 0, -tx * s], [0, s, -ty * s], [0, 0, 1]], dtype=np.float32)


MIXED = ("prospero.vm", "bear.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm", "gyroid-sphere.vm", "hi.vm")


def mixed():
    return np.stack([_place(1.0, 0.0, 0.0), _place(0.6, -0.4, 0.3), _place(0.5, 0.4, 0.4), _place(0.5, 0.3, -0.3),
                     _place(0.45, -0.35, -0.35), _place(0.35, 0.0, 0.1), _place(0.3, 0.55, 0.0), _place(0.4, -0.1, -0.5)])


def grid(n=8, scale=0.12):
    return np.stack([_place(scale, -0.875 + 0.25 * i, -0.875 + 0.25 * j) for j in range(n) for i in range(n)])


COLORS = np.array([[(37 * k) % 256, (91 * k + 40) % 256, (53 * k + 200) % 256] for k in range(256)], dtype=np.uint8)


def _single_cfg(cfg, f):
    return fb.RenderConfig2D(cfg.width, cfg.height, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4), z=f.z,
                             pixel_perfect=cfg.pixel_perfect, tile_sizes=cfg.tile_sizes,
                             var_values=tuple(f.var_values[:f.n_var_values]))


def _singles(shapes, cfg, **per):
    table = fb.scene_table_2d(cfg, len(shapes), **per)
    return [fb.render2d(sh, _single_cfg(cfg, table[k]), stats=True) for k, sh in enumerate(shapes)]


def _summed(singles):
    return {k: [sum(s[k][l] for _, s in singles) for l in range(len(singles[0][1][k]))] for k in CENSUS}


def _check(shapes, cfg, **per):
    """the scene in RGBA against the fold of per-shape renders; returns its index and stats and the singles"""
    cfg = fb.RenderConfig2D(**{**cfg.__dict__, "out_format": "rgba8"})
    colors = COLORS[:len(shapes)]
    img, index, st = fb.render2d_scene(shapes, cfg, colors=colors, stats=True, **per)
    singles = _singles(shapes, cfg, **per)
    want = fold([im for im, _ in singles])
    assert np.array_equal(index, want)
    assert np.array_equal(img, rgba(want, colors))
    return index, st, singles


# ---- 1. bit identity with the fold of per-shape renders ---------------------------------------------------------------
def test_mixed_models(cuda):
    index, st, singles = _check([_shape(cuda, m) for m in MIXED], fb.RenderConfig2D(1024, 1024), world_to_model=mixed())
    assert len(np.unique(index)) >= 7


def test_one_tape_64_times(cuda):
    index, _, _ = _check([_shape(cuda, "hi.vm")] * 64, fb.RenderConfig2D(1024, 1024), world_to_model=grid())
    assert len(np.unique(index)) == 65


def _circle_var(cuda):
    g = fb.Context()
    x, y = g.x(), g.y()
    r, _ = g.var()
    td = g.tape(g.sub(g.sqrt(g.add(g.square(x), g.square(y))), r))
    slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
    return fb.CudaShape(cuda, td), td.n_vars, slot


def test_per_placement_vars_and_z(cuda):
    shape, nv, slot = _circle_var(cuda)
    vv = np.zeros((6, nv), dtype=np.float32)
    vv[:, slot] = np.linspace(0.2, 0.7, 6)
    views = np.stack([_place(1.0, -0.5 + 0.2 * k, 0.3 - 0.12 * k) for k in range(6)])
    _check([shape] * 6, fb.RenderConfig2D(512, 512), var_values=vv, world_to_model=views)
    tangle = _shape(cuda, "tanglecube.vm")
    _check([tangle] * 5, fb.RenderConfig2D(512, 512), z=np.linspace(-0.8, 0.8, 5).astype(np.float32),
           world_to_model=np.stack([_place(0.8, 0.1 * k, -0.1 * k) for k in range(5)]))


def test_ragged_image(cuda):
    _check([_shape(cuda, m) for m in MIXED], fb.RenderConfig2D(1000, 700), world_to_model=mixed())


@pytest.mark.parametrize("ts", [(64, 16, 4), (128, 8)])
def test_tile_sizes(cuda, ts):
    _check([_shape(cuda, m) for m in MIXED], fb.RenderConfig2D(640, 512, tile_sizes=ts), world_to_model=mixed())


def test_pixel_perfect_culls_nothing(cuda):
    """no tile is proven inside, so every shape's census is evaluated in full"""
    _, st, singles = _check([_shape(cuda, m) for m in MIXED[:4]], fb.RenderConfig2D(256, 256, pixel_perfect=True),
                            world_to_model=mixed()[:4])
    assert {k: st[k] for k in CENSUS} == _summed(singles)
    assert st["pixels"] == sum(s["pixels"] for _, s in singles)


def test_oracle_fold(orc, cuda):
    n = 384
    names = ("prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm")
    views = np.stack([_place(1.0, 0.0, 0.0), _place(0.5, 0.3, 0.3), _place(0.5, -0.3, 0.3), _place(0.45, 0.3, -0.3),
                      _place(0.4, -0.3, -0.3)])
    mats = np.stack([fb.pixel_mat(n, n, v) for v in views])
    _, index = fb.render2d_scene([_shape(cuda, m) for m in names], fb.RenderConfig2D(n, n, out_format="mask_u8"),
                                 mats=mats)
    oimgs = [orc.render2d(orc.Tape.from_vm(model_text(m)), n, n, mat=mats[k], threads=8)[0] for k, m in enumerate(names)]
    assert np.array_equal(index, fold(oimgs))
    assert len(np.unique(index)) == 6


# ---- 2. culling is real and safe --------------------------------------------------------------------------------------
def _disc(cuda, r):
    g = fb.Context()
    return fb.CudaShape(cuda, g.tape(g.sub(g.sqrt(g.add(g.square(g.x()), g.square(g.y()))), r)))


def test_covering_shape_culls(cuda):
    """prospero under a disc that fills the frame: whole root tiles are proven inside the disc, so prospero's tiles
    under them are not evaluated; the image is still the fold"""
    _, st, singles = _check([_shape(cuda, "prospero.vm"), _disc(cuda, 1.2)], fb.RenderConfig2D(1024, 1024))
    want = _summed(singles)
    assert sum(st["evaluated"]) < sum(want["evaluated"])
    assert st["pixels"] < sum(s["pixels"] for _, s in singles)


def test_lower_shape_peeks_out_of_partly_covered_tiles(cuda):
    """small discs on top of a large one, their edges inside the large one's tiles: the large disc shows around them"""
    big, small = _disc(cuda, 0.9), _disc(cuda, 1.0)
    views = np.stack([np.eye(3, dtype=np.float32)] + [_place(0.1, -0.5 + 0.25 * k, 0.07 * k) for k in range(5)])
    index, _, _ = _check([big] + [small] * 5, fb.RenderConfig2D(512, 512), world_to_model=views)
    assert (index == 0).sum() > 0.5 * 512 * 512 * 0.6 and all((index == k).any() for k in range(6))


def test_outside_fills_never_cull(cuda):
    """top shapes outside the whole frame prove every tile outside: nothing below them is culled"""
    shapes = [_shape(cuda, "prospero.vm"), _shape(cuda, "hi.vm"), _disc(cuda, 0.3)]
    views = np.stack([np.eye(3, dtype=np.float32), _place(0.5, -4.0, 3.0), _place(1.0, 5.0, 5.0)])
    index, st, singles = _check(shapes, fb.RenderConfig2D(512, 512), world_to_model=views)
    assert (index == 0).any() and set(np.unique(index).tolist()) == {0, NONE}
    assert sum(singles[1][1]["filled_outside"]) > 0 and sum(singles[2][1]["filled_outside"]) > 0
    assert {k: st[k] for k in CENSUS} == _summed(singles)
    assert st["pixels"] == sum(s["pixels"] for _, s in singles)


def test_f_over_2f_gives_the_higher_index(cuda):
    g = fb.Context()
    f = g.sub(g.sqrt(g.add(g.square(g.x()), g.square(g.y()))), 0.6)
    one, two = fb.CudaShape(cuda, g.tape(f)), fb.CudaShape(cuda, g.tape(g.mul(f, 2.0)))
    cfg = fb.RenderConfig2D(512, 512)
    inside = fb.pixel_inside(fb.render2d(one, cfg))
    assert inside.sum() > 1000 and np.array_equal(inside, fb.pixel_inside(fb.render2d(two, cfg)))
    for shapes in ([one, two], [two, one], [one, two, one, two]):
        index, _, _ = _check(shapes, cfg)
        assert (index[inside] == len(shapes) - 1).all() and (index[~inside] == NONE).all()


# ---- 3. determinism ----------------------------------------------------------------------------------------------------
def _stats_fields(st):
    return {k: st[k] for k in CENSUS + ("pixels", "arena_bytes_used", "kernel_launches")}


def test_identical_calls_give_equal_stats(cuda):
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig2D(1024, 1024, out_format="rgba8")
    a = fb.render2d_scene(shapes, cfg, world_to_model=mixed(), stats=True)[2]
    b = fb.render2d_scene(shapes, cfg, world_to_model=mixed(), stats=True)[2]
    assert _stats_fields(a) == _stats_fields(b)
    assert sum(a["evaluated"]) > 0 and a["pixels"] > 0


_CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
import fidget_b200 as fb
from test_gpu_render2d_scene import MIXED, mixed
cuda = fb.CudaContext(0)
shapes = {}
for m in set(MIXED):
    shapes[m] = fb.CudaShape.from_vm(cuda, open(sys.argv[1] + "/models/" + m).read())
img, index, st = fb.render2d_scene([shapes[m] for m in MIXED], fb.RenderConfig2D(1024, 1024, out_format="rgba8"),
                                   world_to_model=mixed(), stats=True)
keys = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified", "pixels", "arena_bytes_used",
        "kernel_launches")
print(json.dumps({"stats": {k: st[k] for k in keys}, "index": int(index.astype(np.uint64).sum()),
                  "img": int(img.astype(np.uint64).sum())}))
"""


def _child(env):
    full = {k: v for k, v in os.environ.items() if not k.startswith("FIDGET_B200_")}
    full.update({"FIDGET_B200_" + k: v for k, v in env.items()})
    out = subprocess.run([sys.executable, "-c", _CHILD, ROOT], capture_output=True, text=True, env=full, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_stats_do_not_depend_on_the_launch_grid():
    base = _child({})
    for env in ({"SM_COUNT": "7"}, {"SM_COUNT": "33", "BLOCKS_PER_SM": "1"}, {"BLOCKS_PER_SM": "3"},
                {"PIXEL_BLOCKS_PER_SM": "1"}, {"COOP_PER_SM": "1"}, {"COOP_PER_SM": "3", "SM_COUNT": "50"}):
        assert _child(env) == base, env


# ---- 4. passes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_pass", [1, 3])
def test_forced_passes_change_nothing(cuda, monkeypatch, per_pass):
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig2D(512, 512, out_format="rgba8")
    one = fb.render2d_scene(shapes, cfg, world_to_model=mixed(), colors=COLORS[:8])
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(per_pass))
    split = fb.render2d_scene(shapes, cfg, world_to_model=mixed(), colors=COLORS[:8])
    assert np.array_equal(split[0], one[0]) and np.array_equal(split[1], one[1])


def test_small_arena_is_an_error(cuda):
    ctx = fb.CudaContext(0)
    shape = fb.CudaShape.from_vm(ctx, model_text("prospero.vm"))
    ctx.set_arena_bytes(1 << 20)
    with pytest.raises(fb.CudaError) as e:
        fb.render2d_scene([shape] * 3, fb.RenderConfig2D(2048, 2048, out_format="rgba8"), world_to_model=mixed()[:3])
    assert e.value.code == -4
    # the exception's traceback holds this frame in a cycle that the collector may free at any later time, the context
    # before its tape; release both now, in order
    del e
    shape.close()
    ctx.close()


# ---- 5. outputs --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["rgba8", "mask_u8", "bitmap_1bit"])
@pytest.mark.parametrize("kind", ["pageable", "pinned", "device", "async"])
def test_outputs(cuda, fmt, kind):
    import torch
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig2D(500, 300, out_format=fmt)
    want_index = fold([fb.render2d(sh, fb.RenderConfig2D(500, 300, world_to_model=v)) for sh, v in zip(shapes, mixed())])
    want = {"rgba8": rgba(want_index, COLORS[:8]), "mask_u8": mask_u8(want_index),
            "bitmap_1bit": bitmap_1bit(want_index)}[fmt]
    if kind == "pageable":
        out, index = np.zeros_like(want), np.zeros_like(want_index)
    else:
        dev = "cpu" if kind == "pinned" else "cuda"
        out = torch.zeros(want.shape, dtype=torch.uint8, device=dev, pin_memory=kind == "pinned")
        index = torch.zeros(want_index.shape, dtype=torch.int16, device=dev, pin_memory=kind == "pinned")
    got = fb.render2d_scene(shapes, cfg, colors=COLORS[:8], world_to_model=mixed(), out=out, index_out=index,
                            asynchronous=kind == "async")
    assert got[0] is out and got[1] is index
    if kind == "async":
        cuda.synchronize()
    o = out if kind == "pageable" else out.cpu().numpy()
    i = index if kind == "pageable" else index.cpu().numpy().view(np.uint16)
    assert np.array_equal(o, want) and np.array_equal(i, want_index)


def _raw(cuda, tapes, table, cfg, out, n=None, index=None, colors=None):
    c = fb.shape._render2d_cfg(cfg, False)
    n = len(tapes) if n is None else n
    handles = None if tapes is None else (C.c_void_p * max(len(tapes), 1))(*[t._h if t is not None else None for t in tapes])
    col = None if colors is None else colors.ctypes.data
    return _lib.load().fc_render2d_scene(cuda._h, handles, table, n, C.byref(c), col, fb.shape._ptr(out),
                                         fb.shape._ptr(index), None)


def test_index_only_and_image_only(cuda):
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig2D(256, 256, out_format="rgba8")
    table = fb.scene_table_2d(cfg, 8, world_to_model=mixed())
    img, index = fb.render2d_scene(shapes, cfg, world_to_model=mixed())
    only_index = np.zeros_like(index)
    assert _raw(cuda, shapes, table, cfg, None, index=only_index) == 0
    assert np.array_equal(only_index, index)
    only_img = np.zeros_like(img)
    assert _raw(cuda, shapes, table, cfg, only_img) == 0
    assert np.array_equal(only_img, img) and np.array_equal(img, rgba(index))   # no colours: white


# ---- 6. refusals, edge cases and cancellation --------------------------------------------------------------------------
def _sentinel(h, w):
    """a device image and index filled with a pattern the call would overwrite: a refused call leaves both untouched"""
    import torch
    return (torch.full((h, w, 4), 7, dtype=torch.uint8, device="cuda"),
            torch.full((h, w), -1, dtype=torch.int16, device="cuda"))


def _untouched(out, index):
    import torch
    torch.cuda.synchronize()
    return (out is None or bool((out == 7).all())) and (index is None or bool((index == -1).all()))


@pytest.mark.parametrize("kw", [dict(root_rows=(0, 1)), dict(interleave=(2, 0)), dict(fused_tail=True),
                                dict(out_format="f32")])
def test_unsupported_settings(cuda, kw):
    shape = _shape(cuda, "hi.vm")
    cfg = fb.RenderConfig2D(256, 256, **{"out_format": "rgba8", **kw})
    out, index = _sentinel(256, 256)
    assert _raw(cuda, [shape] * 2, fb.scene_table_2d(cfg, 2), cfg, out, index=index) == -3
    assert _untouched(out, index)


def test_refusals(cuda):
    hi = _shape(cuda, "hi.vm")
    cfg = fb.RenderConfig2D(64, 64, out_format="rgba8")
    out, index = _sentinel(64, 64)
    table = fb.scene_table_2d(cfg, 2)

    def refused(code, tapes, tab, c=cfg, o=out, i=index, n=None):
        assert _raw(cuda, tapes, tab, c, o, n=n, index=i) == code
        assert _untouched(o, i)
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    refused(-3, [hi, spilled], table)
    g = fb.Context()
    two = fb.CudaShape(cuda, g.tape([g.sub(g.x(), 0.5), g.sub(g.y(), 0.5)]))
    refused(-1, [hi, two], table)
    circle, nv, slot = _circle_var(cuda)
    vt = fb.scene_table_2d(cfg, 2, var_values=np.zeros((2, nv), dtype=np.float32))
    vt[1].n_var_values = 0                                   # the second placement binds nothing
    refused(-1, [circle, circle], vt)
    refused(-1, [hi, None], table)
    refused(-1, None, table, n=2)
    refused(-1, [hi, hi], None)
    refused(-1, [hi, hi], table, o=None, i=None)
    refused(-1, [hi], fb.scene_table_2d(cfg, 1), c=fb.RenderConfig2D(0, 64, out_format="rgba8"))
    refused(-3, [hi] * (_lib.FC_SCENE_MAX_SHAPES + 1), fb.scene_table_2d(cfg, _lib.FC_SCENE_MAX_SHAPES + 1))
    refused(0, [], None, n=0)                                 # no shapes: FC_OK, nothing launched or written


def _run(cuda, tok=None):
    cfg = fb.RenderConfig2D(512, 512, out_format="rgba8", cancel=tok)
    return fb.render2d_scene([_shape(cuda, m) for m in MIXED], cfg, world_to_model=mixed(), stats=True)


def test_cancel_on_entry(cuda):
    tok = fb.CancelToken()
    tok.cancel()
    assert _run(cuda, tok) is None
    assert _lib.load().fc_last_error().decode() == "cancelled before the call started"


@pytest.mark.parametrize("site,item", [("k_scene2d_resolve", 5), ("k_pixels_2d", 0), ("k_interval_level1", 3),
                                       ("k_interval_root_coop", 2)])
def test_poll_site_then_next_call_is_correct(cuda, monkeypatch, site, item):
    want = _run(cuda)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:{item}")
    assert _run(cuda, fb.CancelToken()) is None, "the trigger site was never reached"
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    again = _run(cuda)
    assert np.array_equal(again[0], want[0]) and np.array_equal(again[1], want[1])
    assert _stats_fields(again[2]) == _stats_fields(want[2])
