"""fc_render2d_frames / fb.render2d_frames: many frames of one shape in one call.

Every frame must be bit for bit the fc_render2d of the same settings (image and summed census), for Z stacks,
ShapeVars sweeps and view sequences, every out_format, host and device outputs, pixel_perfect and explicit tile
sizes; the reference's goldens and the oracle hold frame by frame; forcing small passes changes nothing; the
refusals, the arena error, cancellation and asynchronous calls behave as fc_render2d's do."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import fidget_b200 as fb
from conftest import model_text
from fidget_b200 import _lib
from test_gpu_fuzz import build as build_random

pytestmark = pytest.mark.gpu

CENSUS = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")
_PIX = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pixel_render.json")))
_SHAPES = {}


def _shape(cuda, name):
    if name not in _SHAPES:
        _SHAPES[name] = fb.CudaShape.from_vm(cuda, model_text(name))
    return _SHAPES[name]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _singles(shape, cfg, table):
    """render2d of every frame of `table` on its own: (images, summed census, summed pixels)"""
    imgs, census, pixels = [], {k: [0] * 8 for k in CENSUS}, 0
    for f in table:
        c = fb.RenderConfig2D(cfg.width, cfg.height, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4), z=f.z,
                              pixel_perfect=cfg.pixel_perfect, tile_sizes=cfg.tile_sizes, out_format=cfg.out_format,
                              var_values=tuple(f.var_values[:f.n_var_values]))
        img, st = fb.render2d(shape, c, stats=True)
        imgs.append(img)
        for k in CENSUS:
            census[k] = [a + b for a, b in zip(census[k], st[k])]
        pixels += st["pixels"]
    return np.stack(imgs) if imgs else None, census, pixels


def _check_against_singles(shape, cfg, **per_frame):
    table = fb.frame_table(cfg, **per_frame)
    got, st = fb.render2d_frames(shape, cfg, stats=True, **per_frame)
    want, census, pixels = _singles(shape, cfg, table)
    assert got.shape == want.shape
    for k in range(len(table)):
        assert np.array_equal(_bits(got[k]), _bits(want[k])), f"frame {k}"
    for k in CENSUS:
        assert st[k] == census[k], k
    assert st["pixels"] == pixels
    return got, st


# ---- 1. bit-identity with single renders ----------------------------------------------------------------------------
@pytest.mark.parametrize("name,size", [("bear.vm", 512), ("gyroid-sphere.vm", 1024), ("colonnade.vm", 768),
                                       ("tanglecube.vm", 512)])
def test_z_stack_equals_single_renders(cuda, name, size):
    zs = np.linspace(-0.9, 0.9, 32, dtype=np.float32)
    _check_against_singles(_shape(cuda, name), fb.RenderConfig2D(size, size), z=zs)


def test_prospero_views_equal_single_renders(cuda):
    views = []
    for k in range(6):
        s = np.float32(0.9 ** k)
        views.append(np.array([[s, 0, 0.05 * k], [0, s, -0.03 * k], [0, 0, 1]], dtype=np.float32))
    _check_against_singles(_shape(cuda, "prospero.vm"), fb.RenderConfig2D(4096, 4096), world_to_model=np.stack(views))


def _circle_var(cuda):
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    c, _ = ctx.var()
    td = ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y))), c))
    slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
    return fb.CudaShape(cuda, td), td.n_vars, slot


def _radii(n_vars, slot, radii):
    vv = np.zeros((len(radii), n_vars), dtype=np.float32)
    vv[:, slot] = radii
    return vv


def test_variable_sweep(cuda):
    shape, nv, slot = _circle_var(cuda)
    radii = np.linspace(0.05, 1.2, 24, dtype=np.float32)
    _check_against_singles(shape, fb.RenderConfig2D(512, 512), var_values=_radii(nv, slot, radii))


def test_ragged_size(cuda):
    _check_against_singles(_shape(cuda, "bear.vm"), fb.RenderConfig2D(1000, 500), z=np.linspace(-0.5, 0.5, 9))


@pytest.mark.parametrize("tiles,perfect", [((64, 16, 4), False), ((256, 32), False), ((), True), ((64, 8), True)])
def test_tile_sizes_and_pixel_perfect(cuda, tiles, perfect):
    cfg = fb.RenderConfig2D(640, 480, tile_sizes=tiles, pixel_perfect=perfect)
    _check_against_singles(_shape(cuda, "colonnade.vm"), cfg, z=np.linspace(-0.6, 0.6, 7))


@pytest.mark.parametrize("fmt", ["f32", "mask_u8", "bitmap_1bit", "rgba8"])
@pytest.mark.parametrize("device_out", [False, True])
def test_out_formats(cuda, fmt, device_out):
    import torch
    cfg = fb.RenderConfig2D(300, 200, out_format=fmt)
    zs = np.linspace(-0.8, 0.8, 5)
    host, _ = _check_against_singles(_shape(cuda, "gyroid-sphere.vm"), cfg, z=zs)
    if device_out:
        dt = torch.float32 if fmt == "f32" else torch.uint8
        out = torch.zeros(host.shape, dtype=dt, device="cuda")
        fb.render2d_frames(_shape(cuda, "gyroid-sphere.vm"), cfg, z=zs, out=out)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(out.cpu().numpy()), _bits(host))


def test_one_and_zero_frames(cuda):
    shape = _shape(cuda, "bear.vm")
    _check_against_singles(shape, fb.RenderConfig2D(512, 512), z=[0.25])
    img, st = fb.render2d_frames(shape, fb.RenderConfig2D(512, 512), z=np.zeros(0), stats=True)
    assert img.shape == (0, 512, 512) and st["kernel_launches"] == 0 and st["evaluated"] == [0] * 8


# ---- 2. goldens and the oracle ----------------------------------------------------------------------------------------
def _rows(img):
    return ["".join("#" if b else "." for b in r) for r in fb.pixel_inside(img)]


def test_golden_circle_with_bound_var_as_two_frames(cuda):
    shape, nv, slot = _circle_var(cuda)
    imgs = fb.render2d_frames(shape, fb.RenderConfig2D(32, 32), var_values=_radii(nv, slot, [0.75, 0.5]))
    assert _rows(imgs[0]) == _PIX["check_circle_var:EXPECTED_075"]["rows"]
    assert _rows(imgs[1]) == _PIX["check_circle_var:EXPECTED_05"]["rows"]


@pytest.mark.parametrize("name", ["colonnade.vm", "tanglecube.vm"])
def test_z_stack_equals_oracle(orc, cuda, name):
    n = 384
    zs = np.linspace(-0.7, 0.7, 12, dtype=np.float32)
    imgs, st = fb.render2d_frames(_shape(cuda, name), fb.RenderConfig2D(n, n), z=zs, stats=True)
    ot = orc.Tape.from_vm(model_text(name))
    census = None
    for k, z in enumerate(zs):
        o_img, o_st = orc.render2d(ot, n, n, z=float(z), threads=8)
        assert np.array_equal(imgs[k].view(np.uint32), o_img.view(np.uint32)), f"frame {k}"
        census = {c: list(o_st[c]) for c in CENSUS} if census is None else \
            {c: [a + b for a, b in zip(census[c], o_st[c])] for c in CENSUS}
    for c in CENSUS:
        m = min(len(st[c]), len(census[c]))
        assert st[c][:m] == census[c][:m], c


@pytest.mark.parametrize("seed", range(6))
def test_random_csg_z_stacks_equal_oracle(orc, cuda, seed):
    rng = np.random.default_rng(4000 + seed)
    g, o, _ = build_random(orc, cuda, 300 + seed, int(rng.integers(10, 50)), use_z=True)
    n = 256
    zs = rng.uniform(-0.8, 0.8, 8).astype(np.float32)
    imgs = fb.render2d_frames(g, fb.RenderConfig2D(n, n), z=zs)
    for k, z in enumerate(zs):
        o_img, _ = orc.render2d(o, n, n, z=float(z), threads=8)
        assert np.array_equal(imgs[k].view(np.uint32), o_img.view(np.uint32)), f"frame {k}"


# ---- 3. passes ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["f32", "bitmap_1bit"])
@pytest.mark.parametrize("per_pass", [1, 3, 7])
def test_forced_passes_change_nothing(cuda, monkeypatch, fmt, per_pass):
    shape = _shape(cuda, "gyroid-sphere.vm")
    cfg = fb.RenderConfig2D(400, 300, out_format=fmt)
    zs = np.linspace(-0.9, 0.9, 17)
    one, st1 = fb.render2d_frames(shape, cfg, z=zs, stats=True)
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(per_pass))
    split, st = fb.render2d_frames(shape, cfg, z=zs, stats=True)
    assert np.array_equal(_bits(split), _bits(one))
    for k in CENSUS + ("pixels",):
        assert st[k] == st1[k], k
    assert st["arena_bytes_used"] <= st1["arena_bytes_used"]


# ---- 4. refusals and errors ---------------------------------------------------------------------------------------------
def _raw_call(cuda, shape, cfg, table, out):
    c = fb.shape._render2d_cfg(cfg, False)
    return _lib.load().fc_render2d_frames(cuda._h, shape._h, C.byref(c), table, len(table), fb.shape._ptr(out), None)


@pytest.mark.parametrize("kw", [dict(fused_tail=True), dict(root_rows=(0, 1)), dict(interleave=(2, 0))])
def test_unsupported_settings(cuda, kw):
    import torch
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig2D(256, 256, **kw)
    out = torch.zeros((2, 256, 256), device="cuda")
    assert _raw_call(cuda, shape, cfg, fb.frame_table(cfg, z=[0, 0.1]), out) == -3


def test_spilled_tape_is_unsupported(cuda):
    shape = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert shape.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.render2d_frames(shape, fb.RenderConfig2D(128, 128), z=[0.0, 0.5])
    assert e.value.code == -3


def test_missing_var_is_invalid(cuda):
    shape, nv, slot = _circle_var(cuda)
    cfg = fb.RenderConfig2D(64, 64)
    table = fb.frame_table(cfg, var_values=_radii(nv, slot, [0.5, 0.5]))
    table[1].n_var_values = 0                              # the second frame binds nothing
    assert _raw_call(cuda, shape, cfg, table, np.zeros((2, 64, 64), np.float32)) == -1
    assert fb.render2d_frames(shape, cfg, var_values=_radii(nv, slot, [0.5])).shape == (1, 64, 64)


def test_small_arena_then_next_call_is_correct(cuda):
    shape = _shape(cuda, "prospero.vm")
    cfg = fb.RenderConfig2D(1024, 1024)
    zs = np.zeros(4)
    want = fb.render2d_frames(shape, cfg, z=zs)
    ctx = fb.CudaContext(0)
    s = fb.CudaShape.from_vm(ctx, model_text("prospero.vm"))
    ctx.set_arena_bytes(1 << 20)
    with pytest.raises(fb.CudaError) as e:
        fb.render2d_frames(s, cfg, z=zs)
    assert e.value.code == -4
    ctx.set_arena_bytes(1 << 30)
    assert np.array_equal(fb.render2d_frames(s, cfg, z=zs).view(np.uint32), want.view(np.uint32))


# ---- 5. cancellation ------------------------------------------------------------------------------------------------------
def _zooms(n):
    return np.stack([np.array([[0.8 ** k, 0, 0.02 * k], [0, 0.8 ** k, 0], [0, 0, 1]], dtype=np.float32) for k in range(n)])


def _sweep(cuda, tok=None, fmt="f32", shape=None):
    """8 zoom views of prospero at 1024^2: 512 root tiles, of which frames 6 and 7 hold the last 128"""
    cfg = fb.RenderConfig2D(1024, 1024, out_format=fmt, cancel=tok)
    return fb.render2d_frames(shape or _shape(cuda, "prospero.vm"), cfg, world_to_model=_zooms(8), stats=True)


# Two views far from prospero (every root tile proven outside at level 0: no work after level 0 but 64 fill records
# each), then two zoom views.  Whatever a site claims beyond what the empty frames can produce belongs to frame 2 or 3.
_EMPTY = np.array([[0.01, 0, 50.0], [0, 0.01, 50.0], [0, 0, 1]], dtype=np.float32)


def _later(cuda, tok=None, shape=None):
    cfg = fb.RenderConfig2D(1024, 1024, cancel=tok)
    views = np.concatenate([np.stack([_EMPTY, _EMPTY]), _zooms(2)])
    return fb.render2d_frames(shape or _shape(cuda, "prospero.vm"), cfg, world_to_model=views, stats=True)


def _later_frame_item(cuda, site):
    """an item of `site` that only frames 2 and 3 produce, derived from the census of the uncancelled call"""
    _, empty = fb.render2d_frames(_shape(cuda, "prospero.vm"), fb.RenderConfig2D(1024, 1024),
                                  world_to_model=np.stack([_EMPTY, _EMPTY]), stats=True)
    assert empty["ambiguous"] == [0] * 8 and empty["filled_outside"][0] == 128   # the empty frames: level-0 fills only
    _, st = _later(cuda)
    if site == "k_interval_root_coop":      # roots are claimed in order, frame by frame: frame 2 starts at root 128
        return 128 + 32
    if site == "k_interval_level1":         # level-1 jobs are the ambiguous roots, all of frames 2 and 3
        assert st["ambiguous"][0] > 2
        return st["ambiguous"][0] // 2
    if site == "k_pixels_2d":               # leaf jobs: the ambiguous tiles of the last level, all of frames 2 and 3
        assert st["ambiguous"][2] > 2
        return st["ambiguous"][2] // 2
    # k_fill_2d claims (record, 1024-pixel unit) items: 16 per level-0 record, 1 per level-1 / level-2 record.  Items
    # beyond the level-0 launch's total (which holds the empty frames' records) exist only in the level-2 launch.
    l0_items = (st["filled_inside"][0] + st["filled_outside"][0]) * 16
    l2_records = st["filled_inside"][2] + st["filled_outside"][2]
    assert l2_records > l0_items + 2, (l0_items, l2_records)
    return (l0_items + l2_records) // 2


@pytest.mark.parametrize("site", ["k_interval_root_coop", "k_interval_level1", "k_fill_2d", "k_pixels_2d"])
def test_poll_sites_in_a_later_frame(cuda, monkeypatch, site):
    want = _later(cuda)
    item = _later_frame_item(cuda, site)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:{item}")
    assert _later(cuda, fb.CancelToken()) is None, "the trigger site was never reached"
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    again = _later(cuda)
    fresh = fb.CudaContext(0)
    f, _ = _later(fresh, shape=fb.CudaShape.from_vm(fresh, model_text("prospero.vm")))
    assert np.array_equal(again[0].view(np.uint32), f.view(np.uint32))
    assert np.array_equal(again[0].view(np.uint32), want[0].view(np.uint32)) and again[1]["evaluated"] == want[1]["evaluated"]


def _costly(cuda):
    """a shape the intervals cannot prune (a sum of many sines): every pixel runs the whole tape on the device"""
    g = fb.Context()
    x, y = g.x(), g.y()
    acc = None
    for k in range(120):
        t = g.sin(g.add(g.mul(x, 3.0 + 0.37 * k), g.mul(y, 2.0 + 0.11 * k)))
        acc = t if acc is None else g.add(acc, t)
    return fb.CudaShape(cuda, g.tape(g.sub(acc, 0.5)))


@pytest.mark.parametrize("per_pass", [32, 4])
def test_cancel_from_a_thread_into_pageable_host_memory(cuda, monkeypatch, per_pass):
    """A host thread sets the flag while 32 frames render into a numpy array (pageable memory, the default output):
    the call returns None, in one pass and in eight."""
    import threading
    import time
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(per_pass))
    shape = _costly(cuda)
    zs = np.linspace(-0.5, 0.5, 32)

    def run(tok):
        return fb.render2d_frames(shape, fb.RenderConfig2D(2048, 2048, out_format="bitmap_1bit", cancel=tok), z=zs)
    want = run(None)
    t0 = time.perf_counter()
    assert np.array_equal(run(fb.CancelToken()), want)          # an unset flag: the whole result
    t_full = time.perf_counter() - t0
    tok = fb.CancelToken()
    stamp = {}

    def setter():
        time.sleep(0.2 * t_full)
        stamp["set"] = time.perf_counter()
        tok.cancel()
    th = threading.Thread(target=setter)
    th.start()
    r = run(tok)
    t_ret = time.perf_counter()
    th.join()
    assert r is None, t_full
    assert _lib.load().fc_last_error().decode() == "cancelled"
    assert t_ret - stamp["set"] < 0.5 * t_full, (t_ret - stamp["set"], t_full)
    assert np.array_equal(run(None), want)                      # the context stays usable


def test_out_too_small_is_refused(cuda):
    import torch
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig2D(256, 128, out_format="bitmap_1bit")
    with pytest.raises(ValueError):
        fb.render2d_frames(shape, cfg, z=[0.0, 0.5, 0.7], out=np.zeros((2, 128, 32), np.uint8))
    with pytest.raises(ValueError):
        fb.render2d_frames(shape, cfg, z=[0.0, 0.5], out=torch.zeros((2, 128, 64), dtype=torch.uint8, device="cuda")[:, :, ::2])
    out = torch.zeros((3, 128, 32), dtype=torch.uint8, device="cuda")
    assert fb.render2d_frames(shape, cfg, z=[0.0, 0.5, 0.7], out=out) is out


@pytest.mark.parametrize("fmt", ["f32", "bitmap_1bit"])
def test_unset_token_changes_nothing(cuda, fmt):
    a, sa = _sweep(cuda, fb.CancelToken(), fmt)
    b, sb = _sweep(cuda, None, fmt)
    assert np.array_equal(_bits(a), _bits(b))
    for k in CENSUS + ("pixels", "arena_bytes_used"):
        assert sa[k] == sb[k], k


# ---- 6. asynchronous -------------------------------------------------------------------------------------------------------
def test_asynchronous_into_a_cuda_tensor(cuda):
    import torch
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig2D(512, 512)
    zs = np.linspace(-0.5, 0.5, 6)
    want = fb.render2d_frames(shape, cfg, z=zs)
    out = torch.zeros((6, 512, 512), device="cuda")
    assert fb.render2d_frames(shape, cfg, z=zs, out=out, asynchronous=True) is out
    cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
