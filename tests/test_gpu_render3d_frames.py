"""fc_render3d_frames / fb.render3d_frames: many 3D frames of one shape in one call.

Every frame must be bit for bit the fc_render3d of the same settings (depth and all three normal floats, and the summed
census), for orbits, zoom sequences and ShapeVars sweeps, ragged volumes, explicit tile sizes, the full ladder and
clamp=False; forced pass sizes and every kind of output change nothing; a batch fails for arena overflow only where one
frame alone does; the reference's sphere sweep and the oracle hold frame by frame; cancellation and the refusals behave
as fc_render3d's do."""
import ctypes as C

import numpy as np
import pytest

import fidget_b200 as fb
from conftest import model_text, same_f32
from fidget_b200 import _lib

pytestmark = pytest.mark.gpu

CENSUS = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")
# `pixels` without the exact census counts the voxels k_voxels_3d evaluated, which depends on when other warps finish
# the columns a tile skips: it varies between two fc_render3d calls of the same settings, so it is compared only under
# FC_FLAG_EXACT_CENSUS; the census, `grads` and the image do not depend on timing
DETERMINISTIC = CENSUS + ("grads",)
_SHAPES = {}


def _shape(cuda, name):
    key = (id(cuda), name)
    if key not in _SHAPES:
        _SHAPES[key] = (cuda, fb.CudaShape.from_vm(cuda, model_text(name)))
    return _SHAPES[key][1]


def _bits(img):
    return np.ascontiguousarray(img).view(np.uint32)


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]], dtype=np.float32)


def _orbit(n):
    return np.stack([_rot_y(2 * np.pi * k / n) for k in range(n)])


def _zooms(n, shift=0.0):
    return np.stack([np.array([[0.85 ** k, 0, 0, shift * k], [0, 0.85 ** k, 0, -0.5 * shift * k], [0, 0, 0.85 ** k, 0],
                               [0, 0, 0, 1]], dtype=np.float32) for k in range(n)])


def _single_cfg(cfg, f):
    return fb.RenderConfig3D(cfg.width, cfg.height, cfg.depth, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4),
                             tile_sizes=cfg.tile_sizes, clamp=cfg.clamp, exact_census=cfg.exact_census,
                             full_ladder=cfg.full_ladder, var_values=tuple(f.var_values[:f.n_var_values]))


def _singles(shape, cfg, table):
    """render3d of every frame of `table` on its own: (images, summed stats; "launches": those of one call)"""
    imgs, tot = [], {k: [0] * 8 for k in CENSUS}
    tot.update(pixels=0, grads=0, arena=0, launches=0)
    for f in table:
        img, st = fb.render3d(shape, _single_cfg(cfg, f), stats=True)
        imgs.append(img)
        for k in CENSUS:
            tot[k] = [a + b for a, b in zip(tot[k], st[k])]
        tot["pixels"] += st["pixels"]
        tot["grads"] += st["grads"]
        tot["arena"] = max(tot["arena"], st["arena_bytes_used"])
        tot["launches"] = max(tot["launches"], st["kernel_launches"])
    return np.stack(imgs), tot


def _check(shape, cfg, **per_frame):
    table = fb.frame_table_3d(cfg, **per_frame)
    got, st = fb.render3d_frames(shape, cfg, stats=True, **per_frame)
    want, tot = _singles(shape, cfg, table)
    assert got.shape == want.shape == (len(table), cfg.height, cfg.width)
    for k in range(len(table)):
        assert np.array_equal(_bits(got[k]), _bits(want[k])), f"frame {k}"
    for k in DETERMINISTIC + (("pixels",) if cfg.exact_census else ()):
        assert st[k] == tot[k], k
    return got, st, tot


# ---- 1. bit-identity with single renders ------------------------------------------------------------------------------
def test_bear_orbit_256(cuda):
    _check(_shape(cuda, "bear.vm"), fb.RenderConfig3D(256, 256, 256), world_to_model=_orbit(24))


@pytest.mark.parametrize("name", ["colonnade.vm", "tanglecube.vm"])
def test_views_512(cuda, name):
    _check(_shape(cuda, name), fb.RenderConfig3D(512, 512, 512), world_to_model=_orbit(8))


def test_gyroid_sphere_zoom(cuda):
    _check(_shape(cuda, "gyroid-sphere.vm"), fb.RenderConfig3D(384, 384, 384), world_to_model=_zooms(10, 0.03))


def test_prospero_views_1024(cuda):
    _check(_shape(cuda, "prospero.vm"), fb.RenderConfig3D(1024, 1024, 1024), world_to_model=_zooms(4, 0.05))


@pytest.mark.parametrize("name", ["bear.vm", "colonnade.vm"])
def test_ragged_volume(cuda, name):
    """200 x 136 x 72: a tile overhanging a frame's bottom edge must not raise the next frame's heightmap or blocks"""
    _check(_shape(cuda, name), fb.RenderConfig3D(200, 136, 72), world_to_model=_orbit(7))


@pytest.mark.parametrize("kw", [dict(tile_sizes=(64, 16, 4)), dict(tile_sizes=(128, 32)), dict(full_ladder=True),
                                dict(clamp=False)])
def test_tile_sizes_ladder_and_clamp(cuda, kw):
    _check(_shape(cuda, "bear.vm"), fb.RenderConfig3D(320, 240, 200, **kw), world_to_model=_orbit(5))


def _sphere_var(cuda):
    g = fb.Context()
    x, y, z = g.x(), g.y(), g.z()
    r, _ = g.var()
    td = g.tape(g.sub(g.sqrt(g.add(g.add(g.square(x), g.square(y)), g.square(z))), r))
    slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
    return fb.CudaShape(cuda, td), td.n_vars, slot


def _radii(n_vars, slot, radii):
    vv = np.zeros((len(radii), n_vars), dtype=np.float32)
    vv[:, slot] = radii
    return vv


def test_variable_sweep(cuda):
    shape, nv, slot = _sphere_var(cuda)
    _check(shape, fb.RenderConfig3D(256, 256, 256), var_values=_radii(nv, slot, np.linspace(0.05, 1.1, 20)))


# ---- 2. stats ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("census", [False, True])
def test_summed_stats(cuda, census):
    _, st, tot = _check(_shape(cuda, "bear.vm"), fb.RenderConfig3D(256, 384, 256, exact_census=census),
                        world_to_model=_orbit(6))
    assert st["arena_bytes_used"] >= tot["arena"] > 0


# ---- 3. passes and outputs --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_pass", [1, 2, 3])
def test_forced_passes_change_nothing(cuda, monkeypatch, per_pass):
    shape = _shape(cuda, "gyroid-sphere.vm")
    cfg = fb.RenderConfig3D(200, 136, 136)
    one, st1 = fb.render3d_frames(shape, cfg, world_to_model=_orbit(7), stats=True)
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(per_pass))
    split, st = fb.render3d_frames(shape, cfg, world_to_model=_orbit(7), stats=True)
    assert np.array_equal(_bits(split), _bits(one))
    for k in DETERMINISTIC:
        assert st[k] == st1[k], k


@pytest.mark.parametrize("kind", ["device", "pinned", "pageable"])
def test_outputs(cuda, kind):
    import torch
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(256, 200, 128)
    want = fb.render3d_frames(shape, cfg, world_to_model=_orbit(5))
    if kind == "pageable":
        out = np.zeros_like(want)
    else:
        out = torch.zeros((5, 200, 256, 4), dtype=torch.int32, device="cuda" if kind == "device" else "cpu",
                          pin_memory=kind == "pinned")
    assert fb.render3d_frames(shape, cfg, world_to_model=_orbit(5), out=out) is out
    got = out if kind == "pageable" else out.cpu().numpy()
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint32).reshape(-1), _bits(want).reshape(-1))


@pytest.mark.parametrize("case", ["bear orbit", "sphere sweep"])
def test_frames_share_passes(cuda, case):
    """The batch really runs its frames together: a 24-frame call launches a few passes' kernels, not 24 frames'.  Most
    or all root tiles of these frames are ambiguous, which must not shrink the passes to one frame."""
    cfg = fb.RenderConfig3D(256, 256, 256)
    if case == "bear orbit":
        shape, kw = _shape(cuda, "bear.vm"), dict(world_to_model=_orbit(24))
    else:
        shape, nv, slot = _sphere_var(cuda)
        kw = dict(var_values=_radii(nv, slot, np.linspace(0.2, 1.2, 24)))
    _, one = fb.render3d(shape, _single_cfg(cfg, fb.frame_table_3d(cfg, **kw)[0]), stats=True)
    _, st = fb.render3d_frames(shape, cfg, stats=True, **kw)
    if case == "sphere sweep":   # every root octant touches the centre: all 8 roots of each frame are ambiguous
        assert st["ambiguous"][0] == 24 * 8
    assert st["kernel_launches"] <= 4 * one["kernel_launches"], (st["kernel_launches"], one["kernel_launches"])


def test_one_and_zero_frames(cuda):
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(256, 256, 256)
    _check(shape, cfg, world_to_model=_orbit(1))
    img, st = fb.render3d_frames(shape, cfg, mats=np.zeros((0, 4, 4)), stats=True)
    assert img.shape == (0, 256, 256) and st["kernel_launches"] == 0 and st["evaluated"] == [0] * 8


def test_asynchronous_into_a_cuda_tensor(cuda):
    import torch
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(256, 256, 256)
    want = fb.render3d_frames(shape, cfg, world_to_model=_orbit(6))
    out = torch.zeros((6, 256, 256, 4), dtype=torch.int32, device="cuda")
    assert fb.render3d_frames(shape, cfg, world_to_model=_orbit(6), out=out, asynchronous=True) is out
    cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32).reshape(-1), _bits(want).reshape(-1))


# ---- 4. overflow policy -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("forced", [0, 16])
def test_small_arena_batch_equals_singles(cuda, monkeypatch, forced):
    """An arena of 1.5x the largest single frame's use: 16 frames do not fit one pass, and the batch still equals the
    singles (sized from the first frame's use, or, with 16 frames forced into one pass, split in halves on overflow).
    A pass makes the launches of one single call, overflowed passes included, so the launch count says how many ran."""
    cfg = fb.RenderConfig3D(512, 512, 512)
    views = _orbit(16)
    want, tot = _singles(_shape(cuda, "prospero.vm"), cfg, fb.frame_table_3d(cfg, world_to_model=views))
    arena = max(1 << 20, int(1.5 * tot["arena"]))
    assert 16 * tot["arena"] > arena
    ctx = fb.CudaContext(0)
    shape = fb.CudaShape.from_vm(ctx, model_text("prospero.vm"))
    ctx.set_arena_bytes(arena)
    if forced:
        monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(forced))
    got, st = fb.render3d_frames(shape, cfg, world_to_model=views, stats=True)
    assert np.array_equal(_bits(got), _bits(want))
    for k in DETERMINISTIC:
        assert st[k] == tot[k], k
    assert st["arena_bytes_used"] <= arena
    passes, rest = divmod(st["kernel_launches"], tot["launches"])
    assert rest == 0 and passes >= (3 if forced else 2), (st["kernel_launches"], tot["launches"])


def test_arena_too_small_for_one_frame(cuda):
    cfg = fb.RenderConfig3D(1024, 1024, 1024)
    views = _zooms(3, 0.02)
    want = fb.render3d_frames(_shape(cuda, "prospero.vm"), cfg, world_to_model=views)
    ctx = fb.CudaContext(0)
    shape = fb.CudaShape.from_vm(ctx, model_text("prospero.vm"))
    ctx.set_arena_bytes(1 << 20)
    with pytest.raises(fb.CudaError) as e:
        fb.render3d_frames(shape, cfg, world_to_model=views)
    assert e.value.code == -4
    del e   # (its traceback holds this frame: without the cycle, shape is released before its context)
    ctx.set_arena_bytes(1 << 30)
    assert np.array_equal(_bits(fb.render3d_frames(shape, cfg, world_to_model=views)), _bits(want))


# ---- 5. the reference's sphere sweep, and the oracle -------------------------------------------------------------------
def test_golden_sphere_sweep_as_frames(cuda):
    """fidget/tests/voxel_render.rs:13-75 (sphere_var + check_sphere) as the four frames of one call: radius 0.5 and
    0.75 through View3 cameras of scale 1 and 0.5, each within two voxels of the analytic surface"""
    shape, nv, slot = _sphere_var(cuda)
    size = 32
    cfg = fb.RenderConfig3D(size, size, size)
    cases = [(scale, radius) for scale in (1.0, 0.5) for radius in (0.5, 0.75)]
    wm = np.stack([np.diag([s, s, s, 1.0]).astype(np.float32) for s, _ in cases])
    imgs = fb.render3d_frames(shape, cfg, world_to_model=wm, var_values=_radii(nv, slot, [r for _, r in cases]))
    m = fb.screen_to_world_3d(size, size, size).astype(np.float64)
    for k, (scale, radius) in enumerate(cases):
        eps = 2.0 / size / scale * 2.0
        depth = imgs[k]["depth"].astype(np.int64)
        ys, xs = np.mgrid[0:size, 0:size]
        pts = np.stack([xs, ys, depth, np.ones_like(xs)], axis=-1).astype(np.float64) @ m.T
        pos = pts[..., :3] / pts[..., 3:4] * scale
        empty, hit = depth == 0, (depth != 0) & (depth != size)
        assert hit.sum() > 20
        assert (np.hypot(pos[..., 0], pos[..., 1])[empty] + eps > radius).all()
        assert (np.abs(radius - np.linalg.norm(pos, axis=-1))[hit] < eps).all()


@pytest.mark.parametrize("name", ["colonnade.vm", "tanglecube.vm"])
def test_scaled_views_equal_oracle(orc, cuda, name):
    """scale-and-translate views of IEEE models: each frame is the oracle's voxel::render bit for bit, and the exact
    census is the sum of the oracle's front-to-back walks"""
    n = 256
    views = _zooms(5, 0.04)
    mats = np.stack([fb.voxel_mat(n, n, n, v) for v in views])
    imgs, st = fb.render3d_frames(_shape(cuda, name), fb.RenderConfig3D(n, n, n, exact_census=True), mats=mats, stats=True)
    ot = orc.Tape.from_vm(model_text(name))
    census, pixels = {c: [0] * 8 for c in CENSUS}, 0
    for k in range(len(mats)):
        o_img, o_st = orc.render3d(ot, n, n, n, mat=mats[k], threads=8)
        assert np.array_equal(imgs[k]["depth"], o_img["depth"]), f"frame {k}"
        assert same_f32(imgs[k]["normal"], o_img["normal"]), f"frame {k}"
        for c in CENSUS:
            census[c] = [a + b for a, b in zip(census[c], o_st[c])]
        pixels += o_st["pixels"]
    for c in CENSUS:
        assert st[c] == census[c], c
    assert st["pixels"] == pixels


# ---- 6. cancellation --------------------------------------------------------------------------------------------------
def _run(cuda, tok=None):
    cfg = fb.RenderConfig3D(256, 256, 256, cancel=tok)
    return fb.render3d_frames(_shape(cuda, "bear.vm"), cfg, world_to_model=_orbit(8), stats=True)


def test_cancel_on_entry(cuda):
    tok = fb.CancelToken()
    tok.cancel()
    assert _run(cuda, tok) is None
    assert _lib.load().fc_last_error().decode() == "cancelled before the call started"


@pytest.mark.parametrize("site,item", [("k_voxels_3d", 0), ("k_normals_3d", 2048 + 5), ("k_interval_level1", 3)])
def test_poll_site_then_next_call_is_correct(cuda, monkeypatch, site, item):
    """with two frames per pass, k_normals_3d item 2048 + 5 is a patch of the second frame (2048 patches per frame)"""
    want = _run(cuda)
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", "2")
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:{item}")
    assert _run(cuda, fb.CancelToken()) is None, "the trigger site was never reached"
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    again = _run(cuda)
    assert np.array_equal(_bits(again[0]), _bits(want[0]))
    for k in DETERMINISTIC:
        assert again[1][k] == want[1][k], k


def test_unset_token_changes_nothing(cuda):
    a, sa = _run(cuda, fb.CancelToken())
    b, sb = _run(cuda)
    assert np.array_equal(_bits(a), _bits(b))
    for k in DETERMINISTIC + ("arena_bytes_used",):
        assert sa[k] == sb[k], k


# ---- 7. refusals and errors -------------------------------------------------------------------------------------------
def _raw_call(cuda, shape, cfg, table, out):
    c = fb.shape._render3d_cfg(cfg, False)
    return _lib.load().fc_render3d_frames(cuda._h, shape._h, C.byref(c), table, len(table), fb.shape._ptr(out), None)


@pytest.mark.parametrize("kw", [dict(z_range=(0, 128)), dict(root_rows=(0, 1)), dict(interleave=(2, 0))])
def test_unsupported_settings(cuda, kw):
    import torch
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(256, 256, 256, **kw)
    out = torch.zeros((2, 256, 256, 4), dtype=torch.int32, device="cuda")
    assert _raw_call(cuda, shape, cfg, fb.frame_table_3d(cfg, world_to_model=_orbit(2)), out) == -3


def test_spilled_tape_is_unsupported(cuda):
    shape = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert shape.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.render3d_frames(shape, fb.RenderConfig3D(64, 64, 64), world_to_model=_orbit(2))
    assert e.value.code == -3


def test_missing_var_and_multi_output_are_invalid(cuda):
    shape, nv, slot = _sphere_var(cuda)
    cfg = fb.RenderConfig3D(64, 64, 64)
    table = fb.frame_table_3d(cfg, var_values=_radii(nv, slot, [0.5, 0.5]))
    table[1].n_var_values = 0                              # the second frame binds nothing
    assert _raw_call(cuda, shape, cfg, table, np.zeros((2, 64, 64), fb.GEOMETRY_PIXEL)) == -1
    g = fb.Context()
    two = fb.CudaShape(cuda, g.tape([g.sub(g.x(), 0.5), g.sub(g.y(), 0.5)]))
    with pytest.raises(fb.CudaError) as e:
        fb.render3d_frames(two, cfg, world_to_model=_orbit(2))
    assert e.value.code == -1
    lib = _lib.load()
    c = fb.shape._render3d_cfg(cfg, False)
    assert lib.fc_render3d_frames(cuda._h, shape._h, C.byref(c), None, 2, fb.shape._ptr(np.zeros((2, 64, 64), fb.GEOMETRY_PIXEL)),
                                  None) == -1
