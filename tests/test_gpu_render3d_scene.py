"""fc_render3d_scene / fb.render3d_scene: several shapes rendered into one image in one call.

The image and index must be, bit for bit, the fold of the per-shape fb.render3d images (tests/scene_merge.py: the
greatest clamped depth wins, the lowest index on equal depth): for occluding queues, grids and mixed tapes, ragged
volumes, tile sizes, the full ladder, clamp off and per-placement ShapeVars.  Exact ties (f against 2f, raw D - 1
against raw D) pin the tie rule through culling and the column skip; passes, outputs, stats, refusals and cancellation
behave as fc_render3d_frames's do."""
import ctypes as C

import numpy as np
import pytest

import fidget_b200 as fb
from conftest import model_text, same_f32
from fidget_b200 import _lib
from scene_merge import fold

pytestmark = pytest.mark.gpu

CENSUS = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")
_SHAPES = {}


def _shape(cuda, name):
    key = (id(cuda), name)
    if key not in _SHAPES:
        _SHAPES[key] = (cuda, fb.CudaShape.from_vm(cuda, model_text(name)))
    return _SHAPES[key][1]


def _bits(img):
    return np.ascontiguousarray(img).view(np.uint32)


def _place(scale, tx, ty, tz):
    """world -> model of a shape scaled by `scale` and centred at (tx, ty, tz) in world space"""
    s = 1.0 / scale
    return np.array([[s, 0, 0, -tx * s], [0, s, 0, -ty * s], [0, 0, s, -tz * s], [0, 0, 0, 1]], dtype=np.float32)


def queue(n=8):
    """n instances one behind the other along the view axis (front first), each peeking out of the one before"""
    return np.stack([_place(0.5, -0.45 + 0.13 * k, 0.4 - 0.11 * k, 0.45 - 0.13 * k) for k in range(n)])


def grid(n=4):
    return np.stack([_place(0.22, -0.75 + 0.5 * i, -0.75 + 0.5 * j, 0.05 * (i - j)) for j in range(n) for i in range(n)])


MIXED = ("colonnade.vm", "tanglecube.vm", "gyroid-sphere.vm", "bear.vm")


def mixed():
    return np.stack([_place(0.6, -0.3, 0.2, 0.1), _place(0.55, 0.3, 0.25, 0.0), _place(0.5, -0.2, -0.3, 0.2),
                     _place(0.6, 0.25, -0.2, 0.15)])


def _single_cfg(cfg, f):
    return fb.RenderConfig3D(cfg.width, cfg.height, cfg.depth, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4),
                             tile_sizes=cfg.tile_sizes, clamp=cfg.clamp, full_ladder=cfg.full_ladder,
                             var_values=tuple(f.var_values[:f.n_var_values]))


def _singles(shapes, cfg, **per):
    table = fb.scene_table(cfg, len(shapes), **per)
    return [fb.render3d(sh, _single_cfg(cfg, table[k]), stats=True) for k, sh in enumerate(shapes)]


def _check(shapes, cfg, **per):
    got, index, st = fb.render3d_scene(shapes, cfg, stats=True, **per)
    singles = _singles(shapes, cfg, **per)
    want, want_index = fold([img for img, _ in singles])
    assert np.array_equal(_bits(got), _bits(want))
    assert np.array_equal(index, want_index)
    return got, index, st, singles


# ---- 1. bit-identity with the fold of per-shape renders ---------------------------------------------------------------
@pytest.mark.parametrize("n", [256, 512])
def test_queue(cuda, n):
    bear = _shape(cuda, "bear.vm")
    _, index, st, singles = _check([bear] * 8, fb.RenderConfig3D(n, n, n), world_to_model=queue())
    assert len(np.unique(index)) >= 4                   # the instances peek out
    assert sum(sum(s["evaluated"]) for _, s in singles) >= sum(st["evaluated"])   # culled behind the front ones, if any


def test_grid(cuda):
    _check([_shape(cuda, "bear.vm")] * 16, fb.RenderConfig3D(512, 512, 256), world_to_model=grid())


def test_mixed(cuda):
    _, index, _, _ = _check([_shape(cuda, m) for m in MIXED], fb.RenderConfig3D(512, 512, 512), world_to_model=mixed())
    assert len(np.unique(index)) == 4


def test_ragged_volume(cuda):
    shapes = [_shape(cuda, m) for m in MIXED] + [_shape(cuda, "bear.vm")] * 2
    views = np.concatenate([mixed(), queue(2)])
    _check(shapes, fb.RenderConfig3D(200, 136, 72), world_to_model=views)


@pytest.mark.parametrize("kw", [dict(tile_sizes=(64, 16, 4)), dict(tile_sizes=(128, 32)), dict(full_ladder=True),
                                dict(clamp=False)])
def test_tile_sizes_ladder_and_clamp(cuda, kw):
    _check([_shape(cuda, "bear.vm")] * 5, fb.RenderConfig3D(320, 240, 200, **kw), world_to_model=queue(5))


def _sphere_var(cuda):
    g = fb.Context()
    x, y, z = g.x(), g.y(), g.z()
    r, _ = g.var()
    td = g.tape(g.sub(g.sqrt(g.add(g.add(g.square(x), g.square(y)), g.square(z))), r))
    slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
    return fb.CudaShape(cuda, td), td.n_vars, slot


def test_per_placement_vars(cuda):
    shape, nv, slot = _sphere_var(cuda)
    radii = np.linspace(0.1, 0.45, 6)
    vv = np.zeros((6, nv), dtype=np.float32)
    vv[:, slot] = radii
    views = np.stack([_place(1.0, -0.5 + 0.2 * k, 0.1 * k - 0.2, -0.1 * k) for k in range(6)])
    _check([shape] * 6, fb.RenderConfig3D(256, 256, 256), var_values=vv, world_to_model=views)


def test_one_shape_is_render3d(cuda):
    bear = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(512, 512, 512)
    img, index, st = fb.render3d_scene([bear], cfg, stats=True)
    want, wst = fb.render3d(bear, cfg, stats=True)
    assert np.array_equal(_bits(img), _bits(want)) and not index.any()
    assert st["grads"] == wst["grads"]
    assert all(a >= b for a, b in zip(st["evaluated"], wst["evaluated"]))


# ---- 2. ties, pinned exactly -----------------------------------------------------------------------------------------
def _sphere_and_double(cuda):
    g = fb.Context()
    f = g.sub(g.sqrt(g.add(g.add(g.square(g.x()), g.square(g.y())), g.square(g.z()))), 0.6)
    return fb.CudaShape(cuda, g.tape(f)), fb.CudaShape(cuda, g.tape(g.mul(f, 2.0)))


# The tie tests run each pair two ways.  "alone": the default passes, so the first placement runs in a pass of its own.
# "led": both tied placements in ONE pass (FIDGET_B200_FRAMES_PER_PASS=3), behind a leader that shares the tape of the
# higher-index one and stays out of the way.  Level 0 runs per tape in order of first appearance, so the higher-index
# placement's tiles are queued, and mostly evaluated, before the lower-index ones: a tile of the lower index then meets
# the equal depth the higher one already stored, and only the rank comparisons of parent culling and of the column
# skip keep it from being culled or skipped.  Comparing depths alone, as fc_render3d does, hands those pixels to the
# higher index.  The "led" images are large enough (1024 wide) that the leaf tiles of one Z layer run in several waves,
# so such meetings happen on many pixels rather than by chance.
_AWAY = np.array([[1, 0, 0, 5], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float32)   # model x = world x + 5


def _tied(monkeypatch, arrangement, lower, higher, cfg, views=None):
    """render3d_scene of `lower` tied with `higher` (lower index first); returns the image and the index of the pair"""
    if arrangement == "alone":
        kw = {} if views is None else dict(mats=np.stack([views[0], views[0]]))
        return fb.render3d_scene([lower, higher], cfg, **kw)
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", "3")
    img, index = fb.render3d_scene([higher, lower, higher], cfg, **(
        dict(world_to_model=np.stack([_AWAY, np.eye(4, dtype=np.float32), np.eye(4, dtype=np.float32)]))
        if views is None else dict(mats=np.stack(views))))
    if views is None:
        assert not (index == 0)[img["depth"] > 0].any()     # the leader is out of view
    return img, np.where(index > 0, index - 1, 0).astype(np.uint16)


@pytest.mark.parametrize("arrangement", ["alone", "led"])
@pytest.mark.parametrize("kw", [dict(), dict(full_ladder=True), dict(clamp=False)])
def test_f_and_2f_tie(cuda, monkeypatch, kw, arrangement):
    """same zero set and tile decisions, normals exactly twice as large: the lower index wins every pixel"""
    f, f2 = _sphere_and_double(cuda)
    n = 256 if arrangement == "alone" else 1024
    cfg = fb.RenderConfig3D(n, n, n, **kw)
    one, two = fb.render3d(f, cfg), fb.render3d(f2, cfg)
    assert np.array_equal(one["depth"], two["depth"])
    hit = (one["depth"] > 0) & (one["depth"] < n - 1)
    assert hit.sum() > 1000 and not np.array_equal(one["normal"][hit], two["normal"][hit])
    for lower, higher, want in ((f2, f, two), (f, f2, one)):
        img, index = _tied(monkeypatch, arrangement, lower, higher, cfg)
        assert np.array_equal(_bits(img), _bits(want)) and not index.any()


def _half_space(cuda, c):
    g = fb.Context()
    return fb.CudaShape(cuda, g.tape(g.sub(g.z(), c)))


@pytest.mark.parametrize("arrangement", ["alone", "led"])
def test_clamp_tie(cuda, monkeypatch, arrangement):
    """with mats = identity the model z is the voxel z: z < D - 1.5 reaches raw depth D - 1, z < D - 0.5 raw depth D.
    With the clamp both are D and the lower index wins, in both orders; without it raw depth D wins.  (The leader of the
    "led" arrangement is moved 40 voxels down the view axis: it reaches depth 24 only.)"""
    D = 64
    W = 64 if arrangement == "alone" else 1024
    lo, hi = _half_space(cuda, D - 1.5), _half_space(cuda, D - 0.5)
    eye = np.eye(4, dtype=np.float32)
    down = eye.copy()
    down[2, 3] = 40.0                                        # model z = voxel z + 40
    views = [down, eye, eye] if arrangement == "led" else [eye]
    assert (fb.render3d(lo, fb.RenderConfig3D(W, W, D, mat=eye, clamp=False))["depth"] == D - 1).all()
    for lower, higher in ((lo, hi), (hi, lo)):
        img, index = _tied(monkeypatch, arrangement, lower, higher, fb.RenderConfig3D(W, W, D), views)
        assert (img["depth"] == D).all() and not index.any()
        assert (img["normal"] == np.array([0, 0, 1], dtype=np.float32)).all()
        img, index = _tied(monkeypatch, arrangement, lower, higher, fb.RenderConfig3D(W, W, D, clamp=False), views)
        assert (img["depth"] == D).all() and (index == [lower, higher].index(hi)).all()


# ---- 3. against the oracle --------------------------------------------------------------------------------------------
def test_oracle_fold(orc, cuda):
    n = 256
    names = ("colonnade.vm", "quarter.vm", "tanglecube.vm")
    views = np.stack([_place(0.7, -0.2, 0.1, 0.1), _place(0.6, 0.2, 0.0, 0.0), _place(0.6, 0.0, -0.2, 0.2)])
    mats = np.stack([fb.voxel_mat(n, n, n, v) for v in views])
    img, index = fb.render3d_scene([_shape(cuda, m) for m in names], fb.RenderConfig3D(n, n, n), mats=mats)
    oimgs = [orc.render3d(orc.Tape.from_vm(model_text(m)), n, n, n, mat=mats[k], threads=8)[0] for k, m in enumerate(names)]
    want, want_index = fold(oimgs)
    assert np.array_equal(img["depth"], want["depth"])
    assert same_f32(img["normal"], want["normal"])
    assert np.array_equal(index, want_index)


# ---- 4. passes --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_pass", [1, 3])
def test_forced_passes_change_nothing(cuda, monkeypatch, per_pass):
    shapes = [_shape(cuda, m) for m in MIXED] * 2
    views = np.concatenate([mixed(), queue(4)])
    cfg = fb.RenderConfig3D(256, 256, 256)
    one = fb.render3d_scene(shapes, cfg, world_to_model=views)
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(per_pass))
    split = fb.render3d_scene(shapes, cfg, world_to_model=views)
    assert np.array_equal(_bits(split[0]), _bits(one[0])) and np.array_equal(split[1], one[1])


@pytest.mark.parametrize("forced", [0, 8])
def test_small_arena_changes_nothing(cuda, monkeypatch, forced):
    """an arena of 1.5x the largest single shape's use: the eight placements do not fit one pass (with eight forced into
    one, it overflows and is restored and split), and the image is still the fold.  A pass of one tape makes the launches
    of one render3d call, overflowed passes included, so the launch count says how many ran."""
    cfg = fb.RenderConfig3D(512, 512, 512)
    views = queue()
    singles = _singles([_shape(cuda, "prospero.vm")] * 8, cfg, world_to_model=views)
    want, want_index = fold([img for img, _ in singles])
    use = max(s["arena_bytes_used"] for _, s in singles)
    arena = max(1 << 20, int(1.5 * use))
    assert 8 * use > arena
    ctx = fb.CudaContext(0)
    shape = fb.CudaShape.from_vm(ctx, model_text("prospero.vm"))
    ctx.set_arena_bytes(arena)
    if forced:
        monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", str(forced))
    img, index, st = fb.render3d_scene([shape] * 8, cfg, world_to_model=views, stats=True)
    assert np.array_equal(_bits(img), _bits(want)) and np.array_equal(index, want_index)
    assert st["arena_bytes_used"] <= arena
    one = singles[0][1]["kernel_launches"]
    passes, rest = divmod(st["kernel_launches"], one)
    assert rest == 0 and passes >= (3 if forced else 2), (st["kernel_launches"], one)


def test_error_only_where_one_placement_overflows(cuda):
    cfg = fb.RenderConfig3D(1024, 1024, 1024)
    ctx = fb.CudaContext(0)
    shape = fb.CudaShape.from_vm(ctx, model_text("prospero.vm"))
    ctx.set_arena_bytes(1 << 20)
    with pytest.raises(fb.CudaError) as e:
        fb.render3d_scene([shape] * 3, cfg, world_to_model=queue(3))
    assert e.value.code == -4
    del e   # (its traceback holds this frame: without the cycle, shape is released before its context)
    ctx.set_arena_bytes(1 << 30)
    want = fb.render3d_scene([_shape(cuda, "prospero.vm")] * 3, cfg, world_to_model=queue(3))
    got = fb.render3d_scene([shape] * 3, cfg, world_to_model=queue(3))
    assert np.array_equal(_bits(got[0]), _bits(want[0])) and np.array_equal(got[1], want[1])


# ---- 5. stats ---------------------------------------------------------------------------------------------------------
def test_identical_calls_give_equal_stats(cuda):
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig3D(512, 512, 512)
    a = fb.render3d_scene(shapes, cfg, world_to_model=mixed(), stats=True)[2]
    b = fb.render3d_scene(shapes, cfg, world_to_model=mixed(), stats=True)[2]
    for k in CENSUS + ("grads", "arena_bytes_used", "kernel_launches"):
        assert a[k] == b[k], k
    assert a["grads"] > 0 and a["kernel_launches"] > 0


# ---- 6. output memory -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["device", "pinned", "pageable", "async"])
def test_outputs(cuda, kind):
    import torch
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig3D(256, 200, 128)
    want, want_index = fb.render3d_scene(shapes, cfg, world_to_model=mixed())
    if kind == "pageable":
        out, index = np.zeros_like(want), np.zeros_like(want_index)
    else:
        dev = "cpu" if kind == "pinned" else "cuda"
        out = torch.zeros((200, 256, 4), dtype=torch.int32, device=dev, pin_memory=kind == "pinned")
        index = torch.zeros((200, 256), dtype=torch.int16, device=dev, pin_memory=kind == "pinned")
    got = fb.render3d_scene(shapes, cfg, world_to_model=mixed(), out=out, index_out=index, asynchronous=kind == "async")
    assert got[0] is out and got[1] is index
    if kind == "async":
        cuda.synchronize()
    o = out if kind == "pageable" else out.cpu().numpy()
    i = index if kind == "pageable" else index.cpu().numpy().view(np.uint16)
    assert np.array_equal(np.ascontiguousarray(o).view(np.uint32).reshape(-1), _bits(want).reshape(-1))
    assert np.array_equal(i, want_index)


def test_default_index_follows_a_cuda_out(cuda):
    """without index_out a CUDA out gets a CUDA index, so an asynchronous call stays asynchronous"""
    import torch
    shapes = [_shape(cuda, m) for m in MIXED]
    cfg = fb.RenderConfig3D(256, 200, 128)
    want, want_index = fb.render3d_scene(shapes, cfg, world_to_model=mixed())
    out = torch.zeros((200, 256, 4), dtype=torch.int32, device="cuda")
    got, index = fb.render3d_scene(shapes, cfg, world_to_model=mixed(), out=out, asynchronous=True)
    assert got is out and index.is_cuda and index.shape == (200, 256)
    cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32).reshape(-1), _bits(want).reshape(-1))
    assert np.array_equal(index.cpu().numpy().view(np.uint16), want_index)


# ---- 7. refusals and cancellation -------------------------------------------------------------------------------------
def _raw(cuda, tapes, table, cfg, out, n=None, index=None):
    c = fb.shape._render3d_cfg(cfg, False)
    n = len(tapes) if n is None else n
    handles = None if tapes is None else (C.c_void_p * max(len(tapes), 1))(*[t._h if t is not None else None for t in tapes])
    return _lib.load().fc_render3d_scene(cuda._h, handles, table, n, C.byref(c), fb.shape._ptr(out), fb.shape._ptr(index), None)


def _sentinel(h, w):
    """a device image and index filled with a pattern no render writes (NaN normals, depth 0xffffffff, index 0xffff):
    a refused call must leave both untouched, i.e. launch and copy nothing"""
    import torch
    return (torch.full((h, w, 4), -1, dtype=torch.int32, device="cuda"),
            torch.full((h, w), -1, dtype=torch.int16, device="cuda"))


def _untouched(out, index):
    import torch
    torch.cuda.synchronize()
    return bool((out == -1).all()) and bool((index == -1).all())


@pytest.mark.parametrize("kw", [dict(z_range=(0, 128)), dict(root_rows=(0, 1)), dict(interleave=(2, 0)),
                                dict(exact_census=True)])
def test_unsupported_settings(cuda, kw):
    shape = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(256, 256, 256, **kw)
    out, index = _sentinel(256, 256)
    assert _raw(cuda, [shape] * 2, fb.scene_table(cfg, 2), cfg, out, index=index) == -3
    assert _untouched(out, index)


def test_refusals(cuda):
    bear = _shape(cuda, "bear.vm")
    cfg = fb.RenderConfig3D(64, 64, 64)
    out, index = _sentinel(64, 64)
    table = fb.scene_table(cfg, 2)

    def refused(code, tapes, tab, c=cfg, o=out, i=index, n=None):
        assert _raw(cuda, tapes, tab, c, o, n=n, index=i) == code
        assert _untouched(o, i)
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    refused(-3, [bear, spilled], table)
    g = fb.Context()
    two = fb.CudaShape(cuda, g.tape([g.sub(g.x(), 0.5), g.sub(g.y(), 0.5)]))
    refused(-1, [bear, two], table)
    sphere, nv, slot = _sphere_var(cuda)
    vt = fb.scene_table(cfg, 2, var_values=np.zeros((2, nv), dtype=np.float32))
    vt[1].n_var_values = 0                                   # the second placement binds nothing
    refused(-1, [sphere, sphere], vt)
    refused(-1, [bear, None], table)
    refused(-1, None, table, n=2)
    refused(-1, [bear, bear], None)
    refused(-3, [bear] * (_lib.FC_SCENE_MAX_SHAPES + 1), fb.scene_table(cfg, _lib.FC_SCENE_MAX_SHAPES + 1))
    deep = fb.RenderConfig3D(64, 64, _lib.FC_SCENE_MAX_DEPTH + 1)
    refused(-3, [bear], fb.scene_table(deep, 1), c=deep)
    wide = fb.RenderConfig3D(4096, 64, 64, tile_sizes=(2048, 64, 16))   # a root tile edge above FC_SCENE_MAX_ROOT_TILE
    wide_out, wide_index = _sentinel(64, 4096)
    refused(-3, [bear], fb.scene_table(wide, 1), c=wide, o=wide_out, i=wide_index)
    refused(0, [], None, n=0)                                 # no shapes: FC_OK, nothing launched or written


def _run(cuda, tok=None):
    cfg = fb.RenderConfig3D(256, 256, 256, cancel=tok)
    return fb.render3d_scene([_shape(cuda, "bear.vm")] * 8, cfg, world_to_model=queue(), stats=True)


def test_cancel_on_entry(cuda):
    tok = fb.CancelToken()
    tok.cancel()
    assert _run(cuda, tok) is None
    assert _lib.load().fc_last_error().decode() == "cancelled before the call started"


@pytest.mark.parametrize("site,item", [("k_voxels_3d", 0), ("k_normals_3d", 5), ("k_interval_level1", 3)])
def test_poll_site_then_next_call_is_correct(cuda, monkeypatch, site, item):
    want = _run(cuda)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:{item}")
    assert _run(cuda, fb.CancelToken()) is None, "the trigger site was never reached"
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    again = _run(cuda)
    assert np.array_equal(_bits(again[0]), _bits(want[0])) and np.array_equal(again[1], want[1])
    for k in CENSUS + ("grads",):
        assert again[2][k] == want[2][k], k
