"""fc_contour_build_slices (many slices of one shape contoured in one call) against fc_contour_build of every slice:
vertices by bit pattern, offsets, closed flags and per-slice counts -- for Z stacks, views, ShapeVars, forced and
overflowing passes, launch grids, cancellation and refusals -- and a few slices against the numpy oracle as well."""
import ctypes as C

import numpy as np
import pytest

import contour_oracle as co
import fidget_b200 as fb
from conftest import model_text, same_f32
from fidget_b200 import _lib

pytestmark = pytest.mark.gpu

COUNTS = ("n_leaves", "n_vertices", "n_polylines", "n_closed", "n_open")
_MODEL_CACHE = {}


def _model(cuda, name):
    if name not in _MODEL_CACHE:
        _MODEL_CACHE[name] = fb.CudaShape.from_vm(cuda, model_text(name + ".vm"))
    return _MODEL_CACHE[name]


def _slice_kw(k, z=None, world_to_model=None, var_values=None):
    kw = {}
    if z is not None:
        kw["z"] = float(np.float32(z[k]))
    if world_to_model is not None and world_to_model[k] is not None:
        kw["world_to_model"] = np.asarray(world_to_model[k], dtype=np.float32)
    if var_values is not None:
        kw["var_values"] = tuple(float(v) for v in np.asarray(var_values[k], dtype=np.float32))
    return kw


def _same(a, b):
    return same_f32(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def _check_stack(dev, depth, **per):
    """The stack against one fc_contour_build per slice; returns the stack's result"""
    got = fb.contour_slices(dev, depth, **per)
    slices, info, per_slice = got
    n = len(slices)
    for k in range(n):
        want = fb.contour(dev, depth, **_slice_kw(k, **per))
        what = f"slice {k} depth {depth}"
        assert slices[k][1].dtype == np.uint32 and slices[k][2].dtype == bool, what
        assert _same(slices[k], want), what
        for f in COUNTS:
            assert per_slice[k][f] == want[3][f], (what, f)
        assert per_slice[k]["sampler_ms"] == 0 and per_slice[k]["contour_ms"] == 0
    for f in COUNTS:
        assert info[f] == sum(p[f] for p in per_slice), f
    return got


def _z_stack(n):
    """n Z values: a sweep through and past the model (slices that miss it entirely) plus repeated values"""
    return np.concatenate([np.linspace(-1.3, 1.3, n - 4), [0.3, 0.3, -1.5, 0.3]]).astype(np.float32)


@pytest.mark.parametrize("name,depth,n", [("bear", 10, 64), ("gyroid-sphere", 9, 48), ("colonnade", 8, 32),
                                          ("tanglecube", 10, 40), ("bear", 8, 33)])
def test_z_stacks_match_single_builds(cuda, name, depth, n):
    slices, info, per = _check_stack(_model(cuda, name), depth, z=_z_stack(n))
    assert info["n_polylines"] > 0
    z = _z_stack(n)
    reps = [k for k in range(n) if z[k] == np.float32(0.3)]
    assert all(_same(slices[k], slices[reps[0]]) for k in reps)


@pytest.mark.parametrize("name", ("colonnade", "tanglecube"))
def test_stack_matches_the_oracle(orc, cuda, name):
    text = model_text(name + ".vm")
    dev, ref = _model(cuda, name), orc.Tape.from_vm(text)
    z = np.array([-0.55, 0.3, -0.1, 0.8, 0.3], np.float32)
    slices, _, per = fb.contour_slices(dev, 8, z=z)
    for k in range(len(z)):
        want = co.contour(ref, 8, z=float(z[k]))
        assert same_f32(slices[k][0], want.vertices) and np.array_equal(slices[k][1], want.offsets)
        assert np.array_equal(slices[k][2], want.closed)
        assert per[k]["n_leaves"] == want.n_leaves and per[k]["n_open"] == want.n_open


def _rot(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1.0]])


VIEWS = {   # (the views of test_gpu_contour.py)
    "rotate": _rot(30),
    "shear": np.array([[1, 0.4, 0], [0, 1, 0], [0, 0, 1.0]]),
    "mirror_x": np.diag([-1.0, 1.0, 1.0]),
    "scale_translate": np.array([[0.7, 0, 0.15], [0, 1.3, -0.1], [0, 0, 1.0]]),
    "perspective": np.array([[1, 0, 0], [0, 1, 0], [0.3, 0.2, 1.0]]),
    "rot_persp": _rot(-20) @ np.array([[1, 0, 0], [0, 1, 0], [0, 0.3, 1.0]]),
    "identity": np.eye(3),
}


@pytest.mark.parametrize("name", ("quarter", "colonnade", "bear"))
def test_views_in_one_call(cuda, name):
    """Every view, mirror and perspective included, with has_transform = 0 and the identity flagged 1 side by side"""
    views = [np.asarray(m, np.float64).astype(np.float32) for m in VIEWS.values()] + [None, np.eye(3, dtype=np.float32)]
    z = np.array([0.1, -0.3, 0.5, 0.0, -0.6, 0.25, 0.4, 0.35, 0.35], np.float32)
    _check_stack(_model(cuda, name), 8, z=z, world_to_model=views)


def test_non_finite_z_with_and_without_a_transform(cuda):
    """Skipping the transform is not applying the identity: each slice is what its own single build gives"""
    dev = _model(cuda, "quarter")
    z = np.array([np.inf, np.inf, -np.inf, -np.inf, np.nan, -0.0, -0.0], np.float32)
    views = [None, np.eye(3), None, np.eye(3), np.eye(3), None, np.eye(3)]
    _check_stack(dev, 7, z=z, world_to_model=views)


def _var_shape(cuda):
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    r, _ = ctx.var()
    dev = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.add(ctx.abs(x), ctx.square(y)), r)))
    slot = list(dev.slot_keys()).index(next(k for k in dev.slot_keys() if k not in ("x", "y", "z")))
    return dev, slot


def test_shape_vars_per_slice(cuda):
    dev, slot = _var_shape(cuda)
    vv = np.zeros((20, dev.n_vars), np.float32)
    vv[:, slot] = np.linspace(-0.1, 1.4, 20)
    _check_stack(dev, 8, var_values=vv)


def _cone(cuda):
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r = ctx.add(ctx.mul(z, -0.3), 0.3)   # radius 0.3 (1 - z): none above z = 1
    return fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y))), r)))


def test_slices_that_miss_the_shape(cuda):
    """Slices without a contour between slices with one: zero polylines, and their neighbours unchanged"""
    slices, info, per = _check_stack(_cone(cuda), 9, z=np.array([1.5, 0.2, 1.2, 1.2, -0.4, 3.0], np.float32))
    assert [p["n_polylines"] for p in per] == [0, 1, 0, 0, 1, 0]
    assert [len(s[1]) for s in slices] == [1, 2, 1, 1, 2, 1]


def test_deep_cone_stack(cuda):
    """Depth 14: every slice of a cone is a closed circle of the analytic radius, and two builds give the same bits"""
    dev = _cone(cuda)
    z = np.linspace(-0.6, 0.6, 6, dtype=np.float32)
    slices, info, per = fb.contour_slices(dev, 14, z=z)
    for k, (v, off, closed) in enumerate(slices):
        assert closed.tolist() == [True] and per[k]["n_open"] == 0
        r = 0.3 * (1.0 - float(z[k]))
        assert np.abs(np.hypot(v[:, 0].astype(np.float64), v[:, 1]) - r).max() < 2e-5
    again, _, _ = fb.contour_slices(dev, 14, z=z)
    assert all(_same(a, b) for a, b in zip(slices, again))


def _fresh(monkeypatch=None, env=(), arena=None):
    for k, v in env:
        monkeypatch.setenv(k, v)
    c2 = fb.CudaContext(0)
    if arena is not None:
        c2.set_arena_bytes(arena)
    return c2


@pytest.mark.parametrize("env", [("FIDGET_B200_FRAMES_PER_PASS", "1"), ("FIDGET_B200_FRAMES_PER_PASS", "2"),
                                 ("FIDGET_B200_FRAMES_PER_PASS", "3"), ("FIDGET_B200_MAX_TILES_M", "1"),
                                 ("FIDGET_B200_SM_COUNT", "1"), ("FIDGET_B200_SM_COUNT", "7"),
                                 ("FIDGET_B200_BLOCKS_PER_SM", "1"), ("FIDGET_B200_BLOCKS_PER_SM", "13")])
def test_passes_and_launch_grids_give_the_same_bits(cuda, monkeypatch, env):
    z = _z_stack(24)
    want = fb.contour_slices(_model(cuda, "bear"), 9, z=z)
    c2 = _fresh(monkeypatch, [env])
    try:
        dev2 = fb.CudaShape.from_vm(c2, model_text("bear.vm"))
        got = fb.contour_slices(dev2, 9, z=z)
        assert all(_same(a, b) for a, b in zip(got[0], want[0]))
        assert got[2] == want[2] and got[1]["n_vertices"] == want[1]["n_vertices"]
        dev2.close()
    finally:
        c2.close()


def test_small_arena_splits_passes_and_a_lone_overflow_is_reported(cuda):
    """prospero's simplified tapes fill a small arena: a stack the arena cannot hold in one pass is run in smaller
    passes with the same bits, and one whose single slice overflows alone gives that slice's own error"""
    views = np.stack([_rot(a) for a in np.linspace(0, 75, 6)]).astype(np.float32)
    want = fb.contour_slices(_model(cuda, "prospero"), 7, world_to_model=views)
    ok_seen = fail_seen = False
    for arena in (64 << 20, 16 << 20, 4 << 20, 1 << 20):
        c2 = _fresh(arena=arena)
        try:
            dev2 = fb.CudaShape.from_vm(c2, model_text("prospero.vm"))
            singles = []
            for m in views:
                try:
                    fb.contour(dev2, 7, world_to_model=m)
                    singles.append(0)
                except fb.CudaError as e:
                    singles.append(e.code)
            if any(singles):
                with pytest.raises(fb.CudaError) as e:
                    fb.contour_slices(dev2, 7, world_to_model=views)
                assert e.value.code == next(s for s in singles if s)
                fail_seen = True
            else:
                got = fb.contour_slices(dev2, 7, world_to_model=views)
                assert all(_same(a, b) for a, b in zip(got[0], want[0]))
                assert got[2] == want[2]
                ok_seen = True
            dev2.close()
        finally:
            c2.close()
    assert ok_seen and fail_seen


SITES = ["k_interval_level0", "k_interval_level3", "k_contour_leaf", "k_contour_grads", "k_contour_vertices",
         "k_contour_segments", "k_contour_link", "k_contour_emit"]


def _read_is_empty(cuda):
    v = np.zeros((4, 2), np.float32)
    off = np.full(4, 7, np.uint32)
    assert cuda._lib.fc_contour_read(cuda._h, v.ctypes.data, off.ctypes.data, None) == 0
    return off[0] == 0 and (v == 0).all()


@pytest.mark.parametrize("site", SITES)
def test_cancel_at_every_poll_site(cuda, monkeypatch, site):
    dev = _model(cuda, "quarter")
    z = _z_stack(12)
    want = fb.contour_slices(dev, 8, z=z)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:0")
    assert fb.contour_slices(dev, 8, z=z, cancel=fb.CancelToken()) is None
    assert _read_is_empty(cuda)
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    got = fb.contour_slices(dev, 8, z=z, cancel=fb.CancelToken())
    assert all(_same(a, b) for a, b in zip(got[0], want[0]))


@pytest.mark.parametrize("site", ["k_contour_leaf:30", "k_contour_vertices:3", "k_interval_level5:20"])
def test_cancel_inside_forced_passes(cuda, monkeypatch, site):
    """Item numbers restart with every launch: the first pass that reaches the item is cancelled"""
    dev = _model(cuda, "bear")
    z = _z_stack(10)
    want = fb.contour_slices(dev, 8, z=z)
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", "3")
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", site)
    assert fb.contour_slices(dev, 8, z=z, cancel=fb.CancelToken()) is None
    assert _read_is_empty(cuda)
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    got = fb.contour_slices(dev, 8, z=z, cancel=fb.CancelToken())
    assert all(_same(a, b) for a, b in zip(got[0], want[0]))


def test_cancel_before_the_call(cuda):
    tok = fb.CancelToken()
    tok.cancel()
    assert fb.contour_slices(_model(cuda, "quarter"), 8, z=[0.0, 0.5], cancel=tok) is None


def _raw(cuda, dev, depth, table, n):
    c = _lib.FcContourCfg()
    c.depth = depth
    info = _lib.FcContourInfo()
    return cuda._lib.fc_contour_build_slices(cuda._h, dev._h, C.byref(c), table, n, C.byref(info), None), info


def test_refusals(cuda):
    dev = _model(cuda, "quarter")
    with pytest.raises(fb.CudaError) as e:
        fb.contour_slices(dev, 15, z=[0.0, 0.1])
    assert e.value.code == -1
    table = fb.contour_slice_table(z=[0.0, 0.1])
    table[1].n_var_values = 17
    assert _raw(cuda, dev, 6, table, 2)[0] == -1
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    multi = fb.CudaShape(cuda, fb.TapeData(ctx, [x, y]))
    with pytest.raises(fb.CudaError) as e:
        fb.contour_slices(multi, 6, z=[0.0, 0.1])
    assert e.value.code == -1
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.contour_slices(spilled, 6, z=[0.0, 0.1])
    assert e.value.code == -3
    assert _raw(cuda, dev, 6, None, 3)[0] == -1


def test_a_slice_without_its_variable_is_refused(cuda):
    dev, slot = _var_shape(cuda)
    table = fb.contour_slice_table(z=[0.0, 0.0])
    table[0].n_var_values = dev.n_vars
    table[0].var_values[slot] = 0.5
    single = C.c_int32(0)
    try:
        fb.contour(dev, 6)
    except fb.CudaError as e:
        single.value = e.code
    assert single.value != 0
    assert _raw(cuda, dev, 6, table, 2)[0] == single.value


def test_empty_stack(cuda):
    dev = _model(cuda, "quarter")
    fb.contour(dev, 7)
    rc, info = _raw(cuda, dev, 7, None, 0)
    assert rc == 0 and info.n_vertices == 0 and info.n_polylines == 0
    assert _read_is_empty(cuda)
    slices, info, per = fb.contour_slices(dev, 7, z=np.zeros(0, np.float32))
    assert slices == [] and per == [] and info["n_vertices"] == 0


def test_the_last_build_is_what_is_read(cuda):
    dev = _model(cuda, "colonnade")
    z = np.array([0.2, -0.4, 0.6], np.float32)
    stack = fb.contour_slices(dev, 8, z=z)
    single = fb.contour(dev, 8, z=-0.1)
    info = fb.contour_slices(dev, 8, z=z)[1]
    v = np.zeros((info["n_vertices"], 2), np.float32)
    off = np.zeros(info["n_polylines"] + 1, np.uint32)
    assert cuda._lib.fc_contour_read(cuda._h, v.ctypes.data, off.ctypes.data, None) == 0
    assert same_f32(v, np.concatenate([s[0] for s in stack[0]]))
    fb.contour(dev, 8, z=-0.1)
    v = np.zeros((len(single[0]), 2), np.float32)
    off = np.zeros(len(single[1]), np.uint32)
    assert cuda._lib.fc_contour_read(cuda._h, v.ctypes.data, off.ctypes.data, None) == 0
    assert same_f32(v, single[0]) and np.array_equal(off, single[1])


def test_offsets_are_global_over_the_stack(cuda):
    dev = _model(cuda, "hi")
    z = np.zeros(5, np.float32)
    slices, info, per = fb.contour_slices(dev, 8, z=z)
    off = np.zeros(info["n_polylines"] + 1, np.uint32)
    assert cuda._lib.fc_contour_read(cuda._h, None, off.ctypes.data, None) == 0
    base = np.cumsum([0] + [len(s[0]) for s in slices])
    p = 0
    for k, s in enumerate(slices):
        assert np.array_equal(off[p:p + len(s[2]) + 1], s[1] + base[k])
        p += len(s[2])
    assert off[-1] == info["n_vertices"]
