"""fc_measure (volume, centroid, inertia and bounding box from exact integer cell moments) on the device.

- the integers equal the CPU mirror's (the same descent on the oracle's evaluators, tests/csrc/measure_oracle.cc) bit
  for bit for the IEEE models, and a device brute force over every cell centre at depth 9; bear and gyroid-sphere
  (libm opcodes) agree within the renders' 1e-5;
- the float64 results equal exact rational arithmetic on the returned integers within 1e-14;
- known answers at depth 12: the whole cube (sums near 2^64), an axis-aligned dyadic box, a sphere;
- a batch of frames equals one call per frame, whatever the passes; results do not depend on the launch grid;
- cancellation at a level and at the brick kernel, and every refusal."""
import ctypes as C
import math

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib
from conftest import model_text
from measure_ref import brute_sums, derive_exact, ints_of, oracle_measure
from views import _diag, _rot, _translate

pytestmark = pytest.mark.gpu

IEEE_MODELS = ["prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm"]
LIBM_MODELS = ["bear.vm", "gyroid-sphere.vm"]
ROTATE = (_translate(0.1, -0.05, 0.15) @ _rot((1, 2, 3), 25)).astype(np.float32)
VIEWS = {"none": None, "rotate": ROTATE}


# ---- shared fixtures -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shapes(cuda):
    return {name: fb.CudaShape.from_vm(cuda, model_text(name)) for name in IEEE_MODELS + LIBM_MODELS}


@pytest.fixture(scope="module")
def tapes(orc):
    return {name: orc.Tape.from_vm(model_text(name)) for name in IEEE_MODELS + LIBM_MODELS}


def _one(shape, depth, m=None, **kw):
    out = fb.measure(shape, depth, world_to_model=None if m is None else [m], **kw)
    assert out is not None and len(out) == 1
    return out[0]


def _tape(cuda, build):
    ctx = fb.Context()
    return fb.CudaShape(cuda, fb.TapeData(ctx, [build(ctx, ctx.x(), ctx.y(), ctx.z())]))


def _sphere(cuda, r, c=(0.0, 0.0, 0.0)):
    def build(ctx, x, y, z):
        d = [ctx.square(ctx.sub(a, float(ca))) for a, ca in zip((x, y, z), c)]
        return ctx.sub(ctx.sqrt(ctx.add(ctx.add(d[0], d[1]), d[2])), float(r))
    return _tape(cuda, build)


def _sphere_var(cuda):
    """A sphere off the origin whose radius is a ShapeVars variable"""
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    d = ctx.add(ctx.add(ctx.square(ctx.sub(x, 0.3)), ctx.square(ctx.sub(y, 0.1))), ctx.square(z))
    return fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.sub(ctx.sqrt(d), r)]))


# ---- against the oracle and the brute force --------------------------------------------------------------------------
@pytest.mark.parametrize("view", list(VIEWS))
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_ieee_models_match_oracle(orc, shapes, tapes, name, view):
    for depth in (0, 1, 2, 5, 7):
        got = ints_of(_one(shapes[name], depth, VIEWS[view]))
        want = oracle_measure(orc, tapes[name], depth, world_to_model=VIEWS[view])
        assert got == want, (name, view, depth)


@pytest.mark.parametrize("view", list(VIEWS))
@pytest.mark.parametrize("name", LIBM_MODELS)
def test_libm_models_near_oracle(orc, shapes, tapes, name, view):
    for depth in (2, 5, 7):
        got = ints_of(_one(shapes[name], depth, VIEWS[view]))
        want = oracle_measure(orc, tapes[name], depth, world_to_model=VIEWS[view])
        for k in ("n_inside", "n_proven", "n_undecided", "s1", "s2"):
            g, w = np.atleast_1d(np.array(got[k], dtype=np.float64)), np.atleast_1d(np.array(want[k], dtype=np.float64))
            assert np.all(np.abs(g - w) <= 1e-5 * np.maximum(np.abs(w), 1.0)), (name, view, depth, k)
        for k in ("lo", "hi"):
            assert np.all(np.abs(np.array(got[k], dtype=np.int64) - np.array(want[k], dtype=np.int64)) <= 1), (k, depth)


@pytest.mark.parametrize("view", list(VIEWS))
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_ieee_models_match_device_brute_force(shapes, name, view):
    shape, depth = shapes[name], 9
    got = ints_of(_one(shape, depth, VIEWS[view]))
    want = brute_sums(shape.float_slice_eval, shape._axes, shape.info.n_vars, depth,
                      world_to_model=VIEWS[view], slab=16)
    for k in ("n_inside", "s1", "s2", "lo", "hi"):
        assert got[k] == want[k], (name, view, k)


# ---- derived values --------------------------------------------------------------------------------------------------
def _close(got, want, scale, what):
    assert abs(float(got) - float(want)) <= 1e-14 * scale, (what, float(got), float(want))


def _check_derived(row, depth, m):
    ex = derive_exact(ints_of(row), depth, m)
    for k in ("volume", "volume_lo", "volume_hi"):
        _close(row[k], ex[k], max(abs(float(ex[k])), 1e-300), k)
    if ex["centroid"] is None:
        assert row["volume"] == 0
        for k in ("centroid", "inertia", "bbox_min", "bbox_max"):
            assert np.all(np.isnan(row[k])), k
        return
    tscale = 1.0 if m is None else 1.0 + float(np.abs(np.asarray(m, dtype=np.float64)).max()) * 3
    for k in ("centroid", "bbox_min", "bbox_max"):
        for a in range(3):
            _close(row[k][a], ex[k][a], tscale, (k, a))
    iscale = max(abs(float(v)) for v in ex["inertia"])
    for a in range(6):
        _close(row["inertia"][a], ex["inertia"][a], iscale, ("inertia", a))


@pytest.mark.parametrize("name", ["hi.vm", "colonnade.vm", "bear.vm"])
def test_derived_values_exact(shapes, name):
    views = [None, ROTATE, (_translate(0.3, 0.2, -0.1) @ _diag(-1.5, 0.5, 2.0)).astype(np.float32),
             (_rot((0, 0, 1), 90) @ _diag(3.0, 3.0, 3.0)).astype(np.float32),
             _translate(5.0, 5.0, 5.0).astype(np.float32)]   # (the last one moves the shape out of the cube: empty)
    for depth in (3, 6, 8):
        rows = fb.measure(shapes[name], depth, world_to_model=views)
        for k, m in enumerate(views):
            _check_derived(rows[k], depth, m)
    assert rows[-1]["n_inside"] == 0


# ---- known answers at depth 12 ---------------------------------------------------------------------------------------
def _odd_sq(m):
    return m * (4 * m * m - 1) // 3


def _box_sums(i0, i1, j0, j1, k0, k1):
    """fc_measure's sums of the cells [i0, i1] x [j0, j1] x [k0, k1] in closed form"""
    rng = [(i0, i1), (j0, j1), (k0, k1)]
    cnt = [b - a + 1 for a, b in rng]
    s = [(b + 1) ** 2 - a ** 2 for a, b in rng]
    q = [_odd_sq(b + 1) - _odd_sq(a) for a, b in rng]
    n = cnt[0] * cnt[1] * cnt[2]
    return {"n_inside": n, "s1": [s[a] * n // cnt[a] for a in range(3)],
            "s2": [q[a] * n // cnt[a] for a in range(3)] + [s[0] * s[1] * cnt[2], s[0] * s[2] * cnt[1],
                                                             s[1] * s[2] * cnt[0]],
            "lo": [i0, j0, k0], "hi": [i1, j1, k1]}


def test_whole_cube_depth12(cuda):
    # min(|x|, 0) - 1 is the constant -1, and its interval on the cube is [-1, -1]: proven inside at the root
    const = _tape(cuda, lambda ctx, x, y, z: ctx.sub(ctx.min(ctx.abs(x), 0.0), 1.0))
    row = _one(const, 12)
    n = 1 << 12
    want = _box_sums(0, n - 1, 0, n - 1, 0, n - 1)
    got = ints_of(row)
    assert got["n_inside"] == 1 << 36 and got["n_proven"] == 1 << 36 and got["n_undecided"] == 0
    for k in ("s1", "s2", "lo", "hi"):
        assert got[k] == want[k], k
    assert got["s2"][3] == 1 << 60
    assert row["volume"] == 8.0 and np.allclose(row["centroid"], 0.0, atol=1e-15)
    # a unit-density cube of side 2: Ixx = V (1 + 1) / 3
    assert np.allclose(row["inertia"], [16 / 3, 16 / 3, 16 / 3, 0, 0, 0], rtol=1e-14, atol=1e-13)


def test_dyadic_box_depth12(cuda):
    c, half = (0.25, -0.125, 0.375), (0.5, 0.25, 0.5)

    def build(ctx, x, y, z):
        d = [ctx.sub(ctx.abs(ctx.sub(a, ca)), ha) for a, ca, ha in zip((x, y, z), c, half)]
        return ctx.max(ctx.max(d[0], d[1]), d[2])
    row = _one(_tape(cuda, build), 12)
    n, h = 1 << 12, 2.0 / (1 << 12)
    idx = [(int(round((ca - ha + 1) / h)), int(round((ca + ha + 1) / h)) - 1) for ca, ha in zip(c, half)]
    want = _box_sums(*idx[0], *idx[1], *idx[2])
    got = ints_of(row)
    for k in ("n_inside", "s1", "s2", "lo", "hi"):
        assert got[k] == want[k], k
    assert row["volume"] == 8 * half[0] * half[1] * half[2]
    assert np.array_equal(row["centroid"], c) and np.array_equal(row["bbox_min"], np.subtract(c, half))
    assert np.array_equal(row["bbox_max"], np.add(c, half))
    assert got["n_proven"] + got["n_undecided"] <= n ** 3


def test_sphere_depth12(cuda):
    r, c = 0.6, (0.125, -0.0625, 0.25)
    row = _one(_sphere(cuda, r, c), 12)
    h = 2.0 / (1 << 12)
    vol = 4.0 / 3.0 * math.pi * r ** 3
    assert row["volume_lo"] <= vol <= row["volume_hi"]
    assert row["volume_lo"] <= row["volume"] <= row["volume_hi"]
    assert np.all(np.abs(row["centroid"] - np.array(c)) <= h)
    # the voxel solid lies between the spheres of radius r -/+ sqrt(3) h / 2; I = 2/5 V r^2 grows as r^5
    i_true = 0.4 * vol * r * r
    bound = i_true * ((1 + math.sqrt(3) * h / (2 * r)) ** 5 - 1) * 1.5
    assert np.all(np.abs(row["inertia"][:3] - i_true) <= bound)
    assert np.all(np.abs(row["inertia"][3:]) <= bound)


# ---- frames ----------------------------------------------------------------------------------------------------------
def _batch_views(k):
    rng = np.random.default_rng(k)
    out, radii = [], []
    for i in range(k):
        kind = i % 4
        if kind == 0:
            m = _rot(rng.normal(size=3), float(rng.uniform(0, 180)))
        elif kind == 1:
            m = _translate(*rng.uniform(-0.3, 0.3, size=3))
        elif kind == 2:
            m = _diag(-1.0, 1.0, 1.0) @ _translate(*rng.uniform(-0.2, 0.2, size=3))
        else:
            m = None
        out.append(None if m is None else m.astype(np.float32))
        radii.append([float(rng.uniform(0.2, 0.6))] * 4)
    return out, radii


def _same_as_singles(dev, depth, views, radii):
    batch = fb.measure(dev, depth, world_to_model=views, var_values=radii)
    assert len(batch) == len(views)
    for k, (m, vv) in enumerate(zip(views, radii)):
        single = fb.measure(dev, depth, world_to_model=[m], var_values=[vv])
        assert batch[k:k + 1].tobytes() == single.tobytes(), k
    return batch


def test_batch_equals_single_calls(cuda):
    dev = _sphere_var(cuda)
    views, radii = _batch_views(32)
    _same_as_singles(dev, 7, views, radii)


@pytest.mark.parametrize("env", [("FIDGET_B200_MAX_TILES_M", "1"), ("FIDGET_B200_FRAMES_PER_PASS", "3")])
def test_batch_equals_single_calls_small_passes(cuda, monkeypatch, env):
    dev = _sphere_var(cuda)
    views, radii = _batch_views(32)
    want = fb.measure(dev, 8, world_to_model=views, var_values=radii)
    monkeypatch.setenv(*env)
    got = fb.measure(dev, 8, world_to_model=views, var_values=radii)
    assert got.tobytes() == want.tobytes()


def test_batch_with_empty_and_full_frames(cuda):
    dev = _sphere_var(cuda)
    views = [_translate(4.0, 0, 0).astype(np.float32), None, _diag(0.01, 0.01, 0.01).astype(np.float32),
             _rot((0, 1, 0), 30).astype(np.float32), _translate(0, -4.0, 0).astype(np.float32)]
    radii = [[0.5] * 4] * 5
    batch = _same_as_singles(dev, 6, views, radii)
    assert batch[0]["n_inside"] == 0 and batch[4]["n_inside"] == 0
    assert batch[2]["n_inside"] == 1 << 18 and batch[2]["n_proven"] == 1 << 18
    assert list(batch[0]["lo"]) == [0xFFFFFFFF] * 3 and list(batch[0]["hi"]) == [0] * 3
    assert np.isnan(batch[0]["centroid"]).all() and batch[0]["volume"] == 0


# ---- determinism -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob,values", [("FIDGET_B200_SM_COUNT", ["1", "7", "66"]),
                                         ("FIDGET_B200_BLOCKS_PER_SM", ["1", "3", "16"])])
def test_same_bytes_at_any_launch_grid(shapes, monkeypatch, knob, values):
    dev = shapes["colonnade.vm"]
    views = [None, ROTATE]
    want = fb.measure(dev, 8, world_to_model=views).tobytes()
    for v in values:
        monkeypatch.setenv(knob, v)
        ctx = fb.CudaContext(0)   # (the SM count is read when the context is made)
        other = fb.CudaShape.from_vm(ctx, model_text("colonnade.vm"))
        assert fb.measure(other, 8, world_to_model=views).tobytes() == want, (knob, v)
        monkeypatch.delenv(knob)


# ---- cancellation and refusals ---------------------------------------------------------------------------------------
def _raw(cuda, dev, depth, table, n, out, ms=None):
    c = _lib.FcOctreeCfg()
    c.depth = depth
    return cuda._lib.fc_measure(cuda._h, dev._h, C.byref(c), table, n, None if out is None else fb.shape._ptr(out), ms)


@pytest.mark.parametrize("site", ["k_interval_level0:0", "k_interval_level2:0", "k_measure_brick:0",
                                  "k_measure_brick:100"])
def test_cancel(cuda, shapes, monkeypatch, site):
    dev = shapes["colonnade.vm"]
    views = [None, ROTATE, None]
    want = fb.measure(dev, 7, world_to_model=views)
    table = fb.mesh_frame_table(world_to_model=views)
    out = np.frombuffer(b"\xff" * (3 * fb.MEASURE_RESULT.itemsize), dtype=fb.MEASURE_RESULT).copy()
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", site)
    tok = fb.CancelToken()
    rc = cuda._cancellable(tok, lambda: _raw(cuda, dev, 7, table, 3, out))
    assert rc == _lib.FC_ERR_CANCELLED
    assert not out.tobytes().strip(b"\0")
    assert fb.measure(dev, 7, world_to_model=views, cancel=fb.CancelToken()) is None
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    assert fb.measure(dev, 7, world_to_model=views, cancel=fb.CancelToken()).tobytes() == want.tobytes()


def test_cancel_before_the_call(shapes):
    tok = fb.CancelToken()
    tok.cancel()
    assert fb.measure(shapes["hi.vm"], 5, cancel=tok) is None


def test_refusals(cuda, shapes):
    dev = shapes["colonnade.vm"]
    out = np.zeros(2, dtype=fb.MEASURE_RESULT)
    table = fb.mesh_frame_table(world_to_model=[None, ROTATE])
    assert _raw(cuda, dev, 13, table, 2, out) == -1
    assert _raw(cuda, dev, 5, None, 2, out) == -1
    assert _raw(cuda, dev, 5, table, 2, None) == -1
    assert _raw(cuda, dev, 5, None, 0, None) == 0
    table[1].n_var_values = 17
    assert _raw(cuda, dev, 5, table, 2, out) == -1
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    multi = fb.CudaShape(cuda, fb.TapeData(ctx, [x, y]))
    with pytest.raises(fb.CudaError) as e:
        fb.measure(multi, 5)
    assert e.value.code == -1
    with pytest.raises(fb.CudaError) as e:   # the radius has no value
        fb.measure(_sphere_var(cuda), 5)
    assert e.value.code == -1
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.measure(spilled, 5)
    assert e.value.code == -3
    proj = np.eye(4, dtype=np.float32)
    proj[3, 2] = 0.3
    with pytest.raises(fb.CudaError) as e:
        fb.measure(dev, 5, world_to_model=[None, proj])
    assert e.value.code == -3
    # a projective matrix without has_transform is never applied
    table = fb.mesh_frame_table(world_to_model=[None])
    table[0].world_to_model[14] = 0.3
    assert _raw(cuda, dev, 5, table, 1, out[:1]) == 0
    assert fb.measure(dev, 5, world_to_model=np.empty((0, 4, 4))).shape == (0,)


def test_timing(shapes):
    rows, ms = fb.measure(shapes["hi.vm"], 6, world_to_model=[None, ROTATE], timing=True)
    assert ms > 0 and len(rows) == 2
    assert rows.tobytes() == fb.measure(shapes["hi.vm"], 6, world_to_model=[None, ROTATE]).tobytes()
