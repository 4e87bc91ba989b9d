"""fc_raycast (the first inside sample along each ray) on the device.

- every field of every hit equals the CPU mirror's (the same descent on the oracle's evaluators,
  tests/csrc/raycast_oracle.cc) bit for bit, for the IEEE models and every ray family, at the step counts that exercise
  the levels' clipping;
- k is the first sample whose fc_float_slice_eval value is < 0 (IEEE models), within one step of the mirror for the
  libm models; value and grad are fc_float_slice_eval / fc_grad_slice_eval at pos, bit for bit;
- fb.pick over every pixel equals fc_render3d's depth image on identity views of power-of-two sizes;
- ShapeVars; the same bits whatever the launch grid, the passes and the arena; device-resident rays and hits;
- every refusal leaves every hit a miss, cancellation, and an arena too small for one ray."""
import ctypes as C
import os

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib
from conftest import model_text
from raycast_ref import first_inside, make_rays, oracle_raycast, ray_families, sample_points

pytestmark = pytest.mark.gpu

IEEE_MODELS = ["prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm"]
LIBM_MODELS = ["bear.vm", "gyroid-sphere.vm"]
STEPS = (1, 31, 32, 33, 1024, 1025)
MISS = 0xFFFFFFFF


@pytest.fixture(scope="module")
def shapes(cuda):
    return {name: fb.CudaShape.from_vm(cuda, model_text(name)) for name in IEEE_MODELS + LIBM_MODELS}


@pytest.fixture(scope="module")
def tapes(orc):
    return {name: orc.Tape.from_vm(model_text(name)) for name in IEEE_MODELS + LIBM_MODELS}


def _raw(shape, rays, steps, var_values=(), n_values=None, hits=None, info=None):
    """fc_raycast through ctypes: (status, hits as RAY_HIT, info dict)"""
    lib = _lib.load()
    cfg = _lib.FcRaycastCfg()
    cfg.steps = steps
    cfg.n_var_values = len(var_values) if n_values is None else n_values
    for i, v in enumerate(var_values):
        cfg.var_values[i] = float(v)
    n = len(rays)
    if hits is None:
        hits = np.zeros(n, dtype=fb.RAY_HIT)
        hits["k"] = 12345      # garbage that a call must overwrite
        hits["t"] = 7.0
    st = _lib.FcRaycastInfo()
    rc = lib.fc_raycast(shape.cuda._h, shape._h, C.byref(cfg), rays.ctypes.data if n else None, n,
                        hits.ctypes.data if n else None, C.byref(st) if info is None else info)
    return rc, hits, st.as_dict()


def _cast(shape, rays, steps, var_values=()):
    rc, hits, info = _raw(shape, rays, steps, var_values)
    assert rc == 0, _lib.load().fc_last_error().decode()
    return hits, info


def _words(hits):
    return np.ascontiguousarray(hits).view(np.uint32).reshape(len(hits), 10)


def _assert_same(got, want, what):
    g, w = _words(got), _words(want)
    bad = np.nonzero((g != w).any(axis=1))[0]
    assert not len(bad), (what, len(bad), got[bad[:3]], want[bad[:3]])


def _all_misses(hits):
    return np.all(hits["k"] == MISS) and np.all(_words(hits)[:, 1:] == 0)


# ---- against the oracle --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("steps", STEPS)
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_ieee_models_match_oracle(orc, shapes, tapes, name, steps):
    n = 16 if name == "prospero.vm" else 48
    for family, rays in ray_families(11, steps, n).items():
        got, info = _cast(shapes[name], rays, steps)
        want, _ = oracle_raycast(orc, tapes[name], rays, steps)
        _assert_same(got, want, (name, steps, family))
        assert info["n_hits"] == int((want["k"] != MISS).sum())
        assert info["n_proven"] == int(((want["k"] != MISS) & (want["flags"] == 1)).sum())


@pytest.mark.parametrize("name", ["hi.vm", "quarter.vm", "tanglecube.vm"])
def test_max_steps_match_oracle(orc, shapes, tapes, name):
    steps = 1 << 24
    fam = ray_families(5, steps, 6)
    rays = np.concatenate([fam["through"], fam["axis"], fam["inside"]])
    got, info = _cast(shapes[name], rays, steps)
    want, _ = oracle_raycast(orc, tapes[name], rays, steps)
    _assert_same(got, want, name)
    assert info["evaluated"][0] == len(rays) and info["evaluated"][5:] == [0, 0, 0]


@pytest.mark.parametrize("name", LIBM_MODELS)
def test_libm_models_near_oracle(orc, shapes, tapes, name):
    steps = 1025
    for family, rays in ray_families(13, steps, 32).items():
        got, _ = _cast(shapes[name], rays, steps)
        want, _ = oracle_raycast(orc, tapes[name], rays, steps)
        gk, wk = got["k"].astype(np.int64), want["k"].astype(np.int64)
        both = (gk != MISS) & (wk != MISS)
        assert np.all(np.abs(gk[both] - wk[both]) <= 1), (name, family)
        # a hit on one side only lies at the last sample (the other side's miss is one step past it)
        assert np.all(((gk == MISS) == (wk == MISS)) | (np.minimum(gk, wk) >= steps - 1)), (name, family)


# ---- against the device's own evaluators ---------------------------------------------------------------------------
def _slice_values(shape, rays, steps):
    t, x, y, z = sample_points(rays, steps)
    xs, ys, zs = shape._axes
    cols = [np.zeros(x.size, np.float32) for _ in range(max(shape.info.n_vars, 1))]
    for s, v in ((xs, x), (ys, y), (zs, z)):
        if s >= 0:
            cols[s] = v.ravel()
    return shape.float_slice_eval(cols).reshape(len(rays), steps)


@pytest.mark.parametrize("name", IEEE_MODELS)
def test_k_is_first_inside_by_brute_force(shapes, name):
    shape = shapes[name]
    for steps in (33, 1025):
        for family, rays in ray_families(17, steps, 64).items():
            got, _ = _cast(shape, rays, steps)
            want = first_inside(_slice_values(shape, rays, steps))
            assert np.array_equal(got["k"], want), (name, steps, family)


@pytest.mark.parametrize("name", IEEE_MODELS + LIBM_MODELS)
def test_value_and_grad_are_the_slice_evaluators(shapes, name):
    shape = shapes[name]
    rays = np.concatenate(list(ray_families(19, 1025, 64).values()))
    got, _ = _cast(shape, rays, 1025)
    hit = got["k"] != MISS
    assert hit.sum() > 20
    pos = got["pos"][hit]
    xs, ys, zs = shape._axes
    nv = max(shape.info.n_vars, 1)
    cols = [np.zeros(len(pos), np.float32) for _ in range(nv)]
    gcols = [np.zeros((len(pos), 4), np.float32) for _ in range(nv)]
    for a, s in enumerate((xs, ys, zs)):
        if s >= 0:
            cols[s] = np.ascontiguousarray(pos[:, a])
            gcols[s][:, 0] = pos[:, a]
            gcols[s][:, 1 + a] = 1.0
    v = shape.float_slice_eval(cols)
    g = shape.grad_slice_eval(gcols)
    assert np.array_equal(got["value"][hit].view(np.uint32), v.view(np.uint32)), name
    assert np.array_equal(got["grad"][hit].view(np.uint32), np.ascontiguousarray(g[:, 1:]).view(np.uint32)), name


# ---- fb.pick against the renderer ----------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [(256, 256, 256), (512, 256, 128)])
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_pick_equals_render3d_depth(shapes, name, dims):
    w, h, d = dims
    cfg = fb.RenderConfig3D(w, h, d)
    img = fb.render3d(shapes[name], cfg)
    yy, xx = np.mgrid[0:h, 0:w]
    depth, pos, normal = fb.pick(shapes[name], cfg, np.stack([xx.ravel(), yy.ravel()], 1))
    assert np.array_equal(depth.reshape(h, w), img["depth"]), (name, dims)
    assert (depth > 0).any()


def test_pick_refuses_projective(shapes):
    cfg = fb.RenderConfig3D(64, 64, 64)
    m = cfg.matrix().copy()
    m[3, 2] = 0.01
    cfg.mat = m
    with pytest.raises(ValueError):
        fb.pick(shapes["hi.vm"], cfg, [[1, 2]])


# ---- ShapeVars -----------------------------------------------------------------------------------------------------
def _var_sphere(ctx):
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    d = ctx.add(ctx.add(ctx.square(ctx.sub(x, 0.3)), ctx.square(ctx.sub(y, 0.1))), ctx.square(z))
    return ctx.sub(ctx.sqrt(d), r)


def test_shape_vars_sphere(cuda, orc):
    ctx, octx = fb.Context(), orc.Context()
    dev = fb.CudaShape(cuda, fb.TapeData(ctx, [_var_sphere(ctx)]))
    tape = orc.Tape.from_data(octx.tape(_var_sphere(octx)))
    slot = [i for i in range(dev.info.n_vars) if i not in dev._axes][0]
    steps = 4096
    rng = np.random.default_rng(23)
    n = 256
    o = (rng.normal(size=(n, 3)) * 0.2 + [-1.5, 0.1, 0.0]).astype(np.float32)
    di = np.tile(np.float32([1, 0, 0]), (n, 1))
    di[:, 1:] = rng.normal(scale=0.1, size=(n, 2))
    di = (di / np.linalg.norm(di, axis=1, keepdims=True)).astype(np.float32)
    dt = np.float32(3.0 / steps)
    rays = make_rays(o, di, 0.0, dt)
    for radius in (0.25, 0.5, 0.7):
        vals = [0.0] * dev.info.n_vars
        vals[slot] = radius
        got, _ = _cast(dev, rays, steps, vals)
        want, _ = oracle_raycast(orc, tape, rays, steps, vals)
        _assert_same(got, want, radius)
        # the analytic entry: |o + t d - c| = r
        c = np.array([0.3, 0.1, 0.0])
        oc = o.astype(np.float64) - c
        dd = di.astype(np.float64)
        bq = (oc * dd).sum(1)
        disc = bq * bq - ((oc * oc).sum(1) - radius * radius)
        hit = got["k"] != MISS
        assert hit.sum() > 10
        assert np.all(disc[hit] >= -1e-6)
        t_in = -bq[hit] - np.sqrt(np.maximum(disc[hit], 0))
        assert np.all(np.abs(got["t"][hit] - t_in) <= float(dt) * 1.01 + 1e-6), radius


# ---- independence from launch grid, passes and arena ---------------------------------------------------------------
def _env(key, value):
    class _E:
        def __enter__(self):
            self.old = os.environ.get(key)
            os.environ[key] = value

        def __exit__(self, *a):
            if self.old is None:
                os.environ.pop(key, None)
            else:
                os.environ[key] = self.old
    return _E()


def test_same_bits_whatever_the_grid_and_passes(cuda, shapes):
    shape = shapes["prospero.vm"]
    steps = 1025
    rays = np.concatenate(list(ray_families(29, steps, 48).values()))
    want, info = _cast(shape, rays, steps)
    for bps in ("1", "2", "13"):
        with _env("FIDGET_B200_BLOCKS_PER_SM", bps):
            got, _ = _cast(shape, rays, steps)
        _assert_same(got, want, ("blocks per SM", bps))
    with _env("FIDGET_B200_FRAMES_PER_PASS", "7"):
        got, ginfo = _cast(shape, rays, steps)
    _assert_same(got, want, "passes of 7 rays")
    assert ginfo["passes"] >= len(rays) // 7
    try:
        cuda.set_arena_bytes(4 << 20)
        got, ginfo = _cast(shape, rays, steps)
        _assert_same(got, want, "small arena")
        assert ginfo["passes"] > info["passes"]
        cuda.set_arena_bytes(1 << 20)
        # min(x - x, B): the root interval picks x - x, so level 0 simplifies the root tape, whose ~150k clauses
        # (B, a long sum >= 1) do not fit a 1 MiB arena (131072 clauses): one ray alone overflows it
        ctx = fb.Context()
        x, y = ctx.x(), ctx.y()
        acc = ctx.add(ctx.square(y), 1.0)
        for i in range(50000):
            acc = ctx.add(acc, ctx.square(ctx.sub(y, 1e-5 * i)))
        big = fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.min(ctx.sub(x, x), acc)]))
        assert big.info.n_ops > 131072
        one = make_rays([[-0.5, 0.0, 0.0]], [[1.0, 0.0, 0.0]], 0.0, np.float32(1 / 64))
        rc, hits, _ = _raw(big, one, 64)
        assert rc == -4 and _all_misses(hits)     # FC_ERR_ARENA: one ray alone needs more
    finally:
        cuda.set_arena_bytes(1 << 30)
    got, _ = _cast(shape, rays, steps)              # the context stays usable
    _assert_same(got, want, "after FC_ERR_ARENA")


# ---- device-resident I/O -------------------------------------------------------------------------------------------
def test_device_rays_and_hits(shapes):
    import torch
    shape = shapes["colonnade.vm"]
    steps = 1024
    rays = np.concatenate(list(ray_families(31, steps, 64).values()))
    want, _ = _cast(shape, rays, steps)
    o = torch.from_numpy(np.ascontiguousarray(rays["origin"])).cuda()
    d = torch.from_numpy(np.ascontiguousarray(rays["dir"])).cuda()
    t0 = torch.from_numpy(np.ascontiguousarray(rays["t0"])).cuda()
    k, t, pos, value, grad, proven, info = fb.raycast(shape, o, d, t0, float(rays["dt"][0]), steps)
    assert k.is_cuda and pos.is_cuda
    assert np.array_equal(k.cpu().numpy().astype(np.uint32), want["k"])
    for got, w in ((t, want["t"]), (pos, want["pos"]), (value, want["value"]), (grad, want["grad"])):
        assert np.array_equal(got.cpu().numpy().view(np.uint32), np.ascontiguousarray(w).view(np.uint32))
    assert np.array_equal(proven.cpu().numpy(), want["flags"] == 1)
    # host arrays through the Python face give the same
    hk, ht, hpos, hval, hgrad, hprov, _ = fb.raycast(shape, rays["origin"], rays["dir"], rays["t0"], rays["dt"], steps)
    assert np.array_equal(hk, want["k"]) and np.array_equal(hpos.view(np.uint32), want["pos"].view(np.uint32))


def test_unaligned_device_rays_and_hits(shapes):
    """fc_ray and fc_ray_hit are structs of 4-byte words: device tables that start 4 bytes past an 8-byte boundary are
    read and written in place and give the host call's bits"""
    import torch
    shape = shapes["quarter.vm"]
    steps = 1025
    rays = np.concatenate(list(ray_families(41, steps, 64).values()))
    want, _ = _cast(shape, rays, steps)
    n = len(rays)
    rbuf = torch.zeros(n * 8 + 1, dtype=torch.float32, device="cuda")
    rbuf[1:] = torch.from_numpy(np.ascontiguousarray(rays).view(np.float32).reshape(-1)).cuda()
    hbuf = torch.zeros(n * 10 + 1, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert rbuf[1:].data_ptr() % 8 == 4 and hbuf[1:].data_ptr() % 8 == 4
    lib = _lib.load()
    cfg = _lib.FcRaycastCfg()
    cfg.steps = steps
    rc = lib.fc_raycast(shape.cuda._h, shape._h, C.byref(cfg), rbuf[1:].data_ptr(), n, hbuf[1:].data_ptr(), None)
    assert rc == 0, lib.fc_last_error().decode()
    got = hbuf[1:].cpu().numpy().view(fb.RAY_HIT)
    _assert_same(got, want, "unaligned device rays and hits")
    assert float(hbuf[0]) == 0.0                       # nothing written before the table


# ---- refusals and cancellation -------------------------------------------------------------------------------------
def test_refusals_leave_misses(cuda, shapes):
    shape = shapes["hi.vm"]
    good = make_rays([[-1.5, 0.6, 0.0]], [[1.0, 0.0, 0.0]], 0.0, np.float32(1 / 256))

    def bad(**kw):
        r = good.copy()
        for k, v in kw.items():
            r[k] = v
        return r
    cases = [(good, 0), (good, (1 << 24) + 1), (bad(origin=[[np.nan, 0, 0]]), 512), (bad(dir=[[np.inf, 0, 0]]), 512),
             (bad(t0=np.nan), 512), (bad(dt=0.0), 512), (bad(dt=-1.0), 512), (bad(dt=np.inf), 512),
             (bad(dt=np.float32(3e38)), 512)]     # t at the last sample overflows
    for rays, steps in cases:
        rc, hits, _ = _raw(shape, np.concatenate([good, rays]), steps)
        assert rc == -1 and _all_misses(hits), (rays, steps)
    rc, hits, _ = _raw(shape, good, 512, n_values=17)                  # too many values
    assert rc == -1 and _all_misses(hits)
    ctx = fb.Context()
    var_shape = fb.CudaShape(cuda, fb.TapeData(ctx, [_var_sphere(ctx)]))
    rc, hits, _ = _raw(var_shape, good, 512)                           # a bound variable without a value
    assert rc == -1 and _all_misses(hits)
    two = fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.x(), ctx.y()]))
    rc, hits, _ = _raw(two, good, 512)                                 # multi-output
    assert rc == -1 and _all_misses(hits)
    lib = _lib.load()
    cfg = _lib.FcRaycastCfg()
    cfg.steps = 16
    hits = np.zeros(1, dtype=fb.RAY_HIT)
    assert lib.fc_raycast(cuda._h, shape._h, C.byref(cfg), None, 1, hits.ctypes.data, None) == -1
    assert lib.fc_raycast(cuda._h, shape._h, C.byref(cfg), good.ctypes.data, 1, None, None) == -1
    assert lib.fc_raycast(cuda._h, shape._h, C.byref(cfg), None, 0, None, None) == 0
    assert _cast(shape, good, 512)[0]["k"][0] != MISS


def test_spilled_tape_is_unsupported(cuda):
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    terms = [ctx.sub(ctx.mul(ctx.add(x, float(i) * 0.01), ctx.add(y, float(i) * 0.02)), z) for i in range(40)]
    acc = terms[0]
    for t in terms[1:]:
        acc = ctx.min(acc, ctx.add(t, acc))
    shape = fb.CudaShape(cuda, ctx.tape(acc, 4))       # four registers: memory slots
    if not shape.info.mem_count:
        pytest.skip("the tape did not spill")
    good = make_rays([[-1.5, 0.6, 0.0]], [[1.0, 0.0, 0.0]], 0.0, np.float32(1 / 256))
    rc, hits, _ = _raw(shape, good, 512)
    assert rc == -3 and _all_misses(hits)


def test_cancellation(cuda, shapes):
    shape = shapes["prospero.vm"]
    rays = np.concatenate(list(ray_families(37, 1025, 32).values()))
    want, _ = _cast(shape, rays, 1025)
    tok = fb.CancelToken()
    tok.cancel()
    lib = _lib.load()
    rc = cuda._cancellable(tok, lambda: _raw(shape, rays, 1025)[0])
    assert rc == _lib.FC_ERR_CANCELLED
    assert fb.raycast(shape, rays["origin"], rays["dir"], rays["t0"], rays["dt"], 1025, cancel=tok) is None
    for site in ("k_interval_level1:0", "k_ray_leaf:0", "k_ray_hits:0"):
        with _env("FIDGET_B200_CANCEL_AT", site):
            holder = {}

            def call():
                holder["r"] = _raw(shape, rays, 1025)
                return holder["r"][0]
            rc = cuda._cancellable(fb.CancelToken(), call)
        assert rc == _lib.FC_ERR_CANCELLED, (site, lib.fc_last_error())
        assert _all_misses(holder["r"][1]), site
    got, _ = _cast(shape, rays, 1025)                 # the next call succeeds
    _assert_same(got, want, "after cancel")
