"""fc_volume_build / fc_volume_read (sparse narrow-band volumes) on the device.

- IEEE models: bricks, tiles, values and gradients equal the CPU mirror's (tests/csrc/volume_oracle.cc) byte for byte;
  bear and gyroid-sphere (libm opcodes) agree up to a handful of cells near the surface, values within 1e-5;
- at depth 9 against a device brute force: brick values are fc_float_slice_eval's bit for bit, gradients (no
  transform) fc_grad_slice_eval's, every centre within the band is in a brick, every tile on its side of the band;
- at band 0, fc_measure's n_inside is the inside tiles' cells plus the negative brick values, frame by frame;
- a frame batch equals one call per frame, whatever the passes; the bytes do not depend on the launch grid;
- cancellation at the levels, the brick and the gradient kernel; every refusal; reads into host and device memory."""
import ctypes as C

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib
from conftest import model_text
from volume_ref import check_volume, oracle_volume, root_values
from views import _diag, _rot, _translate

pytestmark = pytest.mark.gpu

IEEE_MODELS = ["prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm"]
LIBM_MODELS = ["bear.vm", "gyroid-sphere.vm"]
ROTATE = (_translate(0.1, -0.05, 0.15) @ _rot((1, 2, 3), 25)).astype(np.float32)
PERSPECTIVE = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0.25, 1]], dtype=np.float32)
VIEWS = {"none": None, "rotate": ROTATE, "perspective": PERSPECTIVE}


@pytest.fixture(scope="module")
def shapes(cuda):
    return {name: fb.CudaShape.from_vm(cuda, model_text(name)) for name in IEEE_MODELS + LIBM_MODELS}


@pytest.fixture(scope="module")
def tapes(orc):
    return {name: orc.Tape.from_vm(model_text(name)) for name in IEEE_MODELS + LIBM_MODELS}


def _one(shape, depth, m=None, **kw):
    vol = fb.volume(shape, depth, world_to_model=None if m is None else [m], **kw)
    assert vol is not None
    return vol


def _sphere_var(cuda):
    """A sphere off the origin whose radius is a ShapeVars variable"""
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    d = ctx.add(ctx.add(ctx.square(ctx.sub(x, 0.3)), ctx.square(ctx.sub(y, 0.1))), ctx.square(z))
    return fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.sub(ctx.sqrt(d), r)]))


def _bytes(vol):
    parts = [vol.bricks, vol.values, vol.tiles] + ([vol.grads] if vol.grads is not None else [])
    return b"".join(np.ascontiguousarray(p).tobytes() for p in parts)


# ---- against the oracle ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("view", list(VIEWS))
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_ieee_models_match_oracle(orc, shapes, tapes, name, view):
    m = VIEWS[view]
    big = name == "prospero.vm"
    for depth in (0, 1, 3, 5) if big else (0, 1, 3, 5, 7):
        for band in (0.0, 0.03) if big else (0.0, 0.03, 0.2):
            got = _one(shapes[name], depth, m, band=band, grads=True)
            want = oracle_volume(orc, tapes[name], depth, band=band, world_to_model=m, grads=True)
            for k in ("bricks", "values", "grads", "tiles"):
                assert np.asarray(getattr(got, k)).tobytes() == want[k].tobytes(), (name, view, depth, band, k)
            assert got.info["n_bricks"] == len(want["bricks"]) and got.info["n_tiles"] == len(want["tiles"])
            assert got.info["n_inside_tiles"] == int(want["tiles"][:, 5].sum())
            assert got.info["brick_edge"] == 1 << min(depth, 3) and got.info["passes"] == 1


@pytest.mark.parametrize("view", ["none", "rotate"])
@pytest.mark.parametrize("name", LIBM_MODELS)
def test_libm_models_near_oracle(orc, shapes, tapes, name, view):
    m = VIEWS[view]
    for depth, band in ((3, 0.0), (5, 0.0), (7, 0.0), (7, 0.05)):
        got = _one(shapes[name], depth, m, band=band, grads=True)
        want = oracle_volume(orc, tapes[name], depth, band=band, world_to_model=m, grads=True)
        gb = {tuple(r) for r in got.bricks.tolist()}
        wb = {tuple(r) for r in want["bricks"].tolist()}
        gt = {tuple(r) for r in got.tiles.tolist()}
        wt = {tuple(r) for r in want["tiles"].tolist()}
        assert len(gb ^ wb) <= 8 and len(gt ^ wt) <= 64, (name, view, depth, len(gb ^ wb), len(gt ^ wt))
        gi = {k: i for i, k in enumerate(map(tuple, got.bricks.tolist()))}
        off_cells = cells = 0
        for r, key in enumerate(map(tuple, want["bricks"].tolist())):
            if key not in gi:
                continue
            g, w = got.values[gi[key]], want["values"][r]
            assert np.all(np.abs(g - w) <= 1e-5 * np.maximum(np.abs(w), 1.0)), (name, view, depth, key)
            # (the gradients of libm opcodes differ in their last bits, and more near their singularities: counted)
            gg, wg = got.grads[gi[key]], want["grads"][r]
            with np.errstate(invalid="ignore"):   # (inf - inf where both are infinite)
                off_cells += int(np.any(np.abs(gg - wg) > 1e-5 * np.maximum(np.abs(wg), 1.0), axis=-1).sum())
            cells += g.size
        assert off_cells <= 8 + cells // 1000, (name, view, depth, off_cells, cells)


# ---- against a device brute force ------------------------------------------------------------------------------------
@pytest.mark.parametrize("view", ["none", "rotate"])
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_ieee_models_match_device_brute_force(shapes, name, view):
    shape, depth, band = shapes[name], 9, 0.01
    m = VIEWS[view]
    vol = _one(shape, depth, m, band=band, grads=view == "none")
    v = root_values(shape.float_slice_eval, shape._axes, shape.info.n_vars, depth, world_to_model=m)
    check_volume(vol.bricks, vol.values, vol.tiles, depth, band, v)
    if view == "none" and len(vol.bricks):
        # gradients: fc_grad_slice_eval of the root tape at the world centres of the bricks
        B = 8
        inv = np.float32(1) / np.float32(1 << depth)
        k, j, i = np.meshgrid(np.arange(B), np.arange(B), np.arange(B), indexing="ij")
        base = vol.bricks[:, 1:4].astype(np.int64)
        p = [((2 * (base[:, a, None] + c.ravel()[None, :]) + 1).astype(np.float32) * inv - np.float32(1)).ravel()
             for a, c in enumerate((i, j, k))]
        ins = []
        for s in range(shape.info.n_vars):
            g = np.zeros((p[0].size, 4), dtype=np.float32)
            a = list(shape._axes).index(s)
            g[:, 0] = p[a]
            g[:, 1 + a] = 1
            ins.append(g)
        want = shape.grad_slice_eval(ins)
        np.testing.assert_array_equal(vol.values.reshape(-1), want[:, 0])
        assert np.array_equal(vol.grads.reshape(-1, 3), want[:, 1:]), name


def test_volume_dense_matches_brute_force(shapes):
    shape, band = shapes["hi.vm"], 0.02
    for depth in (2, 5, 7):
        vol = _one(shape, depth, band=band)
        v = root_values(shape.float_slice_eval, shape._axes, shape.info.n_vars, depth)
        B = vol.brick_edge
        in_brick = np.zeros(v.shape, dtype=bool)
        for _, ix, iy, iz in vol.bricks.tolist():
            in_brick[iz:iz + B, iy:iy + B, ix:ix + B] = True
        want = np.where(in_brick, v, np.where(v < 0, np.float32(-1), np.float32(1))).astype(np.float32)
        dense = fb.volume_dense(vol, inside=-1.0, outside=1.0)
        assert dense.tobytes() == want.tobytes(), depth
        dev = fb.volume(shape, depth, band=band, device=True)
        assert fb.volume_dense(dev, inside=-1.0, outside=1.0).cpu().numpy().tobytes() == want.tobytes(), depth


# ---- agreement with fc_measure ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_measure_counts(shapes, name):
    views = [None, ROTATE, _diag(-1.0, 1.0, 1.0).astype(np.float32)]
    for depth in (4, 8):
        vol = fb.volume(shapes[name], depth, world_to_model=views)
        rows = fb.measure(shapes[name], depth, world_to_model=views)
        for f in range(len(views)):
            t = vol.tiles[vol.tiles[:, 0] == f]
            inside = int(sum(1 << (3 * int(lg)) for lg in t[t[:, 5] == 1][:, 4]))
            neg = int((vol.values[vol.bricks[:, 0] == f] < 0).sum())
            assert inside + neg == int(rows[f]["n_inside"]), (name, depth, f)
            assert inside <= int(rows[f]["n_proven"])   # (fc_measure's levels run one depth further)


# ---- frames ----------------------------------------------------------------------------------------------------------
def _batch_views(k):
    rng = np.random.default_rng(k)
    out, radii = [], []
    for i in range(k):
        kind = i % 6
        if kind == 0:
            m = _rot(rng.normal(size=3), float(rng.uniform(0, 180)))
        elif kind == 1:
            m = _translate(*rng.uniform(-0.3, 0.3, size=3))
        elif kind == 2:
            m = _diag(-1.0, 1.0, 1.0) @ _translate(*rng.uniform(-0.2, 0.2, size=3))
        elif kind == 3:
            m = _translate(4.0, 0.0, 0.0)          # empty: the sphere is outside the cube
        elif kind == 4:
            m = _diag(0.01, 0.01, 0.01)            # fully inside
        else:
            m = None
        out.append(None if m is None else m.astype(np.float32))
        radii.append([float(rng.uniform(0.2, 0.6))])
    return out, radii


def _check_batch(dev, depth, band, views, radii, batch):
    off_b = off_t = 0
    for k, (m, vv) in enumerate(zip(views, radii)):
        single = fb.volume(dev, depth, band=band, world_to_model=[m], var_values=[vv], grads=True)
        pf = {key: int(batch.per_frame[key][k]) for key in batch.per_frame}
        assert pf == {"n_bricks": len(single.bricks), "n_tiles": len(single.tiles), "first_brick": off_b,
                      "first_tile": off_t}, k
        sl_b, sl_t = slice(off_b, off_b + pf["n_bricks"]), slice(off_t, off_t + pf["n_tiles"])
        assert np.all(batch.bricks[sl_b, 0] == k) and np.all(batch.tiles[sl_t, 0] == k)
        assert np.array_equal(batch.bricks[sl_b, 1:], single.bricks[:, 1:])
        assert np.array_equal(batch.tiles[sl_t, 1:], single.tiles[:, 1:])
        assert batch.values[sl_b].tobytes() == single.values.tobytes()
        assert batch.grads[sl_b].tobytes() == single.grads.tobytes()
        off_b += pf["n_bricks"]
        off_t += pf["n_tiles"]
    assert off_b == len(batch.bricks) and off_t == len(batch.tiles)


def test_batch_equals_single_calls(cuda):
    dev = _sphere_var(cuda)
    views, radii = _batch_views(32)
    batch = fb.volume(dev, 7, band=0.02, world_to_model=views, var_values=radii, grads=True)
    _check_batch(dev, 7, 0.02, views, radii, batch)
    assert batch.per_frame["n_bricks"][3] == 0 and batch.per_frame["n_bricks"][4] == 0
    assert batch.per_frame["n_tiles"][4] == 1 and batch.tiles[batch.per_frame["first_tile"][4], 5] == 1


@pytest.mark.parametrize("env", [("FIDGET_B200_MAX_TILES_M", "1"), ("FIDGET_B200_FRAMES_PER_PASS", "3")])
def test_batch_equals_single_calls_small_passes(cuda, monkeypatch, env):
    dev = _sphere_var(cuda)
    views, radii = _batch_views(32)
    want = fb.volume(dev, 8, band=0.02, world_to_model=views, var_values=radii, grads=True)
    monkeypatch.setenv(*env)
    got = fb.volume(dev, 8, band=0.02, world_to_model=views, var_values=radii, grads=True)
    assert _bytes(got) == _bytes(want)
    for k in want.per_frame:
        assert np.array_equal(got.per_frame[k], want.per_frame[k])
    assert got.info["passes"] > 1
    _check_batch(dev, 8, 0.02, views[:6], radii[:6], fb.volume(dev, 8, band=0.02, world_to_model=views[:6],
                                                               var_values=radii[:6], grads=True))


# ---- determinism -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob,values", [("FIDGET_B200_SM_COUNT", ["1", "7", "66"]),
                                         ("FIDGET_B200_BLOCKS_PER_SM", ["1", "3", "16"])])
def test_same_bytes_at_any_launch_grid(shapes, monkeypatch, knob, values):
    dev = shapes["colonnade.vm"]
    views = [None, ROTATE]
    want = _bytes(fb.volume(dev, 8, band=0.02, world_to_model=views, grads=True))
    for v in values:
        monkeypatch.setenv(knob, v)
        ctx = fb.CudaContext(0)   # (the SM count is read when the context is made)
        other = fb.CudaShape.from_vm(ctx, model_text("colonnade.vm"))
        assert _bytes(fb.volume(other, 8, band=0.02, world_to_model=views, grads=True)) == want, (knob, v)
        monkeypatch.delenv(knob)


# ---- reads -----------------------------------------------------------------------------------------------------------
def _read(cuda, bricks=None, values=None, grads=None, tiles=None):
    p = fb.shape._ptr
    return cuda._lib.fc_volume_read(cuda._h, *(None if a is None else p(a) for a in (bricks, values, grads, tiles)))


def test_reads(cuda, shapes):
    import torch
    dev = shapes["quarter.vm"]
    host = fb.volume(dev, 7, band=0.05, world_to_model=[None, ROTATE], grads=True)
    on_dev = fb.volume(dev, 7, band=0.05, world_to_model=[None, ROTATE], grads=True, device=True)
    assert on_dev.values.is_cuda and on_dev.bricks.is_cuda and on_dev.tiles.is_cuda
    for k in ("bricks", "values", "grads", "tiles"):
        assert np.array_equal(getattr(on_dev, k).cpu().numpy(), getattr(host, k)), k
    nb, nt = len(host.bricks), len(host.tiles)
    # NULL pointers: each array alone
    vals = np.zeros_like(host.values)
    assert _read(cuda, values=vals) == 0 and np.array_equal(vals, host.values)
    raw_t = np.zeros((nt, 12), dtype=np.uint8)
    assert _read(cuda, tiles=raw_t) == 0
    assert np.array_equal(fb.shape._volume_rows(raw_t, nt, 6, None), host.tiles)
    g = torch.zeros(host.grads.shape, dtype=torch.float32, device="cuda")
    assert _read(cuda, grads=g) == 0 and np.array_equal(g.cpu().numpy(), host.grads)
    assert _read(cuda) == 0
    # a later build replaces the volume; one without gradients refuses a gradient read
    small = fb.volume(dev, 4)
    assert small.grads is None and len(small.bricks) < nb
    assert _read(cuda, grads=np.zeros(10 ** 6, dtype=np.float32)) == -1
    vals = np.zeros((len(small.bricks), 8, 8, 8), dtype=np.float32)
    assert _read(cuda, values=vals) == 0 and np.array_equal(vals, small.values)


def test_timing_and_info(shapes):
    vol = fb.volume(shapes["hi.vm"], 8, band=0.02, world_to_model=[None, ROTATE], timing=True, grads=True)
    assert vol.info["device_ms"] >= vol.info["level_ms"] > 0
    same = fb.volume(shapes["hi.vm"], 8, band=0.02, world_to_model=[None, ROTATE], grads=True)
    assert _bytes(vol) == _bytes(same)
    ev = vol.info["evaluated"]
    assert ev[0] == 2 and all(e % 8 == 0 for e in ev[1:6]) and ev[6] == 0   # levels 0 .. 5 at depth 8
    assert vol.info["n_bricks"] * 512 + sum(1 << (3 * int(lg)) for lg in vol.tiles[:, 4]) == 2 * 8 ** 8


# ---- cancellation and refusals ---------------------------------------------------------------------------------------
def _cfg(depth, band=0.0, flags=0):
    c = _lib.FcVolumeCfg()
    c.depth, c.band, c.flags = depth, band, flags
    return c


def _raw(cuda, dev, cfg, table, n, info=None, per=None):
    return cuda._lib.fc_volume_build(cuda._h, dev._h, C.byref(cfg), table, n, info, per)


@pytest.mark.parametrize("site", ["k_interval_level0:0", "k_interval_level2:0", "k_volume_brick:0", "k_volume_brick:100",
                                  "k_volume_grads:0"])
def test_cancel(cuda, shapes, monkeypatch, site):
    dev = shapes["colonnade.vm"]
    views = [None, ROTATE, None]
    want = fb.volume(dev, 7, band=0.02, world_to_model=views, grads=True)
    assert len(want.bricks) > 100
    table = fb.mesh_frame_table(world_to_model=views)
    info = _lib.FcVolumeInfo()
    per = (_lib.FcVolumeFrameInfo * 3)()
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", site)
    tok = fb.CancelToken()
    rc = cuda._cancellable(tok, lambda: _raw(cuda, dev, _cfg(7, 0.02, _lib.FC_FLAG_VOLUME_GRADS), table, 3,
                                             C.byref(info), per))
    assert rc == _lib.FC_ERR_CANCELLED
    assert not bytes(info).strip(b"\0") and not bytes(per).strip(b"\0")
    vals = np.full(16, 7.0, dtype=np.float32)
    assert _read(cuda, values=vals) == 0 and np.all(vals == 7.0)   # no volume: nothing copied
    assert fb.volume(dev, 7, band=0.02, world_to_model=views, grads=True, cancel=fb.CancelToken()) is None
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    again = fb.volume(dev, 7, band=0.02, world_to_model=views, grads=True, cancel=fb.CancelToken())
    assert _bytes(again) == _bytes(want)


def test_cancel_before_the_call(shapes):
    tok = fb.CancelToken()
    tok.cancel()
    assert fb.volume(shapes["hi.vm"], 5, cancel=tok) is None


def test_refusals(cuda, shapes):
    dev = shapes["colonnade.vm"]
    table = fb.mesh_frame_table(world_to_model=[None, ROTATE])
    assert _raw(cuda, dev, _cfg(13), table, 2) == -1
    assert _raw(cuda, dev, _cfg(5), None, 2) == -1
    for band in (float("nan"), -0.5, float("inf")):
        assert _raw(cuda, dev, _cfg(5, band), table, 2) == -1, band
    assert _raw(cuda, dev, _cfg(5), None, 0) == 0
    table[1].n_var_values = 17
    assert _raw(cuda, dev, _cfg(5), table, 2) == -1
    ctx = fb.Context()
    multi = fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.x(), ctx.y()]))
    with pytest.raises(fb.CudaError) as e:
        fb.volume(multi, 5)
    assert e.value.code == -1
    with pytest.raises(fb.CudaError) as e:   # the radius has no value
        fb.volume(_sphere_var(cuda), 5)
    assert e.value.code == -1
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.volume(spilled, 5)
    assert e.value.code == -3
    # n_frames == 0 leaves an empty volume
    fb.volume(dev, 5)
    empty = fb.volume(dev, 5, world_to_model=np.empty((0, 4, 4)))
    assert len(empty.bricks) == 0 and len(empty.tiles) == 0
    vals = np.full(16, 7.0, dtype=np.float32)
    assert _read(cuda, values=vals) == 0 and np.all(vals == 7.0)
