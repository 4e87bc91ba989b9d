"""fc_contour_build (quadtree dual contouring and polyline linking on the device) against the numpy oracle of the same
definition (tests/contour_oracle.py): vertices, offsets and closed flags bit for bit and in order, plus the structure of
the output, launch grids, cancellation and refusals."""
import numpy as np
import pytest

import contour_oracle as co
import fidget_b200 as fb
from conftest import model_text, same_f32
from mesh_shapes import tape_pair

pytestmark = pytest.mark.gpu

MODELS = ("bear", "colonnade", "gyroid-sphere", "hi", "prospero", "quarter", "tanglecube")
# sin / cos / exp / ln come from CUDA's libdevice on the device and from libm in the oracle (<= 2 ulp apart,
# include/fidget_cuda.h), so the models that use them are compared to within the search's resolution instead of bit for bit
TRANSCENDENTAL = ("bear", "gyroid-sphere")


def _disc(Ctx, r=0.6, cx=0.0, cy=0.0):
    ctx = Ctx()
    x, y = ctx.x(), ctx.y()
    return ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.square(ctx.sub(x, cx)), ctx.square(ctx.sub(y, cy)))), r))


def _pair(orc, cuda, make):
    return fb.CudaShape(cuda, make(fb.Context)), orc.Tape.from_data(make(orc.Context))


_MODEL_CACHE = {}


def _model(orc, cuda, name):
    if name not in _MODEL_CACHE:
        text = model_text(name + ".vm")
        _MODEL_CACHE[name] = (fb.CudaShape.from_vm(cuda, text), orc.Tape.from_vm(text))
    return _MODEL_CACHE[name]


def _check(dev_shape, orc_tape, depth, exact=True, **kw):
    got = fb.contour(dev_shape, depth, **kw)
    want = co.contour(orc_tape, depth, **kw)
    v, off, closed, info = got
    what = f"depth {depth} {kw}"
    if not exact:
        # a corner sample within an ulp of zero may flip a cell; every vertex still has a close counterpart
        from scipy.spatial import cKDTree
        h = 2.0 / (1 << depth)
        assert abs(info["n_leaves"] - want.n_leaves) <= max(2, want.n_leaves // 500), what
        assert abs(info["n_polylines"] - len(want.closed)) <= 2, what
        if len(v) and len(want.vertices):
            assert cKDTree(want.vertices).query(v)[0].max() < h and cKDTree(v).query(want.vertices)[0].max() < h, what
        return got, want
    assert info["n_leaves"] == want.n_leaves, what
    assert np.array_equal(off, want.offsets), what
    assert np.array_equal(closed, want.closed), what
    assert same_f32(v, want.vertices), what
    assert info["n_open"] == want.n_open and info["n_closed"] == int(want.closed.sum()), what
    assert info["n_vertices"] == len(want.vertices) and info["n_polylines"] == len(want.closed), what
    return got, want


@pytest.mark.parametrize("name", MODELS)
def test_models_match_the_oracle(orc, cuda, name):
    depths = (6, 8) if name == "prospero" else (6, 7, 8, 9, 10)
    dev, ref = _model(orc, cuda, name)
    for d in depths:
        _check(dev, ref, d, exact=name not in TRANSCENDENTAL)


@pytest.mark.parametrize("name", ("bear", "gyroid-sphere", "tanglecube", "colonnade"))
def test_z_slices_match_the_oracle(orc, cuda, name):
    dev, ref = _model(orc, cuda, name)
    for z in (-0.55, -0.1, 0.3, 0.8):
        _check(dev, ref, 8, exact=name not in TRANSCENDENTAL, z=z)


@pytest.mark.parametrize("seed", range(48))
def test_random_csg_slices_match_the_oracle(orc, cuda, seed):
    dev_td, ref, _ = tape_pair(orc, fb, seed, 6)
    dev = fb.CudaShape(cuda, dev_td)
    z = float(np.random.default_rng(20_000 + seed).uniform(-0.6, 0.6))
    _check(dev, ref, 5 + seed % 4, z=z)


def test_shape_vars_match_the_oracle(orc, cuda):
    def make(Ctx):
        ctx = Ctx()
        x, y = ctx.x(), ctx.y()
        r, _ = ctx.var()
        return ctx.tape(ctx.sub(ctx.add(ctx.abs(x), ctx.square(y)), r))
    dev, ref = _pair(orc, cuda, make)
    slot = [k for k in dev.slot_keys()].index(next(k for k in dev.slot_keys() if k not in ("x", "y", "z")))
    for r in (0.2, 0.5, 0.9):
        vals = [0.0] * dev.n_vars
        vals[slot] = r
        _check(dev, ref, 7, var_values=tuple(vals))


def _rot(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1.0]])


VIEWS = {
    "rotate": _rot(30),
    "shear": np.array([[1, 0.4, 0], [0, 1, 0], [0, 0, 1.0]]),
    "mirror_x": np.diag([-1.0, 1.0, 1.0]),
    "scale_translate": np.array([[0.7, 0, 0.15], [0, 1.3, -0.1], [0, 0, 1.0]]),
    "perspective": np.array([[1, 0, 0], [0, 1, 0], [0.3, 0.2, 1.0]]),
    "rot_persp": _rot(-20) @ np.array([[1, 0, 0], [0, 1, 0], [0, 0.3, 1.0]]),
    "identity": np.eye(3),
}


@pytest.mark.parametrize("view", VIEWS)
def test_views_match_the_oracle(orc, cuda, view):
    m = np.asarray(VIEWS[view], dtype=np.float64).astype(np.float32)
    for name in ("quarter", "colonnade"):
        dev, ref = _model(orc, cuda, name)
        _check(dev, ref, 7, world_to_model=m)
    dev, ref = _pair(orc, cuda, lambda C: _disc(C, 0.5, 0.1, -0.1))
    _check(dev, ref, 8, world_to_model=m)


def test_mirror_reverses_the_direction_in_model_space(orc, cuda):
    dev, _ = _pair(orc, cuda, lambda C: _disc(C, 0.5))
    v, off, closed, _ = fb.contour(dev, 7, world_to_model=np.diag([-1.0, 1.0, 1.0]))
    p = v.astype(np.float64)
    assert closed.tolist() == [True]
    assert 0.5 * np.sum(p[:, 0] * np.roll(p[:, 1], -1) - np.roll(p[:, 0], -1) * p[:, 1]) < 0


def _structure(got, want, depth):
    v, off, closed, info = got
    n = 1 << depth
    nxt_in = {}
    for k in range(len(closed)):
        ids = list(range(int(off[k]), int(off[k + 1])))
        assert ids, "empty polyline"
        for a, b in zip(ids, ids[1:] + ([ids[0]] if closed[k] else [])):
            assert b not in nxt_in, "a vertex with two incoming segments"
            nxt_in[b] = a
        if not closed[k]:
            for end in (ids[0], ids[-1]):
                iy, ix, _ = want.cells[end]
                assert ix in (0, n - 1) or iy in (0, n - 1), "an open polyline ends inside the square"


@pytest.mark.parametrize("name", ("quarter", "hi", "tanglecube", "colonnade"))
def test_structure(orc, cuda, name):
    dev, ref = _model(orc, cuda, name)
    got, want = _check(dev, ref, 8)
    _structure(got, want, 8)


def test_shapes_inside_the_square_are_closed(orc, cuda):
    dev, ref = _pair(orc, cuda, lambda C: _disc(C, 0.7, 0.1, 0.05))
    got, want = _check(dev, ref, 9)
    _structure(got, want, 9)
    assert got[3]["n_open"] == 0 and got[2].all()


def test_deep_quadtree(orc, cuda):
    """Depth 14 (the maximum): a disc against its own geometry, and the same bits on a second build."""
    dev, _ = _pair(orc, cuda, lambda C: _disc(C, 0.6))
    v, off, closed, info = fb.contour(dev, 14)
    assert closed.tolist() == [True] and info["n_open"] == 0
    assert np.abs(np.hypot(v[:, 0].astype(np.float64), v[:, 1]) - 0.6).max() < 1e-5
    again = fb.contour(dev, 14)
    assert same_f32(again[0], v) and np.array_equal(again[1], off)


def test_prospero_deep(orc, cuda):
    """prospero at depth 12: the canonical order is the same on every build."""
    dev, _ = _model(orc, cuda, "prospero")
    a = fb.contour(dev, 12)
    b = fb.contour(dev, 12)
    assert same_f32(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert a[3]["n_polylines"] > 100


@pytest.mark.parametrize("env", [("FIDGET_B200_SM_COUNT", "1"), ("FIDGET_B200_SM_COUNT", "7"),
                                 ("FIDGET_B200_BLOCKS_PER_SM", "1"), ("FIDGET_B200_BLOCKS_PER_SM", "13"),
                                 ("FIDGET_B200_MAX_TILES_M", "1")])
def test_launch_grids_give_the_same_bits(orc, cuda, monkeypatch, env):
    dev, ref = _model(orc, cuda, "bear")
    want = fb.contour(dev, 9)
    monkeypatch.setenv(*env)
    c2 = fb.CudaContext(0)
    try:
        dev2 = fb.CudaShape.from_vm(c2, model_text("bear.vm"))
        got = fb.contour(dev2, 9)
        assert same_f32(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
        dev2.close()
    finally:
        c2.close()


SITES = ["k_interval_level0", "k_interval_level3", "k_contour_leaf", "k_contour_grads", "k_contour_vertices",
         "k_contour_segments", "k_contour_link", "k_contour_emit"]


@pytest.mark.parametrize("site", SITES)
def test_cancel_at_every_poll_site(orc, cuda, monkeypatch, site):
    dev, _ = _model(orc, cuda, "quarter")
    want = fb.contour(dev, 8)
    tok = fb.CancelToken()
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:0")
    assert fb.contour(dev, 8, cancel=tok) is None
    # a cancelled build leaves no contour
    v = np.zeros((4, 2), np.float32)
    off = np.full(4, 7, np.uint32)
    assert cuda._lib.fc_contour_read(cuda._h, v.ctypes.data, off.ctypes.data, None) == 0
    assert off[0] == 0 and (v == 0).all()
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    got = fb.contour(dev, 8, cancel=fb.CancelToken())
    assert same_f32(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_cancel_before_the_call(orc, cuda):
    dev, _ = _model(orc, cuda, "quarter")
    tok = fb.CancelToken()
    tok.cancel()
    assert fb.contour(dev, 8, cancel=tok) is None


def test_refusals(orc, cuda):
    dev, _ = _model(orc, cuda, "quarter")
    with pytest.raises(fb.CudaError) as e:
        fb.contour(dev, 15)
    assert e.value.code == -1
    with pytest.raises(fb.CudaError) as e:
        fb.contour(dev, 6, var_values=[0.0] * 17)
    assert e.value.code == -1
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    multi = fb.CudaShape(cuda, fb.TapeData(ctx, [x, y]))
    with pytest.raises(fb.CudaError) as e:
        fb.contour(multi, 6)
    assert e.value.code == -1
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.contour(spilled, 6)
    assert e.value.code == -3


def test_svg_of_a_device_contour(orc, cuda):
    import xml.etree.ElementTree as ET
    dev, _ = _model(orc, cuda, "hi")
    v, off, closed, _ = fb.contour(dev, 8)
    root = ET.fromstring(fb.contours_svg(v, off, closed))
    assert len(root.findall("{http://www.w3.org/2000/svg}path")) == len(closed)
