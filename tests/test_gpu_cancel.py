"""Cancellation of renders, octree sampling and meshing (fc_ctx_set_cancel / fb.CancelToken) on the device.

- the reference's own cancel tests (render2d_cancel, cancel_render, test_octree_cancel): a token cancelled before the
  call makes it return None;
- an attached token that is never set changes nothing, bit for bit, stats included;
- every poll site, deterministically: FIDGET_B200_CANCEL_AT=<site>:<n> makes the poll that claims item n cancel the
  call itself, so each site is shown to stop the call cleanly and to leave the context as good as new;
- a token set from a second thread stops a long call well before it would have finished."""
import threading
import time

import numpy as np
import pytest

import fidget_b200 as fb
import mesh_compare
from conftest import model_text, same_f32
from fidget_b200 import _lib

pytestmark = pytest.mark.gpu

_SHAPES = {}


def _shape(ctx, name):
    key = (id(ctx), name)
    if key not in _SHAPES:
        _SHAPES[key] = (ctx, fb.CudaShape.from_vm(ctx, model_text(name)))
    return _SHAPES[key][1]


def _expr_shape(ctx, build):
    g = fb.Context()
    return fb.CudaShape(ctx, g.tape(build(g)))


def _sphere(g, r):
    x, y, z = g.x(), g.y(), g.z()
    return g.sub(g.sqrt(g.add(g.add(g.square(x), g.square(y)), g.square(z))), float(r))


def _last_error():
    return _lib.load().fc_last_error().decode()


# ---- workloads: fn(ctx, token) -> result (None when cancelled) -----------------------------------------------------
def _r2d(fmt="f32", fused=False, stats=False):
    def run(ctx, tok):
        cfg = fb.RenderConfig2D(1024, 1024, out_format=fmt, fused_tail=fused, cancel=tok)
        return fb.render2d(_shape(ctx, "prospero.vm"), cfg, stats=stats)
    return run


def _r3d(model="bear.vm", size=512, census=False):
    def run(ctx, tok):
        cfg = fb.RenderConfig3D(size, size, size, exact_census=census, cancel=tok)
        return fb.render3d(_shape(ctx, model), cfg, stats=True)
    return run


def _octree(ctx, tok):
    return fb.octree_sample(_shape(ctx, "gyroid-sphere.vm"), 7, stats=True, cancel=tok)


def _mesh(model=None, depth=6, collapse=False):
    def run(ctx, tok):
        s = _shape(ctx, model) if model else _sphere_shape(ctx)
        r = fb.mesh(s, depth, collapse=collapse, cancel=tok)
        if r is None:
            return None
        return r + ((fb.mesh_cells(ctx) if collapse else None),)
    return run


def _sphere_shape(ctx):
    key = (id(ctx), "sphere0.9")
    if key not in _SHAPES:
        _SHAPES[key] = (ctx, _expr_shape(ctx, lambda g: _sphere(g, 0.9)))
    return _SHAPES[key][1]


WORKLOADS = {
    "2d": _r2d(stats=True), "2d_fused": _r2d(fused=True, stats=True),
    "3d": _r3d(), "3d_census": _r3d(census=True), "3d_coop": _r3d("prospero.vm", 256),
    "octree": _octree,
    "mesh": _mesh(), "mesh_c": _mesh(collapse=True),
}


def _same(kind, a, b):
    """bit-identical results of one workload"""
    if kind.startswith("mesh"):
        va, ta, ia, ca = a
        vb, tb, ib, cb = b
        mesh_compare.assert_same_mesh(va, ta, vb, tb)
        for k in ("n_leaves", "n_vertices", "n_triangles", "open_edges"):
            assert ia[k] == ib[k], k
        if ca is not None:
            assert mesh_compare.leaf_set(ca) == mesh_compare.leaf_set(cb)
            assert np.array_equal(np.sort(ca.view(np.uint8).reshape(len(ca), -1), axis=0),
                                  np.sort(cb.view(np.uint8).reshape(len(cb), -1), axis=0))
        return
    (ra, sa), (rb, sb) = a, b
    if kind == "octree":
        # the edges a leaf does not mark present carry no data
        for f in ("ix", "iy", "iz", "mask", "n_edges", "present"):
            assert np.array_equal(ra[f], rb[f]), f
        bits = ((ra["present"][:, None].astype(np.uint32) >> np.arange(12, dtype=np.uint32)) & 1).astype(bool)
        for f in ("pos", "grad"):
            assert np.array_equal(ra[f][bits].view(np.uint32), rb[f][bits].view(np.uint32)), f
    elif ra.dtype == fb.GEOMETRY_PIXEL:
        assert np.array_equal(ra.view(np.uint32), rb.view(np.uint32))
    elif ra.dtype == np.float32:
        assert same_f32(ra, rb)
    else:
        assert ra.tobytes() == rb.tobytes()
    sa, sb = dict(sa), dict(sb)
    for d in (sa, sb):
        d.pop("stage_ms", None)
        d.pop("total_ms", None)
        if kind in ("3d", "3d_coop"):
            # without the exact census, the voxels shaded depend on which leaf tiles finish a column first
            d.pop("pixels")
    assert sa == sb


@pytest.fixture(scope="module")
def fresh():
    """results of every workload on a context of their own, without any token"""
    ctx = fb.CudaContext(0)
    cache = {}

    def get(kind):
        if kind not in cache:
            cache[kind] = WORKLOADS[kind](ctx, None)
        return cache[kind]
    return get


@pytest.fixture(scope="module")
def ctx():
    return fb.CudaContext(0)


def _no_mesh(ctx):
    import ctypes as C
    lib = _lib.load()
    n = C.c_size_t()
    assert lib.fc_mesh_write_stl(ctx._h, None, 0, C.byref(n)) == 0 and n.value == 84
    cells = C.c_uint64(7)
    assert lib.fc_mesh_read_cells(ctx._h, None, 0, C.byref(cells)) == 0 and cells.value == 0
    v = np.full(12, 7, dtype=np.float32)
    t = np.full(12, 7, dtype=np.uint32)
    assert lib.fc_mesh_read(ctx._h, fb.shape._ptr(v), fb.shape._ptr(t)) == 0
    assert (v == 7).all() and (t == 7).all()


# ---- 1. the reference's tests, ported -------------------------------------------------------------------------------
def _cancelled_token():
    t = fb.CancelToken()
    t.cancel()
    return t


def test_render2d_cancel(ctx):
    """pixel.rs:508-520"""
    s = fb.CudaShape.from_vm(ctx, model_text("hi.vm"))
    assert fb.render2d(s, fb.RenderConfig2D(128, 128, cancel=_cancelled_token())) is None
    assert "cancelled" in _last_error()
    assert fb.render2d(s, fb.RenderConfig2D(128, 128)) is not None      # the context stays usable


def test_render3d_cancel(ctx):
    """voxel.rs:573-583"""
    s = _expr_shape(ctx, lambda g: g.x())
    assert fb.render3d(s, fb.RenderConfig3D(64, 64, 64, cancel=_cancelled_token())) is None


@pytest.mark.parametrize("kind", ["octree_sample", "mesh", "mesh_collapse"])
def test_octree_cancel(ctx, kind):
    """octree.rs:1688-1704"""
    s = _expr_shape(ctx, lambda g: _sphere(g, 1.0))
    assert fb.mesh(s, 4) is not None                                         # a mesh exists before the call
    tok = _cancelled_token()
    if kind == "octree_sample":
        assert fb.octree_sample(s, 4, cancel=tok) is None
    else:
        assert fb.mesh(s, 4, collapse=kind == "mesh_collapse", cancel=tok) is None
        _no_mesh(ctx)


# ---- 2. a token that is never set changes nothing ------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["f32", "mask_u8", "bitmap_1bit", "rgba8"])
@pytest.mark.parametrize("fused", [False, True])
def test_unset_token_2d(ctx, fmt, fused):
    run = _r2d(fmt, fused, stats=True)
    _same("2d", run(ctx, fb.CancelToken()), run(ctx, None))


@pytest.mark.parametrize("census", [False, True])
def test_unset_token_3d(ctx, census):
    run = _r3d(census=census)
    _same("3d_census" if census else "3d", run(ctx, fb.CancelToken()), run(ctx, None))


def test_unset_token_octree(ctx):
    _same("octree", _octree(ctx, fb.CancelToken()), _octree(ctx, None))


@pytest.mark.parametrize("collapse", [False, True])
def test_unset_token_mesh(ctx, collapse):
    run = _mesh("colonnade.vm", 7, collapse)
    _same("mesh", run(ctx, fb.CancelToken()), run(ctx, None))


# ---- 3. every poll site --------------------------------------------------------------------------------------------
# (site, workload, mid-list item, extra environment)
SITES = [
    ("k_interval_root_coop", "2d", 10, {}),
    ("k_interval_level0", "2d", 1, {"FIDGET_B200_NO_COOP": "1"}),
    ("k_interval_level1", "2d", 5, {}),
    ("k_interval_level2", "2d", 100, {}),
    ("k_fill_2d", "2d", 100, {}),
    ("k_pixels_2d", "2d", 100, {}),
    ("k_tail_2d", "2d_fused", 10, {}),
    ("k_interval_root_coop", "3d_coop", 3, {}),
    ("k_interval_level0", "3d", 1, {"FIDGET_B200_NO_COOP": "1"}),
    ("k_interval_level1", "3d", 5, {}),
    ("k_interval_level2", "3d", 100, {}),
    ("k_voxels_3d", "3d", 100, {}),
    ("k_normals_3d", "3d", 1000, {}),
    ("k_census_3d", "3d_census", 1000, {}),
    ("k_interval_level3", "octree", 10, {}),
    ("k_octree_leaf", "octree", 100, {}),
    ("k_octree_grads", "octree", 100, {}),
] + [(k, "mesh", 10, {}) for k in ("k_mesh_hash", "k_mesh_vertices", "k_mesh_faces0", "k_mesh_faces1", "k_mesh_assign")] + \
    [(k, "mesh_c", 10, {}) for k in ("k_mesh_hash", "k_mesh_vertices", "k_tree_parents", "k_tree_collapse", "k_tree_final",
                                     "k_tree_faces0", "k_tree_faces1", "k_mesh_assign")]


@pytest.mark.parametrize("at", ["first", "mid"])
@pytest.mark.parametrize("site,kind,mid,env", SITES, ids=[f"{s}-{k}" for s, k, _, _ in SITES])
def test_poll_site(ctx, fresh, monkeypatch, site, kind, mid, env, at):
    want = fresh(kind)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:{0 if at == 'first' else mid}")
    assert WORKLOADS[kind](ctx, fb.CancelToken()) is None, "the trigger site was never reached"
    assert _last_error() == "cancelled"
    if kind.startswith("mesh"):
        _no_mesh(ctx)
    for k in list(env) + ["FIDGET_B200_CANCEL_AT"]:
        monkeypatch.delenv(k)
    _same(kind, WORKLOADS[kind](ctx, None), want)


def test_trigger_needs_a_token(ctx, fresh, monkeypatch):
    """the diagnostic acts only when a flag is attached"""
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", "k_pixels_2d:0")
    _same("2d", WORKLOADS["2d"](ctx, None), fresh("2d"))


def test_trigger_rejects_unknown_sites(ctx, monkeypatch):
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", "k_no_such_kernel:0")
    with pytest.raises(fb.CudaError) as e:
        WORKLOADS["2d"](ctx, fb.CancelToken())
    assert e.value.code == -1


# ---- 4. cancel from a second thread --------------------------------------------------------------------------------
def _timed_cancel(run, t_full, frac=0.1):
    """run(token) with the token set from another thread after frac * t_full; -> (result, seconds from set to return)"""
    tok = fb.CancelToken()
    stamp = {}

    def setter():
        time.sleep(frac * t_full)
        stamp["set"] = time.perf_counter()
        tok.cancel()
    th = threading.Thread(target=setter)
    th.start()
    r = run(tok)
    t_ret = time.perf_counter()
    th.join()
    return r, t_ret - stamp["set"]


def _time_once(run):
    t0 = time.perf_counter()
    r = run(None)
    assert r is not None
    return time.perf_counter() - t0


@pytest.fixture(scope="module")
def big_ctx():
    c = fb.CudaContext(0)
    c.set_arena_bytes(8 << 30)          # prospero 4096^3, as bench.py renders it
    return c


def test_cancel_prospero_3d_from_a_thread(big_ctx):
    import torch
    ctx = big_ctx
    s = _shape(ctx, "prospero.vm")
    out = torch.empty((4096, 4096, 4), dtype=torch.float32, device="cuda")

    def run(tok, asynchronous=False):
        return fb.render3d(s, fb.RenderConfig3D(4096, 4096, 4096, cancel=tok), out=out, asynchronous=asynchronous)
    _time_once(run)                                          # warm-up
    t_full = _time_once(run)
    r, latency = _timed_cancel(run, t_full)
    assert r is None
    assert latency <= 0.2 * t_full, (latency, t_full)

    def run_async(tok):
        try:
            run(tok, asynchronous=True)
            ctx.synchronize()
            return out
        except fb.CudaError as e:
            assert e.code == -6
            return None
    r, latency = _timed_cancel(run_async, t_full)
    assert r is None
    assert latency <= 0.2 * t_full, (latency, t_full)
    assert run(None) is not None


def test_cancel_gyroid_mesh_from_a_thread(big_ctx):
    import ctypes as C
    ctx = big_ctx
    s = _shape(ctx, "gyroid-sphere.vm")
    cfg = _lib.FcOctreeCfg()
    cfg.depth = 9
    cfg.flags = _lib.FC_FLAG_MESH_COLLAPSE
    info = _lib.FcMeshInfo()

    def run(tok):   # fc_mesh_build alone: the mesh stays on the device
        rc = ctx._cancellable(tok, lambda: s._lib.fc_mesh_build(ctx._h, s._h, C.byref(cfg), C.byref(info)))
        assert rc in (0, _lib.FC_ERR_CANCELLED), (rc, _last_error())
        return True if rc == 0 else None
    _time_once(run)
    t_full = _time_once(run)
    r, latency = _timed_cancel(run, t_full)
    assert r is None, t_full
    assert latency <= 0.2 * t_full, (latency, t_full)
    _no_mesh(ctx)


# ---- 5. two contexts on two threads --------------------------------------------------------------------------------
def test_two_contexts_two_threads(fresh):
    import torch
    a, b = fb.CudaContext(0), fb.CudaContext(0)
    a.set_arena_bytes(8 << 30)
    want = fresh("3d")
    got, errs = [], []
    out = torch.empty((4096, 4096, 4), dtype=torch.float32, device="cuda")

    def cancelled_side():
        try:
            for _ in range(3):
                tok = fb.CancelToken()
                th = threading.Timer(0.005, tok.cancel)
                th.start()
                r = fb.render3d(_shape(a, "prospero.vm"), fb.RenderConfig3D(4096, 4096, 4096, cancel=tok), out=out)
                th.join()
                assert r is None
        except Exception as e:   # noqa: BLE001 -- reported below
            errs.append(e)

    def clean_side():
        try:
            for _ in range(3):
                got.append(WORKLOADS["3d"](b, None))
        except Exception as e:   # noqa: BLE001
            errs.append(e)
    ts = [threading.Thread(target=cancelled_side), threading.Thread(target=clean_side)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    assert len(got) == 3
    for r in got:
        _same("3d", r, want)
