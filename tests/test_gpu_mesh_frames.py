"""fc_mesh_build_frames (many meshes of one shape in one call) against fc_mesh_build of every frame: vertices bit for
bit and triangles as vertex-position triples (tests/mesh_compare.py), the counts, and with collapse the final leaves and
their vertices -- for ShapeVars sweeps, views, frames that touch the domain's +-Y faces, STL output, forced and
overflowing passes, launch grids, cancellation and refusals -- and a few frames against the oracles as well."""
import ctypes as C

import numpy as np
import pytest

import fidget_b200 as fb
import mesh_compare
import views as V
from conftest import model_text
from fidget_b200 import _lib

pytestmark = pytest.mark.gpu

COUNTS = ("n_leaves", "n_vertices", "n_triangles", "open_edges")
_MODEL_CACHE = {}


def _model(cuda, name):
    if (id(cuda), name) not in _MODEL_CACHE:
        _MODEL_CACHE[(id(cuda), name)] = fb.CudaShape.from_vm(cuda, model_text(name + ".vm"))
    return _MODEL_CACHE[(id(cuda), name)]


def _frame_kw(k, world_to_model=None, var_values=None):
    kw = {}
    if world_to_model is not None and world_to_model[k] is not None:
        kw["world_to_model"] = np.asarray(world_to_model[k], dtype=np.float32)
    if var_values is not None:
        kw["var_values"] = tuple(float(v) for v in np.asarray(var_values[k], dtype=np.float32))
    return kw


def _cells_bytes(cells):
    return np.ascontiguousarray(cells).tobytes()


def _same_frame(a, b, collapse):
    """two (vertices, triangles[, cells]) of one frame are the same mesh"""
    mesh_compare.assert_same_mesh(a[0], a[1], b[0], b[1])
    if collapse:
        assert _cells_bytes(a[-1]) == _cells_bytes(b[-1]), "final leaves differ"


def _check_batch(dev, depth, collapse=False, **per):
    """The batch against one fc_mesh_build per frame; returns the batch's result"""
    got = fb.mesh_frames(dev, depth, collapse=collapse, cells=collapse, **per)
    frames, info, per_frame = got
    for k in range(len(frames)):
        v, t, d = fb.mesh(dev, depth, collapse=collapse, **_frame_kw(k, **per))
        what = f"frame {k} depth {depth} collapse {collapse}"
        want = (v, t, fb.mesh_cells(dev.cuda)) if collapse else (v, t)
        assert frames[k][1].dtype == np.uint32 and (len(frames[k][1]) == 0 or frames[k][1].max() < len(frames[k][0])), what
        _same_frame(frames[k], want, collapse)
        for f in COUNTS:
            assert per_frame[k][f] == d[f], (what, f)
        assert per_frame[k]["n_cells"] == (len(want[2]) if collapse else 0), what
    for f in COUNTS:
        assert info[f] == sum(p[f] for p in per_frame), f
    return got


def _var_shape(cuda, kind):
    """a sphere or a cube whose size is a Context.var(), and the input slot of that variable"""
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    if kind == "sphere":
        e = ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), r)
    else:
        e = ctx.sub(ctx.max(ctx.max(ctx.abs(x), ctx.abs(y)), ctx.abs(z)), r)
    dev = fb.CudaShape(cuda, ctx.tape(e))
    slot = list(dev.slot_keys()).index(next(k for k in dev.slot_keys() if k not in ("x", "y", "z")))
    return dev, slot


def _sizes(n):
    """n sizes: frames that miss the shape (< 0) and frames that cover the whole domain (> sqrt 3) sit between frames
    with a surface"""
    s = np.linspace(0.05, 0.95, n).astype(np.float32)
    s[3::8] = -0.25
    s[6::8] = 1.9
    s[7::16] = 0.5   # repeated frames
    return s


@pytest.mark.parametrize("kind", ["sphere", "cube"])
@pytest.mark.parametrize("collapse", [False, True])
@pytest.mark.parametrize("depth", [1, 2, 3, 4, 5, 6, 7])
def test_shape_var_sweeps(cuda, kind, collapse, depth):
    dev, slot = _var_shape(cuda, kind)
    vv = np.zeros((64, dev.n_vars), np.float32)
    vv[:, slot] = _sizes(64)
    frames, info, per = _check_batch(dev, depth, collapse, var_values=vv)
    if depth >= 2:
        assert [p["n_triangles"] for p in per if p["n_triangles"] == 0] and info["n_triangles"] > 0
    reps = [k for k in range(64) if vv[k, slot] == np.float32(0.5)]
    assert len(reps) > 1
    for k in reps[1:]:
        _same_frame(frames[k], frames[reps[0]], collapse)


def _views(names):
    return [V._f32(V.VIEWS3[n][0]) for n in names]


AFFINE_PERSP = [n for n, (_, kind) in V.VIEWS3.items() if kind in ("affine", "persp")]


@pytest.mark.parametrize("name,depth,collapse", [("colonnade", 5, False), ("colonnade", 6, True), ("bear", 6, False),
                                                 ("bear", 7, True), ("gyroid-sphere", 5, True),
                                                 ("gyroid-sphere", 6, False)])
def test_views_in_one_call(cuda, name, depth, collapse):
    _check_batch(_model(cuda, name), depth, collapse, world_to_model=_views(AFFINE_PERSP))


@pytest.mark.parametrize("collapse", [False, True])
def test_every_catalogue_view(cuda, collapse):
    """strong perspective, degenerate and non-finite views too: each frame is what its own build gives"""
    _check_batch(_model(cuda, "colonnade"), 5, collapse, world_to_model=_views(list(V.VIEWS3)))


@pytest.mark.parametrize("collapse", [False, True])
def test_frames_with_and_without_a_transform(cuda, collapse):
    """has_transform = 0 and the identity flagged as a transform, mixed with views, side by side"""
    m = _views(["rot_y_40", "mirror_x", "persp_z", "shear"])
    table = [None, m[0], np.eye(4, dtype=np.float32), None, m[1], m[2], None, np.eye(4, dtype=np.float32), m[3]]
    _check_batch(_model(cuda, "bear"), 6, collapse, world_to_model=table)


def _column(cuda):
    """max(|x|, |z|) - s: a square column through the whole domain along Y, so every frame has surface cells in the
    top and bottom cell rows, right beside the next frame's in the stacked octree"""
    ctx = fb.Context()
    x, z = ctx.x(), ctx.z()
    s, _ = ctx.var()
    dev = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.max(ctx.abs(x), ctx.abs(z)), s)))
    slot = list(dev.slot_keys()).index(next(k for k in dev.slot_keys() if k not in ("x", "y", "z")))
    return dev, slot


@pytest.mark.parametrize("collapse", [False, True])
@pytest.mark.parametrize("depth", [3, 5, 6])
def test_no_leakage_across_frames(cuda, collapse, depth):
    """Frames reaching the +-Y faces: open edges and triangles equal the single builds, so no cell looked up a
    neighbour of the next frame (which a cell key without the frame would do)"""
    dev, slot = _column(cuda)
    vv = np.zeros((40, dev.n_vars), np.float32)
    vv[:, slot] = np.linspace(0.3, 0.7, 40)
    rot = [V._f32(V._rot((0, 1, 0), a)) if k % 3 == 1 else None for k, a in enumerate(np.linspace(0, 80, 40))]
    frames, info, per = _check_batch(dev, depth, collapse, var_values=vv, world_to_model=rot)
    assert all(p["open_edges"] > 0 for p in per)


@pytest.mark.parametrize("collapse", [False, True])
def test_frames_match_the_oracles(orc, cuda, collapse):
    """A few frames of a batch against the oracles, through mesh_compare, on leaves fb.octree_sample gives that frame"""
    dev = _model(cuda, "colonnade")
    names = ["rot_x_25", "mirror_x", "persp_y"]
    views = _views(names)
    frames, _, per = fb.mesh_frames(dev, 5, world_to_model=views, collapse=collapse, cells=collapse)
    for k, m in enumerate(views):
        leaves = fb.octree_sample(dev, 5, world_to_model=m)
        if collapse:
            v, t, info, _, _ = mesh_compare.compare_collapse(cuda, dev, leaves, 5, world_to_model=m)
            want = (v, t, fb.mesh_cells(cuda))
        else:
            mesh_compare.compare_uniform(dev, leaves, 5, world_to_model=m)
            v, t, info = fb.mesh(dev, 5, world_to_model=m)
            want = (v, t)
        _same_frame(frames[k], want, collapse)
        assert per[k]["n_leaves"] == len(leaves) and per[k]["open_edges"] == info["open_edges"]


def _stl_records(buf):
    body = np.frombuffer(buf[84:], dtype=np.uint8).reshape(-1, 50)
    return sorted(map(bytes, body))


@pytest.mark.parametrize("collapse", [False, True])
def test_stl_one_file_per_frame(cuda, collapse):
    dev, slot = _var_shape(cuda, "sphere")
    vv = np.zeros((9, dev.n_vars), np.float32)
    vv[:, slot] = [0.5, -0.3, 0.8, 0.2, 1.9, 0.6, 0.6, 0.1, 0.9]
    frames, info, per = fb.mesh_frames(dev, 6, var_values=vv, collapse=collapse, stl=True)
    n = C.c_size_t()
    assert dev._lib.fc_mesh_write_stl(cuda._h, None, 0, C.byref(n)) == 0
    assert n.value == 84 * 9 + 50 * info["n_triangles"]
    for k in range(9):
        v, t, d, stl = fb.mesh(dev, 6, var_values=tuple(vv[k]), collapse=collapse, stl=True)
        got = frames[k][2]
        assert len(got) == 84 + 50 * per[k]["n_triangles"] == len(stl)
        assert got[:84] == stl[:84]
        assert _stl_records(got) == _stl_records(stl)


def _fresh(monkeypatch=None, env=(), arena=None):
    for k, v in env:
        monkeypatch.setenv(k, v)
    c2 = fb.CudaContext(0)
    if arena is not None:
        c2.set_arena_bytes(arena)
    return c2


def _same_batch(got, want, collapse):
    assert got[2] == want[2]
    for a, b in zip(got[0], want[0]):
        _same_frame(a, b, collapse)


@pytest.mark.parametrize("env", [("FIDGET_B200_FRAMES_PER_PASS", "1"), ("FIDGET_B200_FRAMES_PER_PASS", "2"),
                                 ("FIDGET_B200_FRAMES_PER_PASS", "3"), ("FIDGET_B200_MAX_TILES_M", "1"),
                                 ("FIDGET_B200_SM_COUNT", "1"), ("FIDGET_B200_SM_COUNT", "7"),
                                 ("FIDGET_B200_BLOCKS_PER_SM", "1"), ("FIDGET_B200_BLOCKS_PER_SM", "13")])
@pytest.mark.parametrize("collapse", [False, True])
def test_passes_and_launch_grids_give_the_same_meshes(cuda, monkeypatch, env, collapse):
    views = _views(AFFINE_PERSP[:10])
    want = fb.mesh_frames(_model(cuda, "bear"), 6, world_to_model=views, collapse=collapse, cells=collapse)
    c2 = _fresh(monkeypatch, [env])
    try:
        dev2 = fb.CudaShape.from_vm(c2, model_text("bear.vm"))
        got = fb.mesh_frames(dev2, 6, world_to_model=views, collapse=collapse, cells=collapse)
        _same_batch(got, want, collapse)
        dev2.close()
    finally:
        c2.close()


def test_small_arena_splits_passes_and_a_lone_overflow_is_reported(cuda):
    """prospero's simplified tapes fill a small arena: a batch the arena cannot hold in one pass is run in smaller
    passes with the same meshes, and one whose single frame overflows alone gives that frame's own error"""
    views = np.stack([V._f32(V._rot((0, 0, 1), a)) for a in np.linspace(0, 75, 6)])
    want = fb.mesh_frames(_model(cuda, "prospero"), 6, world_to_model=views)
    ok_seen = fail_seen = False
    for arena in (512 << 20, 128 << 20, 32 << 20, 8 << 20, 1 << 20):
        c2 = _fresh(arena=arena)
        try:
            dev2 = fb.CudaShape.from_vm(c2, model_text("prospero.vm"))
            singles = []
            for m in views:
                try:
                    fb.mesh(dev2, 6, world_to_model=m)
                    singles.append(0)
                except fb.CudaError as e:
                    singles.append(e.code)
            if any(singles):
                with pytest.raises(fb.CudaError) as e:
                    fb.mesh_frames(dev2, 6, world_to_model=views)
                assert e.value.code == next(s for s in singles if s)
                fail_seen = True
            else:
                _same_batch(fb.mesh_frames(dev2, 6, world_to_model=views), want, False)
                ok_seen = True
            dev2.close()
        finally:
            c2.close()
    assert ok_seen and fail_seen


def _no_mesh(cuda):
    n = C.c_size_t()
    assert cuda._lib.fc_mesh_write_stl(cuda._h, None, 0, C.byref(n)) == 0 and n.value == 84
    cells = C.c_uint64(7)
    assert cuda._lib.fc_mesh_read_cells(cuda._h, None, 0, C.byref(cells)) == 0 and cells.value == 0
    v = np.full(12, 7, dtype=np.float32)
    t = np.full(12, 7, dtype=np.uint32)
    assert cuda._lib.fc_mesh_read(cuda._h, v.ctypes.data, t.ctypes.data) == 0
    assert (v == 7).all() and (t == 7).all()


SITES = [(s, False) for s in ("k_interval_level0", "k_interval_level3", "k_octree_leaf", "k_octree_grads", "k_mesh_hash",
                               "k_mesh_vertices", "k_mesh_faces0", "k_mesh_faces1", "k_mesh_assign")] + \
        [(s, True) for s in ("k_mesh_hash", "k_mesh_vertices", "k_tree_parents", "k_tree_collapse", "k_tree_final",
                             "k_tree_faces0", "k_tree_faces1", "k_mesh_assign")]


@pytest.mark.parametrize("site,collapse", SITES, ids=[f"{s}-{'c' if c else 'u'}" for s, c in SITES])
def test_cancel_at_every_poll_site(cuda, monkeypatch, site, collapse):
    dev = _model(cuda, "colonnade")
    views = _views(AFFINE_PERSP[:8])
    want = fb.mesh_frames(dev, 6, world_to_model=views, collapse=collapse, cells=collapse)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:0")
    assert fb.mesh_frames(dev, 6, world_to_model=views, collapse=collapse, cancel=fb.CancelToken()) is None
    _no_mesh(cuda)
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    _same_batch(fb.mesh_frames(dev, 6, world_to_model=views, collapse=collapse, cells=collapse,
                               cancel=fb.CancelToken()), want, collapse)


@pytest.mark.parametrize("site", ["k_octree_leaf:30", "k_mesh_vertices:3", "k_interval_level4:20", "k_tree_faces1:5"])
def test_cancel_inside_forced_passes(cuda, monkeypatch, site):
    """Item numbers restart with every launch: the first pass that reaches the item is cancelled"""
    dev = _model(cuda, "bear")
    views = _views(AFFINE_PERSP[:7])
    monkeypatch.setenv("FIDGET_B200_FRAMES_PER_PASS", "3")
    fb.mesh(dev, 5)
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", site)
    assert fb.mesh_frames(dev, 6, world_to_model=views, collapse=True, cancel=fb.CancelToken()) is None
    _no_mesh(cuda)


def test_cancel_before_the_call(cuda):
    dev = _model(cuda, "colonnade")
    fb.mesh(dev, 5)
    tok = fb.CancelToken()
    tok.cancel()
    assert fb.mesh_frames(dev, 5, world_to_model=_views(["rot_x_25", "shear"]), cancel=tok) is None
    _no_mesh(cuda)


def _raw(cuda, dev, depth, table, n, flags=0):
    c = _lib.FcOctreeCfg()
    c.depth = depth
    c.flags = flags
    info = _lib.FcMeshInfo()
    return cuda._lib.fc_mesh_build_frames(cuda._h, dev._h, C.byref(c), table, n, C.byref(info), None), info


def test_refusals_leave_no_mesh(cuda):
    dev = _model(cuda, "colonnade")
    fb.mesh(dev, 5)
    with pytest.raises(fb.CudaError) as e:
        fb.mesh_frames(dev, 13, world_to_model=_views(["rot_x_25", "shear"]))
    assert e.value.code == -1
    _no_mesh(cuda)
    table = fb.mesh_frame_table(world_to_model=_views(["rot_x_25", "shear"]))
    table[1].n_var_values = 17
    assert _raw(cuda, dev, 5, table, 2)[0] == -1
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    multi = fb.CudaShape(cuda, fb.TapeData(ctx, [x, y]))
    with pytest.raises(fb.CudaError) as e:
        fb.mesh_frames(multi, 5, world_to_model=[None, None])
    assert e.value.code == -1
    spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
    assert spilled.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.mesh_frames(spilled, 5, world_to_model=[None, None])
    assert e.value.code == -3
    assert _raw(cuda, dev, 5, None, 3)[0] == -1


def test_a_frame_without_its_variable_is_refused(cuda):
    dev, slot = _var_shape(cuda, "sphere")
    table = fb.mesh_frame_table(var_values=np.zeros((2, 0), np.float32))
    table[0].n_var_values = dev.n_vars
    table[0].var_values[slot] = 0.5
    with pytest.raises(fb.CudaError) as e:
        fb.mesh(dev, 5)
    assert _raw(cuda, dev, 5, table, 2)[0] == e.value.code != 0


def test_empty_batch(cuda):
    dev = _model(cuda, "colonnade")
    fb.mesh(dev, 5)
    rc, info = _raw(cuda, dev, 5, None, 0)
    assert rc == 0 and info.n_vertices == 0 and info.n_triangles == 0
    _no_mesh(cuda)
    frames, info, per = fb.mesh_frames(dev, 5, var_values=np.zeros((0, 0), np.float32))
    assert frames == [] and per == [] and info["n_vertices"] == 0


@pytest.mark.parametrize("collapse", [False, True])
def test_the_last_build_is_what_is_read(cuda, collapse):
    dev = _model(cuda, "colonnade")
    views = _views(["rot_x_25", "mirror_x", "persp_z"])
    batch = fb.mesh_frames(dev, 6, world_to_model=views, collapse=collapse, cells=collapse)
    single = fb.mesh(dev, 6, collapse=collapse, stl=True)
    info = fb.mesh_frames(dev, 6, world_to_model=views, collapse=collapse)[1]
    v = np.zeros((info["n_vertices"], 3), np.float32)
    t = np.zeros((info["n_triangles"], 3), np.uint32)
    assert cuda._lib.fc_mesh_read(cuda._h, v.ctypes.data, t.ctypes.data) == 0
    for got, want in zip(fb.split_mesh_frames(v, t, batch[2]), batch[0]):
        _same_frame(got, want[:2], False)
    again = fb.mesh(dev, 6, collapse=collapse, stl=True)
    mesh_compare.assert_same_mesh(again[0], again[1], single[0], single[1])
    assert all(again[2][f] == single[2][f] for f in COUNTS)
    assert again[3][:84] == single[3][:84] and _stl_records(again[3]) == _stl_records(single[3])
