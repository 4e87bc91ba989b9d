"""The refusals of the four render batches (fc_render2d_frames, fc_render2d_scene, fc_render3d_frames,
fc_render3d_scene), called through ctypes: for each defect, and for pairs of defects whose order decides the answer,
the status code, the exact fc_last_error() text, and that a sentinel-filled device `out` (and `index`) is untouched.
"""
import ctypes as C

import numpy as np
import pytest

import fidget_b200 as fb
from conftest import model_text
from fidget_b200 import _lib

pytestmark = pytest.mark.gpu

CALLS = ("frames2d", "scene2d", "frames3d", "scene3d")
N = 2      # frames or shapes of a call
W = 64     # image side (and volume depth)
SENTINEL = 0xA5
_SHAPES = {}


def _shapes(cuda):
    """A sphere of var radius (with its var count and slot), colonnade at 3 registers (spilled), a two-output tape"""
    if id(cuda) not in _SHAPES:
        g = fb.Context()
        x, y, z = g.x(), g.y(), g.z()
        r, _ = g.var()
        td = g.tape(g.sub(g.sqrt(g.add(g.add(g.square(x), g.square(y)), g.square(z))), r))
        slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
        spilled = fb.CudaShape.from_vm(cuda, model_text("colonnade.vm"), 3)
        assert spilled.info.mem_count > 0
        g2 = fb.Context()
        two = fb.CudaShape(cuda, g2.tape([g2.sub(g2.x(), 0.5), g2.sub(g2.y(), 0.5)]))
        _SHAPES[id(cuda)] = (cuda, fb.CudaShape(cuda, td), td.n_vars, slot, spilled, two)
    return _SHAPES[id(cuda)][1:]


def _table(call, n, nv):
    vv = np.full((n, nv), 0.5, dtype=np.float32)
    if call.endswith("2d"):
        return fb.frame_table(fb.RenderConfig2D(W, W), var_values=vv)
    return fb.frame_table_3d(fb.RenderConfig3D(W, W, W), var_values=vv)


def _args(cuda, call):
    """The arguments of a valid call: a dict each case edits.  A frame batch's tape is tapes[0], its only entry."""
    import torch
    sphere, nv, _, _, _ = _shapes(cuda)
    scene = call.startswith("scene")
    if call.endswith("2d"):
        cfg = fb.shape._render2d_cfg(fb.RenderConfig2D(W, W, out_format="rgba8"), False)
        px = 4
    else:
        cfg = fb.shape._render3d_cfg(fb.RenderConfig3D(W, W, W), False)
        px = 16
    return dict(cfg=cfg, tapes=[sphere] * (N if scene else 1), table=_table(call, N, nv), n=N,
                out=torch.full(((1 if scene else N) * W * W * px,), SENTINEL, dtype=torch.uint8, device="cuda"),
                index=torch.full((W * W,), -1, dtype=torch.int16, device="cuda") if scene else None)


def _run(cuda, call, a):
    lib, ptr = _lib.load(), fb.shape._ptr
    cfg = None if a["cfg"] is None else C.byref(a["cfg"])
    tapes = a["tapes"]
    if call == "frames2d":
        return lib.fc_render2d_frames(cuda._h, tapes[0]._h, cfg, a["table"], a["n"], ptr(a["out"]), None)
    if call == "frames3d":
        return lib.fc_render3d_frames(cuda._h, tapes[0]._h, cfg, a["table"], a["n"], ptr(a["out"]), None)
    handles = None if tapes is None else (C.c_void_p * len(tapes))(*[t._h if t is not None else None for t in tapes])
    if call == "scene2d":
        return lib.fc_render2d_scene(cuda._h, handles, a["table"], a["n"], cfg, None, ptr(a["out"]), ptr(a["index"]), None)
    return lib.fc_render3d_scene(cuda._h, handles, a["table"], a["n"], cfg, ptr(a["out"]), ptr(a["index"]), None)


def _untouched(a):
    import torch
    torch.cuda.synchronize()
    return (a["out"] is None or bool((a["out"] == SENTINEL).all())) and (a["index"] is None or bool((a["index"] == -1).all()))


# ---- the edits -------------------------------------------------------------------------------------------------------
def _cfg(**fields):
    def edit(cuda, call, a):
        for k, v in fields.items():
            setattr(a["cfg"], k, getattr(a["cfg"], k) | v if k == "flags" else v)
    return edit


def _set(**fields):
    def edit(cuda, call, a):
        a.update(fields)
    return edit


def _tape(which):
    def edit(cuda, call, a):
        _, _, _, spilled, two = _shapes(cuda)
        a["tapes"][-1] = {"spilled": spilled, "two": two, "none": None}[which]
    return edit


def _frame_vars(count):
    def edit(cuda, call, a):
        a["table"][N - 1].n_var_values = count
    return edit


def _too_many(cuda, call, a):
    sphere, nv, _, _, _ = _shapes(cuda)
    n = _lib.FC_SCENE_MAX_SHAPES + 1
    a.update(tapes=[sphere] * n, table=_table(call, n, nv), n=n)


def _both(*edits):
    def edit(cuda, call, a):
        for e in edits:
            e(cuda, call, a)
    return edit


INVALID, UNSUPPORTED = -1, -3
SPILL = (UNSUPPORTED, "renderers need a tape without memory spills (<= 255 registers)")


def _cases(call):
    """name -> (edit, expected status, expected fc_last_error text, {slot}: the var's input slot) of `call`'s refusals"""
    two_d, scene = call.endswith("2d"), call.startswith("scene")
    noun = "scenes" if scene else "frame batches"
    rows = (UNSUPPORTED, f"root row bands are not supported by {noun}")
    interleave = (UNSUPPORTED, f"the tile interleave is not supported by {noun}")
    null = (INVALID, "null argument")
    c = {
        "null_cfg": (_set(cfg=None),) + null,
        "null_out": (_set(out=None, index=None),) + null,
        "null_table": (_set(table=None),) + null,
        "row_band": (_cfg(root_row_end=1),) + rows,
        "interleave": (_cfg(root_stride=2),) + interleave,
        "row_band_then_interleave": (_cfg(root_row_begin=0, root_row_end=1, root_stride=2),) + rows,
        "spilled": (_tape("spilled"),) + SPILL,
        "two_outputs": (_tape("two"), INVALID, "ShapeTape has multiple outputs"),
        "too_many_vars": (_frame_vars(_lib.FC_MAX_VARS + 1), INVALID, "n_var_values above FC_MAX_VARS"),
        "missing_var": (_frame_vars(0), INVALID, "missing value for bound variable in input slot {slot}"),
    }
    if scene:
        c["null_tapes"] = (_set(tapes=None),) + null
        c["null_tape"] = (_tape("none"), INVALID, "null tape in the scene")
        c["too_many_shapes"] = (_too_many, UNSUPPORTED, "more than FC_SCENE_MAX_SHAPES shapes")
        c["too_many_shapes_then_row_band"] = (_both(_too_many, _cfg(root_row_end=1)), UNSUPPORTED,
                                              "more than FC_SCENE_MAX_SHAPES shapes")
    if two_d:
        fused = (UNSUPPORTED, f"FC_FLAG_FUSED_TAIL is not supported by {noun}")
        unknown = (INVALID, "unknown out_format")
        c["fused_tail"] = (_cfg(flags=_lib.FC_FLAG_FUSED_TAIL),) + fused
        c["unknown_format"] = (_cfg(out_format=4),) + unknown
        c["fused_tail_then_row_band"] = (_cfg(flags=_lib.FC_FLAG_FUSED_TAIL, root_row_end=1),) + fused
        c["interleave_then_unknown_format"] = (_cfg(root_stride=2, out_format=4),) + interleave
        # a frame batch checks the tape first, a scene its cfg first (then every placement's tape)
        c["spilled_and_fused_tail"] = (_both(_tape("spilled"), _cfg(flags=_lib.FC_FLAG_FUSED_TAIL)),) + \
            (fused if scene else SPILL)
        if scene:
            c["f32"] = (_cfg(out_format=_lib.FC_OUT_F32), UNSUPPORTED,
                        "a 2D scene keeps no distances: FC_OUT_F32 is not supported")
    else:
        slab = (UNSUPPORTED, f"Z slabs are not supported by {noun}")
        c["z_slab"] = (_cfg(z_end=32),) + slab
        c["z_slab_then_row_band"] = (_cfg(z_begin=0, z_end=32, root_row_end=1),) + slab
        c["spilled_and_z_slab"] = (_both(_tape("spilled"), _cfg(z_end=32)),) + (slab if scene else SPILL)
        if scene:
            census = (UNSUPPORTED, "the exact census is not supported by scenes")
            c["exact_census"] = (_cfg(flags=_lib.FC_FLAG_EXACT_CENSUS),) + census
            c["exact_census_then_z_slab"] = (_cfg(flags=_lib.FC_FLAG_EXACT_CENSUS, z_end=32),) + census
    return c


CASES = [(call, name) for call in CALLS for name in _cases(call)]


@pytest.mark.parametrize("call", CALLS)
def test_valid_call_writes_out(cuda, call):
    """(the sentinel check below can see a write: the unedited call overwrites it)"""
    a = _args(cuda, call)
    assert _run(cuda, call, a) == 0, _lib.load().fc_last_error().decode()
    assert not _untouched(a)


@pytest.mark.parametrize("call,name", CASES)
def test_refusal(cuda, call, name):
    edit, code, msg = _cases(call)[name]
    a = _args(cuda, call)
    edit(cuda, call, a)
    assert _run(cuda, call, a) == code
    assert _lib.load().fc_last_error().decode() == msg.format(slot=_shapes(cuda)[2])
    assert _untouched(a)
