"""Every kernel gives the same bits at any launch grid.

Grids are sized from the context's SM count (persistent CTAs and warps claiming jobs, grid-stride loops, the TMA slice
ring) and from per-SM knobs.  On the full device with small renders each CTA or warp takes about one unit of work, so
the code that runs only for a second, fourth or n-th unit -- reused choice scratch, shared rows and registers, a
refilled TMA stage waiting on parity 1, a cooperative CTA's second round of root tiles -- would go untested.  Here the
same workload runs on contexts that size their grids for 1, 3 and 16 SMs and for all but one of the device's SMs
(FIDGET_B200_SM_COUNT: launch geometry only, the kernels still run on the whole device), and with each per-SM knob below
and above its default:

  * IEEE models equal the CPU oracle bit for bit (images, depth and normals, octree leaves, slices, solver results)
    with the census level by level where it is deterministic;
  * libm models (bear, gyroid-sphere) equal the same call on a default context bit for bit (the oracle's libm differs
    by ulps; other tests hold the default context to it within a tolerance).

Not compared: kernel launch counts, timings, arena use, the 3D census without exact_census (culling depends on timing)
and mesh vertex order (meshes are compared as multisets).  Coverage is asserted, not assumed: each launch shape has a
case whose cooperative level-0 CTAs take several rounds (read from the FIDGET_B200_COOP_DEBUG line), 2D and 3D cases
with more level jobs than the grid has warps, and f32 and gradient slices whose TMA CTAs run past their third tile
(read from the FIDGET_B200_SLICE_DEBUG line)."""
import io
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import fidget_b200 as fb
import solve_oracle as so
import solver_cases as sc
from conftest import ROOT, model_text, same_f32
from mesh_compare import assert_same_mesh

pytestmark = pytest.mark.gpu

EMULATED = (1, 3, 16, -1)                        # -1: all but one of the device's SMs (131 on an H100 SXM)
EMULATED_IDS = ["sm1", "sm3", "sm16", "sm_all_but_one"]
WARPS_PER_BLOCK = 4                              # kernels.cuh: warps of an interval-level CTA
BLOCKS_PER_SM, LAST_LEVEL_BLOCKS_PER_SM = 6, 8   # render.cu defaults
TMA_STAGES = 3                                   # bulk.cu: the TMA slice kernel's ring of stages
CENSUS = ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")
KNOBS = ("FIDGET_B200_SM_COUNT", "FIDGET_B200_BLOCKS_PER_SM", "FIDGET_B200_LAST_LEVEL_BLOCKS_PER_SM",
         "FIDGET_B200_PIXEL_BLOCKS_PER_SM", "FIDGET_B200_VOXEL_BLOCKS_PER_SM", "FIDGET_B200_COOP_PER_SM",
         "FIDGET_B200_COOP_THREADS", "FIDGET_B200_NO_COOP", "FIDGET_B200_NO_ZSORT", "FIDGET_B200_SERIAL_FILL",
         "FIDGET_B200_TAIL_PAINTS", "FIDGET_B200_LEVEL_FUSED_PATH", "FIDGET_B200_FUSE", "FIDGET_B200_NO_TMA",
         "FIDGET_B200_COOP_DEBUG", "FIDGET_B200_SLICE_DEBUG", "FIDGET_B200_NO_CULL", "FIDGET_B200_FULL_LADDER", "FIDGET_B200_FRAMES_PER_PASS")
COOP_LINE = re.compile(r"coop: .* (\d+) CTAs/SM x (\d+) threads .*, (\d+) roots, occupancy \d+ CTAs/SM, (\d+) SMs")
SLICE_LINE = re.compile(r"slice: (?:TMA kernel, (\d+) points, (\d+) full tiles, (\d+) CTAs, (\d+) SMs|per-thread kernel)")


def _real_sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sphere(Ctx, r):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    return ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), ctx.constant(r)))


def _place(scale, tx, ty, tz):
    s = 1.0 / scale
    return np.array([[s, 0, 0, -tx * s], [0, s, 0, -ty * s], [0, 0, s, -tz * s], [0, 0, 0, 1]], dtype=np.float32)


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]], dtype=np.float32)


ORBIT = np.stack([_rot_y(2 * np.pi * k / 3) for k in range(3)])
GRID2 = np.stack([_place(0.45, -0.5 + i, -0.5 + j, 0.1 * (i - j)) for j in range(2) for i in range(2)])
Z_STACK = np.array([-0.45, -0.1, 0.25, 0.6], dtype=np.float32)


def _shape(cuda, name):
    if name.startswith("sphere"):
        return fb.CudaShape(cuda, _sphere(fb.Context, float(name[len("sphere"):])))
    return fb.CudaShape.from_vm(cuda, model_text(name))


def _oracle_tape(orc, name):
    if name.startswith("sphere"):
        return orc.Tape.from_data(_sphere(orc.Context, float(name[len("sphere"):])))
    return orc.Tape.from_vm(model_text(name))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


# ---- the workload ------------------------------------------------------------------------------------------------
# 2D: name -> (model, width, height, RenderConfig2D keywords).  bear is libm: compared with the default context.
CASES_2D = {
    "prospero1024": ("prospero.vm", 1024, 1024, {}),
    "prospero512_32_8": ("prospero.vm", 512, 512, dict(tile_sizes=(32, 8))),       # 256 roots: coop rounds at S <= 16
    "prospero512_8": ("prospero.vm", 512, 512, dict(tile_sizes=(8,))),             # 4096 roots: coop rounds at S > 96
    "prospero1024_32_8_2": ("prospero.vm", 1024, 1024, dict(tile_sizes=(32, 8, 2))),   # ~5.5k level-2 jobs
    "hi300x200": ("hi.vm", 300, 200, {}),
    "colonnade512_fused": ("colonnade.vm", 512, 512, dict(fused_tail=True)),
    "colonnade256_pp": ("colonnade.vm", 256, 256, dict(pixel_perfect=True, z=0.3)),
    "bear512": ("bear.vm", 512, 512, {}),
}
LIBM = ("bear.vm", "gyroid-sphere.vm")
# 3D with exact_census (IEEE, against the oracle's census level by level); prospero 512^3 has more jobs per level
# than the grids for all but one SM of an H100 have warps
CASES_3D_EXACT = {"prospero256": ("prospero.vm", 256), "colonnade256": ("colonnade.vm", 256),
                  "prospero512": ("prospero.vm", 512)}
# model -> whether its tape fits the TMA slice kernel (colonnade's 42 registers exceed its 40)
SLICE_MODELS = {"hi.vm": True, "colonnade.vm": False, "bear.vm": True}
SLICE_SIZES = (4097, 100003)
BIG_F32, BIG_GRAD = (1 << 22) + 3, (1 << 20) + 3


class Want:
    """What each case must give, computed once for the module: the oracle's outputs, and for libm models the same
    call on the session's default context with every tuning knob unset."""

    def __init__(self, orc, cuda):
        self.orc, self.cuda = orc, cuda
        self._memo = {}
        self._tapes = {}
        self._shapes = {}

    def _get(self, key, fn):
        if key not in self._memo:
            self._memo[key] = fn()
        return self._memo[key]

    def tape(self, name):
        if name not in self._tapes:
            self._tapes[name] = _oracle_tape(self.orc, name)
        return self._tapes[name]

    def default(self, key, fn):
        """fn(shape getter) on the default context, knobs unset"""
        def run():
            with pytest.MonkeyPatch.context() as mp:
                for k in KNOBS:
                    mp.delenv(k, raising=False)
                return fn(self._shape)
        return self._get(("default",) + key, run)

    def _shape(self, name):
        if name not in self._shapes:
            self._shapes[name] = _shape(self.cuda, name)
        return self._shapes[name]

    def render2d(self, case):
        name, w, h, kw = CASES_2D[case]
        if name in LIBM:
            return self.default(("2d", case), lambda sh: fb.render2d(sh(name), fb.RenderConfig2D(w, h, **kw), stats=True))
        ts = kw.get("tile_sizes") or (128, 32, 8)
        return self._get(("2d", case), lambda: self.orc.render2d(self.tape(name), w, h, tile_sizes=ts, threads=8,
                                                                  z=kw.get("z", 0.0),
                                                                  pixel_perfect=kw.get("pixel_perfect", False)))

    def z_stack(self, k):
        return self._get(("z", k), lambda: self.orc.render2d(self.tape("colonnade.vm"), 256, 256, z=float(Z_STACK[k]),
                                                              threads=8)[0])

    def render3d(self, name, w, h, d):
        return self._get(("3d", name, w, h, d), lambda: self.orc.render3d(self.tape(name), w, h, d, threads=8))

    def octree(self, name, depth):
        return self._get(("octree", name, depth), lambda: self.orc.octree_sample(self.tape(name), depth))

    def float_slice(self, name, n):
        return self._get(("f32", name, n), lambda: self.tape(name).float_slice_eval(_points(n, self.tape(name).n_vars)))

    def grad_slice(self, name, n):
        return self._get(("grad", name, n), lambda: self.tape(name).grad_slice_eval(_grad_points(n, self.tape(name).n_vars)))

    def solve(self):
        def run():
            ctx = self.orc.Context()
            case = sc.rosenbrock_chain(ctx, 3)
            keys = case.free + case.fixed
            tds = [ctx.tape(r) for r in case.roots]
            vals, res = so.solve_batch([self.orc.Tape.from_data(t) for t in tds], [sc.slot_map(t, keys) for t in tds],
                                       len(case.free), _solver_starts(case), 0)
            return vals, res["status"], res["iterations"], res["err"]
        return self._get(("solve",), run)


@pytest.fixture(scope="module")
def want(orc, cuda):
    return Want(orc, cuda)


class Rig:
    """A fresh CudaContext whose grids are sized for `sm` SMs (None: the device's own count), with its shapes, the
    FIDGET_B200_COOP_DEBUG and FIDGET_B200_SLICE_DEBUG lines of its calls and what the coverage assertions need."""

    def __init__(self, monkeypatch, capfd, sm):
        self.mp, self.capfd = monkeypatch, capfd
        self.real_sm = _real_sm_count()
        if sm is None:
            monkeypatch.delenv("FIDGET_B200_SM_COUNT", raising=False)
        else:
            monkeypatch.setenv("FIDGET_B200_SM_COUNT", str(sm))
        self.cuda = fb.CudaContext(0)            # (the count is read once, here)
        monkeypatch.delenv("FIDGET_B200_SM_COUNT", raising=False)
        self.sm = sm if sm is not None else self.real_sm
        self._shapes, self._others = {}, []
        self.coop = []                           # (CTAs/SM, threads, roots, SMs) of each cooperative launch
        self.slices = []                         # (points, full tiles, CTAs, SMs) of each TMA slice, None per-thread
        self.jobs_over_warps = {2: [], 3: []}    # (case, level, jobs, warps) where a warp takes several jobs
        self.jobs_under_warps = {2: [], 3: []}
        monkeypatch.setenv("FIDGET_B200_COOP_DEBUG", "1")
        monkeypatch.setenv("FIDGET_B200_SLICE_DEBUG", "1")

    def shape(self, name):
        if name not in self._shapes:
            self._shapes[name] = _shape(self.cuda, name)
        return self._shapes[name]

    def watch(self, fn):
        """fn() with the debug lines of the cooperative kernel and of the slices collected"""
        self.capfd.readouterr()
        out = fn()
        err = self.capfd.readouterr().err
        for m in COOP_LINE.finditer(err):
            self.coop.append(tuple(int(v) for v in m.groups()))
        for m in SLICE_LINE.finditer(err):
            self.slices.append(tuple(int(v) for v in m.groups()) if m.group(1) else None)
        return out

    def knob(self, name, default):
        v = os.environ.get("FIDGET_B200_" + name)
        return int(v) if v else default

    def count_jobs(self, dim, case, ambiguous, n_levels):
        """level l (>= 1) claims one job per ambiguous tile of level l - 1; its grid has this many warps"""
        bps = self.knob("BLOCKS_PER_SM", BLOCKS_PER_SM)
        for l in range(1, n_levels):
            last = dim == 3 and l == n_levels - 1
            per_sm = max(bps, self.knob("LAST_LEVEL_BLOCKS_PER_SM", LAST_LEVEL_BLOCKS_PER_SM)) if last else bps
            warps = self.sm * per_sm * WARPS_PER_BLOCK
            rec = (case, l, ambiguous[l - 1], warps)
            (self.jobs_over_warps if ambiguous[l - 1] > warps else self.jobs_under_warps)[dim].append(rec)

    def track(self, shape):
        self._others.append(shape)
        return shape

    def close(self):
        # every tape is released before its context, also those a failed assertion's traceback still holds
        for sh in list(self._shapes.values()) + self._others:
            sh.close()
        self._shapes.clear()
        self._others.clear()
        self.cuda.close()


@pytest.fixture
def rigs(monkeypatch, capfd):
    made = []

    def make(sm=None):
        """sm: an SM count, -1 for all but one of the device's SMs, None for all of them"""
        real = _real_sm_count()
        sm = real - 1 if sm == -1 else sm
        if sm is not None and not 1 <= sm < real:
            pytest.skip(f"the device has {real} SMs: {sm} is not a smaller launch shape")
        made.append(Rig(monkeypatch, capfd, sm))
        return made[-1]
    yield make
    for r in made:
        r.close()


# ---- the groups of cases -----------------------------------------------------------------------------------------
def _census_eq(got, want, what):
    for k in CENSUS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    assert got["pixels"] == want["pixels"], (what, "pixels", got["pixels"], want["pixels"])


def check_2d(rig, want, cases=tuple(CASES_2D), tail_paints=("0", "1")):
    for case in cases:
        name, w, h, kw = CASES_2D[case]
        for paints in (tail_paints if kw.get("fused_tail") else (None,)):
            if paints is not None:
                rig.mp.setenv("FIDGET_B200_TAIL_PAINTS", paints)
            img, st = rig.watch(lambda: fb.render2d(rig.shape(name), fb.RenderConfig2D(w, h, **kw), stats=True))
            w_img, w_st = want.render2d(case)
            what = (case, rig.sm, paints)
            bad = np.argwhere(_bits(img) != _bits(w_img))
            assert not len(bad), (what, "first differing pixels (row, col)", bad[:5].tolist())
            _census_eq(st, w_st, what)
            if not kw.get("fused_tail") and not os.environ.get("FIDGET_B200_FUSE"):
                n_levels = len(kw.get("tile_sizes") or (128, 32, 8))
                rig.count_jobs(2, case, st["ambiguous"], n_levels)


def check_frames_2d(rig, want):
    imgs = rig.watch(lambda: fb.render2d_frames(rig.shape("colonnade.vm"), fb.RenderConfig2D(256, 256), z=Z_STACK))
    for k in range(len(Z_STACK)):
        assert np.array_equal(_bits(imgs[k]), _bits(want.z_stack(k))), ("z stack frame", k, rig.sm)


def _cmp_geometry(got, exp, what):
    bad = np.argwhere(got["depth"] != exp["depth"])
    assert not len(bad), (what, "first differing depth pixels", bad[:5].tolist())
    assert same_f32(got["normal"], exp["normal"]), what


def check_3d(rig, want, exact=tuple(CASES_3D_EXACT)):
    for case in exact:
        name, n = CASES_3D_EXACT[case]
        img, st = rig.watch(lambda: fb.render3d(rig.shape(name), fb.RenderConfig3D(n, n, n, exact_census=True),
                                                stats=True))
        o_img, o_st = want.render3d(name, n, n, n)
        _cmp_geometry(img, o_img, (case, rig.sm))
        _census_eq(st, o_st, (case, rig.sm))
        rig.count_jobs(3, case, st["ambiguous"], 5)          # exact census: the full ladder (128, 64, 32, 16, 8)
    img = rig.watch(lambda: fb.render3d(rig.shape("sphere0.7"), fb.RenderConfig3D(100, 60, 90)))
    _cmp_geometry(img, want.render3d("sphere0.7", 100, 60, 90)[0], ("sphere", rig.sm))
    cfg = fb.RenderConfig3D(256, 256, 256)
    img = rig.watch(lambda: fb.render3d(rig.shape("bear.vm"), cfg))
    _cmp_geometry(img, want.default(("bear3d",), lambda sh: fb.render3d(sh("bear.vm"), cfg)), ("bear", rig.sm))
    frames = rig.watch(lambda: fb.render3d_frames(rig.shape("colonnade.vm"), cfg, world_to_model=ORBIT))
    exp = want.default(("orbit",), lambda sh: fb.render3d_frames(sh("colonnade.vm"), cfg, world_to_model=ORBIT))
    for k in range(len(ORBIT)):
        _cmp_geometry(frames[k], exp[k], ("orbit view", k, rig.sm))
    scfg = fb.RenderConfig3D(256, 256, 256)
    img, index = rig.watch(lambda: fb.render3d_scene([rig.shape("colonnade.vm")] * 4, scfg, world_to_model=GRID2))
    e_img, e_index = want.default(("scene",), lambda sh: fb.render3d_scene([sh("colonnade.vm")] * 4, scfg,
                                                                           world_to_model=GRID2))
    _cmp_geometry(img, e_img, ("scene", rig.sm))
    assert np.array_equal(index, e_index), ("scene index", rig.sm)


def _cmp_leaves(g, o, what):
    assert len(g) == len(o), (what, len(g), len(o))
    for k in ("ix", "iy", "iz", "mask", "n_edges", "present"):
        bad = np.flatnonzero(g[k] != o[k])
        assert not len(bad), (what, k, "first differing leaves", o[bad[:3]][["ix", "iy", "iz"]].tolist())
    present = ((o["present"][:, None] >> np.arange(12)[None, :]) & 1).astype(bool)
    assert same_f32(g["pos"][present], o["pos"][present]), what
    assert same_f32(g["grad"][present], o["grad"][present]), what


def check_octree(rig, want):
    for name in ("sphere0.6", "colonnade.vm"):
        g, gst = fb.octree_sample(rig.shape(name), 5, stats=True)
        o, ost = want.octree(name, 5)
        _cmp_leaves(g, o, (name, rig.sm))
        for k in ("evaluated", "full", "empty", "ambiguous"):
            assert gst[k][:6] == ost[k][:6], (name, rig.sm, k)
        assert (gst["leaf_empty"], gst["leaf_full"], gst["leaf_surface"]) == \
            (ost["leaf_empty"], ost["leaf_full"], ost["leaf_surface"]), (name, rig.sm)
    g = fb.octree_sample(rig.shape("gyroid-sphere.vm"), 6)
    _cmp_leaves(g, want.default(("gyroid",), lambda sh: fb.octree_sample(sh("gyroid-sphere.vm"), 6)), ("gyroid", rig.sm))


def check_mesh(rig, want):
    for collapse in (False, True):
        verts, tris, info = fb.mesh(rig.shape("colonnade.vm"), 5, collapse=collapse)
        e_verts, e_tris, e_info = want.default(("mesh", collapse),
                                               lambda sh: fb.mesh(sh("colonnade.vm"), 5, collapse=collapse))
        assert info["open_edges"] == e_info["open_edges"], (collapse, rig.sm)
        assert_same_mesh(verts, tris, e_verts, e_tris)


def _points(n, nv):
    rng = np.random.default_rng(n)
    return [rng.uniform(-1, 1, n).astype(np.float32) for _ in range(nv)]


def _grad_points(n, nv):
    pts = _points(n, nv)
    rng = np.random.default_rng(n + 1)
    out = []
    for k in range(nv):
        g = np.zeros((n, 4), dtype=np.float32)
        g[:, 0] = pts[k]
        g[:, 1 + k % 3] = 1.0
        g[:, 1:] += rng.uniform(-1, 1, (n, 3)).astype(np.float32)
        out.append(g)
    return out


def check_slices(rig, want, cases):
    """cases: (model, n, grad).  Each slice from host arrays through the per-thread kernel (FIDGET_B200_NO_TMA=1),
    from device tensors (every variable 16-byte aligned) through the TMA kernel where the model fits it, and the
    oracle: the same bits (bear: the device paths with each other).  The FIDGET_B200_SLICE_DEBUG line of each call
    shows which kernel ran.  Returns (what, full tiles, CTAs) of each TMA run."""
    import torch
    runs = []
    for name, n, grad in cases:
        shape = rig.shape(name)
        args = _grad_points(n, shape.n_vars) if grad else _points(n, shape.n_vars)
        ev = shape.grad_slice_eval if grad else shape.float_slice_eval
        what = (name, n, "grad" if grad else "f32", rig.sm)
        rig.mp.setenv("FIDGET_B200_NO_TMA", "1")
        slow = np.asarray(rig.watch(lambda: ev(args)))
        assert rig.slices[-1] is None, (what, rig.slices[-1])
        rig.mp.delenv("FIDGET_B200_NO_TMA")
        dev = [torch.from_numpy(a).cuda() for a in args]
        fast = rig.watch(lambda: ev(dev)).cpu().numpy()
        line = rig.slices[-1]
        if SLICE_MODELS[name]:
            assert line is not None and line[0] == n and line[3] == rig.sm, (what, "took the per-thread kernel", line)
            runs.append((what, line[1], line[2]))
        else:
            assert line is None, (what, line)
        bad = np.argwhere(_bits(fast) != _bits(slow))
        assert not len(bad), (what, "device slice vs per-thread kernel, first differing points", bad[:5].tolist())
        if name not in LIBM:
            exp = want.grad_slice(name, n) if grad else want.float_slice(name, n)
            assert same_f32(fast, exp), what
    return runs


def _assert_tma_ring(runs, kind):
    """some CTA of a TMA run of this kind evaluated more than TMA_STAGES tiles: refilled a stage, waited on parity 1"""
    assert any(what[2] == kind and tiles > TMA_STAGES * ctas for what, tiles, ctas in runs), \
        (f"no {kind} slice made a TMA CTA run more than {TMA_STAGES} tiles", runs)


def _solver_starts(case):
    rng = np.random.default_rng(3)
    rows = np.tile(np.array(case.start, dtype=np.float32), (4096, 1))
    rows[:, :len(case.free)] = rng.uniform(-1.5, 1.5, (4096, len(case.free))).astype(np.float32)
    return rows


def check_solver(rig, want):
    ctx = fb.Context()
    case = sc.rosenbrock_chain(ctx, 3)
    shapes = [rig.track(fb.CudaShape(rig.cuda, ctx.tape(r))) for r in case.roots]
    vals, status, iters, err = fb.solve_batch(shapes, case.free, case.fixed, _solver_starts(case))
    rv, rs, ri, re_ = want.solve()
    assert np.array_equal(status, rs), rig.sm
    assert np.array_equal(iters, ri), rig.sm
    assert same_f32(vals, rv), rig.sm
    assert same_f32(err, re_), rig.sm


# ---- (a) emulated SM counts ---------------------------------------------------------------------------------------
def _assert_coop_rounds(rig):
    assert rig.coop, "no render took the cooperative level-0 kernel"
    assert all(sms == rig.sm for _, _, _, sms in rig.coop), (rig.sm, rig.coop)
    assert any(roots > rig.sm * per_sm for per_sm, _, roots, _ in rig.coop), \
        ("no cooperative launch had more root tiles than CTAs", rig.sm, rig.coop)


@pytest.mark.parametrize("sm", EMULATED + (None,), ids=EMULATED_IDS + ["real"])
def test_2d_at_any_sm_count(want, rigs, sm):
    rig = rigs(sm)
    check_2d(rig, want)
    check_frames_2d(rig, want)
    _assert_coop_rounds(rig)
    assert rig.jobs_over_warps[2], ("no 2D level had more jobs than warps", rig.jobs_under_warps[2])
    if sm is None:
        assert rig.jobs_under_warps[2], "the default grid should also see a level with fewer jobs than warps"


@pytest.mark.parametrize("sm", EMULATED + (None,), ids=EMULATED_IDS + ["real"])
def test_3d_at_any_sm_count(want, rigs, sm):
    rig = rigs(sm)
    check_3d(rig, want)
    assert rig.coop and all(sms == rig.sm for _, _, _, sms in rig.coop), (rig.sm, rig.coop)
    assert rig.jobs_over_warps[3], ("no 3D level had more jobs than warps", rig.jobs_under_warps[3])
    if sm is None:
        assert rig.jobs_under_warps[3]


@pytest.mark.parametrize("sm", EMULATED, ids=EMULATED_IDS)
def test_octree_and_mesh_at_any_sm_count(want, rigs, sm):
    rig = rigs(sm)
    check_octree(rig, want)
    check_mesh(rig, want)


@pytest.mark.parametrize("sm", EMULATED, ids=EMULATED_IDS)
def test_slices_at_any_sm_count(want, rigs, sm):
    rig = rigs(sm)
    cases = [(m, n, grad) for m in SLICE_MODELS for n in SLICE_SIZES for grad in (False, True)]
    if rig.sm == rig.real_sm - 1:   # so many CTAs take at most one ring of 100003 points: the long slices as well
        cases += [(m, BIG_GRAD if grad else BIG_F32, grad) for m in ("hi.vm", "bear.vm") for grad in (False, True)]
    runs = check_slices(rig, want, cases)
    _assert_tma_ring(runs, "f32")
    _assert_tma_ring(runs, "grad")


@pytest.mark.parametrize("sm", EMULATED, ids=EMULATED_IDS)
def test_solver_at_any_sm_count(want, rigs, sm):
    check_solver(rigs(sm), want)


# ---- (b) per-SM knobs on the real SM count ------------------------------------------------------------------------
KNOB_RUNS = [
    ({"BLOCKS_PER_SM": "1"}, ("2d", "3d", "octree")),
    ({"BLOCKS_PER_SM": "16"}, ("2d", "3d", "octree")),
    ({"LAST_LEVEL_BLOCKS_PER_SM": "24"}, ("3d",)),
    ({"VOXEL_BLOCKS_PER_SM": "1"}, ("3d",)),
    ({"VOXEL_BLOCKS_PER_SM": "32"}, ("3d",)),
    ({"PIXEL_BLOCKS_PER_SM": "1"}, ("2d",)),
    ({"PIXEL_BLOCKS_PER_SM": "32"}, ("2d",)),
    ({"COOP_PER_SM": "1"}, ("2d", "3d")),
    ({"COOP_PER_SM": "2"}, ("2d", "3d")),
    ({"COOP_THREADS": "64"}, ("2d", "3d")),
    ({"COOP_THREADS": "96"}, ("2d", "3d")),
    ({"COOP_THREADS": "160"}, ("2d", "3d")),
    ({"NO_COOP": "1"}, ("2d", "3d")),
    ({"NO_ZSORT": "1"}, ("3d",)),
    ({"SERIAL_FILL": "1"}, ("2d",)),
    ({"FUSE": "1"}, ("2d",)),
]


@pytest.mark.parametrize("env,groups", KNOB_RUNS, ids=["-".join(f"{k}={v}" for k, v in e.items()) for e, _ in KNOB_RUNS])
def test_per_sm_knob(want, rigs, env, groups, monkeypatch):
    rig = rigs()
    for k, v in env.items():
        monkeypatch.setenv("FIDGET_B200_" + k, v)
    if "2d" in groups:
        check_2d(rig, want)
        check_frames_2d(rig, want)
    if "3d" in groups:
        check_3d(rig, want)
    if "octree" in groups:
        check_octree(rig, want)
    if "COOP_THREADS" in env:
        assert rig.coop and all(t == int(env["COOP_THREADS"]) for _, t, _, _ in rig.coop), rig.coop
    if "COOP_PER_SM" in env:
        assert rig.coop and all(p <= int(env["COOP_PER_SM"]) for p, _, _, _ in rig.coop), rig.coop
        _assert_coop_rounds(rig)
    if "NO_COOP" in env:
        assert not rig.coop
    if "FUSE" in env:   # the switch is the flag: one fused tail launch per render
        name, w, h, kw = CASES_2D["prospero1024"]
        _, st = fb.render2d(rig.shape(name), fb.RenderConfig2D(w, h, **kw), stats=True)
        monkeypatch.delenv("FIDGET_B200_FUSE")
        _, flagged = fb.render2d(rig.shape(name), fb.RenderConfig2D(w, h, fused_tail=True, **kw), stats=True)
        _, plain = fb.render2d(rig.shape(name), fb.RenderConfig2D(w, h, **kw), stats=True)
        assert st["kernel_launches"] == flagged["kernel_launches"] < plain["kernel_launches"]


def test_long_slices_on_the_real_sm_count(want, rigs):
    """f32 needs more than TMA_STAGES x 132 SMs x 8 CTAs x 1024 points, gradients x 256 points, before any CTA of
    any occupancy reaches its fourth tile"""
    rig = rigs()
    assert BIG_F32 > TMA_STAGES * rig.sm * 8 * 1024 and BIG_GRAD > TMA_STAGES * rig.sm * 8 * 256
    runs = check_slices(rig, want, [(m, BIG_GRAD if grad else BIG_F32, grad) for m in ("hi.vm", "bear.vm")
                                    for grad in (False, True)])
    assert len(runs) == 4 and all(tiles > TMA_STAGES * ctas for _, tiles, ctas in runs), runs


_FUSED_PATH_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import fidget_b200 as fb
cuda = fb.CudaContext(0)
with open(sys.argv[2]) as f:
    shape = fb.CudaShape.from_vm(cuda, f.read())
img = fb.render2d(shape, fb.RenderConfig2D(int(sys.argv[3]), int(sys.argv[3]), tile_sizes=tuple(map(int, sys.argv[4:]))))
np.save(sys.stdout.buffer, img)
"""


@pytest.mark.parametrize("case", ["prospero512_32_8", "prospero1024_32_8_2"])
def test_level_fused_path(want, case, tmp_path):
    """FIDGET_B200_LEVEL_FUSED_PATH=1 (read once per process, so in a process of its own) runs the per-level
    launches with the fused tail's code path: the same image"""
    name, w, _, kw = CASES_2D[case]
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env["FIDGET_B200_LEVEL_FUSED_PATH"] = "1"
    out = subprocess.run([sys.executable, "-c", _FUSED_PATH_CHILD, ROOT, os.path.join(ROOT, "models", name), str(w)] +
                         [str(t) for t in kw["tile_sizes"]], env=env, check=True, capture_output=True).stdout
    img = np.load(io.BytesIO(out))
    assert np.array_equal(_bits(img), _bits(want.render2d(case)[0]))
