"""Every opcode, in each of its clause forms, through each device interpreter: the cooperative level-0 kernel (tapes of
>= 64 clauses), the level / pixel / tail kernels of 2D renders, the voxel and normal kernels of 3D renders, the TMA
slice kernels, the octree sampler and the solver.  Each result is checked against the CPU oracle (bit for bit where the
reference is IEEE-exact) and against the float64 numpy reference of op_reference.py, which shares no code with either:

  IEEE opcodes   bit-exact, images and census;
  libm opcodes   (sin cos tan asin acos atan exp ln atan2) within the CUDA Programming Guide's documented ulp bounds;
                 fills must still be sound, except at pixels whose float64 value lies within that bound of 0."""
import zlib

import numpy as np
import pytest

import fidget_b200 as fb
import op_reference as R
import solve_oracle as so
import solver_cases as sc
from conftest import same_f32
from scene_merge import fold

pytestmark = pytest.mark.gpu

SIZES = [(256, 256), (200, 136)]
CONFIGS = {"default": {}, "tiles": {"tile_sizes": (64, 16, 4)}, "perfect": {"pixel_perfect": True},
           "fused": {"fused_tail": True}}
FILL_MASK, FILL_TAG = np.uint32(0xFF << 9), np.uint32(0xF6 << 9)


def _same_pixels(a, b):
    """Per-pixel equality of RawDistancePixel images: equal bits, or both a NaN that is not a fill."""
    ab, bb = a.view(np.uint32), b.view(np.uint32)
    plain_nan = lambda img, bits: np.isnan(img) & ((bits & FILL_MASK) != FILL_TAG)  # noqa: E731
    return (ab == bb) | (plain_nan(a, ab) & plain_nan(b, bb))


def _is_fill(img):
    return np.isnan(img) & ((img.view(np.uint32) & FILL_MASK) == FILL_TAG)


class OpCase:
    """One opcode's 2D / 3D op shapes, on the device and in the oracle, plus per-size float64 pixel references."""

    def __init__(self, orc, cuda, op):
        self.op = op
        self.orc, self.cuda = orc, cuda
        seed = zlib.crc32(op.encode()) & 0xFFFF
        self.g = {}
        self.o = {}
        self.parts = {}
        for dim in (2, 3):
            gctx, groot, gprims = R.op_shape(fb.Context, op, seed, dim=dim)
            octx, oroot, _ = R.op_shape(orc.Context, op, seed, dim=dim)
            self.g[dim] = fb.CudaShape(cuda, gctx.tape(groot))
            self.o[dim] = orc.Tape.from_data(octx.tape(oroot))
            self.parts[dim] = (gctx, octx, gprims, R.op_shape(orc.Context, op, seed, dim=dim)[2])
        self._pp = {}

    def pixel_reference(self, w, h):
        """(device pixel-perfect image, f32 numpy image, float64 numpy image, tolerance) at w x h, from pixel-perfect
        renders of each primitive's argument and disc tapes (themselves checked bit for bit against the oracle)."""
        if (w, h) in self._pp:
            return self._pp[(w, h)]
        gctx, octx, gprims, oprims = self.parts[2]
        cfg = fb.RenderConfig2D(w, h, pixel_perfect=True)

        def render(node_g, node_o):
            img = fb.render2d(fb.CudaShape(self.cuda, gctx.tape(node_g)), cfg)
            ref, _ = self.orc.render2d(self.orc.Tape.from_data(octx.tape(node_o)), w, h, pixel_perfect=True)
            assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), "argument tape differs from the oracle"
            return img

        terms32, terms64, masks, tol = [], [], [], np.zeros((h, w))
        for gp, op_ in zip(gprims, oprims):
            vals = []
            for ga, oa in zip(gp.args, op_.args):
                vals.append(np.full((h, w), ga, dtype=np.float32) if isinstance(ga, float) else render(ga, oa))
            masks.append(render(gp.mask, op_.mask))
            terms32.append(R.f32(self.op, *vals))
            t64 = R.f64(self.op, *vals)
            terms64.append(t64)
            if self.op in R.LIBM:
                with np.errstate(all="ignore"):
                    tol = np.maximum(tol, np.nan_to_num(R.ULP_BOUND[self.op] * R.ulp(t64), nan=0.0))
        img = fb.render2d(self.g[2], cfg)
        ref32 = R.combine(gprims, terms32, masks)
        ref64 = R.combine(gprims, terms64, masks)
        with np.errstate(all="ignore"):
            tol = tol + R.ulp(ref64)
        self._pp[(w, h)] = (img, ref32, ref64, tol)
        return self._pp[(w, h)]

    def accept(self, w, h, img):
        """Pixels of a libm-op render ``img`` that (b) and (c) accept: values within tolerance of the float64
        reference, and fills whose sign agrees with it or whose float64 value lies within tolerance of 0."""
        _, _, ref64, tol = self.pixel_reference(w, h)
        fill = _is_fill(img)
        inside = fb.pixel_inside(img)
        with np.errstate(all="ignore"):
            near = np.abs(ref64) <= tol
            val_ok = (np.isnan(img) & np.isnan(ref64)) | (img == ref64) | (np.abs(img.astype(np.float64) - ref64) <= tol)
            fill_ok = ~np.isnan(ref64) & (near | np.where(inside, ref64 < 0, ref64 > 0))
        return np.where(fill, fill_ok, val_ok)


_CASES = {}


@pytest.fixture
def case(orc, cuda, op):
    if op not in _CASES:
        _CASES[op] = OpCase(orc, cuda, op)
    return _CASES[op]


# ---- (a) 2D renders against the oracle, with and without the cooperative level-0 kernel ----------------------------
@pytest.mark.parametrize("op", R.ALL_OPS)
def test_render2d_vs_oracle(case, op, monkeypatch, capfd):
    for w, h in SIZES:
        for name, kw in CONFIGS.items():
            ts = kw.get("tile_sizes", (128, 32, 8))
            want, want_st = case.orc.render2d(case.o[2], w, h, pixel_perfect=kw.get("pixel_perfect", False),
                                              tile_sizes=ts, threads=8)
            for coop in (True, False):
                monkeypatch.setenv("FIDGET_B200_NO_COOP", "0" if coop else "1")
                monkeypatch.setenv("FIDGET_B200_COOP_DEBUG", "1")
                capfd.readouterr()
                got, st = fb.render2d(case.g[2], fb.RenderConfig2D(w, h, **kw), stats=True)
                err = capfd.readouterr().err
                if not kw.get("pixel_perfect"):
                    assert ("coop:" in err) == coop, (name, coop, err[-300:])
                what = (op, (w, h), name, coop)
                if op in R.LIBM:
                    ok = _same_pixels(got, want) | case.accept(w, h, got)
                    assert ok.all(), (what, np.argwhere(~ok)[:5])
                else:
                    assert _same_pixels(got, want).all(), (what, np.argwhere(~_same_pixels(got, want))[:5])
                    for k in ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified", "pixels"):
                        assert st[k] == want_st[k], (what, k, st[k], want_st[k])


# ---- (b) pixel values against the float64 reference -----------------------------------------------------------------
@pytest.mark.parametrize("op", R.ALL_OPS)
def test_pixel_values_vs_float64(case, op):
    for w, h in SIZES:
        img, ref32, ref64, tol = case.pixel_reference(w, h)
        if op in R.LIBM:
            assert np.array_equal(np.isnan(img), np.isnan(ref64)), (op, (w, h))
            with np.errstate(all="ignore"):
                err = np.abs(img.astype(np.float64) - ref64)
            fin = ~np.isnan(ref64)
            ok = (img == ref64) | (err <= tol)
            assert ok[fin].all(), (op, (w, h), np.argwhere(fin & ~ok)[:5])
        else:
            assert same_f32(img, ref32), (op, (w, h), np.argwhere(~_same_pixels(img, ref32))[:5])


# ---- (c) fills are sound, checked against the pixel-perfect values ---------------------------------------------------
@pytest.mark.parametrize("op", R.ALL_OPS)
def test_fills_sound(case, op):
    kinds = set()
    for w, h in SIZES:
        pp, _, ref64, tol = case.pixel_reference(w, h)
        img = fb.render2d(case.g[2], fb.RenderConfig2D(w, h))
        fill = _is_fill(img)
        inside = fb.pixel_inside(img)
        with np.errstate(all="ignore"):
            ok = ~np.isnan(pp) & np.where(inside, pp < 0, pp > 0)
            if op in R.LIBM:
                ok |= np.abs(ref64) <= tol
        bad = fill & ~ok
        assert not bad.any(), (op, (w, h), np.argwhere(bad)[:5], pp[bad][:5])
        kinds |= {"in"} if (fill & inside).any() else set()
        kinds |= {"out"} if (fill & ~inside).any() else set()
        kinds |= {"nan"} if np.isnan(pp).any() else set()
    # the shape is doing its job: both kinds of fill occur (NaN regions only where the op makes them)
    assert {"in", "out"} <= kinds, (op, kinds)


# ---- (d) 3D renders -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", R.ALL_OPS)
def test_render3d_vs_oracle(case, op):
    for w, h, d in ((128, 128, 128), (100, 72, 90)):
        got = fb.render3d(case.g[3], fb.RenderConfig3D(w, h, d))
        want, _ = case.orc.render3d(case.o[3], w, h, d, threads=8)
        assert (want["depth"] > 0).any(), "empty image"
        if op not in R.LIBM:
            assert np.array_equal(got["depth"], want["depth"]), (op, (w, h, d))
            assert same_f32(got["normal"], want["normal"]), (op, (w, h, d))
            continue
        dd = np.abs(got["depth"].astype(np.int64) - want["depth"].astype(np.int64))
        assert dd.max() <= 1 and (dd > 0).mean() <= 1e-3, (op, (w, h, d), dd.max(), (dd > 0).mean())
        same = (dd == 0) & (want["depth"] > 0)
        a, b = got["normal"][same].astype(np.float64), want["normal"][same].astype(np.float64)
        na, nb = np.linalg.norm(a, axis=1), np.linalg.norm(b, axis=1)
        good = np.isfinite(na) & np.isfinite(nb) & (nb > 1e-3) & (nb < 1e4)
        cos = np.sum(a[good] * b[good], axis=1) / (na[good] * nb[good])
        assert (cos >= 1 - 1e-4).mean() >= 0.999, (op, (w, h, d), np.sort(cos)[:5])


# ---- (e) the TMA slice kernels against the plain slice kernels, the oracle and the numpy reference -------------------
def _single_op_tapes(op):
    """(form, imm, device shape built from fb.Context, tape data) for every clause form of ``op``"""
    out = []
    if op in R.UNARY:
        ctx = fb.Context()
        return [("r", None, ctx.tape(ctx.unary(op, ctx.x())))]
    ctx = fb.Context()
    out.append(("rr", None, ctx.tape(ctx.binary(op, ctx.x(), ctx.y()))))
    for form in R.FORMS[op]:
        for k in (0.75, -2.0):
            c = fb.Context()
            if form == "ri":
                out.append(("ri", k, c.tape(c.binary(op, c.x(), c.constant(k)))))
            elif form == "ir":
                out.append(("ir", k, c.tape(c.binary(op, c.constant(k), c.x()))))
    return out


def _slice_points(rng, n):
    from test_gpu_known_answers import SPECIAL
    xs, ys = [a.ravel() for a in np.meshgrid(SPECIAL, SPECIAL)]
    x = np.concatenate([xs, rng.uniform(-3, 3, n)])[:n].astype(np.float32)
    y = np.concatenate([ys, np.round(rng.uniform(-3, 3, n) * 2) / 2])[:n].astype(np.float32)
    return x, y


def _both_paths(monkeypatch, fn):
    out = []
    for no_tma in ("0", "1"):
        monkeypatch.setenv("FIDGET_B200_NO_TMA", no_tma)
        out.append(np.asarray(fn()))
    return out


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_slices_tma(cuda, orc, op, monkeypatch):
    rng = np.random.default_rng(zlib.crc32(op.encode()))
    for n in (4096, 4097, 12289):
        x, y = _slice_points(rng, n)
        g = np.zeros((n, 4), dtype=np.float32)
        g[:, 0], g[:, 1] = x, 1.0
        g[:, 1:] += (rng.uniform(-1, 1, (n, 3)) * (rng.random((n, 1)) < 0.5)).astype(np.float32)
        gy = np.zeros((n, 4), dtype=np.float32)
        gy[:, 0], gy[:, 2] = y, 1.0
        for form, imm, td in _single_op_tapes(op):
            shape = fb.CudaShape(cuda, td)
            vx, vy, _ = td.var_slots()
            vals, grads = [None] * td.n_vars, [None] * td.n_vars
            vals[vx], grads[vx] = x, g
            if vy >= 0:
                vals[vy], grads[vy] = y, gy
            f_tma, f_plain = _both_paths(monkeypatch, lambda: shape.float_slice_eval(vals))
            g_tma, g_plain = _both_paths(monkeypatch, lambda: shape.grad_slice_eval(grads))
            what = (op, form, imm, n)
            assert same_f32(f_tma, f_plain) and same_f32(g_tma, g_plain), what
            args = (x, y) if form == "rr" else (x, np.full(n, imm, np.float32)) if form == "ri" else \
                (np.full(n, imm, np.float32), x) if form == "ir" else (x,)
            want = R.f32(op, *args)
            gwant = R.grad(op, form, g, gy if form == "rr" else None, imm)
            if op in R.LIBM:
                assert R.ulp_distance(f_tma, want).max() <= R.ULP_BOUND[op], what
                assert R.ulp_distance(g_tma[:, 0], want).max() <= R.ULP_BOUND[op], what
            else:
                assert same_f32(f_tma, want), (what, np.argwhere(~((f_tma == want) | np.isnan(want)))[:4])
                assert same_f32(g_tma, gwant), what
        # the whole op shape: IEEE ops bit for bit against the oracle
        if op not in R.LIBM:
            gctx, root, _ = R.op_shape(fb.Context, op, 7, dim=3)
            octx, oroot, _ = R.op_shape(orc.Context, op, 7, dim=3)
            td = gctx.tape(root)
            shape, o = fb.CudaShape(cuda, td), orc.Tape.from_data(octx.tape(oroot))
            pts = [rng.uniform(-1.2, 1.2, n).astype(np.float32) for _ in range(td.n_vars)]
            gpts = []
            for k, p in enumerate(pts):
                a = np.zeros((n, 4), dtype=np.float32)
                a[:, 0], a[:, 1 + k] = p, 1.0
                gpts.append(a)
            f_tma, f_plain = _both_paths(monkeypatch, lambda: shape.float_slice_eval(pts))
            g_tma, g_plain = _both_paths(monkeypatch, lambda: shape.grad_slice_eval(gpts))
            assert same_f32(f_tma, f_plain) and same_f32(g_tma, g_plain), (op, n, "shape")
            assert same_f32(f_tma, o.float_slice_eval(pts)), (op, n, "shape")
            assert same_f32(g_tma, o.grad_slice_eval(gpts)), (op, n, "shape")


# ---- (f) octree sampling -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", R.IEEE)
def test_octree_vs_oracle(case, op):
    o_leaves, o_st = case.orc.octree_sample(case.o[3], 5)
    g_leaves, g_st = fb.octree_sample(case.g[3], 5, stats=True)
    assert len(g_leaves) == len(o_leaves) > 0
    for f in ("ix", "iy", "iz", "mask", "n_edges", "present"):
        assert np.array_equal(g_leaves[f], o_leaves[f]), f
    present = ((o_leaves["present"][:, None] >> np.arange(12)[None, :]) & 1).astype(bool)
    for f in ("pos", "grad"):
        assert same_f32(g_leaves[f][present], o_leaves[f][present]), f
    for k in ("evaluated", "full", "empty", "ambiguous"):
        assert g_st[k][:6] == o_st[k][:6], k


# ---- (g) the solver ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", R.IEEE)
def test_solver_vs_oracle(cuda, orc, op):
    rng = np.random.default_rng(zlib.crc32(op.encode()))
    starts = rng.uniform(-2, 2, (24, 2)).astype(np.float32)
    starts[:4] = [[0.0, 0.0], [1.0, -1.0], [0.5, 0.5], [-1.5, 2.0]]
    keys = ["x", "y"]
    for max_iters in (1, 3):
        ctx = fb.Context()
        g = fb.CudaShape(cuda, ctx.tape(R.scalar_residual(ctx, op, ctx.x(), ctx.y())))
        dev = fb.solve_batch([g], keys, [], starts, max_iters)
        octx = orc.Context()
        td = octx.tape(R.scalar_residual(octx, op, octx.x(), octx.y()))
        vals, res = so.solve_batch([orc.Tape.from_data(td)], [sc.slot_map(td, keys)], 2, starts, max_iters)
        assert np.array_equal(dev[1], res["status"]), (op, max_iters)
        assert np.array_equal(dev[2], res["iterations"]), (op, max_iters)
        assert same_f32(dev[0], vals) and same_f32(dev[3], res["err"]), (op, max_iters)


# ---- (h) the frame and scene instantiations on a tape of every opcode ------------------------------------------------
def test_instantiations_every_op(cuda):
    ctx, root = R.every_op_shape(fb.Context)
    shape = fb.CudaShape(cuda, ctx.tape(root))
    assert shape.size() >= 64
    # 2D frames: Z slices
    cfg = fb.RenderConfig2D(200, 136)
    zs = np.array([-0.4, -0.05, 0.2, 0.55], dtype=np.float32)
    frames = fb.render2d_frames(shape, cfg, z=zs)
    for k, z in enumerate(zs):
        single = fb.render2d(shape, fb.RenderConfig2D(200, 136, z=float(z)))
        assert np.array_equal(frames[k].view(np.uint32), single.view(np.uint32)), ("2d frame", k)
    # 3D frames: views
    cfg3 = fb.RenderConfig3D(128, 96, 112)
    views = []
    for k in range(4):
        a = 0.4 * k
        m = np.eye(4, dtype=np.float32)
        m[0, 0], m[0, 2], m[2, 0], m[2, 2] = np.cos(a), -np.sin(a), np.sin(a), np.cos(a)
        views.append(m)
    views = np.stack(views).astype(np.float32)
    frames = fb.render3d_frames(shape, cfg3, world_to_model=views)
    for k in range(4):
        single = fb.render3d(shape, fb.RenderConfig3D(128, 96, 112, world_to_model=views[k]))
        assert np.array_equal(frames[k]["depth"], single["depth"]), ("3d frame", k)
        assert same_f32(frames[k]["normal"], single["normal"]), ("3d frame", k)
    # a 2-placement scene against the fold of single renders
    place = np.stack([views[0], views[2]])
    img, index = fb.render3d_scene([shape, shape], cfg3, world_to_model=place)
    singles = [fb.render3d(shape, fb.RenderConfig3D(128, 96, 112, world_to_model=place[k])) for k in range(2)]
    want, want_index = fold(singles)
    assert np.array_equal(img["depth"], want["depth"]) and same_f32(img["normal"], want["normal"])
    assert np.array_equal(index, want_index)
