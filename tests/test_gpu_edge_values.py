"""Every device evaluator on the f32 edge catalogue (edge_values.py): subnormals, rounding boundaries, the ends of the
range, NaN payloads and the arguments where exp, ln, asin, acos and the trig functions overflow, underflow or leave
their domain, as registers, as immediates and as render inputs.

  (a) interpreted bulk evaluators (TMA and per-thread slices, gradients, point and interval evaluation): against
      op_reference (IEEE opcodes bit for bit, libm opcodes within ULP_BOUND of float64) and against the oracle
  (b) compiled tapes: float, gradient and interval results equal to the interpreters', bit for bit
  (c) ri / ir clauses with edge immediates, through (a), (b) and (d)
  (d) 2D renders: one frame per catalogue value or pair, the values bound to Context.var()s, so the level kernels see
      point intervals and the pixel kernels the values; and axis-driven routes s * x + v across each edge

What these catch that the rest of the suite does not: -ftz=true in build.sh or in the tape compiler's NVRTC options,
-fmad=true in the NVRTC options, and roundf written as floorf(x + 0.5f)."""
import zlib

import numpy as np
import pytest

import edge_values as E
import fidget_b200 as fb
import op_reference as R
from test_gpu_interp_ops import _both_paths, _is_fill

pytestmark = pytest.mark.gpu

F = np.float32
LENGTHS = (4097, 3 * 4096 + 5)          # ragged; >= 4096 so that the TMA slice kernel takes them


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _report(fails):
    assert not fails, "\n".join(str(f) for f in fails[:12]) + f"\n({len(fails)} failures)"


def _where(mask, *cols):
    return [tuple(np.asarray(c)[i].tolist() for c in cols) for i in np.flatnonzero(~mask)[:3]]


def _agree(op, got, want):
    """Per element, device result against the oracle's: IEEE opcodes bit for bit, libm opcodes within ULP_BOUND"""
    return E.close_ulps(got, want, R.ULP_BOUND[op]) if op in R.LIBM else E.same_bits(got, want)


def _pairs(cuda, orc, op):
    return [(form, imm, gtd, fb.CudaShape(cuda, gtd), orc.Tape.from_data(otd))
            for (form, imm, gtd), (_, _, otd) in zip(E.op_tapes(fb.Context, op), E.op_tapes(orc.Context, op))]


# ---- (a) + (c) interpreted bulk evaluators ----------------------------------------------------------------------------
@pytest.mark.parametrize("op", R.ALL_OPS)
def test_bulk_evaluators(cuda, orc, op, monkeypatch):
    fails = []
    for form, imm, td, g, o in _pairs(cuda, orc, op):
        vx, vy, _ = td.var_slots()
        vals, ins, _ = E.inputs(td, form)
        gin = E.grad_inputs(td, form, _seed(op, form, imm))
        for n in LENGTHS:
            what = (op, form, imm, n)
            v = [np.resize(a, n) for a in vals]
            args = E.operands(form, [np.resize(a, n) for a in ins], imm)
            f_tma, f_plain = _both_paths(monkeypatch, lambda: g.float_slice_eval(v))
            if not E.same_bits(f_tma, f_plain).all():
                fails.append((what, "float: TMA != per-thread", _where(E.same_bits(f_tma, f_plain), *args)))
            ok = E.value_ok(op, f_tma, args)
            if not ok.all():
                fails.append((what, "float vs op_reference", _where(ok, *args, f_tma)))
            ok = _agree(op, f_tma, o.float_slice_eval(v))
            if not ok.all():
                fails.append((what, "float vs oracle", _where(ok, *args, f_tma)))
            gv = [np.resize(a, (n, 4)) for a in gin]
            g_tma, g_plain = _both_paths(monkeypatch, lambda: g.grad_slice_eval(gv))
            if not E.same_bits(g_tma, g_plain).all():
                fails.append((what, "grad: TMA != per-thread"))
            ok = E.grad_ok(op, form, g_tma, gv[vx], gv[vy] if form == "rr" else None, imm, args)
            if not ok.all():
                fails.append((what, "grad vs op_reference", _where(ok, *args, g_tma)))
            og = o.grad_slice_eval(gv)
            ok = _agree(op, g_tma[:, 0], og[:, 0])
            if op in R.LIBM:
                ok &= E.close_ulps(g_tma[:, 1:], og[:, 1:], E.GRAD_ULPS[op]).all(axis=1)
            else:
                ok &= E.same_bits(g_tma, og).all(axis=1)
            if not ok.all():
                fails.append((what, "grad vs oracle", _where(ok, *args, g_tma, og)))
        # point evaluation with choices, on a seeded subset
        rng = np.random.default_rng(_seed(op, form, imm))
        for i in rng.choice(len(vals[0]), min(len(vals[0]), 96), replace=False):
            p = np.array([a[i] for a in vals], F)
            go, gc, gs = g.point_eval(p)
            oo, oc, os_ = o.point_eval(p)
            if not (_agree(op, go[:1], np.array([oo], F)).all() and np.array_equal(gc, oc) and gs == os_):
                fails.append(((op, form, imm), "point", p.tolist(), go[0], oo, gc, oc, gs, os_))
        # intervals: every box against op_reference (containment), a seeded subset against the oracle
        b = E.boxes(td.n_vars, 600, _seed(op, form, imm, "boxes"))
        out, ch, simp = g.interval_eval_batch(b, want_choices=True)
        ordered = b[:, [vx, vy]] if form == "rr" else b
        ok = E.contains(op, form, ordered, out[:, 0], imm, _seed(op, form, imm, "samples"))
        if not ok.all():
            fails.append(((op, form, imm), "interval containment",
                          [(ordered[i].tolist(), out[i, 0].tolist()) for i in np.flatnonzero(~ok)[:3]]))
        for i in rng.choice(len(b), 120, replace=False):
            oo, oc, os_ = o.interval_eval(b[i])
            if not (_agree(op, out[i, 0], oo).all() and np.array_equal(ch[i], oc) and bool(simp[i]) == os_):
                fails.append(((op, form, imm), "interval vs oracle", b[i].tolist(), out[i, 0].tolist(), oo.tolist(),
                              ch[i].tolist(), oc.tolist()))
    _report(fails)


# ---- (b) + (c) compiled tapes -------------------------------------------------------------------------------------
def _multi_tapes(op):
    """Tapes of ``op`` for the tape compiler: the plain form, then every kept immediate of a form as one output each
    (one NVRTC compile per form)"""
    out = []
    tapes = E.op_tapes(fb.Context, op)
    for form in R.FORMS[op]:
        c = fb.Context()
        if form in ("r", "rr"):
            out.append((form, tapes[0][2]))
            continue
        imms = [imm for f, imm, _ in tapes if f == form]
        x = c.x()
        roots = [c.binary(op, x, c.constant(float(k))) if form == "ri" else c.binary(op, c.constant(float(k)), x)
                 for k in imms]
        out.append((form, c.tape(roots)))
    return out


def _compiled_vs_interpreter(shape, vals, grads, boxes, what, fails):
    comp = shape.compile()
    for kind, got, want in (("float", comp.float_slice_eval(vals), shape.float_slice_eval(vals)),
                            ("grad", comp.grad_slice_eval(grads), shape.grad_slice_eval(grads))):
        got, want = np.asarray(got), np.asarray(want)
        if not E.same_bits(got, want).all():
            bad = ~E.same_bits(got, want)
            fails.append((what, kind, int(bad.sum()), got[bad][:3].tolist(), want[bad][:3].tolist()))
    go, gc, gs = comp.interval_eval_batch(boxes, want_choices=True)
    wo, wc, ws = shape.interval_eval_batch(boxes, want_choices=True)
    if not (E.same_bits(go, wo).all() and np.array_equal(gc, wc) and np.array_equal(gs, ws)):
        fails.append((what, "interval", int((~E.same_bits(go, wo)).sum())))
    comp.close()


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_compiled_tapes(cuda, op):
    fails = []
    for form, td in _multi_tapes(op):
        shape = fb.CudaShape(cuda, td)
        vals, _, _ = E.inputs(td, "rr" if form == "rr" else "r")
        grads = E.grad_inputs(td, "rr" if form == "rr" else "r", _seed(op, form))
        b = E.boxes(td.n_vars, 2000, _seed(op, form, "boxes"))
        _compiled_vs_interpreter(shape, vals, grads, b, (op, form, td.output_count), fails)
    _report(fails)


@pytest.mark.parametrize("route", E.ROUTES, ids=[r[0] for r in E.ROUTES])
def test_compiled_routes(cuda, route):
    """s * x + v and the route's ops, one output each: a contraction of s * x + v changes the exp route's values"""
    name, s, v, _, ops = route
    c = fb.Context()
    arg = c.add(c.mul(c.x(), float(s)), float(v))
    td = c.tape([c.sub(E.route_term(c, op, imm, arg), float(F(level))) for op, imm, level in ops] + [arg])
    rng = np.random.default_rng(_seed(name))
    x = np.concatenate([E.VALUES, rng.uniform(-1, 1, 5000)]).astype(F)
    g = np.zeros((len(x), 4), F)
    g[:, 0], g[:, 1] = x, 1.0
    g[:, 1:] += rng.uniform(-2, 2, (len(x), 3)).astype(F)
    b = E.boxes(1, 2000, _seed(name, "boxes"))
    fails = []
    _compiled_vs_interpreter(fb.CudaShape(cuda, td), [x], [g], b, name, fails)
    _report(fails)


# ---- (d) + (c) 2D renders with the values as ShapeVars ------------------------------------------------------------
W, H = 24, 16
CONFIGS = {"default": {}, "perfect": {"pixel_perfect": True}, "fused": {"fused_tail": True},
           "tiles": {"tile_sizes": (64, 16, 4)}}


def _var_tape(op, form, imm, pad):
    """(shape, slot of a, slot of b or None, slot of the pad var or None): op over Context.var()s, ``pad`` wraps it as
    and(p, term) with p = 65 * c over 64 clauses (c bound to 1), so the cooperative level-0 kernel (tapes of >= 64
    clauses) takes it; p is never 0 and its interval never holds 0, so and() passes the term through unchanged"""
    c = fb.Context()
    a, va = c.var()
    b, vb = c.var() if form == "rr" else (None, None)
    if form == "r":
        term = c.unary(op, a)
    elif form == "rr":
        term = c.binary(op, a, b)
    else:
        k = c.constant(float(imm))
        term = c.binary(op, a, k) if form == "ri" else c.binary(op, k, a)
    vc = None
    if pad:
        p, vc = c.var()
        q = p
        for _ in range(64):
            q = c.add(q, p)
        term = c.binary("and", q, term)
    td = c.tape(term)
    slot = {vid: i for i, (_, vid) in enumerate(td.vars())}
    return td, slot[va], slot.get(vb), slot.get(vc)


def _frame_checks(op, imgs, a, b, imm, form, what, fails):
    """Each frame k is the constant op(a[k], b[k]): pixels equal to it (libm within ULP_BOUND of float64), fills with
    its sign (libm: or within tolerance of 0)"""
    args = E.operands(form, (a, b) if form == "rr" else (a,), imm)
    ref32 = R.f32(op, *args)
    pix = imgs.reshape(len(a), -1)
    fill = _is_fill(pix)
    inside = fb.pixel_inside(pix)
    ref = np.broadcast_to(ref32[:, None], pix.shape)
    if op in R.LIBM:
        ref64 = np.broadcast_to(R.f64(op, *args)[:, None], pix.shape)
        val_ok = E.libm_error(pix, ref64) <= R.ULP_BOUND[op]
        with np.errstate(all="ignore"):
            near = np.abs(ref64) <= R.ULP_BOUND[op] * R.ulp(ref64)
        sign_ok = ~np.isnan(ref64) & (near | np.where(inside, ref64 < 0, ref64 > 0))
    else:
        val_ok = E.same_bits(pix, ref)
        with np.errstate(all="ignore"):
            sign_ok = ~np.isnan(ref) & np.where(inside, ref < 0, ref > 0)
    ok = np.where(fill, sign_ok, val_ok).all(axis=1)
    if not ok.all():
        k = np.flatnonzero(~ok)[:3]
        fails.append((what, [(tuple(x[i].tolist() for x in args), ref32[i].tolist(), pix[i, :2].tolist(),
                              bool(fill[i].any())) for i in k]))
    return fill.any()


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_render_frames(cuda, op, monkeypatch, capfd):
    fails = []
    plain = [("rr", None)] if op in R.BINARY else [("r", None)]
    imms = [(form, imm) for form, imm, _ in E.op_tapes(fb.Context, op) if form in ("ri", "ir")]
    filled = False
    for form, imm in plain + imms:
        pads = (False, True) if imm is None else (False,)
        for pad in pads:
            td, sa, sb, sc = _var_tape(op, form, imm, pad)
            shape = fb.CudaShape(cuda, td)
            a, b = E.pairs() if form == "rr" else (E.VALUES, None)
            vv = np.zeros((len(a), td.n_vars), F)
            vv[:, sa] = a
            if sb is not None:
                vv[:, sb] = b
            if sc is not None:
                vv[:, sc] = 1.0
            configs = CONFIGS if imm is None else {k: CONFIGS[k] for k in ("default", "perfect")}
            for name, kw in configs.items():
                monkeypatch.setenv("FIDGET_B200_COOP_DEBUG", "1")
                capfd.readouterr()
                if kw.get("fused_tail"):      # frame batches do not take the fused tail: single renders of a subset
                    pick = np.random.default_rng(_seed(op, form, pad)).choice(len(a), 48, replace=False)
                    imgs = np.stack([fb.render2d(shape, fb.RenderConfig2D(W, H, var_values=tuple(vv[k]), **kw))
                                     for k in pick])
                    fa, fb_ = a[pick], None if b is None else b[pick]
                else:
                    imgs = fb.render2d_frames(shape, fb.RenderConfig2D(W, H, **kw), var_values=vv)
                    fa, fb_ = a, b
                err = capfd.readouterr().err
                if pad and not kw.get("pixel_perfect") and "coop:" not in err:
                    fails.append(((op, form, name), "padded tape did not take the cooperative level-0 kernel"))
                filled |= _frame_checks(op, imgs, fa, fb_, imm, form, (op, form, imm, name, pad), fails)
    monkeypatch.delenv("FIDGET_B200_COOP_DEBUG")
    _report(fails)
    assert filled, "no frame was filled: the level kernels never decided a tile"


@pytest.mark.parametrize("route", E.ROUTES, ids=[r[0] for r in E.ROUTES])
def test_render_routes(cuda, orc, route):
    """op(s * x + v) - level over the image, against the f32 / float64 reference of each pixel's argument, the argument
    itself rendered pixel-perfect and checked bit for bit against the oracle (as OpCase.pixel_reference does)"""
    name, s, v, edge, ops = route
    w, h = 256, 40
    fails = []
    arg_img = None
    for op, imm, level in ops:
        tapes = []
        for Ctx in (fb.Context, orc.Context):
            c = Ctx()
            arg = c.add(c.mul(c.x(), float(s)), float(v))
            tapes.append((c.tape(arg), c.tape(c.sub(E.route_term(c, op, imm, arg), float(F(level))))))
        if arg_img is None:
            arg_img = fb.render2d(fb.CudaShape(cuda, tapes[0][0]), fb.RenderConfig2D(w, h, pixel_perfect=True))
            want, _ = orc.render2d(orc.Tape.from_data(tapes[1][0]), w, h, pixel_perfect=True)
            assert E.same_bits(arg_img, want).all(), (name, "argument differs from the oracle")
            assert arg_img.min() < edge < arg_img.max(), (name, arg_img.min(), arg_img.max())
        args = (arg_img,) if imm is None else (arg_img, np.full_like(arg_img, imm))
        lv = F(level)
        with np.errstate(all="ignore"):
            ref32 = R.f32("sub", R.f32(op, *args), np.full_like(arg_img, lv))
            t64 = R.f64(op, *args)
            ref64 = t64 - np.float64(lv)
            tol = R.ULP_BOUND.get(op, 0) * R.ulp(t64) + R.ulp(ref64)
        shape = fb.CudaShape(cuda, tapes[0][1])
        for cfg, kw in CONFIGS.items():
            img = fb.render2d(shape, fb.RenderConfig2D(w, h, **kw))
            fill = _is_fill(img)
            inside = fb.pixel_inside(img)
            with np.errstate(all="ignore"):
                if op in R.LIBM:
                    val_ok = (np.isnan(img) & np.isnan(ref64)) | (img.astype(np.float64) == ref64) | \
                        (np.abs(img.astype(np.float64) - ref64) <= tol)
                    sign_ok = ~np.isnan(ref64) & ((np.abs(ref64) <= tol) | np.where(inside, ref64 < 0, ref64 > 0))
                else:
                    val_ok = E.same_bits(img, ref32)
                    sign_ok = ~np.isnan(ref32) & np.where(inside, ref32 < 0, ref32 > 0)
            ok = np.where(fill, sign_ok, val_ok)
            if kw.get("pixel_perfect"):
                ok &= ~fill
            if not ok.all():
                idx = [tuple(i) for i in np.argwhere(~ok)[:3]]
                fails.append(((name, op, cfg), [(arg_img[i].item(), img[i].item(), ref32[i].item()) for i in idx]))
    _report(fails)
