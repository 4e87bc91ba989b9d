"""The numpy opcode reference (op_reference.py) against the CPU oracle, and the op shapes' tapes: the reference equals
the oracle bit for bit on every IEEE opcode in every clause form (values and gradients), is within 1 ulp of it on the
libm opcodes, and each op shape carries its opcode in each intended form on a tape long enough for the cooperative
level-0 schedule."""
import zlib

import numpy as np
import pytest

import op_reference as R
from conftest import same_f32

SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 0.5, -0.5, 2.0, -2.0, 1.5, -1.5, 3.25, -7.75, 1e-3, -1e-3, 10.0, -10.0,
                    100.0, 0.99999, -0.99999, 6.2831855, 3.1415927, 1.5707964, -3.1415927, 4.712389,
                    1e-30, 1e30, np.inf, -np.inf, np.nan], dtype=np.float32)
IMMS = (0.75, -2.0, 0.0, 1.0)


def _points(op, rng, n_random=2000):
    """Operand arrays: every pair of SPECIAL values, plus random values at several magnitudes and exact integers."""
    xs, ys = [a.ravel() for a in np.meshgrid(SPECIAL, SPECIAL)]
    r = np.concatenate([rng.uniform(-4, 4, n_random), rng.uniform(-1e4, 1e4, n_random // 4),
                        np.round(rng.uniform(-5, 5, n_random // 4) * 2) / 2]).astype(np.float32)
    s = np.concatenate([rng.uniform(-4, 4, n_random), rng.uniform(-3, 3, n_random // 4),
                        np.round(rng.uniform(-5, 5, n_random // 4))]).astype(np.float32)
    return np.concatenate([xs, r]), np.concatenate([ys, s])


def _tapes(orc, op):
    """(form, imm, oracle tape) for every clause form, the immediates of IMMS for ri / ir.  A clause the Context
    folds away (x + 0, x * 1, ...) is left out: its tape no longer runs the opcode."""
    from fidget_b200.host import OP
    return [t for t in _all_tapes(orc, op) if any(o == OP[op] for o, _ in _clauses(t[2].bytecode().words))]


def _all_tapes(orc, op):
    out = []
    ctx = orc.Context()
    if op in R.UNARY:
        out.append(("r", None, orc.Tape.from_data(ctx.tape(ctx.unary(op, ctx.x())))))
        return out
    out.append(("rr", None, orc.Tape.from_data(ctx.tape(ctx.binary(op, ctx.x(), ctx.y())))))
    for k in IMMS:
        for form in R.FORMS[op]:
            if form == "ri":
                c = orc.Context()
                out.append(("ri", k, orc.Tape.from_data(c.tape(c.binary(op, c.x(), c.constant(k))))))
            elif form == "ir":
                c = orc.Context()
                out.append(("ir", k, orc.Tape.from_data(c.tape(c.binary(op, c.constant(k), c.x())))))
    return out


def _by_slot(tape, x, y):
    """x and y values in the tape's input slot order"""
    vx, vy, _ = tape.data.var_slots()
    out = [None, None]
    out[vx], out[vy] = x, y
    return out


def _ref_f32(op, form, imm, a, b):
    if form == "r":
        return R.f32(op, a)
    if form == "rr":
        return R.f32(op, a, b)
    k = np.full_like(a, imm)
    return R.f32(op, a, k) if form == "ri" else R.f32(op, k, a)


def _grad_inputs(rng, a, b):
    """[n, 4] gradients of two registers with mixed derivative vectors (zeros, units, random, NaN-free)."""
    n = len(a)
    ga = np.zeros((n, 4), dtype=np.float32)
    gb = np.zeros((n, 4), dtype=np.float32)
    ga[:, 0], gb[:, 0] = a, b
    ga[:, 1] = 1.0
    gb[:, 2] = 1.0
    ga[:, 1:] += (rng.uniform(-2, 2, (n, 3)) * (rng.random((n, 1)) < 0.5)).astype(np.float32)
    gb[:, 1:] += (rng.uniform(-2, 2, (n, 3)) * (rng.random((n, 1)) < 0.5)).astype(np.float32)
    ga[::11, 1:] = -0.0
    return ga, gb


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_reference_matches_oracle(orc, op):
    rng = np.random.default_rng(zlib.crc32(op.encode()))
    a, b = _points(op, rng)
    for form, imm, tape in _tapes(orc, op):
        args = [a] if form in ("r", "ri", "ir") else _by_slot(tape, a, b)
        got = tape.float_slice_eval(args)
        want = _ref_f32(op, form, imm, a, b)
        if op in R.LIBM:
            d = R.ulp_distance(got, want)
            assert d.max() <= 1, (op, form, imm, a[d.argmax()], got[d.argmax()], want[d.argmax()])
        else:
            bad = ~((np.isnan(got) & np.isnan(want)) | (got.view(np.uint32) == want.view(np.uint32)))
            assert not bad.any(), (op, form, imm, a[bad][:4], b[bad][:4], got[bad][:4], want[bad][:4])
        # gradients
        ga, gb = _grad_inputs(rng, a, b)
        gargs = [ga] if len(args) == 1 else _by_slot(tape, ga, gb)
        g_got = tape.grad_slice_eval(gargs)
        g_want = R.grad(op, form, ga, gb if form == "rr" else None, imm)
        if op in R.LIBM:
            v = R.ulp_distance(g_got[:, 0], g_want[:, 0])
            assert v.max() <= 1, (op, form, imm)
            fin = np.isfinite(g_want[:, 1:]) & np.isfinite(g_got[:, 1:])
            with np.errstate(invalid="ignore"):
                rel = np.abs(g_got[:, 1:].astype(np.float64) - g_want[:, 1:]) / np.maximum(1.0, np.abs(g_want[:, 1:]))
            assert rel[fin].max(initial=0) <= 1e-5, (op, form, imm)
        else:
            assert same_f32(g_got, g_want), (op, form, imm, np.argwhere(~((np.isnan(g_got) & np.isnan(g_want)) |
                                                                          (g_got == g_want)))[:4])


def test_analytic_derivatives_match_difference_quotients():
    """d_analytic against central differences in float64, away from kinks and poles."""
    rng = np.random.default_rng(5)
    x = rng.uniform(0.2, 0.8, 200)
    y = rng.uniform(0.3, 0.9, 200)
    h = 1e-6
    for op in ("neg", "recip", "sqrt", "square", "sin", "cos", "tan", "asin", "acos", "atan", "exp", "ln",
               "add", "sub", "mul", "div", "atan2"):
        da, db = R.d_analytic(op, x, y if op in R.BINARY else None)
        f = (lambda u, v: R.f64(op, u, v)) if op in R.LIBM else None
        exact = {"neg": lambda u, v: -u, "recip": lambda u, v: 1 / u, "sqrt": lambda u, v: np.sqrt(u),
                 "square": lambda u, v: u * u, "add": lambda u, v: u + v, "sub": lambda u, v: u - v,
                 "mul": lambda u, v: u * v, "div": lambda u, v: u / v}
        f = f or exact[op]
        na = (f(x + h, y) - f(x - h, y)) / (2 * h)
        assert np.allclose(da, na, rtol=1e-6, atol=1e-6), op
        if op in R.BINARY:
            nb = (f(x, y + h) - f(x, y - h)) / (2 * h)
            assert np.allclose(db, nb, rtol=1e-6, atol=1e-6), op


def test_ulp_distance():
    one = np.float32(1.0)
    assert R.ulp_distance(one, np.nextafter(one, np.float32(2))) == 1
    assert R.ulp_distance(np.float32(0.0), np.float32(-0.0)) == 0
    assert R.ulp_distance(np.float32(np.nan), np.float32(np.nan)) == 0
    assert R.ulp_distance(np.float32(np.nan), one) > 1e9
    tiny = np.float32(1e-45)
    assert R.ulp_distance(tiny, -tiny) == 2


def _clauses(words):
    """(opcode, form) of every clause of a bytecode (start/end markers dropped)."""
    out = []
    for w in words[2:-2:2]:
        op, lhs, rhs = int(w) & 0xFF, (int(w) >> 16) & 0xFF, (int(w) >> 24) & 0xFF
        form = "ir" if lhs == 0xFF else "ri" if rhs == 0xFF else "rr"
        out.append((op, form))
    return out


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("op", R.ALL_OPS)
def test_op_shape_tape(orc, op, dim):
    from fidget_b200.host import OP
    ctx, root, prims = R.op_shape(orc.Context, op, 0, dim=dim)
    td = ctx.tape(root)
    bc = orc.Tape.from_data(td).bytecode()
    assert bc.mem_count == 0, "spilled"
    cl = _clauses(bc.words)
    assert len(cl) >= 64, len(cl)
    got = {form for o, form in cl if o == OP[op]}
    want = {"rr" if f == "r" else f for f in R.FORMS[op]}
    if op in R.UNARY:
        assert got, op
    else:
        assert got == want, (op, got, want)
    assert len(prims) >= 12 and sorted({p.form for p in prims}) == sorted(R.FORMS[op])
    # the same shape in the product's Context gives the same bytecode
    import fidget_b200 as fb
    c2, r2, _ = R.op_shape(fb.Context, op, 0, dim=dim)
    assert np.array_equal(c2.tape(r2).bytecode().words, td.bytecode().words)
