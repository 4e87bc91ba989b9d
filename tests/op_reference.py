"""An independent numpy restatement of every opcode of the reference VM, and the shapes that route each opcode
through the device interpreters.

Written from fidget-core's ``types/float.rs`` (min/max/and/or/compare/not), ``types/grad.rs`` and the gradient arms
of ``vm/mod.rs`` (which side of an immediate clause becomes ``Grad::from(imm)``), ``rng/mod.rs`` (the rand / mix hash)
and SURVEY.md Appendix A.  It imports neither the oracle nor the package's kernels: each f32 result is computed in
float64 (or uint32 for the hash) and rounded once to f32.  For add, sub, mul, div, sqrt and fmod that single rounding
of the float64 result is the correctly rounded f32 result (53 >= 2 * 24 + 2 bits, so the double rounding is
innocuous), which is what IEEE 754 asks of the reference's f32 operations; libm opcodes are the float64 function
rounded once, i.e. (almost always) correctly rounded, which the device's libdevice is not required to be."""
import numpy as np

F = np.float32

UNARY = ["neg", "abs", "recip", "sqrt", "square", "floor", "ceil", "round", "not", "rand",
         "sin", "cos", "tan", "asin", "acos", "atan", "exp", "ln"]
BINARY = ["add", "sub", "mul", "div", "atan2", "compare", "mix", "mod", "min", "max", "and", "or"]
ALL_OPS = UNARY + BINARY
LIBM = {"sin", "cos", "tan", "asin", "acos", "atan", "exp", "ln", "atan2"}
IEEE = [op for op in ALL_OPS if op not in LIBM]

# Maximum error of the single-precision functions, in ulps, from the CUDA C++ Programming Guide (appendix
# "Mathematical Functions", table "Single-Precision Mathematical Standard Library Functions with Maximum ULP Error",
# default compilation without -use_fast_math):
#     sinf 2, cosf 2, tanf 4, asinf 2, acosf 2, atanf 2, atan2f 3, expf 2, logf 1
# These are the Guide's documented bounds, not measurements of this build.
ULP_BOUND = {"sin": 2, "cos": 2, "tan": 4, "asin": 2, "acos": 2, "atan": 2, "atan2": 3, "exp": 2, "ln": 1}

# Clause forms as they appear in the bytecode: commutative opcodes put an immediate on the right, and and/or with an
# immediate on the left fold away in the Context, so they have no imm/reg clause.
FORMS = {op: ["r"] for op in UNARY}
FORMS.update({op: ["rr", "ri", "ir"] for op in BINARY})
for _op in ("add", "mul", "min", "max", "and", "or"):
    FORMS[_op] = ["rr", "ri"]

_M32 = np.uint64(0xFFFFFFFF)


def _bits(a):
    return np.ascontiguousarray(a, dtype=F).view(np.uint32).astype(np.uint64)


def _hash(v):
    """rng::hash (Jarzynski & Olano's PCG hash) on uint32 values held in uint64."""
    state = (v * np.uint64(747796405) + np.uint64(2891336453)) & _M32
    word = (((state >> ((state >> np.uint64(28)) + np.uint64(4))) ^ state) * np.uint64(277803737)) & _M32
    return (word >> np.uint64(22)) ^ word


def _rand(a):
    h = _hash(_bits(a))
    one_two = ((h >> np.uint64(9)) | np.uint64(0x3F800000)).astype(np.uint32).view(F)
    return (one_two.astype(np.float64) - 1.0).astype(F)     # exact: a value of [1, 2) minus 1


def _mix(a, b):
    return ((_hash((_bits(a) + _hash(_bits(b))) & _M32)).astype(np.uint32)).view(F)


def _rem_euclid(a, b):
    """f32::rem_euclid: r = a % b (fmod, exact); r < 0 ? r + |b| : r, the sum rounded once."""
    r = np.fmod(a, b)
    return np.where(r < 0, r + np.abs(b), r)


def _div_euclid(a, b):
    """f32::div_euclid: q = trunc(a / b) with a / b rounded to f32; one step down (b > 0) or up when a % b < 0."""
    q = np.trunc(F(a) / F(b)).astype(np.float64)
    r = np.fmod(a, b)
    return np.where(r < 0, np.where(b > 0, q - 1.0, q + 1.0), q)


def _round(a):
    """f32::round: half away from zero.  For |a| < 2^23, a +- 0.5 is exact in float64; larger f32 are integers."""
    return np.where(np.abs(a) >= 2.0 ** 23, a, np.trunc(a + np.copysign(0.5, a)))


def _min(a, b):
    """FloatExt::min_choice: a < b -> a; b < a -> b; otherwise NaN if either is NaN, else b."""
    return np.where(a < b, a, np.where(b < a, b, np.where(np.isnan(a) | np.isnan(b), np.nan, b)))


def _max(a, b):
    return np.where(a > b, a, np.where(b > a, b, np.where(np.isnan(a) | np.isnan(b), np.nan, b)))


def _compare(a, b):
    """f32::partial_cmp as i8 as f32: -1 / 0 / +1, NaN when unordered."""
    return np.where(a < b, -1.0, np.where(a > b, 1.0, np.where(a == b, 0.0, np.nan)))


def f32(op, a, b=None):
    """The reference VM's f32 result of ``op`` on f32 arrays ``a`` (and ``b``), as float32."""
    a = np.asarray(a, dtype=F)
    if op == "rand":
        return _rand(a)
    if op == "mix":
        return _mix(a, np.broadcast_to(np.asarray(b, dtype=F), a.shape))
    x = a.astype(np.float64)
    y = None if b is None else np.asarray(b, dtype=F).astype(np.float64)
    with np.errstate(all="ignore"):
        r = {
            "neg": lambda: -x, "abs": lambda: np.abs(x), "recip": lambda: 1.0 / x, "sqrt": lambda: np.sqrt(x),
            "square": lambda: x * x, "floor": lambda: np.floor(x), "ceil": lambda: np.ceil(x),
            "round": lambda: _round(x), "not": lambda: np.where(x == 0.0, 1.0, 0.0),
            "sin": lambda: np.sin(x), "cos": lambda: np.cos(x), "tan": lambda: np.tan(x),
            "asin": lambda: np.arcsin(x), "acos": lambda: np.arccos(x), "atan": lambda: np.arctan(x),
            "exp": lambda: np.exp(x), "ln": lambda: np.log(x),
            "add": lambda: x + y, "sub": lambda: x - y, "mul": lambda: x * y, "div": lambda: x / y,
            "atan2": lambda: np.arctan2(x, y), "compare": lambda: _compare(x, y), "mod": lambda: _rem_euclid(x, y),
            "min": lambda: _min(x, y), "max": lambda: _max(x, y),
            "and": lambda: np.where(x == 0.0, x, y), "or": lambda: np.where(x != 0.0, x, y),
        }[op]()
        return np.asarray(r).astype(F)


def f64(op, a, b=None):
    """``op`` in float64 without the final rounding (libm opcodes), for error bounds."""
    with np.errstate(all="ignore"):
        x = np.asarray(a, dtype=np.float64)
        y = None if b is None else np.asarray(b, dtype=np.float64)
        fn = {"sin": np.sin, "cos": np.cos, "tan": np.tan, "asin": np.arcsin, "acos": np.arccos, "atan": np.arctan,
              "exp": np.exp, "ln": np.log}
        if op in fn:
            return fn[op](x)
        if op == "atan2":
            return np.arctan2(x, y)
        return f32(op, a, b).astype(np.float64)


# ---------------------------------------------------------------------------
# Gradients: Grad {v, dx, dy, dz} arithmetic of types/grad.rs, every step an f32 operation in the reference's order.
def _g(a):
    a = np.asarray(a, dtype=F).reshape(-1, 4)
    return a[:, 0], a[:, 1:]


def _pack(v, d):
    out = np.empty((len(v), 4), dtype=F)
    out[:, 0] = v
    out[:, 1:] = d
    return out


def _const(k, n):
    return np.full(n, k, dtype=F), np.zeros((n, 3), dtype=F)


def grad(op, form, a, b=None, imm=None):
    """The reference VM's gradient result (``vm/mod.rs`` gradient arms, ``types/grad.rs``) for a clause of ``form``
    ("r", "rr", "ri", "ir"): ``a`` / ``b`` are [n, 4] register values, ``imm`` the immediate of an ri / ir clause.
    IEEE opcodes are exact; libm values are float64 rounded once (compare those within ULP_BOUND)."""
    with np.errstate(all="ignore"):
        if form == "ri":
            va, da = _g(a)
            vb, db = _const(imm, len(va))
        elif form == "ir":
            vb, db = _g(a if b is None else b)
            va, da = _const(imm, len(vb))
        else:
            va, da = _g(a)
            vb, db = _g(b) if b is not None else (None, None)
        col = lambda v: v[:, None]  # noqa: E731
        n = len(va)
        zero = np.zeros((n, 3), dtype=F)
        if op == "neg":
            return _pack(-va, -da)
        if op == "abs":
            neg = col(va < 0)
            return _pack(np.where(va < 0, -va, va), np.where(neg, -da, da))
        if op == "sqrt":
            v = np.sqrt(va)
            return _pack(v, da / (F(2) * col(v)))
        if op == "square":
            return _mul(va, da, va, da)
        if op == "recip":
            return _div(np.ones(n, dtype=F), zero, va, da)
        if op in ("floor", "ceil", "round", "not", "rand"):
            return _pack(f32(op, va), zero)
        if op in ("compare", "mix"):
            return _pack(f32(op, va, vb), zero)
        if op in LIBM and op != "atan2":
            v = f32(op, va)
            x = va.astype(np.float64)
            dv = {"sin": lambda: np.cos(x), "cos": lambda: -np.sin(x), "tan": lambda: 1.0 / np.cos(x) ** 2,
                  "asin": lambda: 1.0 / np.sqrt(1.0 - x * x), "acos": lambda: -1.0 / np.sqrt(1.0 - x * x),
                  "atan": lambda: 1.0 / (x * x + 1.0), "exp": lambda: v.astype(np.float64),   # the VM's own f32 value
                  "ln": lambda: 1.0 / x}[op]()
            return _pack(v, (da.astype(np.float64) * col(dv)).astype(F))
        if op == "atan2":
            # IEEE steps in the VM's order, in f32: d = x * x + y * y underflows and overflows where the VM's does
            d = vb * vb + va * va
            return _pack(f32("atan2", va, vb), (col(vb) * da - col(va) * db) / col(d))
        if op == "add":
            return _pack(va + vb, da + db)
        if op == "sub":
            return _pack(va - vb, da - db)
        if op == "mul":
            if form == "ri":      # MulRegImm: Grad * f32 scales all four components
                k = F(imm)
                return _pack(va * k, da * k)
            return _mul(va, da, vb, db)
        if op == "div":
            return _div(va, da, vb, db)
        if op == "mod":
            e = _div_euclid(va.astype(np.float64), vb.astype(np.float64)).astype(F)
            return _pack(f32("mod", va, vb), da - db * col(e))
        if op in ("min", "max"):
            nan = np.isnan(va) | np.isnan(vb)
            left = (va < vb) if op == "min" else (va > vb)
            v = np.where(nan, np.nan, np.where(left, va, vb)).astype(F)
            d = np.where(col(nan), F(0), np.where(col(left), da, db)).astype(F)
            return _pack(v, d)
        if op in ("and", "or"):
            left = (va == 0) if op == "and" else (va != 0)
            return _pack(np.where(left, va, vb), np.where(col(left), da, db))
    raise KeyError(op)


def _mul(va, da, vb, db):
    col = lambda v: v[:, None]  # noqa: E731
    return _pack(va * vb, col(va) * db + col(vb) * da)


def _div(va, da, vb, db):
    col = lambda v: v[:, None]  # noqa: E731
    d = vb * vb                       # powi(2)
    return _pack(va / vb, (col(vb) * da - col(va) * db) / col(d))


def d_analytic(op, a, b=None):
    """float64 partial derivatives (d/da, d/db) of the exact function ``op`` at (a, b); for unary ops d/db is 0."""
    with np.errstate(all="ignore"):
        x = np.asarray(a, dtype=np.float64)
        y = np.zeros_like(x) if b is None else np.asarray(b, dtype=np.float64)
        one, zero = np.ones_like(x), np.zeros_like(x)
        table = {
            "neg": (-one, zero), "abs": (np.sign(x), zero), "recip": (-1.0 / (x * x), zero),
            "sqrt": (0.5 / np.sqrt(x), zero), "square": (2.0 * x, zero),
            "sin": (np.cos(x), zero), "cos": (-np.sin(x), zero), "tan": (1.0 / np.cos(x) ** 2, zero),
            "asin": (1.0 / np.sqrt(1.0 - x * x), zero), "acos": (-1.0 / np.sqrt(1.0 - x * x), zero),
            "atan": (1.0 / (1.0 + x * x), zero), "exp": (np.exp(x), zero), "ln": (1.0 / x, zero),
            "add": (one, one), "sub": (one, -one), "mul": (y, x), "div": (1.0 / y, -x / (y * y)),
            "atan2": (y / (x * x + y * y), -x / (x * x + y * y)),
        }
        if op in table:
            return table[op]
        if op in ("floor", "ceil", "round", "not", "rand", "compare", "mix"):
            return zero, zero
        if op == "mod":
            return one, -np.floor(x / y)
        if op in ("min", "max"):
            left = (x < y) if op == "min" else (x > y)
            return left.astype(np.float64), (~left).astype(np.float64)
        if op in ("and", "or"):
            left = (x == 0) if op == "and" else (x != 0)
            return left.astype(np.float64), (~left).astype(np.float64)
    raise KeyError(op)


def ulp_distance(a, b):
    """Distance between f32 values in units in the last place: the number of f32 values between them (+-0 count as
    one value); 0 where both are NaN, and a huge number where only one is."""
    a = np.ascontiguousarray(a, dtype=F)
    b = np.ascontiguousarray(b, dtype=F)

    def ordinal(x):
        i = x.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    d = np.abs(ordinal(a) - ordinal(b))
    na, nb = np.isnan(a), np.isnan(b)
    return np.where(na & nb, 0, np.where(na | nb, 1 << 40, d))


def ulp(x):
    """Spacing of f32 at |x| (float64)."""
    x = np.abs(np.asarray(x, dtype=np.float64))
    with np.errstate(all="ignore"):
        return np.spacing(np.minimum(x, np.finfo(F).max).astype(F)).astype(np.float64)


# ---------------------------------------------------------------------------
# Shapes: a union of primitives, each routing the op in one of its forms through affine maps of the axes.
#
# Per op: (scale, offset, jitter, pre, level, (imm of ri, imm of ir)).  An argument is
# scale * (direction . p) + offset + U(-jitter, jitter) for a random unit direction, then ``pre`` ("floor" gives
# plateaus, where and/or/not meet exact zeros, compare meets ties and rand/mix meet constant seeds).  The offsets put
# each op's interesting points inside the image: for sqrt/ln the negative argument only reaches a corner (NaN there),
# asin/acos leave [-1, 1] near two corners, tan crosses its poles at +-pi/2, floor/ceil/round/mod step several times.
SPEC = {
    "neg": (1.0, 0.0, 0.4, None, 0.3, ()), "abs": (1.0, 0.0, 0.4, None, 0.3, ()),
    "recip": (1.0, 0.0, 0.4, None, 2.0, ()), "sqrt": (1.0, 1.2, 0.0, None, 0.6, ()),
    "square": (1.0, 0.0, 0.4, None, 0.2, ()), "floor": (2.5, 0.1, 0.3, None, 0.5, ()),
    "ceil": (2.5, 0.1, 0.3, None, 0.5, ()), "round": (2.5, 0.1, 0.3, None, 0.5, ()),
    "not": (2.0, 0.5, 0.3, "floor", 0.5, ()), "rand": (2.0, 0.0, 0.5, "floor", 0.5, ()),
    "sin": (4.0, 0.0, 1.0, None, 0.2, ()), "cos": (4.0, 0.0, 1.0, None, 0.2, ()),
    "tan": (2.5, 0.0, 0.3, None, 0.5, ()), "asin": (0.83, 0.0, 0.0, None, 0.2, ()),
    "acos": (0.83, 0.0, 0.0, None, 1.2, ()), "atan": (4.0, 0.0, 1.0, None, 0.3, ()),
    "exp": (2.0, 0.0, 0.5, None, 1.5, ()), "ln": (1.0, 1.2, 0.0, None, -0.5, ()),
    "add": (1.0, 0.0, 0.4, None, 0.3, (0.75, -0.5)), "sub": (1.0, 0.0, 0.4, None, 0.3, (0.75, -0.5)),
    "mul": (1.5, 0.0, 0.4, None, 0.2, (-1.5, 0.75)), "div": (1.0, 0.0, 0.4, None, 0.5, (0.75, -0.5)),
    "atan2": (1.0, 0.0, 0.4, None, 0.5, (0.25, -0.5)), "compare": (2.0, 0.0, 0.5, "floor", 0.5, (1.0, -1.0)),
    "mix": (2.0, 0.0, 0.5, "floor", 1.0, (1.0, -2.0)), "mod": (2.5, 0.0, 0.5, None, 0.3, (0.75, -2.0)),
    "min": (1.0, 0.0, 0.4, None, 0.2, (0.25, 0.25)), "max": (1.0, 0.0, 0.4, None, 0.2, (-0.25, -0.25)),
    "and": (2.0, 0.5, 0.3, "floor", 0.3, (0.75, 0.0)), "or": (2.0, -0.5, 0.3, "floor", 0.3, (0.75, 0.0)),
}
# the second argument of and/or stays continuous (only the first decides the choice)
_PRE_B = {"and": None, "or": None}


class Prim:
    """One primitive: value = max(op(args) - level, mask).  ``args`` are nodes (register operands) or floats
    (immediates) in operand order; ``arg_nodes`` are the register operands, ``mask`` a disc, all IEEE-only."""

    def __init__(self, form, args, level, mask, term):
        self.form, self.args, self.level, self.mask, self.term = form, args, level, mask, term

    @property
    def arg_nodes(self):
        return [a for a in self.args if not isinstance(a, float)]


def op_shape(Ctx, op, seed, dim=2, n_prims=12):
    """(ctx, root, prims): the union of ``n_prims`` primitives that each route ``op`` through one of its FORMS,
    built identically in any Context class (``fb.Context`` or ``orc.Context``) from ``seed``."""
    ctx = Ctx()
    root, prims = op_prims(ctx, op, seed, dim, n_prims)
    return ctx, root, prims


def every_op_shape(Ctx, dim=3):
    """(ctx, root): a union with one primitive per clause form of every opcode.  rand and mix only ever see floors of
    coordinates, never a NaN made inside the tape (whose payload the platform chooses)."""
    ctx = Ctx()
    root = None
    for i, op in enumerate(ALL_OPS):
        r, _ = op_prims(ctx, op, 50 + i, dim, len(FORMS[op]))
        root = r if root is None else ctx.min(root, r)
    return ctx, root


def op_prims(ctx, op, seed, dim, n_prims):
    """Adds op_shape's primitives to ``ctx``; returns (root, prims)."""
    rng = np.random.default_rng([seed, ALL_OPS.index(op), dim])
    axes = [ctx.x(), ctx.y()] + ([ctx.z()] if dim == 3 else [])
    scale, offset, jitter, pre, level, imms = SPEC[op]
    forms = FORMS[op]

    def c(v):
        return float(F(v))

    def affine(pre_kind):
        d = rng.normal(size=dim)
        d /= np.linalg.norm(d)
        u = ctx.mul(axes[0], c(scale * d[0]))
        for ax, w in zip(axes[1:], d[1:]):
            u = ctx.add(u, ctx.mul(ax, c(scale * w)))
        u = ctx.add(u, c(offset + rng.uniform(-jitter, jitter) + 1e-3 * rng.uniform(0.5, 1.0)))
        return ctx.floor(u) if pre_kind == "floor" else u

    def disc():
        ctr = rng.uniform(-0.7, 0.7, size=dim)
        s = None
        for ax, k in zip(axes, ctr):
            t = ctx.square(ctx.sub(ax, c(k)))
            s = t if s is None else ctx.add(s, t)
        return ctx.sub(ctx.sqrt(s), c(rng.uniform(0.3, 0.7)))

    prims = []
    root = None
    for i in range(n_prims):
        form = forms[i % len(forms)]
        pre_b = _PRE_B.get(op, pre)
        if form == "r":
            args = [affine(pre)]
            term = ctx.unary(op, args[0])
        elif form == "rr":
            args = [affine(pre), affine(pre_b)]
            term = ctx.binary(op, args[0], args[1])
        elif form == "ri":
            args = [affine(pre), c(imms[0])]
            term = ctx.binary(op, args[0], args[1])
        else:
            args = [c(imms[1]), affine(pre_b)]
            term = ctx.binary(op, args[0], args[1])
        lv = c(level)
        mask = disc()
        p = ctx.max(ctx.sub(term, lv), mask)
        prims.append(Prim(form, args, lv, mask, term))
        root = p if root is None else ctx.min(root, p)
    return root, prims


def combine(prims, terms, masks):
    """Finish the CSG in numpy: ``terms[i]`` / ``masks[i]`` = value of prim i's op term / disc at each point (f32, or
    float64 for an unrounded reference); returns min over i of max(term - level, mask) with the reference's NaN rules,
    in the dtype of ``terms``."""
    out = None
    for p, t, m in zip(prims, terms, masks):
        dt = t.dtype
        with np.errstate(all="ignore"):
            s = (t - dt.type(p.level)).astype(dt)
        v = _max(s.astype(np.float64), m.astype(np.float64)).astype(dt)
        out = v if out is None else _min(out.astype(np.float64), v.astype(np.float64)).astype(dt)
    return out


def scalar_residual(ctx, op, x, y, k=0.75):
    """A one- or two-variable residual built around ``op`` for the solver: op(x, y) - k (or op(x) + y * 0.5 - k)."""
    if op in UNARY:
        return ctx.sub(ctx.add(ctx.unary(op, x), ctx.mul(y, 0.5)), k)
    return ctx.sub(ctx.binary(op, x, y), k)

