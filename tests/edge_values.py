"""A catalogue of f32 edge values, each with the reason it is there, and the pairs and interval boxes built from it.

f32 kernels go wrong at a few places that ordinary inputs never reach: subnormals (flushed to zero by -ftz=true),
values next to a rounding boundary (``floorf(x + 0.5f)`` is not ``roundf``), the ends of the range, and the arguments
at which a libm function overflows, underflows or leaves its domain.  test_edge_values_oracle.py pins the CPU side on
these values and test_gpu_edge_values.py feeds them to every device evaluator."""
import numpy as np

import op_reference as R

F = np.float32


def _bits(u):
    return np.array([u], dtype=np.uint32).view(F)[0]


def _next(a, toward):
    return np.nextafter(F(a), F(toward))


# (value, reason).  Values are f32; a decimal literal is the f32 nearest to it.
CATALOGUE = [
    # ---- zeros and subnormals
    (F(0.0), "+0"),
    (F(-0.0), "-0: signed zero through min/max, atan2, recip, sqrt, and/or"),
    (_bits(0x00000001), "smallest subnormal 2^-149 (1e-45)"),
    (_bits(0x80000001), "smallest negative subnormal"),
    (F(1e-40), "a subnormal in the middle of the range"),
    (F(-1e-40), "a negative subnormal"),
    (_bits(0x00400000), "2^-127, half the smallest normal: a subnormal power of two"),
    (_bits(0x007FFFFF), "largest subnormal"),
    (_bits(0x00800000), "smallest normal 2^-126"),
    (_bits(0x80800000), "smallest negative normal"),
    (_bits(0x00800001), "smallest normal + 1 ulp"),
    (F(1e-38), "a normal just above the smallest: 1e-38 / 1e3 lands in the subnormals"),
    (F(1e-20), "1e-20 squared is a subnormal"),
    (F(1e-30), "tiny normal"),
    # ---- rounding boundaries
    (_next(0.5, 0), "largest f32 below 0.5: floorf(x + 0.5f) rounds it up to 1"),
    (F(0.5), "0.5 rounds away from zero"),
    (_next(0.5, 1), "smallest f32 above 0.5"),
    (F(-0.5), "-0.5 rounds away from zero"),
    (-_next(0.5, 0), "largest f32 above -0.5"),
    (F(1.5), "1.5: a tie between 1 and 2"),
    (F(-1.5), "-1.5: a tie between -1 and -2"),
    (F(2.5), "2.5: a tie that round-half-even would send down"),
    (F(-2.5), "-2.5: a tie that round-half-even would send up"),
    (F(8388607.5), "2^23 - 0.5: the last half-integer, x + 0.5 is exact"),
    (F(-8388607.5), "-(2^23 - 0.5)"),
    (F(8388608.0), "2^23: from here on every f32 is an integer"),
    (F(8388609.0), "2^23 + 1: x + 0.5 rounds to the even 2^23 + 2"),
    (F(16777217.0), "2^24 + 1 as f32, which is 2^24: integers stop being exact"),
    (F(16777218.0), "2^24 + 2: the f32 after 2^24"),
    # ---- range ends
    (F(3.4028235e38), "FLT_MAX: doubling, squaring or adding it overflows"),
    (F(-3.4028235e38), "-FLT_MAX"),
    (F(np.inf), "+inf"),
    (F(-np.inf), "-inf"),
    (_bits(0x7FC00000), "the canonical quiet NaN"),
    (_bits(0x7FC01234), "a quiet NaN with a payload: rand and mix hash its bits"),
    (_bits(0xFFC00001), "a negative quiet NaN with a payload"),
    # ---- exp
    (F(88.72283), "exp just below its overflow threshold ln(FLT_MAX) = 88.7228391: finite"),
    (F(88.72284), "exp just above its overflow threshold: inf"),
    (F(-87.33654), "exp near ln(2^-126): the edge of the normal range"),
    (F(-103.27893), "exp deep in the subnormals (about 2^-149 * e^0.7)"),
    (F(-103.97208), "exp at ln(2^-150): rounds to 2^-149 or to 0"),
    (F(-104.0), "exp below ln(2^-150): 0"),
    # ---- ln, asin, acos
    (F(1.0), "1: ln 1 = 0, asin / acos at their domain edge"),
    (F(-1.0), "-1: asin / acos at their domain edge"),
    (_next(1, 0), "1 - 1 ulp: ln just below 0, asin / acos just inside the domain"),
    (_next(1, 2), "1 + 1 ulp: ln just above 0, asin / acos just outside the domain (NaN)"),
    (-_next(1, 0), "-(1 - 1 ulp)"),
    (-_next(1, 2), "-(1 + 1 ulp)"),
    # ---- trig
    (F(1e4), "a large trig argument: Payne-Hanek free but not Cody-Waite exact"),
    (F(105414350.0), "a large trig argument close to a multiple of pi/2"),
    (F(1e30), "a huge argument: trig needs full range reduction; 1e30 mod 3"),
    (F(-1e30), "a huge negative argument"),
    (F(1.5707964), "f32(pi/2): cos is tiny, tan is huge"),
    (F(-1.5707964), "f32(-pi/2)"),
    (F(3.1415927), "f32(pi): sin is tiny and negative"),
    (F(4.712389), "f32(3pi/2)"),
    (F(6.2831855), "f32(2pi)"),
    # ---- mod divisors, and ordinary inexact values (a fused multiply-add changes their products)
    (F(2.0), "2: 2^24 + 1 mod 2"),
    (F(3.0), "3: 1e30 mod 3"),
    (F(-3.0), "a negative divisor: rem_euclid adds |b|"),
    (F(0.1), "an inexact decimal"),
    (F(1.0 / 3.0), "1/3: products and quotients round"),
]
VALUES = np.array([v for v, _ in CATALOGUE], dtype=F)
NOT_NAN = VALUES[~np.isnan(VALUES)]

# Pairs (a, b) aimed at one result: products and quotients in the subnormals, sums cancelling to a subnormal, overflow.
TARGETED = np.array([
    (1e-20, 1e-20),                                   # a * b = 1e-40
    (1e-38, 1e3),                                     # a / b = 1e-41
    (1e-20, -1e-20),
    (_bits(0x00800000), _bits(0x807FFFFF)),           # a + b = 2^-149
    (_bits(0x00800001), _bits(0x80800000)),           # a + b = 2^-149
    (_bits(0x00800001), _bits(0x00800000)),           # a - b = 2^-149
    (F(1.0000001e-38), F(-1e-38)),                    # a + b: a few subnormal ulps
    (F(3.4028235e38), 2.0),                           # a * b = inf
    (F(3.4028235e38), F(3.4028235e38)),               # a + b = inf
    (F(3.4028235e38), 0.5),                           # a / b = inf
    (F(16777217.0), 2.0),                             # a mod b
    (F(1e30), 3.0),                                   # a mod b
    (F(1e30), F(-3.0)),
    (F(-1e30), 3.0),
    (F(1.0), _bits(0x00000001)),                      # a mod (smallest subnormal), a / b = inf
    (F(-1e-40), F(1e-45)),
], dtype=F)

# Immediates of ri / ir clauses: a value of each family (the host stores an immediate as f32 bits, a NaN payload too)
IMMEDIATES = np.array([
    0.0, -0.0, _bits(0x00000001), F(-1e-40), _bits(0x00800000), _next(0.5, 0), F(-2.5), F(8388609.0),
    F(3.4028235e38), F(-np.inf), _bits(0x7FC01234), F(88.72284), F(-103.97208), _next(1, 2), F(1e30), F(-3.0),
    F(0.1),
], dtype=F)


def pairs():
    """(a, b) f32 arrays: the full product of the catalogue, then the targeted pairs."""
    a, b = [g.ravel() for g in np.meshgrid(VALUES, VALUES, indexing="ij")]
    return np.concatenate([a, TARGETED[:, 0]]), np.concatenate([b, TARGETED[:, 1]])


def boxes(n_vars, n, seed):
    """[m, n_vars, 2] interval boxes with catalogue endpoints: every point box [v, v] (NaN ones included) on each
    variable, then ``n`` boxes whose endpoints are two catalogue values in order."""
    rng = np.random.default_rng(seed)
    pts = np.repeat(VALUES[:, None, None], 2, axis=2)                 # [k, 1, 2]
    point = np.concatenate([np.broadcast_to(np.roll(pts, s, axis=0), (len(VALUES), 1, 2))
                            for s in range(n_vars)], axis=1) if n_vars > 1 else pts
    lo = rng.choice(NOT_NAN, (n, n_vars))
    hi = rng.choice(NOT_NAN, (n, n_vars))
    lo, hi = np.fmin(lo, hi), np.fmax(lo, hi)
    return np.concatenate([point, np.stack([lo, hi], -1)]).astype(F)


def interior(b, k, seed):
    """``k`` f32 samples per box of [m, 2] intervals, endpoints included: [m, k + 2].  Samples are spread both
    linearly and in f32 order, so that a box like [1e-45, 1e30] is sampled in its subnormals too."""
    rng = np.random.default_rng(seed)
    lo, hi = b[:, 0].astype(F), b[:, 1].astype(F)

    def ordinal(x):
        i = x.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    def from_ordinal(o):
        o = o.astype(np.int64)
        return np.where(o < 0, (-o) | 0x80000000, o).astype(np.uint32).view(F)

    t = rng.random((len(b), k))
    half = k // 2
    with np.errstate(all="ignore"):
        lin = (lo[:, None].astype(np.float64) * (1 - t[:, :half]) + hi[:, None].astype(np.float64) * t[:, :half])
        lin = np.clip(np.nan_to_num(lin, nan=0.0), lo[:, None], hi[:, None]).astype(F)
        olo, ohi = ordinal(lo)[:, None], ordinal(hi)[:, None]
        ords = np.floor(olo + (ohi - olo) * t[:, half:]).astype(np.int64)
    out = np.concatenate([lo[:, None], hi[:, None], lin, from_ordinal(ords)], axis=1)
    point = (lo.view(np.uint32) == hi.view(np.uint32))[:, None]       # [-0, -0] holds -0 only
    return np.where(np.isnan(lo)[:, None] | np.isnan(hi)[:, None], np.nan, np.where(point, lo[:, None], out)).astype(F)


# Axis-driven 2D routes: the argument s * x + v (x over [-1, 1] across the image) crosses ``edge`` inside the image.
# (name, s, v, edge, [(op, imm or None, level)]); the rendered value is op(arg[, imm]) - level, which puts a sign change
# where the op's result crosses ``level``.  The exp route's s * x is inexact: a fused multiply-add changes s * x + v.
ROUTES = [
    ("subnormal", F(2e-38), F(0.0), F(1.1754942e-38),
     [("sqrt", None, 1e-20), ("recip", None, 1e38), ("neg", None, 1e-40), ("square", None, 0.0), ("ln", None, -88.0),
      ("mul", F(3.0), 1e-39), ("div", F(0.1), 1e-38), ("mod", F(1e-38), 1e-39)]),
    ("half", F(2.0 ** -18), F(0.5), F(0.5), [("round", None, 0.5), ("floor", None, 0.5), ("ceil", None, 0.5)]),
    ("2^23", F(8.0), F(8388608.0), F(8388608.0),
     [("round", None, 8388608.0), ("floor", None, 8388607.5), ("ceil", None, 8388608.5), ("mod", F(2.0), 0.5)]),
    ("exp underflow", F(10.0), F(-95.0), F(-103.97208), [("exp", None, 1e-40)]),
]


def route_term(ctx, op, imm, arg):
    """op(arg) or op(arg, imm) in ``ctx``"""
    return ctx.unary(op, arg) if imm is None else ctx.binary(op, arg, ctx.constant(float(imm)))


# ---- the tapes and the checks shared by the CPU and GPU suites ------------------------------------------------------
def op_tapes(Ctx, op, immediates=IMMEDIATES):
    """(form, imm, tape data) for every clause form of ``op`` in context class ``Ctx``: "r" / "rr" over the axes, then
    "ri" / "ir" with each immediate whose clause survives the host's constant folding as that opcode and form (x + 0,
    x * 1 and 0 and x fold away; 0 - x becomes neg x)."""
    if op in R.UNARY:
        c = Ctx()
        return [("r", None, c.tape(c.unary(op, c.x())))]
    c = Ctx()
    out = [("rr", None, c.tape(c.binary(op, c.x(), c.y())))]
    for form in R.FORMS[op][1:]:
        for k in immediates:
            c = Ctx()
            k = float(k)
            td = c.tape(c.binary(op, c.x(), c.constant(k)) if form == "ri" else c.binary(op, c.constant(k), c.x()))
            clause = td.dump().splitlines()[1]   # input, op, output
            if len(td) == 3 and clause.startswith(op.capitalize() + " ") and ("<- #" in clause) == (form == "ir"):
                out.append((form, F(k), td))
    return out


def inputs(td, form):
    """(vals per tape input slot, operands in op order, n): the catalogue for "r", ri / ir clauses, every pair for
    "rr".  Slots come from ``td.var_slots()``: the tape numbers its inputs in its own order."""
    vx, vy, _ = td.var_slots()
    if form == "rr":
        a, b = pairs()
        vals = [None] * td.n_vars
        vals[vx], vals[vy] = a, b
        return vals, (a, b), len(a)
    return [VALUES], (VALUES,), len(VALUES)


def operands(form, ins, imm):
    """The op's operands in order for ``form`` from ``inputs``' operand tuple."""
    if form == "ri":
        return ins[0], np.full(len(ins[0]), imm, F)
    if form == "ir":
        return np.full(len(ins[0]), imm, F), ins[0]
    return ins


def grad_inputs(td, form, seed):
    """[n, 4] gradient inputs per slot: values as ``inputs``, d/d(own axis) = 1, half the rows with added random
    derivative parts (inexact products: a fused multiply-add changes them)."""
    rng = np.random.default_rng(seed)
    vals, _, n = inputs(td, form)
    out = []
    for k, v in enumerate(vals):
        g = np.zeros((n, 4), F)
        g[:, 0] = v
        g[:, 1 + k] = 1.0
        g[:, 1:] += (rng.uniform(-2, 2, (n, 3)) * (rng.random((n, 1)) < 0.5)).astype(F)
        g[::7, 1:] = rng.choice(VALUES, (len(g[::7]), 3))
        out.append(g)
    return out


def libm_error(got, ref64):
    """|got - ref64| in ulps of f32 at ref64 (an infinite ``got`` counts as +-2^128); 0 where both are NaN or equal,
    inf where only one is NaN."""
    g = np.asarray(got, F).astype(np.float64)
    r = np.asarray(ref64, np.float64)
    with np.errstate(all="ignore"):
        same = (g == r) | (np.isnan(g) & np.isnan(r))
        gg = np.where(np.isinf(g), np.sign(g) * 2.0 ** 128, g)
        rr = np.clip(r, -2.0 ** 128, 2.0 ** 128)
        err = np.abs(gg - rr) / R.ulp(rr)
    return np.where(same, 0.0, np.where(np.isnan(g) | np.isnan(r), np.inf, err))


def value_ok(op, got, args):
    """Per element: ``got`` is the reference f32 ``op(*args)`` bit for bit (any NaN for a NaN) for an IEEE opcode, or
    within ULP_BOUND ulps of the float64 value for a libm opcode."""
    got = np.asarray(got, F)
    if op in R.LIBM:
        return libm_error(got, R.f64(op, *args)) <= R.ULP_BOUND[op]
    want = R.f32(op, *args)
    return (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))


def same_bits(a, b):
    """Per element: equal bits, or both NaN."""
    a, b = np.ascontiguousarray(a, F), np.ascontiguousarray(b, F)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def close_ulps(a, b, n):
    """Per element: ``a`` and ``b`` at most ``n`` f32 steps apart (both NaN counts as equal)."""
    return R.ulp_distance(a, b) <= n


def contains(op, form, box, out, imm, seed, k=16):
    """Per box: the interval ``out`` [m, 2] of ``op`` over ``box`` [m, n_vars, 2] (operand order) holds the f32
    reference value at the box's endpoints and at ``k`` interior samples, wherever that value is not NaN.  A NaN
    interval holds everything.  libm opcodes may miss by ULP_BOUND ulps (their endpoints are libm values too)."""
    m = len(box)
    samples = [interior(box[:, i], k, seed + i) for i in range(box.shape[1])]
    if form == "ri":
        args = (samples[0], np.full_like(samples[0], imm))
    elif form == "ir":
        args = (np.full_like(samples[0], imm), samples[0])
    else:
        args = tuple(samples)
    v = R.f32(op, *[a.ravel() for a in args]).reshape(m, -1)
    lo, hi = out[:, 0:1], out[:, 1:2]
    slack = R.ULP_BOUND.get(op, 0)
    with np.errstate(all="ignore"):
        inside = (v >= lo) & (v <= hi)
        if slack:
            inside |= (R.ulp_distance(v, np.broadcast_to(lo, v.shape)) <= slack) | \
                (R.ulp_distance(v, np.broadcast_to(hi, v.shape)) <= slack)
    ok = inside | np.isnan(v) | np.isnan(lo) | np.isnan(hi)
    if op == "atan2":
        # at the origin atan2 of reals has no value; the f32 one (0, +-pi) comes from the zeros' signs, which an
        # interval [-0, b] does not carry (the reference's corners treat -0 as 0)
        ok |= (args[0] == 0).reshape(m, -1) & (args[1] == 0).reshape(m, -1)
    return ok.all(axis=1)


# Partial derivatives of the libm opcodes are f32 chains (cos(x) * dx, dx / (c * c), dx / sqrt(1 - x * x), ...) around
# one libm value, where op_reference.grad rounds the float64 derivative once: a few roundings plus the libm error.
GRAD_ULPS = {op: 2 * b + 2 for op, b in R.ULP_BOUND.items()}


def grad_ok(op, form, got, ga, gb, imm, args):
    """Per row: the gradient ``got`` [n, 4] of ``op`` on register inputs ``ga`` (``gb``) is op_reference.grad: IEEE
    opcodes bit for bit; libm values within ULP_BOUND of float64 (``args``: the operand values), partials within
    GRAD_ULPS of the once-rounded float64 partial."""
    want = R.grad(op, form, ga, gb, imm)
    if op not in R.LIBM:
        return same_bits(got, want).all(axis=1)
    return value_ok(op, got[:, 0], args) & close_ulps(got[:, 1:], want[:, 1:], GRAD_ULPS[op]).all(axis=1)
