"""fc_solve_batch on the device: fidget-solver's own test cases, bit-for-bit agreement with the CPU oracle
(oracle/solve.cc) on values, exit, iteration count and error for tapes of IEEE operations, batch independence, and the
API's edge cases."""
import ctypes as C

import numpy as np
import pytest

import solve_oracle as so
import solver_cases as sc
from conftest import same_f32

pytestmark = pytest.mark.gpu


def device_solve(cuda, build, starts=None, max_iters=None, as_torch=False):
    import fidget_b200 as fb
    ctx = fb.Context()
    built = build(ctx)
    case, check = built if isinstance(built, tuple) else (built, None)
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    vals = np.array([case.start] if starts is None else starts, dtype=np.float32)
    if as_torch:
        import torch
        vals = torch.from_numpy(vals).cuda()
    out = fb.solve_batch(shapes, case.free, case.fixed, vals, max_iters)
    if as_torch:
        out = tuple(o.cpu().numpy() for o in out)
    return case, check, out


def oracle_solve(orc, build, starts=None, max_iters=None):
    ctx = orc.Context()
    built = build(ctx)
    case = built[0] if isinstance(built, tuple) else built
    keys = case.free + case.fixed
    tds = [ctx.tape(r) for r in case.roots]
    vals, res = so.solve_batch([orc.Tape.from_data(t) for t in tds], [sc.slot_map(t, keys) for t in tds],
                                len(case.free), [case.start] if starts is None else starts, max_iters or 0)
    return vals, res["status"], res["iterations"], res["err"]


def assert_same(dev, ref):
    vals, status, iters, err = dev
    rv, rs, ri, re_ = ref
    assert np.array_equal(status, rs), (status, rs)
    assert np.array_equal(iters, ri), (iters, ri)
    assert same_f32(vals, rv)
    assert same_f32(err, re_)


def check_both(cuda, orc, build, starts=None, max_iters=None):
    _, _, dev = device_solve(cuda, build, starts, max_iters)
    ref = oracle_solve(orc, build, starts, max_iters)
    assert_same(dev, ref)
    return dev


def rel_eq(a, b, eps=np.finfo(np.float32).eps):
    d = abs(a - b)
    return d <= eps or d <= max(abs(a), abs(b)) * eps


# ---- the reference's cases ---------------------------------------------------------------------------------------
def test_basic_solver(cuda, orc):
    import fidget_b200 as fb
    ctx = fb.Context()
    shape = fb.CudaShape(cuda, ctx.tape(ctx.add(ctx.x(), ctx.y())))
    sol = fb.solve([shape], {"x": fb.Free(0.0), "y": fb.Fixed(-1.0)})
    assert list(sol) == ["x"] and rel_eq(sol["x"], 1.0)
    check_both(cuda, orc, sc.basic_solver)


def test_four_vars(cuda, orc):
    import fidget_b200 as fb
    ctx = fb.Context()
    case = sc.four_vars_independent(ctx)
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    sol = fb.solve(shapes, {k: fb.Free(v) for k, v in zip(case.free, case.start)})
    assert [rel_eq(sol[k], float(i)) for i, k in enumerate(case.free)] == [True] * 4
    _, _, (vals, _, _, _) = device_solve(cuda, sc.four_vars_at_once)
    assert rel_eq(float(np.float32(np.float32(vals[0, 0] + vals[0, 1]) + vals[0, 2]) + vals[0, 3]), 0.0)
    check_both(cuda, orc, sc.four_vars_at_once)
    check_both(cuda, orc, sc.four_vars_independent)


def test_xy_nonlinear_and_no_solution(cuda, orc):
    vals = check_both(cuda, orc, sc.xy_nonlinear)[0]
    x, y = vals[0]
    assert rel_eq(float(x * np.float32(3) + y), 5.0)
    vals = check_both(cuda, orc, sc.one_var_no_solution)[0]
    assert rel_eq(float(vals[0, 0]), 1.5)


@pytest.mark.parametrize("start", [(0.0, 0.0), (1.0, 1.0)])
def test_solve_banana(cuda, orc, start):
    vals = check_both(cuda, orc, lambda ctx: sc.banana(ctx, start))[0]
    assert rel_eq(float(vals[0, 0]), 1.0) and rel_eq(float(vals[0, 1]), 1.0)


@pytest.mark.parametrize("start", [(0.0, 0.0), (1.0, 1.5)])
def test_solve_circle(cuda, orc, start):
    vals = check_both(cuda, orc, lambda ctx: sc.circle(ctx, start))[0]
    assert rel_eq(float(vals[0, 0]), 0.0) and rel_eq(float(vals[0, 1]), 0.0)


@pytest.mark.parametrize("n,count", [(2, 50), (10, 20), (50, 3)])
def test_linear_systems(cuda, orc, n, count):
    for seed in range(count):
        build = lambda ctx: sc.linear(ctx, n, np.random.default_rng([n, seed]))   # noqa: E731
        _, check, dev = device_solve(cuda, build)
        assert sc.linear_ok(check, dev[0][0]), (n, seed)
        assert_same(dev, oracle_solve(orc, build))


# ---- device = oracle on seeded batches ---------------------------------------------------------------------------
def starts_for(case, count, seed, lo=-1.5, hi=1.5):
    rng = np.random.default_rng(seed)
    rows = np.tile(np.array(case.start, dtype=np.float32), (count, 1))
    rows[:, :len(case.free)] = rng.uniform(lo, hi, (count, len(case.free))).astype(np.float32)
    return rows


FAMILIES = [("linear", n) for n in (1, 2, 3, 4, 7, 50, 64)] + [("quadratic", n) for n in (1, 2, 3, 4, 7)] + \
           [("rosenbrock", n) for n in (2, 3, 4, 7)] + [("sphere", n) for n in (1, 2, 3, 4, 7)]


@pytest.mark.parametrize("family,n", FAMILIES, ids=[f"{f}{n}" for f, n in FAMILIES])
def test_batches_match_the_oracle_bit_for_bit(cuda, orc, family, n):
    def build(ctx):
        rng = np.random.default_rng([7, n])
        if family == "linear":
            return sc.linear(ctx, n, rng)
        if family == "quadratic":
            return sc.quadratic(ctx, n, rng)
        return sc.rosenbrock_chain(ctx, n) if family == "rosenbrock" else sc.sphere(ctx, n)
    case = build(orc.Context())
    case = case[0] if isinstance(case, tuple) else case
    starts = starts_for(case, 4 if n >= 50 else 48, [11, n])
    check_both(cuda, orc, build, starts)


def test_banana_and_circle_batches(cuda, orc):
    check_both(cuda, orc, sc.banana, starts_for(sc.banana(orc.Context()), 256, 3, -3.0, 3.0))
    check_both(cuda, orc, sc.circle, starts_for(sc.circle(orc.Context()), 256, 4, -3.0, 3.0))


def test_transcendental_ops_agree_within_tolerance(cuda, orc):
    """sin / exp come from libdevice on the device and libm in the oracle (<= 2 ulp apart).  The exits agree, except
    that FC_SOLVE_UNCHANGED and FC_SOLVE_STALLED may swap.  Both mean the iterate stopped moving at rounding level;
    which test fires first depends on the last bits of the ulp-different values (measured on H100: 3 of these 64
    problems swap).  Where both sides found a root (err < 1e-10), the roots agree within 1e-4; elsewhere the end point
    depends on the whole path (measured: one problem stops 40 apart)."""
    from fidget_b200 import _lib
    starts = starts_for(sc.transcendental(orc.Context()), 64, 5, -1.0, 1.0)
    _, _, (vals, status, iters, err) = device_solve(cuda, sc.transcendental, starts)
    rv, rs, _, re_ = oracle_solve(orc, sc.transcendental, starts)
    settled = (_lib.FC_SOLVE_UNCHANGED, _lib.FC_SOLVE_STALLED)
    same = (status == rs) | (np.isin(status, settled) & np.isin(rs, settled))
    assert same.all(), (status, rs)
    assert (status == rs).mean() >= 0.9
    converged = (err < 1e-10) & (re_ < 1e-10)
    assert converged.mean() >= 0.8
    diff = np.max(np.abs(vals - rv), axis=1)
    assert np.all(diff[converged] < 1e-4), (diff, status)


def test_problem_alone_equals_problem_in_a_batch_of_4096(cuda, orc):
    starts = starts_for(sc.banana(orc.Context()), 4096, 9, -4.0, 4.0)
    full = check_both(cuda, orc, sc.banana, starts)
    for i in (0, 1, 777, 2048, 4095):
        _, _, one = device_solve(cuda, sc.banana, starts[i:i + 1])
        assert same_f32(one[0][0], full[0][i]) and one[1][0] == full[1][i] and one[2][0] == full[2][i]
        assert same_f32(one[3], full[3][i:i + 1])


# ---- edge cases --------------------------------------------------------------------------------------------------
def test_unused_free_parameter_stays_put(cuda, orc):
    def build(ctx):
        case = sc.banana(ctx)
        case.free.append("z")
        case.start.append(0.3)
        return case
    vals = check_both(cuda, orc, build)[0]
    assert vals[0, 2] == np.float32(0.3) and rel_eq(float(vals[0, 0]), 1.0)


def test_fixed_parameters_are_read_per_problem(cuda, orc):
    def build(ctx):
        (a, ka), (b, kb) = ctx.var(), ctx.var()
        x, y = ctx.x(), ctx.y()
        return sc.Case([ctx.sub(x, a), ctx.sub(y, ctx.mul(b, x))], ["x", "y"], [ka, kb], [0.0, 0.0, 0.0, 0.0])
    rng = np.random.default_rng(12)
    starts = np.zeros((64, 4), dtype=np.float32)
    starts[:, 2:] = rng.uniform(-2, 2, (64, 2)).astype(np.float32)
    vals = check_both(cuda, orc, build, starts)[0]
    assert np.array_equal(vals[:, 2:], starts[:, 2:])
    assert np.allclose(vals[:, 0], starts[:, 2], atol=1e-5)
    assert np.allclose(vals[:, 1], starts[:, 2] * starts[:, 3], atol=1e-5)


def test_host_and_device_values_agree(cuda, orc):
    starts = starts_for(sc.banana(orc.Context()), 128, 13, -3.0, 3.0)
    _, _, host = device_solve(cuda, sc.banana, starts)
    _, _, dev = device_solve(cuda, sc.banana, starts, as_torch=True)
    assert same_f32(host[0], dev[0]) and np.array_equal(host[1], dev[1]) and np.array_equal(host[2], dev[2])
    assert same_f32(host[3], dev[3])


def test_zero_problems_launch_nothing(cuda):
    import fidget_b200 as fb
    from fidget_b200 import _lib
    ctx = fb.Context()
    shape = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.x(), 1.0)))
    vals, status, iters, err = fb.solve_batch([shape], ["x"], [], np.zeros((0, 1), np.float32))
    assert vals.shape == (0, 1) and len(status) == len(iters) == len(err) == 0
    cfg = _lib.FcSolveCfg(1, 1, 0)
    sp = np.zeros(1, np.int32)
    rc = cuda._lib.fc_solve_batch(cuda._h, (C.c_void_p * 1)(shape._h), 1,
                                  (C.POINTER(C.c_int32) * 1)(sp.ctypes.data_as(C.POINTER(C.c_int32))),
                                  C.byref(cfg), None, 0, None)
    assert rc == 0


def test_max_iters_one_gives_the_oracle_state(cuda, orc):
    from fidget_b200 import _lib
    dev = check_both(cuda, orc, sc.banana, max_iters=1)
    assert dev[1][0] == _lib.FC_SOLVE_MAX_ITERS and dev[2][0] == 1


def test_limits_and_invalid_bindings(cuda):
    import fidget_b200 as fb
    ctx = fb.Context()
    vs, keys = [], []
    for _ in range(65):
        node, vid = ctx.var()
        vs.append(node)
        keys.append(vid)
    s = vs[0]
    for v in vs[1:]:
        s = ctx.add(s, v)
    shape = fb.CudaShape(cuda, ctx.tape(s))
    with pytest.raises(fb.CudaError) as e:
        fb.solve_batch([shape], keys, [], np.zeros((1, 65), np.float32))
    assert e.value.code == -3                                          # n_free = 65: FC_ERR_UNSUPPORTED
    xy = fb.CudaShape(cuda, ctx.tape(ctx.add(ctx.x(), ctx.y())))
    with pytest.raises(fb.CudaError) as e:
        fb.solve([xy], {"x": fb.Free(0.0)})                            # y is bound to nothing
    assert e.value.code == -1


def test_spilled_tape_is_unsupported(cuda):
    import fidget_b200 as fb
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    terms = [ctx.mul(ctx.add(x, float(i)), ctx.sub(y, float(i))) for i in range(12)]
    root = terms[0]
    for t in terms[1:]:
        root = ctx.max(root, t)
    shape = fb.CudaShape(cuda, ctx.tape(root, n_regs=3))
    assert shape.info.mem_count > 0
    with pytest.raises(fb.CudaError) as e:
        fb.solve([shape], {"x": fb.Free(0.0), "y": fb.Free(0.0)})
    assert e.value.code == -3


def test_nan_constraint_ends_like_the_oracle(cuda, orc):
    """sqrt of a negative start: NaN residuals.  Only the defined exits are compared: exit and iteration count."""
    def build(ctx):
        x, y = ctx.x(), ctx.y()
        return sc.Case([ctx.sub(ctx.sqrt(x), 1.0), ctx.sub(y, 2.0)], ["x", "y"], [], [-4.0, 0.0])
    _, _, dev = device_solve(cuda, build, max_iters=40)
    ref = oracle_solve(orc, build, max_iters=40)
    assert dev[1][0] == ref[1][0] and dev[2][0] == ref[2][0]


def test_blob_shapes_bind_axes_only(cuda):
    import fidget_b200 as fb
    ctx = fb.Context()
    circle = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.square(ctx.x()), ctx.square(ctx.y()))), 1.0)))
    loaded = fb.CudaShape.from_blob(cuda, circle.serialize())
    params = {"x": fb.Free(0.5), "y": fb.Free(0.25)}
    assert fb.solve([loaded], params) == fb.solve([circle], params)
    node, _ = ctx.var()
    with_var = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.x(), node)))
    with pytest.raises(ValueError, match="blob"):
        fb.CudaShape.from_blob(cuda, with_var.serialize()).slot_keys()
