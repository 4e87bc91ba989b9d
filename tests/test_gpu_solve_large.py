"""fc_solve_large_batch on the device: bit for bit what fc_solve_batch gives on every problem both take, bit for bit what
the CPU oracle (oracle/solve.cc) gives beyond fc_solve_batch's limits, the same bits at every cluster size and SM count,
convergence up to 1024 free parameters, the API's limits and errors, and cancellation of both solver entry points."""
import ctypes as C

import numpy as np
import pytest

import solve_oracle as so
import solver_cases as sc
import solver_large_cases as lc
from conftest import same_f32

pytestmark = pytest.mark.gpu


def _build(build, ctx):
    built = build(ctx)
    return built if isinstance(built, tuple) else (built, None)


def device_run(cuda, fn, build, starts=None, max_iters=None, as_torch=False, cancel=None):
    """fb.<fn>(...) on the case `build` makes; returns (case, check, output)"""
    import fidget_b200 as fb
    ctx = fb.Context()
    case, check = _build(build, ctx)
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    vals = np.array([case.start] if starts is None else starts, dtype=np.float32)
    if as_torch:
        import torch
        vals = torch.from_numpy(vals).cuda()
    out = getattr(fb, fn)(shapes, case.free, case.fixed, vals, max_iters, cancel=cancel)
    if as_torch and out is not None:
        out = tuple(o.cpu().numpy() for o in out)
    return case, check, out


def oracle_run(orc, build, starts=None, max_iters=None):
    ctx = orc.Context()
    case, _ = _build(build, ctx)
    keys = case.free + case.fixed
    tds = [ctx.tape(r) for r in case.roots]
    vals, res = so.solve_batch([orc.Tape.from_data(t) for t in tds], [sc.slot_map(t, keys) for t in tds],
                               len(case.free), [case.start] if starts is None else starts, max_iters or 0)
    return vals, res["status"], res["iterations"], res["err"]


def assert_same(a, b):
    assert np.array_equal(a[1], b[1]), (a[1], b[1])
    assert np.array_equal(a[2], b[2]), (a[2], b[2])
    assert same_f32(a[0], b[0])
    assert same_f32(a[3], b[3])


def starts_for(case, count, seed, lo=-1.5, hi=1.5):
    rng = np.random.default_rng(seed)
    rows = np.tile(np.array(case.start, dtype=np.float32), (count, 1))
    rows[:, :len(case.free)] = rng.uniform(lo, hi, (count, len(case.free))).astype(np.float32)
    return rows


def family(name, n):
    def build(ctx):
        rng = np.random.default_rng([7, n])
        if name == "linear":
            return sc.linear(ctx, n, rng)
        if name == "quadratic":
            return sc.quadratic(ctx, n, rng)
        return sc.rosenbrock_chain(ctx, n) if name == "rosenbrock" else sc.sphere(ctx, n)
    return build


# ---- the same bits as fc_solve_batch --------------------------------------------------------------------------------
SMALL = [("linear", n) for n in (1, 2, 3, 4, 7, 50, 64)] + [("quadratic", n) for n in (1, 2, 3, 4, 7)] + \
        [("rosenbrock", n) for n in (2, 3, 4, 7)] + [("sphere", n) for n in (1, 2, 3, 4, 7)]


@pytest.mark.parametrize("name,n", SMALL, ids=[f"{f}{n}" for f, n in SMALL])
def test_same_bits_as_solve_batch(cuda, orc, name, n):
    build = family(name, n)
    case, _ = _build(build, orc.Context())
    starts = starts_for(case, 4 if n >= 50 else 48, [11, n])
    _, _, small = device_run(cuda, "solve_batch", build, starts)
    _, _, large = device_run(cuda, "solve_large_batch", build, starts)
    assert_same(large, small)


@pytest.mark.parametrize("build,count,seed,lo,hi", [
    (sc.banana, 256, 3, -3.0, 3.0), (sc.circle, 256, 4, -3.0, 3.0), (sc.transcendental, 64, 5, -1.0, 1.0),
    (sc.basic_solver, 1, 0, 0.0, 0.0), (sc.four_vars_at_once, 1, 0, 0.0, 3.0), (sc.xy_nonlinear, 1, 0, 0.0, 0.0),
    (sc.one_var_no_solution, 1, 0, 0.0, 0.0)], ids=["banana", "circle", "transcendental", "basic", "four_vars",
                                                     "xy_nonlinear", "no_solution"])
def test_reference_cases_same_bits_as_solve_batch(cuda, orc, build, count, seed, lo, hi):
    case, _ = _build(build, orc.Context())
    starts = starts_for(case, count, seed, lo, hi) if count > 1 else None
    _, _, small = device_run(cuda, "solve_batch", build, starts)
    _, _, large = device_run(cuda, "solve_large_batch", build, starts)
    assert_same(large, small)


# ---- the same bits as the oracle, beyond fc_solve_batch ------------------------------------------------------------
SKETCH_AT = {65: (11, 4), 96: (8, 7), 128: (8, 9)}   # n -> (W, H); a sketch's n is even: 66 stands for 65
LARGE = [(f, n) for n in (65, 96, 128) for f in ("linear", "rosenbrock", "sphere", "sketch")]


@pytest.mark.parametrize("name,n", LARGE, ids=[f"{f}{n}" for f, n in LARGE])
def test_same_bits_as_the_oracle(cuda, orc, name, n):
    if name == "sketch":
        w, h = SKETCH_AT[n]
        build = lambda ctx: lc.sketch(ctx, w, h, seed=n)[0]   # noqa: E731
        case = build(orc.Context())
        starts = lc.sketch_starts(case, 2 if n == 65 else 1, n)
    else:
        build = family(name, n)
        case, _ = _build(build, orc.Context())
        starts = starts_for(case, 2 if n == 65 else 1, [13, n], -1.0, 1.0)
    _, _, dev = device_run(cuda, "solve_large_batch", build, starts)
    assert_same(dev, oracle_run(orc, build, starts))


# ---- the same bits at any launch shape -------------------------------------------------------------------------------
def _sketch400(ctx):
    return lc.sketch(ctx, 20, 11, seed=4)[0]


def test_same_bits_at_every_cluster_size_and_sm_count(cuda, orc, monkeypatch):
    import fidget_b200 as fb
    case = _sketch400(orc.Context())
    assert len(case.free) == 400
    starts = lc.sketch_starts(case, 3, 400)
    _, _, want = device_run(cuda, "solve_large_batch", _sketch400, starts, max_iters=3)
    for c in (1, 2, 4, 8, 16):
        monkeypatch.setenv("FIDGET_B200_SOLVE_CLUSTER", str(c))
        _, _, got = device_run(cuda, "solve_large_batch", _sketch400, starts, max_iters=3)
        assert_same(got, want)
    monkeypatch.delenv("FIDGET_B200_SOLVE_CLUSTER")
    for sm in (1, 3, 16):
        monkeypatch.setenv("FIDGET_B200_SM_COUNT", str(sm))
        other = fb.CudaContext(0)                 # (the SM count is read when the context is made)
        monkeypatch.delenv("FIDGET_B200_SM_COUNT")
        _, _, got = device_run(other, "solve_large_batch", _sketch400, starts, max_iters=3)
        assert_same(got, want)
        other.close()


def test_problem_alone_equals_problem_in_a_batch_of_64(cuda, orc):
    build = lambda ctx: lc.sketch(ctx, 8, 7, seed=64)[0]   # noqa: E731
    starts = lc.sketch_starts(build(orc.Context()), 64, 64)
    _, _, full = device_run(cuda, "solve_large_batch", build, starts)
    for i in (0, 1, 37, 63):
        _, _, one = device_run(cuda, "solve_large_batch", build, starts[i:i + 1])
        assert_same(one, tuple(x[i:i + 1] for x in full))


# ---- convergence where no oracle is affordable ---------------------------------------------------------------------
@pytest.mark.parametrize("n", [512, 1024])
def test_large_linear_systems_converge(cuda, n):
    _, check, (vals, status, iters, err) = device_run(
        cuda, "solve_large_batch", lambda ctx: sc.linear(ctx, n, np.random.default_rng([n, 0])))
    assert sc.linear_ok(check, vals[0]), (status, iters, err)


def test_1000_free_sketch_converges(cuda):
    import fidget_b200 as fb
    w, h = 25, 21
    ctx = fb.Context()
    case, edges = lc.sketch(ctx, w, h, seed=1000)
    assert len(case.free) == 1000
    _, _, (vals, status, iters, err) = device_run(cuda, "solve_large_batch", lambda c: lc.sketch(c, w, h, seed=1000)[0])
    start = np.array(case.start, dtype=np.float32)
    assert np.array_equal(vals[0, 1000:].view(np.uint32), start[1000:].view(np.uint32))   # the fixed row, bit for bit
    got = lc.sketch_residuals(w, h, edges, vals[0])
    assert np.max(np.abs(got)) < 1e-4, (np.max(np.abs(got)), status, iters, err)


# ---- limits and errors ----------------------------------------------------------------------------------------------
def _sum_of(ctx, n):
    vs, keys = [], []
    for _ in range(n):
        node, vid = ctx.var()
        vs.append(node)
        keys.append(vid)
    s = vs[0]
    for v in vs[1:]:
        s = ctx.add(s, v)
    return s, keys


def test_limits_and_invalid_arguments(cuda):
    import fidget_b200 as fb
    ctx = fb.Context()
    s, keys = _sum_of(ctx, 1025)
    shape = fb.CudaShape(cuda, ctx.tape(s))
    for free, fixed, cons in ((keys, [], [shape]),                              # 1025 free
                              (keys[:1024], keys[1024:], [shape] * 4097)):      # 4097 constraints
        with pytest.raises(fb.CudaError) as e:
            fb.solve_large_batch(cons, free, fixed, np.zeros((1, 1025), np.float32))
        assert e.value.code == -3                                              # FC_ERR_UNSUPPORTED
    x = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.x(), 1.0)))
    extra = [ctx.var()[1] for _ in range(16384)]
    with pytest.raises(fb.CudaError) as e:                                     # 16385 parameters
        fb.solve_large_batch([x], ["x"], extra, np.zeros((1, 16385), np.float32))
    assert e.value.code == -3
    xy = fb.CudaShape(cuda, ctx.tape(ctx.add(ctx.x(), ctx.y())))
    with pytest.raises(fb.CudaError) as e:                                     # y is bound to nothing
        fb.solve_large_batch([xy], ["x"], [], np.zeros((1, 1), np.float32))
    assert e.value.code == -1
    with pytest.raises(fb.CudaError) as e:                                     # no free parameter
        fb.solve_large_batch([xy], [], ["x", "y"], np.zeros((1, 2), np.float32))
    assert e.value.code == -1


def test_zero_problems_launch_nothing(cuda):
    import fidget_b200 as fb
    from fidget_b200 import _lib
    ctx = fb.Context()
    shape = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.x(), 1.0)))
    vals, status, iters, err = fb.solve_large_batch([shape], ["x"], [], np.zeros((0, 1), np.float32))
    assert vals.shape == (0, 1) and len(status) == len(iters) == len(err) == 0
    cfg = _lib.FcSolveCfg(1, 1, 0)
    sp = np.zeros(1, np.int32)
    rc = cuda._lib.fc_solve_large_batch(cuda._h, (C.c_void_p * 1)(shape._h), 1,
                                        (C.POINTER(C.c_int32) * 1)(sp.ctypes.data_as(C.POINTER(C.c_int32))),
                                        C.byref(cfg), None, 0, None)
    assert rc == 0


def test_host_and_device_values_agree(cuda, orc):
    build = lambda ctx: lc.sketch(ctx, 8, 7, seed=5)[0]   # noqa: E731
    starts = lc.sketch_starts(build(orc.Context()), 8, 5)
    _, _, host = device_run(cuda, "solve_large_batch", build, starts)
    _, _, dev = device_run(cuda, "solve_large_batch", build, starts, as_torch=True)
    assert_same(dev, host)


def test_solve_routes_100_free_to_the_large_solver(cuda):
    import fidget_b200 as fb
    ctx = fb.Context()
    case, _ = lc.sketch(ctx, 10, 6, seed=100)
    assert len(case.free) == 100
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    params = {k: fb.Free(v) for k, v in zip(case.free, case.start)}
    params.update({k: fb.Fixed(v) for k, v in zip(case.fixed, case.start[len(case.free):])})
    got = fb.solve(shapes, params)
    vals = fb.solve_large_batch(shapes, case.free, case.fixed, np.array([case.start], np.float32))[0]
    assert list(got) == case.free
    assert same_f32(np.array(list(got.values()), np.float32), vals[0, :100])


# ---- cancellation ----------------------------------------------------------------------------------------------------
def _raw(cuda, fn, shapes, case, vals, token):
    """fc_<fn> on `vals` (a host array or a CUDA tensor, solved in place) with `token` attached; returns the status"""
    from fidget_b200 import _lib
    keys = case.free + case.fixed
    maps = [np.array([keys.index(k) for k in s.slot_keys()], dtype=np.int32) for s in shapes]
    tapes = (C.c_void_p * len(shapes))(*[s._h for s in shapes])
    sp = (C.POINTER(C.c_int32) * len(maps))(*[m.ctypes.data_as(C.POINTER(C.c_int32)) for m in maps])
    cfg = _lib.FcSolveCfg(len(keys), len(case.free), 0)
    res = np.zeros((vals.shape[0], 4), np.int32)
    ptr = vals.data_ptr() if hasattr(vals, "data_ptr") else vals.ctypes.data
    call = getattr(cuda._lib, "fc_" + fn)
    return cuda._cancellable(token, lambda: call(cuda._h, tapes, len(shapes), sp, C.byref(cfg), C.c_void_p(ptr),
                                                 vals.shape[0], res.ctypes.data_as(C.c_void_p)))


CANCEL = [("solve_batch", "k_solve", sc.banana, 512),
          ("solve_large_batch", "k_solve_large", lambda ctx: lc.sketch(ctx, 8, 7, seed=6)[0], 24)]


@pytest.mark.parametrize("fn,site,build,count", CANCEL, ids=["solve_batch", "solve_large_batch"])
def test_cancellation(cuda, orc, monkeypatch, fn, site, build, count):
    import torch
    import fidget_b200 as fb
    case = build(orc.Context())
    starts = lc.sketch_starts(case, count, 6) if len(case.free) > 2 else starts_for(case, count, 6, -3.0, 3.0)
    ctx = fb.Context()
    case = build(ctx)
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    # a token cancelled before the call: None, host values untouched
    token = fb.CancelToken()
    token.cancel()
    assert getattr(fb, fn)(shapes, case.free, case.fixed, starts, cancel=token) is None
    vals = starts.copy()
    assert _raw(cuda, fn, shapes, case, vals, token) == -6
    assert np.array_equal(vals.view(np.uint32), starts.view(np.uint32))
    # cancelled by the poll that claims problem 5: FC_ERR_CANCELLED, host values untouched
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", f"{site}:5")
    vals = starts.copy()
    assert _raw(cuda, fn, shapes, case, vals, fb.CancelToken()) == -6
    assert np.array_equal(vals.view(np.uint32), starts.view(np.uint32))
    assert getattr(fb, fn)(shapes, case.free, case.fixed, starts, cancel=fb.CancelToken()) is None
    # device values: every row untouched or fully solved
    dvals = torch.from_numpy(starts.copy()).cuda()
    assert _raw(cuda, fn, shapes, case, dvals, fb.CancelToken()) == -6
    rows = dvals.cpu().numpy()
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    # the next call on the same context: the bits of a fresh context
    got = getattr(fb, fn)(shapes, case.free, case.fixed, starts, cancel=fb.CancelToken())
    fresh = fb.CudaContext(0)
    _, _, want = device_run(fresh, fn, build, starts)
    fresh.close()
    assert_same(got, want)
    for i in range(count):
        assert same_f32(rows[i], starts[i]) or same_f32(rows[i], got[0][i]), i
    assert same_f32(rows[5], starts[5])                                       # the cancelling claim solved nothing


# ---- the cluster path against k_solve, and cancellation after a zero-residual exit -------------------------------------
@pytest.mark.parametrize("c", [2, 4])
@pytest.mark.parametrize("name,n", [("linear", 50), ("linear", 64), ("quadratic", 7), ("rosenbrock", 7)],
                         ids=["linear50", "linear64", "quadratic7", "rosenbrock7"])
def test_multi_cta_clusters_same_bits_as_solve_batch(cuda, orc, monkeypatch, name, n, c):
    """Problems fc_solve_batch takes, forced through clusters of several CTAs"""
    build = family(name, n)
    case, _ = _build(build, orc.Context())
    starts = starts_for(case, 4 if n >= 50 else 16, [17, n])
    _, _, small = device_run(cuda, "solve_batch", build, starts)
    monkeypatch.setenv("FIDGET_B200_SOLVE_CLUSTER", str(c))
    _, _, large = device_run(cuda, "solve_large_batch", build, starts)
    assert_same(large, small)


def test_cancel_at_the_claim_after_a_zero_residual_exit(cuda, orc, monkeypatch):
    """One cluster of two CTAs in flight: problem 0 starts at rest (every residual exactly 0, so it leaves at the
    residual test) and the claim of problem 1 cancels the call.  The cancel flag is written only after every CTA has
    read it for problem 0, so the cluster stops together."""
    import fidget_b200 as fb
    monkeypatch.setenv("FIDGET_B200_SM_COUNT", "1")
    one = fb.CudaContext(0)                       # (one cluster in flight: it takes problems 0, 1, 2, ... in turn)
    monkeypatch.delenv("FIDGET_B200_SM_COUNT")
    ctx = fb.Context()
    case = lc.sketch(ctx, 8, 7, seed=3, noise=0.0)[0]                        # 96 free: two CTAs per cluster
    shapes = [fb.CudaShape(one, ctx.tape(r)) for r in case.roots]
    starts = lc.sketch_starts(case, 4, 3)
    starts[0] = np.array(case.start, np.float32)                             # at rest
    _, _, (_, status, iters, err) = device_run(one, "solve_large_batch", lambda c: lc.sketch(c, 8, 7, seed=3, noise=0.0)[0],
                                               starts[:1])
    assert status[0] == 0 and iters[0] == 0 and err[0] == 0                 # FC_SOLVE_ZERO_RESIDUAL
    monkeypatch.setenv("FIDGET_B200_CANCEL_AT", "k_solve_large:1")
    vals = starts.copy()
    assert _raw(one, "solve_large_batch", shapes, case, vals, fb.CancelToken()) == -6
    assert np.array_equal(vals.view(np.uint32), starts.view(np.uint32))
    monkeypatch.delenv("FIDGET_B200_CANCEL_AT")
    got = fb.solve_large_batch(shapes, case.free, case.fixed, starts)        # the context is as good as new
    _, _, want = device_run(cuda, "solve_large_batch", lambda c: lc.sketch(c, 8, 7, seed=3, noise=0.0)[0], starts)
    assert_same(got, want)
    one.close()
