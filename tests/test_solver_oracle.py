"""CPU oracle of the batched Levenberg-Marquardt solver (oracle/solve.cc, the restatement of fc_solve_batch): it
passes fidget-solver's own tests (fidget-solver/src/lib.rs), its Jacobi pseudo-inverse agrees with a float64 one, and
the C ABI's solver structs and constants are mirrored exactly by the ctypes face.  No GPU needed."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import solver_cases as sc
from oracle import oracle as orc
import solve_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def orc_solve(build, max_iters=0):
    ctx = orc.Context()
    built = build(ctx)
    case, check = built if isinstance(built, tuple) else (built, None)
    keys = case.free + case.fixed
    tds = [ctx.tape(r) for r in case.roots]
    vals, res = so.solve_batch([orc.Tape.from_data(t) for t in tds], [sc.slot_map(t, keys) for t in tds],
                                len(case.free), [case.start], max_iters)
    return dict(zip(case.free, vals[0][:len(case.free)].tolist())), res[0], check


def rel_eq(a, b, eps=np.finfo(np.float32).eps):
    """approx::relative_eq! with its f32 defaults (epsilon = max_relative = f32::EPSILON)."""
    d = abs(a - b)
    return d <= eps or d <= max(abs(a), abs(b)) * eps


def test_basic_solver():
    sol, _, _ = orc_solve(sc.basic_solver)
    assert list(sol) == ["x"] and rel_eq(sol["x"], 1.0)


def test_four_vars_at_once():
    sol, _, _ = orc_solve(sc.four_vars_at_once)
    assert len(sol) == 4
    out = np.float32(0)
    for v in sol.values():
        out = np.float32(out + np.float32(v))
    assert rel_eq(float(out), 0.0)


def test_four_vars_independent():
    sol, _, _ = orc_solve(sc.four_vars_independent)
    assert [rel_eq(v, float(i)) for i, v in enumerate(sol.values())] == [True] * 4


def test_xy_nonlinear():
    sol, _, _ = orc_solve(sc.xy_nonlinear)
    x, y = np.float32(sol["x"]), np.float32(sol["y"])
    two, three = np.float32(2), np.float32(3)
    assert rel_eq(float((x * two + y * three) * (x - y)), 2.0, eps=4 * np.finfo(np.float32).eps)
    assert rel_eq(float(x * three + y), 5.0)


def test_one_var_no_solution():
    sol, res, _ = orc_solve(sc.one_var_no_solution)
    assert rel_eq(sol["x"], 1.5)
    assert res["status"] != orc_status("MAX_ITERS")


@pytest.mark.parametrize("start", [(0.0, 0.0), (1.0, 1.0)])
def test_solve_banana(start):
    sol, _, _ = orc_solve(lambda ctx: sc.banana(ctx, start))
    assert rel_eq(sol["x"], 1.0) and rel_eq(sol["y"], 1.0)


@pytest.mark.parametrize("start", [(0.0, 0.0), (1.0, 1.5)])
def test_solve_circle(start):
    sol, _, _ = orc_solve(lambda ctx: sc.circle(ctx, start))
    assert rel_eq(sol["x"], 0.0) and rel_eq(sol["y"], 0.0)


@pytest.mark.parametrize("n,count", [(2, 200), (10, 50), (50, 4)], ids=["small", "medium", "big"])
def test_linear(n, count):
    """small/medium/big_linear with seeded systems: squared residual < 1e-3 and every row within 1e-2."""
    for seed in range(count):
        rng = np.random.default_rng([n, seed])
        sol, _, check = orc_solve(lambda ctx: sc.linear(ctx, n, rng))
        assert sc.linear_ok(check, list(sol.values())), (n, seed)


@pytest.mark.parametrize("n,count", [(2, 300), (5, 60), (10, 20)], ids=["small", "medium", "large"])
def test_quadratic(n, count):
    """many_quadratic: local minima are allowed, but at least 90 % of the seeded systems are solved."""
    ok = 0
    for seed in range(count):
        rng = np.random.default_rng([100 + n, seed])
        sol, _, check = orc_solve(lambda ctx: sc.quadratic(ctx, n, rng))
        ok += sc.quadratic_ok(check, list(sol.values()))
    assert ok >= count * 9 // 10, (ok, count)


def orc_status(name):
    from fidget_b200 import _lib
    return getattr(_lib, "FC_SOLVE_" + name)


def test_max_iters_stops_the_loop():
    full, res_full, _ = orc_solve(lambda ctx: sc.banana(ctx))
    one, res_one, _ = orc_solve(lambda ctx: sc.banana(ctx), max_iters=1)
    assert res_full["iterations"] > 1
    assert res_one["status"] == orc_status("MAX_ITERS") and res_one["iterations"] == 1
    assert one != full


# ---- the Jacobi pseudo-inverse against float64 --------------------------------------------------------------------
def psd_corpus():
    """Seeded symmetric PSD float32 matrices up to 64 x 64 with eigenvalues in [1e-3, 1] x scale, plus copies with
    zero rows and columns (a free parameter no constraint uses)."""
    out = []
    for n in (1, 2, 3, 4, 5, 7, 8, 16, 31, 33, 50, 64):
        for seed in range(6):
            rng = np.random.default_rng([n, seed])
            q, _ = np.linalg.qr(rng.standard_normal((n, n)))
            lam = 10.0 ** rng.uniform(-3, 0, n)
            scale = 10.0 ** rng.uniform(-2, 3)
            a = ((q * lam) @ q.T) * scale
            a32 = np.float32(a)
            a32 = np.triu(a32) + np.triu(a32, 1).T                   # exactly symmetric
            b = np.float32(rng.standard_normal(n) * scale)
            if seed == 5 and n > 1:
                dead = rng.choice(n, size=max(1, n // 4), replace=False)
                a32[dead, :] = 0
                a32[:, dead] = 0
                out.append((a32, b, dead))
            else:
                out.append((a32, b, None))
    return out


# largest ||x - x64|| / (cond(A) * eps32 * ||x64||) measured over this corpus: 0.55 (a 2 x 2 matrix); the bound
# leaves a margin of ~4x
PINV_BOUND = 2.0


def test_jacobi_pinv_matches_float64():
    eps = float(np.finfo(np.float32).eps)
    worst = 0.0
    for a32, b, dead in psd_corpus():
        a64 = a32.astype(np.float64)
        w = np.linalg.eigvalsh(a64)
        kept = np.abs(w) > eps
        cond = np.abs(w[kept]).max() / np.abs(w[kept]).min()
        x64 = np.linalg.pinv(a64, rcond=eps / np.abs(w).max(), hermitian=True) @ b.astype(np.float64)
        x = so.sym_pinv_apply(a32, b)
        assert np.all(np.isfinite(x))
        if dead is not None:
            assert np.all(x[dead] == 0.0)                          # exact zero column: exactly dropped
        err = np.linalg.norm(x - x64) / (cond * eps * max(np.linalg.norm(x64), 1e-30))
        worst = max(worst, err)
    assert worst < PINV_BOUND, worst


def test_jacobi_pinv_terminates_on_nan_and_inf():
    a = np.full((8, 8), np.nan, dtype=np.float32)
    assert np.all(np.isnan(so.sym_pinv_apply(a, np.ones(8, np.float32))))
    a = np.eye(5, dtype=np.float32)
    a[1, 2] = a[2, 1] = np.inf
    so.sym_pinv_apply(a, np.ones(5, np.float32))                  # returns (after the sweep cap)


# ---- C ABI mirrors ---------------------------------------------------------------------------------------------
def test_solver_structs_match_the_c_compiler(tmp_path):
    from fidget_b200 import _lib
    src = tmp_path / "solve_hdr.c"
    src.write_text('#include <stdio.h>\n#include "fidget_cuda.h"\nint main(void) {\n'
                   '  printf("%zu %zu\\n", sizeof(fc_solve_cfg), sizeof(fc_solve_result));\n  return 0;\n}\n')
    exe = tmp_path / "solve_hdr"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I",
                           os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_lib.FcSolveCfg), C.sizeof(_lib.FcSolveResult)] == [12, 16]
    assert so.SOLVE_RESULT.itemsize == 16


def test_solver_defines_are_mirrored():
    from fidget_b200 import _lib
    text = open(os.path.join(ROOT, "include", "fidget_cuda.h")).read()
    defines = dict(re.findall(r"^#define\s+(FC_SOLVE_\w+)\s+(\d+)u?\b", text, re.M))
    assert len(defines) == 9
    for name, value in defines.items():
        assert getattr(_lib, name) == int(value), name
    assert "fc_solve_batch" in _lib.CUDA_API
