"""fc_solve_large_batch without a GPU: the C symbol, its ctypes and Rust faces, the Python wrappers' argument handling,
the launch planner (solve_plan.h, through a host program), and the CPU oracle on a sketch larger than fc_solve_batch
takes, held to a float64 residual."""
import inspect
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import fidget_b200 as fb
import solve_oracle as so
import solver_large_cases as lc
from fidget_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


def test_symbol_signature_and_limits():
    h = _read("include", "fidget_cuda.h")
    assert re.search(r"int32_t\s+fc_solve_large_batch\s*\(\s*fc_ctx\s*\*\s*ctx\s*,\s*const\s+fc_tape\s*\*\s*const\s*\*\s*"
                     r"constraints\s*,\s*uint32_t\s+n_constraints\s*,\s*const\s+int32_t\s*\*\s*const\s*\*\s*slot_param\s*,"
                     r"\s*const\s+fc_solve_cfg\s*\*\s*cfg\s*,\s*float\s*\*\s*values\s*,\s*uint64_t\s+n_problems\s*,\s*"
                     r"fc_solve_result\s*\*\s*results\s*\)", h)
    for name, value in (("FREE", 1024), ("CONSTRAINTS", 4096), ("PARAMS", 16384)):
        assert re.search(rf"#define\s+FC_SOLVE_LARGE_MAX_{name}\s+\(16 \* FC_SOLVE_MAX_{name}\)", h)
        assert getattr(_lib, f"FC_SOLVE_LARGE_MAX_{name}") == value
    assert _lib.CUDA_API["fc_solve_large_batch"] == _lib.CUDA_API["fc_solve_batch"]
    assert hasattr(_lib.load(), "fc_solve_large_batch")
    rs = _read("bindings", "rust", "ffi.rs")
    assert "pub fn fc_solve_large_batch(" in rs
    for name in ("FREE", "CONSTRAINTS", "PARAMS"):
        assert f"pub const FC_SOLVE_LARGE_MAX_{name}: u32 = 16 * FC_SOLVE_MAX_{name};" in rs


def test_limit_macros_evaluate_to_the_limits(tmp_path):
    src = tmp_path / "limits.c"
    src.write_text('#include <stdio.h>\n#include "fidget_cuda.h"\nint main(void) {\n'
                   '  printf("%d %d %d\\n", FC_SOLVE_LARGE_MAX_FREE, FC_SOLVE_LARGE_MAX_CONSTRAINTS, '
                   'FC_SOLVE_LARGE_MAX_PARAMS);\n  return 0;\n}\n')
    exe = tmp_path / "limits"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I",
                           os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [1024, 4096, 16384] == [_lib.FC_SOLVE_LARGE_MAX_FREE, _lib.FC_SOLVE_LARGE_MAX_CONSTRAINTS,
                                          _lib.FC_SOLVE_LARGE_MAX_PARAMS]


def test_null_context_is_invalid():
    import ctypes as C
    cfg = _lib.FcSolveCfg(1, 1, 0)
    assert _lib.load().fc_solve_large_batch(None, None, 0, None, C.byref(cfg), None, 0, None) == -1   # FC_ERR_INVALID


def test_cancel_keywords_default_to_no_token():
    for fn in (fb.solve, fb.solve_batch, fb.solve_large_batch):
        assert inspect.signature(fn).parameters["cancel"].default is None
    assert list(inspect.signature(fb.solve_large_batch).parameters) == \
        list(inspect.signature(fb.solve_batch).parameters)


def test_python_argument_validation():
    with pytest.raises(ValueError, match="solve_large_batch needs at least one constraint"):
        fb.solve_large_batch([], ["x"], [], np.zeros((1, 1), np.float32))
    with pytest.raises(TypeError, match="Free"):
        fb.solve([], {"x": 1.0})


# ---- the launch planner ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("solve_plan") / "solve_plan_check")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O1",
                    "-I", os.path.join(ROOT, "fidget_b200", "csrc", "cuda"), "-o", exe,
                    os.path.join(ROOT, "tests", "csrc", "solve_plan_check.cu")], check=True, capture_output=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines()
    return {k: [int(v) for v in rest.split()] for k, rest in (line.split(" ", 1) for line in out)}


def _floats(m, n_params, n):
    return n_params + 4 * n + 2 * m + m * n + 3 * n * n


def test_cluster_size_rule(plan):
    # one CTA per 64 free columns, rounded up to a power of two, at most 16
    assert plan["cluster"] == [1, 1, 2, 2, 4, 4, 8, 8, 16, 16]
    assert plan["forced"] == [1, 3, 8, 16, 16, 16]


def test_workspace_bytes(plan):
    assert plan["slice_floats"] == [_floats(4096, 16384, 1024), _floats(1, 1, 1), _floats(149, 120, 100)]
    assert plan["slice_bytes"] == [-(-4 * f // 256) * 256 for f in plan["slice_floats"]]
    assert 28 << 20 < plan["slice_bytes"][0] < 29 << 20             # about 28 MiB per cluster at the limits


def test_clusters_in_flight(plan):
    budget_clusters = (512 << 20) // plan["slice_bytes"][0]
    assert budget_clusters == 18
    assert plan["clusters"] == [1, 8, budget_clusters, 1, 1, 5, 1]


# ---- the oracle beyond fc_solve_batch's limits ------------------------------------------------------------------
def test_oracle_solves_a_70_free_sketch(orc):
    w, h = 7, 6
    ctx = orc.Context()
    case, edges = lc.sketch(ctx, w, h, seed=1)
    assert len(case.free) == 70
    keys = case.free + case.fixed
    tds = [ctx.tape(r) for r in case.roots]
    import solver_cases as sc
    vals, res = so.solve_batch([orc.Tape.from_data(t) for t in tds], [sc.slot_map(t, keys) for t in tds],
                               len(case.free), [case.start])
    start = np.array(case.start, dtype=np.float32)
    assert np.array_equal(vals[0, 70:].view(np.uint32), start[70:].view(np.uint32))   # the fixed row, bit for bit
    start_res = lc.sketch_residuals(w, h, edges, start)
    got = lc.sketch_residuals(w, h, edges, vals[0])
    assert np.max(np.abs(start_res)) > 1e-2
    assert np.max(np.abs(got)) < 1e-4, (np.max(np.abs(got)), res)
    assert res["err"][0] < 1e-8
