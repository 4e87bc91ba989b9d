"""Throughput of the batched constraint solver (fc_solve_batch) against the two ways of solving without it.  One JSON
line per measurement, written to --out, each carrying the card's name and power limit.

    python scripts/bench_solve.py --out profiles/solve_bench.jsonl

Workloads: fidget-solver's quadratic system with n = 10 (10 constraints of 110 terms) and linear system with n = 50
(50 constraints of 50 terms), both seeded, with seeded starting points in [0, 1).  For n_problems in {1, 1024, 65536}:
  device       fc_solve_batch on device values: device time between CUDA events around the call (median of the
               repeats, after a warm-up call) and problems / s;
  host_loop    n_problems = 1 only: the same Levenberg-Marquardt loop driven from the host, one fc_grad_slice_eval per
               constraint per iteration and one fc_point_eval per constraint per step attempt (what a Rust caller of the
               CudaFunction shim in INTEGRATION.md does today), numpy for the small linear algebra; host wall time;
  oracle_cpu   the C++ oracle (oracle/solve.cc via tests/solve_oracle.py, one thread, -O2) per problem, host wall time over a few problems."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def build(ctx, kind):
    import solver_cases as sc
    rng = np.random.default_rng(2024)
    return (sc.quadratic(ctx, 10, rng) if kind == "quadratic10" else sc.linear(ctx, 50, rng))[0]


def starts(case, n):
    rng = np.random.default_rng(n)
    return rng.random((n, len(case.free)), dtype=np.float32)


def device_run(fb, cuda, kind, n, repeats):
    import torch
    from fidget_b200 import _lib
    ctx = fb.Context()
    case = build(ctx, kind)
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    maps = [np.array([case.free.index(k) for k in s.slot_keys()], dtype=np.int32) for s in shapes]
    tapes = (C.c_void_p * len(shapes))(*[s._h for s in shapes])
    sp = (C.POINTER(C.c_int32) * len(maps))(*[m.ctypes.data_as(C.POINTER(C.c_int32)) for m in maps])
    cfg = _lib.FcSolveCfg(len(case.free), len(case.free), 0)
    init = torch.from_numpy(starts(case, n)).cuda()
    vals = torch.empty_like(init)
    res = torch.zeros((n, 4), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()
    torch.cuda.synchronize()
    cuda.set_stream(stream.cuda_stream)
    times = []
    try:
        for rep in range(repeats + 1):
            vals.copy_(init)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            rc = cuda._lib.fc_solve_batch(cuda._h, tapes, len(shapes), sp, C.byref(cfg), C.c_void_p(vals.data_ptr()), n,
                                          C.c_void_p(res.data_ptr()))
            b.record(stream)
            assert rc == 0, cuda._lib.fc_last_error()
            b.synchronize()
            if rep:
                times.append(a.elapsed_time(b))
    finally:
        cuda.set_stream(None)
    r = res.cpu().numpy()
    return {"device_ms": statistics.median(times), "device_ms_all": times,
            "problems_per_s": n / (statistics.median(times) / 1e3),
            "status_counts": np.bincount(r[:, 0], minlength=6).tolist(), "iterations_mean": float(r[:, 1].mean()),
            "iterations_max": int(r[:, 1].max())}


def host_loop(fb, cuda, kind):
    """The LM loop of fidget-solver's solve with every evaluation a synchronous evaluator call."""
    ctx = fb.Context()
    case = build(ctx, kind)
    shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    n = len(case.free)
    keys = [s.slot_keys() for s in shapes]
    cur = starts(case, 1)[0].copy()
    G = (n + 2) // 3
    t0 = time.perf_counter()
    damping, prev_err, err_buf = np.float32(1), np.float32(np.inf), [np.float32(0)] * 4
    it = 0
    grad_calls = point_calls = 0
    for it in range(1000):
        J = np.zeros((len(shapes), n), np.float32)
        r = np.zeros(len(shapes), np.float32)
        for k, s in enumerate(shapes):
            ins = []
            for key in keys[k]:
                gi = case.free.index(key)
                g = np.zeros((G, 4), np.float32)
                g[:, 0] = cur[gi]
                g[gi // 3, 1 + gi % 3] = 1.0
                ins.append(g)
            out = s.grad_slice_eval(ins)
            grad_calls += 1
            for gi in range(n):
                J[k, gi] = out[gi // 3, 1 + gi % 3]
            r[k] = out[0, 0]
        if np.all(r == 0):
            break
        jtj, jtr = J.T @ J, J.T @ r
        while True:
            adj = jtj + damping * np.diag(np.diag(jtj))
            delta = np.linalg.pinv(adj, rcond=np.finfo(np.float32).eps / max(np.abs(adj).max(), 1e-30)) @ jtr
            err = np.float32(0)
            for k, s in enumerate(shapes):
                v, _, _ = s.point_eval(np.array([cur[case.free.index(key)] - delta[case.free.index(key)]
                                                 for key in keys[k]], np.float32))
                point_calls += 1
                err = np.float32(err + v[0] * v[0])
            if err > prev_err:
                damping = np.float32(damping * 1.5)
            else:
                damping = np.float32(damping / 3)
                break
        new = (cur - delta).astype(np.float32)
        changed = bool(np.any(new != cur))
        cur = new
        err_buf[it % 4] = err
        if not changed or err == 0 or damping == 0 or all(e == err_buf[0] for e in err_buf):
            break
        prev_err = err
    ms = (time.perf_counter() - t0) * 1e3
    return {"host_ms": ms, "iterations": it + 1, "grad_calls": grad_calls, "point_calls": point_calls,
            "ms_per_call": ms / max(grad_calls + point_calls, 1)}


def oracle_cpu(kind, count):
    import solver_cases as sc
    import solve_oracle as so
    from oracle import oracle as orc
    ctx = orc.Context()
    case = build(ctx, kind)
    tds = [ctx.tape(r) for r in case.roots]
    tapes = [orc.Tape.from_data(t) for t in tds]
    maps = [sc.slot_map(t, case.free) for t in tds]
    vals = starts(case, count)
    t0 = time.perf_counter()
    so.solve_batch(tapes, maps, len(case.free), vals)
    return {"ms_per_problem": (time.perf_counter() - t0) * 1e3 / count, "problems": count}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "solve_bench.jsonl"))
    ap.add_argument("--sizes", default="1,1024,65536")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch  # noqa: F401
    import fidget_b200 as fb
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    cuda = fb.CudaContext(0)
    lines = []
    for kind in ("quadratic10", "linear50"):
        for n in [int(s) for s in args.sizes.split(",")]:
            d = device_run(fb, cuda, kind, n, args.repeats if n < 65536 else max(1, args.repeats // 2))
            lines.append({"workload": kind, "mode": "device", "n_problems": n, "gpu": gpu, **d})
            print(json.dumps(lines[-1]), flush=True)
        lines.append({"workload": kind, "mode": "host_loop", "n_problems": 1, "gpu": gpu, **host_loop(fb, cuda, kind)})
        print(json.dumps(lines[-1]), flush=True)
        lines.append({"workload": kind, "mode": "oracle_cpu", "gpu": gpu, **oracle_cpu(kind, 16)})
        print(json.dumps(lines[-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
