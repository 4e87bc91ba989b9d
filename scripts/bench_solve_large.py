"""Time of the cluster solver (fc_solve_large_batch) on problems fc_solve_batch cannot take, and of both solver entry
points where both can.  One JSON line per measurement, written to --out, each carrying the card's name and power limit.

    python scripts/bench_solve_large.py --out profiles/solve_large_bench.jsonl [--parent <parent tree, built>]

  large        fc_solve_large_batch on device values, device time between CUDA events around the call (median of
               --repeats after a warm-up call): sketches (tests/solver_large_cases.py) with 64, 128, 256, 512 and 1024
               free parameters, one problem and a batch of 16, and fidget-solver's linear system at n = 512 and 1024;
               exits and iteration counts alongside (above 256 free parameters one call, without a warm-up);
  oracle_cpu   the C++ oracle (oracle/solve.cc, one thread) per problem, host wall time, where it is affordable
               (n <= 128); "not run" elsewhere;
  entry_points fc_solve_batch and fc_solve_large_batch on linear n = 50 with 1 and 1024 problems (outputs compared);
  parent       with --parent: scripts/bench_solve.py's device workloads (quadratic10, linear50 at 1 and 1024 problems)
               in fresh processes alternating between the parent commit's tree (its library built) and this one,
               --rounds each."""
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SKETCH = {64: (8, 5), 128: (8, 9), 256: (16, 9), 512: (16, 17), 1024: (32, 17)}   # n_free -> (W, H)


def sketch_case(ctx, n):
    import solver_large_cases as lc
    w, h = SKETCH[n]
    return lc.sketch(ctx, w, h, seed=n)[0]


def linear_case(ctx, n):
    import solver_cases as sc
    return sc.linear(ctx, n, np.random.default_rng(2024))[0]


def starts_of(case, count):
    import solver_large_cases as lc
    if count == 1:
        return np.array([case.start], np.float32)
    return lc.sketch_starts(case, count, 7) if case.fixed else \
        np.random.default_rng(count).random((count, len(case.free)), dtype=np.float32)


def device_time(fb, cuda, fn, case, init, repeats, warmup=1):
    """fc_<fn> on a device copy of `init`, `warmup` untimed calls first: (median ms, all ms, values, results)"""
    import torch
    from fidget_b200 import _lib
    ctx_shapes = case._shapes
    keys = case.free + case.fixed
    maps = [np.array([keys.index(k) for k in s.slot_keys()], dtype=np.int32) for s in ctx_shapes]
    tapes = (C.c_void_p * len(ctx_shapes))(*[s._h for s in ctx_shapes])
    sp = (C.POINTER(C.c_int32) * len(maps))(*[m.ctypes.data_as(C.POINTER(C.c_int32)) for m in maps])
    cfg = _lib.FcSolveCfg(len(keys), len(case.free), 0)
    d_init = torch.from_numpy(init).cuda()
    vals = torch.empty_like(d_init)
    res = torch.zeros((init.shape[0], 4), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()
    torch.cuda.synchronize()
    cuda.set_stream(stream.cuda_stream)
    call = getattr(cuda._lib, "fc_" + fn)
    times = []
    try:
        for rep in range(repeats + warmup):
            vals.copy_(d_init)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            rc = call(cuda._h, tapes, len(ctx_shapes), sp, C.byref(cfg), C.c_void_p(vals.data_ptr()), init.shape[0],
                      C.c_void_p(res.data_ptr()))
            b.record(stream)
            assert rc == 0, cuda._lib.fc_last_error()
            b.synchronize()
            if rep >= warmup:
                times.append(a.elapsed_time(b))
    finally:
        cuda.set_stream(None)
    return statistics.median(times), times, vals.cpu().numpy(), res.cpu().numpy()


def prepared(fb, cuda, make, n):
    ctx = fb.Context()
    case = make(ctx, n)
    case._shapes = [fb.CudaShape(cuda, ctx.tape(r)) for r in case.roots]
    return case


def summary(res):
    return {"status_counts": np.bincount(res[:, 0], minlength=6).tolist(), "iterations_mean": float(res[:, 1].mean()),
            "iterations_max": int(res[:, 1].max()), "err_max": float(res.view(np.float32)[:, 2].max())}


def oracle_ms(make, n, init):
    import solver_cases as sc
    import solve_oracle as so
    from oracle import oracle as orc
    ctx = orc.Context()
    case = make(ctx, n)
    keys = case.free + case.fixed
    tds = [ctx.tape(r) for r in case.roots]
    t0 = time.perf_counter()
    so.solve_batch([orc.Tape.from_data(t) for t in tds], [sc.slot_map(t, keys) for t in tds], len(case.free), init)
    return (time.perf_counter() - t0) * 1e3 / len(init)


def parent_rounds(parent, rounds, repeats):
    """bench_solve.py's device workloads in fresh processes, alternating the parent's tree and this one"""
    snippet = ("import json, sys; sys.path.insert(0, {scripts!r}); import bench_solve as b; import fidget_b200 as fb; "
               "cuda = fb.CudaContext(0); "
               "print(json.dumps({{f'{{k}}/{{n}}': b.device_run(fb, cuda, k, n, {repeats})['device_ms'] "
               "for k in ('quadratic10', 'linear50') for n in (1, 1024)}}))")
    runs = {"parent": [], "this": []}
    for _ in range(rounds):
        for who in ("parent", "this"):
            tree = os.path.abspath(parent) if who == "parent" else ROOT
            env = dict(os.environ)
            env.pop("FIDGET_B200_LIB", None)
            code = snippet.format(scripts=os.path.join(tree, "scripts"), repeats=repeats)
            out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=tree)
            if out.returncode:
                raise SystemExit(out.stderr[-2000:])
            runs[who].append(json.loads(out.stdout.strip().splitlines()[-1]))
    lines = []
    for key in runs["this"][0]:
        p = [r[key] for r in runs["parent"]]
        t = [r[key] for r in runs["this"]]
        pm, tm = statistics.median(p), statistics.median(t)
        lines.append({"mode": "parent", "workload": key, "parent_ms": p, "this_ms": t,
                      "parent_spread_pct": round(100 * (max(p) - min(p)) / pm, 2),
                      "this_vs_parent_pct": round(100 * (tm / pm - 1), 2)})
    return lines


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "solve_large_bench.jsonl"))
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sizes", default="64,128,256,512,1024")
    ap.add_argument("--parent", help="tree of the parent commit with its library built (./build.sh)")
    ap.add_argument("--skip-large", action="store_true", help="only the parent and entry-point comparisons")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    open(args.out, "w").close()

    def emit(rec):   # line by line: a long run keeps what it measured
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        with open(args.out, "a") as f:
            f.write(json.dumps(rec) + "\n")

    if args.parent:
        for rec in parent_rounds(args.parent, args.rounds, args.repeats):
            emit(rec)
    import fidget_b200 as fb
    cuda = fb.CudaContext(0)
    for count in (1, 1024):
        case = prepared(fb, cuda, linear_case, 50)
        init = starts_of(case, count)
        small = device_time(fb, cuda, "solve_batch", case, init, args.repeats)
        large = device_time(fb, cuda, "solve_large_batch", case, init, args.repeats)
        same = bool(np.array_equal(small[2].view(np.uint32), large[2].view(np.uint32)) and
                    np.array_equal(small[3], large[3]))
        emit({"mode": "entry_points", "workload": "linear50", "n_problems": count, "solve_batch_ms": small[0],
              "solve_large_batch_ms": large[0], "solve_batch_ms_all": small[1], "solve_large_batch_ms_all": large[1],
              "same_bits": same, **summary(large[3])})
    if args.skip_large:
        return
    work = [("sketch", n, c) for n in [int(s) for s in args.sizes.split(",")] for c in (1, 16)]
    work += [("linear", n, 1) for n in (512, 1024)]
    for kind, n, count in work:
        make = sketch_case if kind == "sketch" else linear_case
        case = prepared(fb, cuda, make, n)
        init = starts_of(case, count)
        # a call of seconds needs no warm-up and few repeats: one above 256 free parameters
        big = n > 256
        ms, all_ms, _, res = device_time(fb, cuda, "solve_large_batch", case, init, 1 if big else args.repeats,
                                         0 if big else 1)
        emit({"mode": "large", "workload": f"{kind}{n}", "n_free": n, "n_constraints": len(case.roots),
              "n_problems": count, "device_ms": ms, "device_ms_all": all_ms, "ms_per_problem": ms / count, **summary(res)})
        if count == 1:
            emit({"mode": "oracle_cpu", "workload": f"{kind}{n}", "n_free": n,
                  "ms_per_problem": oracle_ms(make, n, init) if n <= 128 else "not run"})


if __name__ == "__main__":
    main()
