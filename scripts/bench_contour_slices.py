"""Slice stacks (fc_contour_build_slices) against a loop of fc_contour_build over the same slices: device time (the
FC_FLAG_TIMING sums of sampler_ms + contour_ms) and wall time of each way with the read into host arrays, median of 5
after two warm-ups.  The two outputs are asserted identical in the run, slice by slice.  Workloads: bear as 256 Z slices
at depth 10 and 12, gyroid-sphere 128 slices at 12, colonnade 64 slices at 10, a 64-value ShapeVars sweep of a wavy
disc at 12, and prospero in 16 views at 12.  One JSON line each, with the card and power limit read in the same run.
Writes profiles/contour_slices_bench.jsonl (or the path given).

  python scripts/bench_contour_slices.py [out.jsonl]
  python scripts/bench_contour_slices.py --small      one small stack (hi, 4 slices at depth 8), for compute-sanitizer
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import fidget_b200 as fb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPS, WARMUP = 5, 2


def machine():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def model(cuda, name):
    with open(os.path.join(ROOT, "models", name + ".vm")) as f:
        return fb.CudaShape.from_vm(cuda, f.read())


def wavy_disc(cuda):
    """sqrt(x^2 + y^2) - r - 0.08 sin(7x) cos(7y), r a ShapeVars variable; returns the shape and r's slot"""
    ctx = fb.Context()
    x, y = ctx.x(), ctx.y()
    r, _ = ctx.var()
    wave = ctx.mul(ctx.mul(ctx.sin(ctx.mul(x, 7.0)), ctx.cos(ctx.mul(y, 7.0))), 0.08)
    shape = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.sub(ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y))), r), wave)))
    slot = list(shape.slot_keys()).index(next(k for k in shape.slot_keys() if k not in ("x", "y", "z")))
    return shape, slot


def rot(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1.0]], np.float32)


def workloads(cuda):
    bear = model(cuda, "bear")
    yield "bear 256 z slices depth 10", bear, 10, {"z": np.linspace(-0.9, 0.9, 256, dtype=np.float32)}
    yield "bear 256 z slices depth 12", bear, 12, {"z": np.linspace(-0.9, 0.9, 256, dtype=np.float32)}
    yield "gyroid-sphere 128 z slices depth 12", model(cuda, "gyroid-sphere"), 12, \
        {"z": np.linspace(-0.9, 0.9, 128, dtype=np.float32)}
    yield "colonnade 64 z slices depth 10", model(cuda, "colonnade"), 10, \
        {"z": np.linspace(-0.9, 0.9, 64, dtype=np.float32)}
    disc, slot = wavy_disc(cuda)
    vv = np.zeros((64, disc.n_vars), np.float32)
    vv[:, slot] = np.linspace(0.2, 0.8, 64)
    yield "wavy disc 64-value ShapeVars sweep depth 12", disc, 12, {"var_values": vv}
    yield "prospero 16 views depth 12", model(cuda, "prospero"), 12, \
        {"world_to_model": np.stack([rot(a) for a in np.linspace(0, 90, 16)])}


def per_slice_kw(per, k):
    kw = {}
    if "z" in per:
        kw["z"] = float(per["z"][k])
    if "world_to_model" in per:
        kw["world_to_model"] = per["world_to_model"][k]
    if "var_values" in per:
        kw["var_values"] = tuple(float(v) for v in per["var_values"][k])
    return kw


def n_of(per):
    return len(next(iter(per.values())))


def run_batched(shape, depth, per):
    t0 = time.perf_counter()
    slices, info, _ = fb.contour_slices(shape, depth, **per)
    return (time.perf_counter() - t0) * 1e3, info["sampler_ms"] + info["contour_ms"], slices, info


def run_loop(shape, depth, per):
    t0 = time.perf_counter()
    out, dev = [], 0.0
    for k in range(n_of(per)):
        v, off, closed, info = fb.contour(shape, depth, **per_slice_kw(per, k))
        out.append((v, off, closed))
        dev += info["sampler_ms"] + info["contour_ms"]
    return (time.perf_counter() - t0) * 1e3, dev, out


def same(a, b):
    return all(np.array_equal(x[0].view(np.uint32), y[0].view(np.uint32)) and np.array_equal(x[1], y[1])
               and np.array_equal(x[2], y[2]) for x, y in zip(a, b)) and len(a) == len(b)


def bench(shape, depth, per):
    for _ in range(WARMUP):
        run_batched(shape, depth, per)
        run_loop(shape, depth, per)
    bw, bd, lw, ld = [], [], [], []
    for _ in range(REPS):
        w, d, slices, info = run_batched(shape, depth, per)
        bw.append(w)
        bd.append(d)
        w, d, loop = run_loop(shape, depth, per)
        lw.append(w)
        ld.append(d)
        assert same(slices, loop), "the batched output differs from the loop's"
    rec = {"n_slices": n_of(per), "depth": depth,
           "batched_device_ms": float(np.median(bd)), "loop_device_ms": float(np.median(ld)),
           "batched_wall_ms": float(np.median(bw)), "loop_wall_ms": float(np.median(lw)),
           "batched_wall_ms_min": float(np.min(bw)), "batched_wall_ms_max": float(np.max(bw)),
           "loop_wall_ms_min": float(np.min(lw)), "loop_wall_ms_max": float(np.max(lw)),
           "n_leaves": info["n_leaves"], "n_vertices": info["n_vertices"], "n_polylines": info["n_polylines"],
           "outputs_identical": True}
    rec["device_speedup"] = rec["loop_device_ms"] / rec["batched_device_ms"]
    rec["wall_speedup"] = rec["loop_wall_ms"] / rec["batched_wall_ms"]
    return rec


def main():
    cuda = fb.CudaContext(0)
    cuda.set_stream(torch.cuda.current_stream().cuda_stream)
    if "--small" in sys.argv:
        shape = model(cuda, "hi")
        per = {"z": np.array([0.0, 0.2, -0.3, 0.0], np.float32)}
        slices, info, _ = fb.contour_slices(shape, 8, **per)
        assert same(slices, run_loop(shape, 8, per)[2])
        print(json.dumps({"small": True, "n_vertices": info["n_vertices"], "n_polylines": info["n_polylines"]}))
        return
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out_path = args[0] if args else os.path.join(ROOT, "profiles", "contour_slices_bench.jsonl")
    mach = machine()
    lines = []
    for name, shape, depth, per in workloads(cuda):
        rec = {"workload": name, **mach, **bench(shape, depth, per)}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    with open(out_path, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
