"""2D contours (fc_contour_build) on the sample models: device time of the quadtree sampler and of the contour stages
(FC_FLAG_TIMING events inside the library) and wall time of the whole build with the read into host arrays, median of 5
after two warm-up builds; leaf, vertex and polyline counts; and, in the same session for scale, fc_render2d of the same
shape into a device-resident 2^D x 2^D f32 image (device time between CUDA events, median of 5).  Workloads: prospero at
depth 10, 12 and 14, hi and quarter at 12, bear and gyroid-sphere sliced at z = 0 at 12.  One JSON line each, with the
card and power limit read in the same run.  Writes profiles/contour_bench.jsonl (or the path given).

  python scripts/bench_contour.py [out.jsonl]
  python scripts/bench_contour.py --small      one small build (hi at depth 8), for compute-sanitizer
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
WORKLOADS = [("prospero", 10, 0.0), ("prospero", 12, 0.0), ("prospero", 14, 0.0), ("hi", 12, 0.0), ("quarter", 12, 0.0),
             ("bear", 12, 0.0), ("gyroid-sphere", 12, 0.0)]
REPS, WARMUP = 5, 2


def machine():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def shape_of(cuda, name):
    with open(os.path.join(ROOT, "models", name + ".vm")) as f:
        return fb.CudaShape.from_vm(cuda, f.read())


def bench_contour(shape, depth, z):
    for _ in range(WARMUP):
        fb.contour(shape, depth, z=z)
    dev_s, dev_c, wall = [], [], []
    for _ in range(REPS):
        t0 = time.perf_counter()
        v, off, closed, info = fb.contour(shape, depth, z=z)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev_s.append(info["sampler_ms"])
        dev_c.append(info["contour_ms"])
    return {"sampler_ms": float(np.median(dev_s)), "contour_ms": float(np.median(dev_c)),
            "wall_ms": float(np.median(wall)), "wall_ms_min": float(np.min(wall)), "wall_ms_max": float(np.max(wall)),
            "n_leaves": info["n_leaves"], "n_vertices": info["n_vertices"], "n_polylines": info["n_polylines"],
            "n_closed": info["n_closed"], "n_open": info["n_open"]}


def bench_render2d(shape, depth, z):
    side = 1 << depth
    img = torch.empty((side, side), dtype=torch.float32, device="cuda")
    cfg = fb.RenderConfig2D(side, side, z=z)
    stream = torch.cuda.current_stream()
    for _ in range(WARMUP):
        fb.render2d(shape, cfg, out=img)
    ms = []
    for _ in range(REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fb.render2d(shape, cfg, out=img)
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def main():
    cuda = fb.CudaContext(0)
    cuda.set_stream(torch.cuda.current_stream().cuda_stream)
    if "--small" in sys.argv:
        v, off, closed, info = fb.contour(shape_of(cuda, "hi"), 8)
        print(json.dumps({"small": True, "n_vertices": info["n_vertices"], "n_polylines": info["n_polylines"]}))
        return
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out_path = args[0] if args else os.path.join(ROOT, "profiles", "contour_bench.jsonl")
    mach = machine()
    shapes = {}
    lines = []
    for name, depth, z in WORKLOADS:
        if name not in shapes:
            shapes[name] = shape_of(cuda, name)
        rec = {"workload": f"{name} depth {depth} z {z}", **mach}
        rec.update(bench_contour(shapes[name], depth, z))
        rec["render2d_f32_ms"] = bench_render2d(shapes[name], depth, z)
        rec["render2d_side"] = 1 << depth
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    with open(out_path, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
