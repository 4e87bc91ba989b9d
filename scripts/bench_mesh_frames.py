"""Mesh frame batches (fc_mesh_build_frames) against a loop of fc_mesh_build over the same frames: device time (the
FC_FLAG_TIMING sums of sampler_ms + mesh_ms) and wall time of each way with the read into host arrays, median of 5 after
two warm-ups.  The two outputs are asserted identical in the run, frame by frame (vertices bit for bit, triangles as
vertex-position triples, both as multisets: fc_mesh_build writes in atomic order).  Workloads: a 64-value ShapeVars
sweep of a sphere at depth 6, uniform and collapsed; bear in 32 turntable views at depth 7; gyroid-sphere in 16 views at
depth 7 with collapse; colonnade in 32 views at depth 6.  One JSON line each, with the card and power limit read in the
same run.  Writes profiles/mesh_frames_bench.jsonl (or the path given).

  python scripts/bench_mesh_frames.py [out.jsonl]
  python scripts/bench_mesh_frames.py --small      one small batch (sphere sweep, 4 frames at depth 4)
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


def sphere(cuda):
    """sqrt(x^2 + y^2 + z^2) - r, r a ShapeVars variable; returns the shape and r's slot"""
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    shape = fb.CudaShape(cuda, ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), r)))
    slot = list(shape.slot_keys()).index(next(k for k in shape.slot_keys() if k not in ("x", "y", "z")))
    return shape, slot


def turntable(n, tilt=20.0):
    """n views about Y, tilted about X"""
    out = []
    for a in np.linspace(0.0, 360.0, n, endpoint=False):
        t, s = np.deg2rad(a), np.deg2rad(tilt)
        ry = np.array([[np.cos(t), 0, np.sin(t), 0], [0, 1, 0, 0], [-np.sin(t), 0, np.cos(t), 0], [0, 0, 0, 1.0]])
        rx = np.array([[1, 0, 0, 0], [0, np.cos(s), -np.sin(s), 0], [0, np.sin(s), np.cos(s), 0], [0, 0, 0, 1.0]])
        out.append((rx @ ry).astype(np.float32))
    return np.stack(out)


def workloads(cuda):
    sph, slot = sphere(cuda)
    vv = np.zeros((64, sph.n_vars), np.float32)
    vv[:, slot] = np.linspace(0.1, 0.95, 64)
    yield "sphere 64-value ShapeVars sweep depth 6", sph, 6, False, {"var_values": vv}
    yield "sphere 64-value ShapeVars sweep depth 6 collapse", sph, 6, True, {"var_values": vv}
    yield "bear 32 turntable views depth 7", model(cuda, "bear"), 7, False, {"world_to_model": turntable(32)}
    yield "gyroid-sphere 16 views depth 7 collapse", model(cuda, "gyroid-sphere"), 7, True, {"world_to_model": turntable(16)}
    yield "colonnade 32 views depth 6", model(cuda, "colonnade"), 6, False, {"world_to_model": turntable(32)}


def frame_kw(per, k):
    kw = {}
    if "world_to_model" in per:
        kw["world_to_model"] = per["world_to_model"][k]
    if "var_values" in per:
        kw["var_values"] = tuple(float(v) for v in per["var_values"][k])
    return kw


def n_of(per):
    return len(next(iter(per.values())))


def run_batched(shape, depth, collapse, per):
    t0 = time.perf_counter()
    frames, info, _ = fb.mesh_frames(shape, depth, collapse=collapse, **per)
    return (time.perf_counter() - t0) * 1e3, info["sampler_ms"] + info["mesh_ms"], frames, info


def run_loop(shape, depth, collapse, per):
    t0 = time.perf_counter()
    out, dev = [], 0.0
    for k in range(n_of(per)):
        v, t, info = fb.mesh(shape, depth, collapse=collapse, **frame_kw(per, k))
        out.append((v, t))
        dev += info["sampler_ms"] + info["mesh_ms"]
    return (time.perf_counter() - t0) * 1e3, dev, out


def mesh_key(v, t):
    """the mesh as a multiset: its vertex bit patterns as sorted rows, and its triangles as sorted rows of vertex ranks
    (a vertex's place among the distinct bit patterns), each triangle rotated to start at its smallest (first, second)"""
    vb = np.ascontiguousarray(v, dtype=np.float32).reshape(-1, 3).view(np.uint32)
    order = np.lexsort(vb.T[::-1])
    rows = vb[order]
    rank = np.empty(len(vb), np.int64)
    rank[order] = np.cumsum(np.r_[False, (rows[1:] != rows[:-1]).any(axis=1)])
    r = rank[np.asarray(t, dtype=np.int64).reshape(-1, 3)]
    n = np.int64(max(len(vb), 1))
    rot = np.stack([np.roll(r, -k, axis=1) for k in range(3)])            # [3, m, 3]
    best = (rot[:, :, 0] * n + rot[:, :, 1]).argmin(axis=0)
    tri = rot[best, np.arange(len(r))]
    return rows, tri[np.lexsort(tri.T[::-1])] if len(tri) else tri


def same(a, b):
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        kx, ky = mesh_key(*x[:2]), mesh_key(*y[:2])
        if not (np.array_equal(kx[0], ky[0]) and np.array_equal(kx[1], ky[1])):
            return False
    return True


def bench(shape, depth, collapse, per):
    for _ in range(WARMUP):
        t0 = time.perf_counter()
        run_batched(shape, depth, collapse, per)
        t1 = time.perf_counter()
        run_loop(shape, depth, collapse, per)
        print(f"  warm-up: batched {t1 - t0:.2f} s, loop {time.perf_counter() - t1:.2f} s", file=sys.stderr, flush=True)
    bw, bd, lw, ld = [], [], [], []
    for _ in range(REPS):
        w, d, frames, info = run_batched(shape, depth, collapse, per)
        bw.append(w)
        bd.append(d)
        w, d, loop = run_loop(shape, depth, collapse, per)
        lw.append(w)
        ld.append(d)
    assert same(frames, loop), "the batched output differs from the loop's"
    rec = {"n_frames": n_of(per), "depth": depth, "collapse": collapse,
           "batched_device_ms": float(np.median(bd)), "loop_device_ms": float(np.median(ld)),
           "batched_wall_ms": float(np.median(bw)), "loop_wall_ms": float(np.median(lw)),
           "batched_wall_ms_min": float(np.min(bw)), "batched_wall_ms_max": float(np.max(bw)),
           "loop_wall_ms_min": float(np.min(lw)), "loop_wall_ms_max": float(np.max(lw)),
           "n_leaves": info["n_leaves"], "n_vertices": info["n_vertices"], "n_triangles": info["n_triangles"],
           "outputs_identical": True}
    rec["device_speedup"] = rec["loop_device_ms"] / rec["batched_device_ms"]
    rec["wall_speedup"] = rec["loop_wall_ms"] / rec["batched_wall_ms"]
    return rec


def main():
    cuda = fb.CudaContext(0)
    cuda.set_stream(torch.cuda.current_stream().cuda_stream)
    if "--small" in sys.argv:
        shape, slot = sphere(cuda)
        vv = np.zeros((4, shape.n_vars), np.float32)
        vv[:, slot] = [0.3, 0.5, -0.2, 0.8]
        per = {"var_values": vv}
        frames, info, _ = fb.mesh_frames(shape, 4, **per)
        assert same(frames, run_loop(shape, 4, False, per)[2])
        print(json.dumps({"small": True, "n_vertices": info["n_vertices"], "n_triangles": info["n_triangles"]}))
        return
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out_path = args[0] if args else os.path.join(ROOT, "profiles", "mesh_frames_bench.jsonl")
    mach = machine()
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    with open(out_path, "w") as f:
        for name, shape, depth, collapse, per in workloads(cuda):
            rec = {"workload": name, **mach, **bench(shape, depth, collapse, per)}
            print(json.dumps(rec), flush=True)
            f.write(json.dumps(rec) + "\n")
            f.flush()


if __name__ == "__main__":
    main()
