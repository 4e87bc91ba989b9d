"""fc_raycast: random rays through bear and prospero, against a device brute force, and fb.pick against fc_render3d.

Workloads, each one JSON line with the card and its power limit read in the same run:
- 2^20 random rays x 4096 steps through the [-1, 1]^3 cube on bear and prospero: device time (FC_FLAG_TIMING, the
  levels, leaves and hits of every pass), and the samples the descent evaluated (segments at every level plus leaf
  samples) against rays x steps;
- the same descent on 2^14 rays x 4096 steps against a brute force: every sample built with torch f32 ops on the device
  (t = t0 + k dt, x = o + t d, one rounding each) and evaluated with fc_float_slice_eval, its first inside sample per
  ray asserted equal to fc_raycast's k;
- fb.pick of all 1024^2 pixels of an identity view against fc_render3d at 1024^3, the depth images asserted equal.
Device times are CUDA events (both calls' FC_FLAG_TIMING), median of 5 after two warm-ups; the ray casts also
report the wall time of the call, host pass planning and copies included.  Writes profiles/raycast_bench.jsonl (or the path given).

  python scripts/bench_raycast.py [out.jsonl]
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


def random_rays(n, steps, seed):
    """Rays from a sphere of radius 2 towards random points of the cube, 4 units of t over the steps"""
    rng = np.random.default_rng(seed)
    o = rng.normal(size=(n, 3))
    o = (2.0 * o / np.linalg.norm(o, axis=1, keepdims=True)).astype(np.float32)
    d = rng.uniform(-0.8, 0.8, size=(n, 3)) - o
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    return o, d, np.float32(0.0), np.float32(4.0 / steps)


def cast_ms(shape, o, d, t0, dt, steps):
    """fc_raycast's device time (FC_FLAG_TIMING, summed over passes) and the wall time of the whole call, host pass
    planning and copies included: (device ms, wall ms, the last result), medians of REPS"""
    ms, wall, out = [], [], None
    for i in range(WARMUP + REPS):
        t = time.perf_counter()
        out = fb.raycast(shape, o, d, t0, dt, steps, timing=True)
        w = (time.perf_counter() - t) * 1e3
        if i >= WARMUP:
            ms.append(out[-1]["device_ms"])
            wall.append(w)
    return float(np.median(ms)), float(np.median(wall)), out


def render3d_ms(shape, cfg):
    """fc_render3d's device time (FC_FLAG_TIMING: first level to the last normal), into a device image, median of REPS"""
    cfg.timing = True
    dev = torch.empty((cfg.height, cfg.width, 4), dtype=torch.float32, device="cuda")
    ms = []
    for i in range(WARMUP + REPS):
        torch.cuda.synchronize()
        _, st = fb.render3d(shape, cfg, out=dev, stats=True)
        if i >= WARMUP:
            ms.append(st["stage_ms"][15])
    cfg.timing = False
    return float(np.median(ms))


def brute_k(shape, o, d, t0, dt, steps, chunk=1 << 12):
    """First inside sample per ray over every sample, on the device: (k as numpy uint32, the float slice calls' ms)"""
    dev = torch.device("cuda")
    ks, ms = [], 0.0
    kk = torch.arange(steps, device=dev, dtype=torch.float32)
    axes, n_vars = shape._axes, shape.info.n_vars
    for r0 in range(0, len(o), chunk):
        ot = torch.from_numpy(o[r0:r0 + chunk]).to(dev)
        dd = torch.from_numpy(d[r0:r0 + chunk]).to(dev)
        t = t0 + kk[None, :] * dt                       # (two kernels: one rounding each)
        xyz = [(ot[:, a:a + 1] + t * dd[:, a:a + 1]).reshape(-1).contiguous() for a in range(3)]
        ins = [xyz[axes.index(s)] if s in axes else torch.zeros_like(xyz[0]) for s in range(n_vars)]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        vals = shape.float_slice_eval(ins)
        torch.cuda.synchronize()
        b.record()
        torch.cuda.synchronize()
        ms += a.elapsed_time(b)
        ins_m = (vals < 0).reshape(-1, steps)
        k = torch.argmax(ins_m.to(torch.int8), dim=1).to(torch.int64)
        k = torch.where(ins_m.any(dim=1), k, torch.full_like(k, 0xFFFFFFFF))
        ks.append(k.cpu().numpy().astype(np.uint32))
    return np.concatenate(ks), ms


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "raycast_bench.jsonl")
    cuda = fb.CudaContext(0)
    mach = machine()
    rows = []
    steps = 4096
    for name in ("bear", "prospero"):
        shape = model(cuda, name)
        o, d, t0, dt = random_rays(1 << 20, steps, 1)
        ms, wall, r = cast_ms(shape, o, d, t0, dt, steps)
        info = r[-1]
        evaluated = sum(info["evaluated"]) + info["leaf_samples"]
        rows.append({"bench": "raycast", "model": name, "rays": 1 << 20, "steps": steps, "device_ms": ms, "wall_ms": wall,
                     "hits": info["n_hits"], "proven": info["n_proven"], "passes": info["passes"],
                     "segments_per_level": info["evaluated"], "leaf_samples": info["leaf_samples"],
                     "evaluated_over_samples": evaluated / float((1 << 20) * steps), **mach})
        print(json.dumps(rows[-1]), flush=True)
    for name in ("bear", "prospero"):
        shape = model(cuda, name)
        o, d, t0, dt = random_rays(1 << 14, steps, 2)
        ms, _, r = cast_ms(shape, o, d, t0, dt, steps)
        want, brute_ms = brute_k(shape, o, d, t0, dt, steps)
        same = bool(np.array_equal(r[0], want))
        near = bool(np.all(np.abs(r[0].astype(np.int64) - want.astype(np.int64)) <= 1))
        rows.append({"bench": "raycast_vs_brute_force", "model": name, "rays": 1 << 14, "steps": steps,
                     "raycast_device_ms": ms, "brute_force_device_ms": brute_ms, "k_equal": same,
                     "k_within_one_step": near, **mach})
        print(json.dumps(rows[-1]), flush=True)
        if name == "prospero":
            assert same, "raycast k differs from the brute force"
    for name in ("prospero", "bear"):
        shape = model(cuda, name)
        cfg = fb.RenderConfig3D(1024, 1024, 1024)
        yy, xx = np.mgrid[0:1024, 0:1024]
        px = np.stack([xx.ravel(), yy.ravel()], 1)
        render_ms = render3d_ms(shape, cfg)
        img = fb.render3d(shape, cfg)
        origins, dirs = fb.pick_rays(cfg, px)
        ms, wall, r = cast_ms(shape, origins, dirs, 0.0, 1.0, 1024)
        depth = fb.pick(shape, cfg, px)[0].reshape(1024, 1024)
        same = bool(np.array_equal(depth, img["depth"]))
        rows.append({"bench": "pick_vs_render3d", "model": name, "pixels": 1 << 20, "depth": 1024,
                     "pick_raycast_device_ms": ms, "pick_raycast_wall_ms": wall, "render3d_device_ms": render_ms,
                     "depth_equal": same, **mach})
        print(json.dumps(rows[-1]), flush=True)
        if name == "prospero":
            assert same, "fb.pick differs from fc_render3d's depth image"
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    with open(out_path, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
