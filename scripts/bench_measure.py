"""fc_measure against a device brute force at the same depth, and a ShapeVars sweep batched against one call per frame.

The brute force evaluates every cell centre -1 + (2i + 1) 2^-D with fc_float_slice_eval, Z slabs of 2^24 cells at a
time on device tensors, and reduces the inside cells to fc_measure's integers with torch int64 sums; the two sides'
integers are asserted equal.  Both sides' device time comes from CUDA events (fc_measure: its FC_FLAG_TIMING
device_ms, the levels and the brick kernel), median of 5 after two warm-ups, plus the wall time of the call.  The
batch's rows are asserted equal to the single calls'.  Workloads: bear, gyroid-sphere and colonnade at depths 8 and
10; a 64-frame sweep of a sphere's radius at depth 8.  One JSON line each, with the card and its power limit read in
the same run.  Writes profiles/measure_bench.jsonl (or the path given).

  python scripts/bench_measure.py [out.jsonl]
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


def ints(row):
    return {k: [int(v) for v in row[k]] if np.ndim(row[k]) else int(row[k])
            for k in ("n_inside", "s1", "s2", "lo", "hi")}


def brute(shape, depth):
    """fc_measure's integers over every cell centre, on the device"""
    n = 1 << depth
    dev = torch.device("cuda")
    odd = (2 * torch.arange(n, device=dev, dtype=torch.int64) + 1)
    c = ((2 * torch.arange(n, device=dev, dtype=torch.int64) + 1).to(torch.float32) * (1.0 / n) - 1.0)
    slab = max(1, (1 << 24) // (n * n))
    out = {"n_inside": 0, "s1": [0, 0, 0], "s2": [0] * 6, "lo": [0xFFFFFFFF] * 3, "hi": [0] * 3}
    cx_all = torch.zeros(n, device=dev, dtype=torch.int64)
    cy_all = torch.zeros(n, device=dev, dtype=torch.int64)
    cz_all = torch.zeros(n, device=dev, dtype=torch.int64)
    uv = uw = vw = 0
    axes, n_vars = shape._axes, shape.info.n_vars
    for k0 in range(0, n, slab):
        k1 = min(n, k0 + slab)
        z, y, x = torch.meshgrid(c[k0:k1], c, c, indexing="ij")
        ins = []
        for s in range(n_vars):
            ins.append((x if s == axes[0] else y if s == axes[1] else z).reshape(-1).contiguous())
        # (the evaluator runs on the context's stream, torch on its own: the inputs must be ready before it starts
        # and stay alive until it ends)
        torch.cuda.synchronize()
        vals = shape.float_slice_eval(ins)
        torch.cuda.synchronize()
        m = (vals < 0).reshape(k1 - k0, n, n).to(torch.int64)
        w = odd[k0:k1]
        cx_all += m.sum(dim=(0, 1))
        cy_all += m.sum(dim=(0, 2))
        cz_all[k0:k1] += m.sum(dim=(1, 2))
        # (torch has no int64 matmul on the device: the products are elementwise, then summed)
        uv += int((m.sum(dim=0) * odd[:, None] * odd[None, :]).sum())
        uw += int((m.sum(dim=1) * w[:, None] * odd[None, :]).sum())
        vw += int((m.sum(dim=2) * w[:, None] * odd[None, :]).sum())
    dot = lambda a, b: int((a * b).sum())   # noqa: E731
    out["n_inside"] = int(cz_all.sum())
    out["s1"] = [dot(cx_all, odd), dot(cy_all, odd), dot(cz_all, odd)]
    out["s2"] = [dot(cx_all, odd * odd), dot(cy_all, odd * odd), dot(cz_all, odd * odd), uv, uw, vw]
    for a, cnt in enumerate((cx_all, cy_all, cz_all)):
        nz = torch.nonzero(cnt).flatten()
        if len(nz):
            out["lo"][a], out["hi"][a] = int(nz[0]), int(nz[-1])
    return out


def timed(fn):
    """median device ms (CUDA events) and wall ms of fn() over REPS runs after WARMUP"""
    dev, wall = [], []
    r = None
    for i in range(WARMUP + REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        r = fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= WARMUP:
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(e0.elapsed_time(e1))
    return float(np.median(dev)), float(np.median(wall)), r


def measure_timed(shape, depth, **kw):
    dev, wall = [], []
    rows = None
    for i in range(WARMUP + REPS):
        t0 = time.perf_counter()
        rows, ms = fb.measure(shape, depth, timing=True, **kw)
        if i >= WARMUP:
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(ms)
    return float(np.median(dev)), float(np.median(wall)), rows


def sphere_var(cuda):
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    d = ctx.add(ctx.add(ctx.square(ctx.sub(x, 0.1)), ctx.square(y)), ctx.square(ctx.sub(z, -0.05)))
    return fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.sub(ctx.sqrt(d), r)]))


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "measure_bench.jsonl")
    cuda = fb.CudaContext(0)
    info = machine()
    lines = []
    for name in ("bear", "gyroid-sphere", "colonnade"):
        shape = model(cuda, name)
        for depth in (8, 10):
            m_dev, m_wall, rows = measure_timed(shape, depth)
            b_dev, b_wall, want = timed(lambda: brute(shape, depth))
            got = ints(rows[0])
            assert got == want, (name, depth, got, want)
            lines.append({"bench": "measure", "model": name, "depth": depth, "n_inside": got["n_inside"],
                          "brute_n_inside": want["n_inside"], "integers_equal": got == want,
                          "n_proven": int(rows[0]["n_proven"]), "n_undecided": int(rows[0]["n_undecided"]),
                          "measure_device_ms": round(m_dev, 3), "measure_wall_ms": round(m_wall, 3),
                          "brute_device_ms": round(b_dev, 3), "brute_wall_ms": round(b_wall, 3),
                          "device_speedup": round(b_dev / m_dev, 2), **info})
            print(json.dumps(lines[-1]), flush=True)
    shape = sphere_var(cuda)
    radii = [[float(r)] * 4 for r in np.linspace(0.2, 0.8, 64)]
    depth = 8
    bt_dev, bt_wall, batch = measure_timed(shape, depth, var_values=radii)

    def loop():
        rows, ms = [], 0.0
        for vv in radii:
            r, t = fb.measure(shape, depth, var_values=[vv], timing=True)
            rows.append(r)
            ms += t
        return np.concatenate(rows), ms
    dev, wall = [], []
    for i in range(WARMUP + REPS):
        t0 = time.perf_counter()
        singles, ms = loop()
        if i >= WARMUP:
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(ms)
    assert singles.tobytes() == batch.tobytes()
    lines.append({"bench": "measure_frames", "model": "sphere radius sweep", "depth": depth, "frames": len(radii),
                  "batch_device_ms": round(bt_dev, 3), "batch_wall_ms": round(bt_wall, 3),
                  "loop_device_ms": round(float(np.median(dev)), 3), "loop_wall_ms": round(float(np.median(wall)), 3),
                  **info})
    print(json.dumps(lines[-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
