"""fc_volume_build against the dense alternative: fc_float_slice_eval (and with gradients fc_grad_slice_eval) over every
cell centre -1 + (2i + 1) 2^-D, in device-resident Z slabs of 2^24 cells.

Workloads: a sphere of radius 0.5 and bear at depths 9 and 10, gyroid-sphere at depth 9; band 0 and a band of 4 cells;
with and without gradients.  The volume's device time is its FC_FLAG_TIMING device_ms (levels, sorts, bricks and
gradients) with level_ms, the interval levels alone, beside fc_measure's device time at the same depth; the dense side's
is CUDA events around the slab loop.  Median of 5 after two warm-ups.  At depth 9 every brick value is asserted equal to
the dense value at its cell, bit for bit.  One JSON line each, with the card and its power limit read in the same run.
Writes profiles/volume_bench.jsonl (or the path given).

  python scripts/bench_volume.py [out.jsonl]
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import fidget_b200 as fb
from bench_measure import REPS, WARMUP, machine, measure_timed, model, timed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sphere(cuda):
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    d = ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))
    return fb.CudaShape(cuda, fb.TapeData(ctx, [ctx.sub(ctx.sqrt(d), 0.5)]))


def dense(shape, depth, grads, keep=False):
    """every cell centre through the slice evaluators, Z slab by Z slab; with keep the [z, y, x] values"""
    n = 1 << depth
    dev = torch.device("cuda")
    c = (2 * torch.arange(n, device=dev, dtype=torch.int64) + 1).to(torch.float32) * (1.0 / n) - 1.0
    slab = max(1, (1 << 24) // (n * n))
    axes, n_vars = shape._axes, shape.info.n_vars
    out = torch.empty((n, n, n), dtype=torch.float32, device=dev) if keep else None
    for k0 in range(0, n, slab):
        k1 = min(n, k0 + slab)
        z, y, x = torch.meshgrid(c[k0:k1], c, c, indexing="ij")
        cols = [(x if s == axes[0] else y if s == axes[1] else z).reshape(-1).contiguous() for s in range(n_vars)]
        torch.cuda.synchronize()   # (the evaluators run on the context's stream)
        vals = shape.float_slice_eval(cols)
        if grads:
            g = []
            for s in range(n_vars):
                a = torch.zeros((cols[s].numel(), 4), dtype=torch.float32, device=dev)
                a[:, 0] = cols[s]
                a[:, 1 + list(axes).index(s)] = 1
                g.append(a)
            torch.cuda.synchronize()
            shape.grad_slice_eval(g)
        torch.cuda.synchronize()
        if keep:
            out[k0:k1] = vals.reshape(k1 - k0, n, n)
    return out


def volume_timed(shape, depth, band, grads):
    dev, lvl, wall = [], [], []
    vol = None
    for i in range(WARMUP + REPS):
        t0 = time.perf_counter()
        vol = fb.volume(shape, depth, band=band, grads=grads, timing=True, device=True)
        if i >= WARMUP:
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(vol.info["device_ms"])
            lvl.append(vol.info["level_ms"])
    return float(np.median(dev)), float(np.median(lvl)), float(np.median(wall)), vol


def check(vol, want):
    B = vol.brick_edge
    b = vol.bricks[:, 1:4].long()
    r = torch.arange(B, device=b.device)
    iz = (b[:, 2, None, None, None] + r[None, :, None, None]).expand(-1, B, B, B)
    iy = (b[:, 1, None, None, None] + r[None, None, :, None]).expand(-1, B, B, B)
    ix = (b[:, 0, None, None, None] + r[None, None, None, :]).expand(-1, B, B, B)
    return bool(torch.equal(want[iz, iy, ix].view(torch.int32), vol.values.view(torch.int32)))


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "volume_bench.jsonl")
    cuda = fb.CudaContext(0)
    info = machine()
    lines = []
    work = [("sphere r=0.5", sphere(cuda), (9, 10)), ("bear", model(cuda, "bear"), (9, 10)),
            ("gyroid-sphere", model(cuda, "gyroid-sphere"), (9,))]
    for name, shape, depths in work:
        for depth in depths:
            m_dev, _, _ = measure_timed(shape, depth)
            want = dense(shape, depth, False, keep=True) if depth == 9 else None
            for cells in (0, 4):
                band = cells * 2.0 / (1 << depth)
                for grads in (False, True):
                    v_dev, v_lvl, v_wall, vol = volume_timed(shape, depth, band, grads)
                    d_dev, d_wall, _ = timed(lambda: dense(shape, depth, grads))
                    ok = check(vol, want) if want is not None else None
                    if want is not None:
                        assert ok, (name, depth, band)
                    nb = vol.info["n_bricks"]
                    lines.append({"bench": "volume", "model": name, "depth": depth, "band_cells": cells, "band": band,
                                  "grads": grads, "n_bricks": nb, "n_tiles": vol.info["n_tiles"],
                                  "volume_bytes": nb * vol.brick_edge ** 3 * 4 * (1 + 3 * grads),
                                  "dense_bytes": 8 ** depth * 4 * (1 + 3 * grads),
                                  "volume_device_ms": round(v_dev, 3), "volume_level_ms": round(v_lvl, 3),
                                  "volume_wall_ms": round(v_wall, 3), "measure_device_ms": round(m_dev, 3),
                                  "dense_device_ms": round(d_dev, 3), "dense_wall_ms": round(d_wall, 3),
                                  "device_speedup": round(d_dev / v_dev, 2), "brick_values_equal_dense": ok, **info})
                    print(json.dumps(lines[-1]), flush=True)
            del want
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
