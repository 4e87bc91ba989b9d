"""What one call per scene saves: fc_render3d_scene against K fc_render3d calls into device buffers plus the same fold
on the device in torch (the greatest depth wins, the lowest index on equal depth), and that the single-shape path
(fc_render3d on bear 1024^3 and prospero 4096^3, bench.py's value) holds against the parent build.  One JSON line per
measurement, appended to --out, each carrying the card's name and power limit (read in the same run).

    mkdir -p build/parent && git archive <parent commit> | tar -x -C build/parent && (cd build/parent && ./build.sh)
    python scripts/bench_scene.py --parent build/parent --out profiles/scene_bench.jsonl

Per workload, `--repeats` times each (median and range reported):
  - device time: both ways enqueued asynchronously into device tensors, timed with CUDA events on the stream;
  - end to end: host wall time of synchronous calls, the image and index landing in pinned host memory.
Workloads: queue (8 bears one behind the other along the view axis, each peeking out: the occlusion case) at 512^3 and
1024^3; grid (16 bears on a 4 x 4 grid, little overlap) at 1024^3; mixed (colonnade, tanglecube, gyroid-sphere and bear
overlapping: four distinct tapes) at 512^3; one shape (bear 1024^3, a scene of one against fc_render3d).  The parent
comparison alternates the two builds round by round in one run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_frames import _model, _stats, bench_value  # noqa: E402
from bench_frames3d import _compare, single_ms  # noqa: E402


def _place(scale, tx, ty, tz):
    """world -> model of a shape scaled by `scale` and centred at (tx, ty, tz) in world space"""
    s = 1.0 / scale
    return np.array([[s, 0, 0, -tx * s], [0, s, 0, -ty * s], [0, 0, s, -tz * s], [0, 0, 0, 1]], dtype=np.float32)


def workloads(fb, cuda):
    bear = fb.CudaShape.from_vm(cuda, _model("bear.vm"))
    queue = np.stack([_place(0.5, -0.45 + 0.13 * k, 0.4 - 0.11 * k, 0.45 - 0.13 * k) for k in range(8)])
    grid = np.stack([_place(0.22, -0.75 + 0.5 * i, -0.75 + 0.5 * j, 0.05 * (i - j)) for j in range(4) for i in range(4)])
    mixed = [fb.CudaShape.from_vm(cuda, _model(m)) for m in ("colonnade.vm", "tanglecube.vm", "gyroid-sphere.vm")] + [bear]
    mixed_views = np.stack([_place(0.6, -0.3, 0.2, 0.1), _place(0.55, 0.3, 0.25, 0.0), _place(0.5, -0.2, -0.3, 0.2),
                            _place(0.6, 0.25, -0.2, 0.15)])
    return [("queue 8 bears 512^3", [bear] * 8, fb.RenderConfig3D(512, 512, 512), queue),
            ("queue 8 bears 1024^3", [bear] * 8, fb.RenderConfig3D(1024, 1024, 1024), queue),
            ("grid 16 bears 1024^3", [bear] * 16, fb.RenderConfig3D(1024, 1024, 1024), grid),
            ("mixed 4 tapes 512^3", mixed, fb.RenderConfig3D(512, 512, 512), mixed_views),
            ("one shape bear 1024^3", [bear], fb.RenderConfig3D(1024, 1024, 1024), np.eye(4, dtype=np.float32)[None])]


def measure(fb, cuda, shapes, cfg, views, repeats):
    import torch
    n = len(shapes)
    table = fb.scene_table(cfg, n, world_to_model=views)
    singles = [fb.RenderConfig3D(cfg.width, cfg.height, cfg.depth, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4))
               for f in table]
    h, w = cfg.height, cfg.width
    dev = torch.empty((h, w, 4), dtype=torch.int32, device="cuda")
    dev_index = torch.empty((h, w), dtype=torch.int16, device="cuda")
    per_shape = torch.empty((n, h, w, 4), dtype=torch.int32, device="cuda")
    pinned = torch.empty((h, w, 4), dtype=torch.int32, pin_memory=True)
    pinned_index = torch.empty((h, w), dtype=torch.int16, pin_memory=True)
    stream = torch.cuda.current_stream()
    cuda.set_stream(stream.cuda_stream)

    def scene(out, index, asynchronous):
        assert fb.render3d_scene(shapes, cfg, world_to_model=views, out=out, index_out=index,
                                 asynchronous=asynchronous) is not None

    def calls(out, index, asynchronous):
        """K fc_render3d into device buffers, then the fold in torch (and, for a host out, the copies)"""
        for k, c in enumerate(singles):
            assert fb.render3d(shapes[k], c, out=per_shape[k], asynchronous=True) is not None
        acc = per_shape[0].clone()
        idx = torch.zeros((h, w), dtype=torch.int16, device="cuda")
        for k in range(1, n):
            take = ~(acc[..., 3] >= per_shape[k][..., 3])   # depths < 2^31: int32 order is the uint32 order
            acc = torch.where(take[..., None], per_shape[k], acc)
            idx = torch.where(take, torch.full_like(idx, k), idx)
        out.copy_(acc, non_blocking=True)
        index.copy_(idx, non_blocking=True)
        if not asynchronous:
            torch.cuda.synchronize()

    # the two ways agree bit for bit before anything is timed
    scene(dev, dev_index, False)
    ref, ref_index = dev.clone(), dev_index.clone()
    calls(dev, dev_index, False)
    assert torch.equal(ref, dev) and torch.equal(ref_index, dev_index)

    def device_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn(dev, dev_index, True)   # warm
        torch.cuda.synchronize()
        e0.record(stream)
        fn(dev, dev_index, True)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def host_ms(fn):
        fn(pinned, pinned_index, False)
        t0 = time.perf_counter()
        fn(pinned, pinned_index, False)
        return (time.perf_counter() - t0) * 1e3

    _, _, st = fb.render3d_scene(shapes, cfg, world_to_model=views, stats=True)
    single_st = [fb.render3d(shapes[k], c, stats=True)[1] for k, c in enumerate(singles)]
    rec = {"shapes": n, "scene_evaluated": sum(st["evaluated"]),
           "calls_evaluated": sum(sum(s["evaluated"]) for s in single_st),
           "scene_kernel_launches": st["kernel_launches"], "calls_kernel_launches": sum(s["kernel_launches"] for s in single_st)}
    for what, timer in (("device", device_ms), ("end_to_end_pinned_host", host_ms)):
        a, b = [], []
        for _ in range(repeats):   # alternate the two ways
            a.append(timer(scene))
            b.append(timer(calls))
        rec[f"{what}_scene_ms"] = _stats(a)
        rec[f"{what}_calls_and_fold_ms"] = _stats(b)
        rec[f"{what}_speedup"] = round(statistics.median(b) / statistics.median(a), 3)
    cuda.set_stream(None)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="tree of the parent commit with its library built (./build.sh)")
    ap.add_argument("--rounds", type=int, default=3, help="alternating runs per build")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10, help="fc_render3d calls per single-shape timing")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--skip-scenes", action="store_true", help="only the parent comparison")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "scene_bench.jsonl"))
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    lines = []
    if args.parent:
        trees = {"parent": os.path.abspath(args.parent), "this": ROOT}
        lines.append(_compare("bench.py value (prospero 4096^2, Mvoxels/s)", gpu, args.rounds,
                              lambda w: bench_value(trees[w], args.steps, args.warmup)))
        for model, size in (("bear.vm", 1024), ("prospero.vm", 4096)):
            lines.append(_compare(f"fc_render3d {model} {size}^3 device ms", gpu, args.rounds,
                                  lambda w: single_ms(trees[w], model, size, args.reps)))
        for rec in lines:
            print(json.dumps(rec), flush=True)
    if not args.skip_scenes:
        import fidget_b200 as fb
        cuda = fb.CudaContext(0)
        cuda.set_arena_bytes(8 << 30)   # a small bear at 1024^3 alone takes more than the default 1 GiB
        for label, shapes, cfg, views in workloads(fb, cuda):
            rec = {"what": "scene", "workload": label, "gpu": gpu, "repeats": args.repeats}
            rec.update(measure(fb, cuda, shapes, cfg, views, args.repeats))
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
