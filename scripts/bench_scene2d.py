"""What one call per 2D draw list saves: fc_render2d_scene against K fc_render2d calls into device images plus the same
fold in torch on the device (the last shape inside a pixel wins, its colour painted opaque), and that the single-shape
paths hold against the parent build (bench.py's value, fc_render2d on prospero 4096^2, the bear slice stack of
bench_frames.py).  One JSON line per measurement, appended to --out, each carrying the card's name and power limit
(read in the same run).

    mkdir -p build/parent && git archive <parent commit> | tar -x -C build/parent && (cd build/parent && ./build.sh)
    python scripts/bench_scene2d.py --parent build/parent --out profiles/scene2d_bench.jsonl

Per workload, `--repeats` times each (median and range reported), the two ways alternated:
  - device time: both ways enqueued asynchronously into device tensors, timed with CUDA events on the stream;
  - end to end: host wall time of synchronous calls, the RGBA image and the index landing in pinned host memory.
Workloads (4096^2, RGBA): a viewer-like draw list of 8 overlapping placements of the models (Z = 0 slices of the 3D
ones); 256 small placements of hi.vm on a 16 x 16 grid; prospero under a frame-filling disc drawn on top (the culling
case); a scene of one prospero against fc_render2d itself."""
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
from bench_frames3d import _compare  # noqa: E402


def _place(scale, tx, ty):
    s = 1.0 / scale
    return np.array([[s, 0, -tx * s], [0, s, -ty * s], [0, 0, 1]], dtype=np.float32)


def workloads(fb, cuda):
    models = {m: fb.CudaShape.from_vm(cuda, _model(m)) for m in
              ("prospero.vm", "bear.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm", "gyroid-sphere.vm")}
    names = ("prospero.vm", "bear.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm", "gyroid-sphere.vm", "hi.vm")
    views = np.stack([_place(1.0, 0.0, 0.0), _place(0.6, -0.4, 0.3), _place(0.5, 0.4, 0.4), _place(0.5, 0.3, -0.3),
                      _place(0.45, -0.35, -0.35), _place(0.35, 0.0, 0.1), _place(0.3, 0.55, 0.0), _place(0.4, -0.1, -0.5)])
    grid = np.stack([_place(0.06, -0.9375 + 0.125 * i, -0.9375 + 0.125 * j) for j in range(16) for i in range(16)])
    g = fb.Context()
    disc = fb.CudaShape(cuda, g.tape(g.sub(g.sqrt(g.add(g.square(g.x()), g.square(g.y()))), 1.2)))
    eye = np.eye(3, dtype=np.float32)
    cfg = fb.RenderConfig2D(4096, 4096, out_format="rgba8")
    return [("viewer draw list 8 models 4096^2", [models[m] for m in names], cfg, views),
            ("hi.vm 256 placements 16x16 grid 4096^2", [models["hi.vm"]] * 256, cfg, grid),
            ("prospero under a frame-filling disc 4096^2", [models["prospero.vm"], disc], cfg, np.stack([eye, eye])),
            ("one shape prospero 4096^2", [models["prospero.vm"]], cfg, eye[None])]


def measure(fb, cuda, shapes, cfg, views, repeats):
    import torch
    n = len(shapes)
    table = fb.scene_table_2d(cfg, n, world_to_model=views)
    singles = [fb.RenderConfig2D(cfg.width, cfg.height, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4), z=f.z)
               for f in table]
    colors = np.array([[(37 * k) % 256, (91 * k + 40) % 256, (53 * k + 200) % 256] for k in range(n)], dtype=np.uint8)
    h, w = cfg.height, cfg.width
    dev = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    dev_index = torch.empty((h, w), dtype=torch.int16, device="cuda")
    per_shape = torch.empty((h, w), dtype=torch.float32, device="cuda")   # one image at a time: K of them may not fit
    table_t = torch.from_numpy(np.concatenate([colors, np.full((n, 1), 255, np.uint8)], axis=1)).cuda()
    pinned = torch.empty((h, w, 4), dtype=torch.uint8, pin_memory=True)
    pinned_index = torch.empty((h, w), dtype=torch.int16, pin_memory=True)
    stream = torch.cuda.current_stream()
    cuda.set_stream(stream.cuda_stream)

    def scene(out, index, asynchronous):
        assert fb.render2d_scene(shapes, cfg, colors=colors, world_to_model=views, out=out, index_out=index,
                                 asynchronous=asynchronous) is not None

    def calls(out, index, asynchronous):
        """K fc_render2d into a device image, each folded into the index in torch (RawDistancePixel::inside), then the
        colours looked up (and, for a host out, the copies)"""
        idx = torch.full((h, w), -1, dtype=torch.int16, device="cuda")
        for k, c in enumerate(singles):
            assert fb.render2d(shapes[k], c, out=per_shape, asynchronous=True) is not None
            bits = per_shape.view(torch.int32)
            fill = torch.isnan(per_shape) & ((bits & (0xFF << 9)) == (0xF6 << 9))
            inside = torch.where(fill, (bits & 1) == 1, per_shape < 0)
            idx = torch.where(inside, torch.full_like(idx, k), idx)
        hit = idx >= 0
        img = torch.where(hit[..., None], table_t[idx.long().clamp(min=0)], torch.zeros((), dtype=torch.uint8, device="cuda"))
        out.copy_(img, non_blocking=True)
        index.copy_(idx, non_blocking=True)   # -1 is FC_SCENE2D_NONE's bits
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

    _, _, st = fb.render2d_scene(shapes, cfg, world_to_model=views, stats=True)
    single_st = [fb.render2d(shapes[k], c, stats=True)[1] for k, c in enumerate(singles)]
    rec = {"shapes": n, "scene_evaluated": sum(st["evaluated"]),
           "calls_evaluated": sum(sum(s["evaluated"]) for s in single_st),
           "scene_pixels": st["pixels"], "calls_pixels": sum(s["pixels"] for s in single_st),
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


# device ms of one fc_render2d (prospero 4096^2, f32, device image) or one fc_render2d_frames call (bear, 256 Z slices at
# 1024^2 as 1-bit bitmaps, bench_frames.py's slice stack), median of `reps`, in the tree given as the working directory
_SINGLE = r"""
import json, sys
import numpy as np
sys.path.insert(0, ".")
import torch
import fidget_b200 as fb
what, reps = sys.argv[1], int(sys.argv[2])
cuda = fb.CudaContext(0)
if what == "prospero":
    shape = fb.CudaShape.from_vm(cuda, open("models/prospero.vm").read())
    cfg = fb.RenderConfig2D(4096, 4096)
    out = torch.empty((4096, 4096), dtype=torch.float32, device="cuda")
    call = lambda: fb.render2d(shape, cfg, out=out, asynchronous=True)
else:
    shape = fb.CudaShape.from_vm(cuda, open("models/bear.vm").read())
    cfg = fb.RenderConfig2D(1024, 1024, out_format="bitmap_1bit")
    z = np.linspace(-1.0, 1.0, 256, dtype=np.float32)
    out = torch.empty((256, 1024, 128), dtype=torch.uint8, device="cuda")
    call = lambda: fb.render2d_frames(shape, cfg, z=z, out=out, asynchronous=True)
stream = torch.cuda.current_stream()
cuda.set_stream(stream.cuda_stream)
for _ in range(3):
    call()
torch.cuda.synchronize()
ms = []
for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    call()
    e1.record(stream)
    torch.cuda.synchronize()
    ms.append(e0.elapsed_time(e1))
print(json.dumps({"ms": sorted(ms)[len(ms) // 2]}))
"""


def single_ms(tree, what, reps):
    env = dict(os.environ)
    env.pop("FIDGET_B200_LIB", None)
    r = subprocess.run([sys.executable, "-c", _SINGLE, what, str(reps)], capture_output=True, text=True, env=env, cwd=tree)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode or not line:
        raise SystemExit(f"{what} timing failed in {tree}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return json.loads(line[-1])["ms"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="tree of the parent commit with its library built (./build.sh)")
    ap.add_argument("--rounds", type=int, default=3, help="alternating runs per build")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20, help="calls per single-shape timing")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--skip-scenes", action="store_true", help="only the parent comparison")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "scene2d_bench.jsonl"))
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    lines = []
    if args.parent:
        trees = {"parent": os.path.abspath(args.parent), "this": ROOT}
        lines.append(_compare("bench.py value (prospero 4096^2, Mvoxels/s)", gpu, args.rounds,
                              lambda w: bench_value(trees[w], args.steps, args.warmup)))
        lines.append(_compare("fc_render2d prospero.vm 4096^2 f32 device ms", gpu, args.rounds,
                              lambda w: single_ms(trees[w], "prospero", args.reps)))
        lines.append(_compare("fc_render2d_frames bear.vm 256 x 1024^2 bitmap device ms per call", gpu, args.rounds,
                              lambda w: single_ms(trees[w], "bear_slices", args.reps)))
        for rec in lines:
            print(json.dumps(rec), flush=True)
    if not args.skip_scenes:
        import fidget_b200 as fb
        cuda = fb.CudaContext(0)
        for label, shapes, cfg, views in workloads(fb, cuda):
            rec = {"what": "scene2d", "workload": label, "gpu": gpu, "repeats": args.repeats}
            rec.update(measure(fb, cuda, shapes, cfg, views, args.repeats))
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
