"""What batching 2D frames saves: fc_render2d_frames against a loop of fc_render2d over the same frames, and that
bench.py's single-frame value holds against the parent build.  One JSON line per measurement, appended to --out,
each carrying the card's name and power limit (read in the same run).

    mkdir -p build/parent && git archive <parent commit> | tar -x -C build/parent && (cd build/parent && ./build.sh)
    python scripts/bench_frames.py --parent build/parent --out profiles/frames_bench.jsonl

Per workload, `--repeats` times each (median and range reported):
  - device time: both ways enqueued asynchronously into a device tensor, timed with CUDA events on the stream;
  - end to end: host wall time of synchronous calls into pinned host memory (the slicer's case: bitmaps on the host).
Workloads: bear and gyroid-sphere, 256 Z slices at 1024^2 as 1-bit bitmaps; a ShapeVars sweep, 64 frames at 512^2;
prospero at 4096^2, 16 zoom views (f32)."""
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


def _model(name):
    with open(os.path.join(ROOT, "models", name)) as f:
        return f.read()


def _swept_shape(fb, cuda):
    """A ShapeVars sweep target: rings of a var-controlled radius cut by a wavy band"""
    g = fb.Context()
    x, y = g.x(), g.y()
    r, _ = g.var()
    ring = g.sub(g.abs(g.sub(g.sqrt(g.add(g.square(x), g.square(y))), r)), 0.05)
    band = g.sub(g.abs(g.sub(y, g.mul(g.sin(g.mul(x, 6.0)), 0.3))), 0.1)
    td = g.tape(g.min(ring, band))
    slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
    return fb.CudaShape(cuda, td), td.n_vars, slot


def workloads(fb, cuda):
    out = []
    for name in ("bear.vm", "gyroid-sphere.vm"):
        out.append((f"slice {name} 256 x 1024^2 bitmap", fb.CudaShape.from_vm(cuda, _model(name)),
                    fb.RenderConfig2D(1024, 1024, out_format="bitmap_1bit"),
                    dict(z=np.linspace(-1.0, 1.0, 256, dtype=np.float32))))
    shape, nv, slot = _swept_shape(fb, cuda)
    vv = np.zeros((64, nv), dtype=np.float32)
    vv[:, slot] = np.linspace(0.1, 0.9, 64)
    out.append(("var sweep 64 x 512^2 f32", shape, fb.RenderConfig2D(512, 512), dict(var_values=vv)))
    views = np.stack([np.array([[0.85 ** k, 0, 0.01 * k], [0, 0.85 ** k, 0.01 * k], [0, 0, 1]], dtype=np.float32)
                      for k in range(16)])
    out.append(("prospero 16 zoom views x 4096^2 f32", fb.CudaShape.from_vm(cuda, _model("prospero.vm")),
                fb.RenderConfig2D(4096, 4096), dict(world_to_model=views)))
    return out


def _stats(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def measure(fb, cuda, label, shape, cfg, per_frame, repeats):
    import torch
    table = fb.frame_table(cfg, **per_frame)
    n = len(table)
    singles = [fb.RenderConfig2D(cfg.width, cfg.height, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4), z=f.z,
                                 out_format=cfg.out_format, var_values=tuple(f.var_values[:f.n_var_values]))
               for f in table]
    dims, dtype = fb.shape._image_shape_2d(cfg)
    tdt = torch.float32 if dtype == np.float32 else torch.uint8
    dev = torch.empty((n,) + dims, dtype=tdt, device="cuda")
    pinned = torch.empty((n,) + dims, dtype=tdt, pin_memory=True)
    stream = torch.cuda.current_stream()
    cuda.set_stream(stream.cuda_stream)

    def batch(out, asynchronous):
        assert fb.render2d_frames(shape, cfg, out=out, asynchronous=asynchronous, **per_frame) is not None

    def loop(out, asynchronous):
        for k, c in enumerate(singles):
            assert fb.render2d(shape, c, out=out[k], asynchronous=asynchronous) is not None

    # the two ways agree bit for bit before anything is timed
    batch(dev, False)
    ref = dev.clone()
    loop(dev, False)
    assert torch.equal(ref.view(torch.uint8) if tdt == torch.float32 else ref, dev.view(torch.uint8) if tdt == torch.float32 else dev)

    def device_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn(dev, True)   # warm
        cuda.synchronize()
        e0.record(stream)
        fn(dev, True)
        e1.record(stream)
        cuda.synchronize()
        return e0.elapsed_time(e1)

    def host_ms(fn):
        fn(pinned, False)
        t0 = time.perf_counter()
        fn(pinned, False)
        return (time.perf_counter() - t0) * 1e3

    rec = {"workload": label, "frames": n}
    for what, timer in (("device", device_ms), ("end_to_end_pinned_host", host_ms)):
        b, lp = [], []
        for _ in range(repeats):   # alternate the two ways
            b.append(timer(batch) / n)
            lp.append(timer(loop) / n)
        rec[f"{what}_batched_ms_per_frame"] = _stats(b)
        rec[f"{what}_loop_ms_per_frame"] = _stats(lp)
        rec[f"{what}_speedup"] = round(statistics.median(lp) / statistics.median(b), 3)
    cuda.set_stream(None)
    return rec


def bench_value(tree, steps, warmup):
    env = dict(os.environ)
    env.pop("FIDGET_B200_LIB", None)
    r = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
                        str(warmup)], capture_output=True, text=True, env=env, cwd=tree)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode or not line:
        raise SystemExit(f"bench.py failed in {tree}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return json.loads(line[-1])["value"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="tree of the parent commit with its library built (./build.sh)")
    ap.add_argument("--rounds", type=int, default=4, help="alternating bench.py runs per build")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "frames_bench.jsonl"))
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    lines = []
    if args.parent:
        vals = {"parent": [], "this": []}
        for _ in range(args.rounds):
            vals["parent"].append(bench_value(os.path.abspath(args.parent), args.steps, args.warmup))
            vals["this"].append(bench_value(ROOT, args.steps, args.warmup))
        p, t = statistics.median(vals["parent"]), statistics.median(vals["this"])
        lines.append({"what": "bench.py value (prospero 4096^2, Mvoxels/s)", "gpu": gpu, "rounds": args.rounds,
                      "parent": [round(v, 1) for v in vals["parent"]], "this": [round(v, 1) for v in vals["this"]],
                      "parent_spread_pct": round(100 * (max(vals["parent"]) - min(vals["parent"])) / p, 2),
                      "this_vs_parent_pct": round(100 * (t / p - 1), 2)})
    import fidget_b200 as fb
    cuda = fb.CudaContext(0)
    for label, shape, cfg, per_frame in workloads(fb, cuda):
        rec = measure(fb, cuda, label, shape, cfg, per_frame, args.repeats)
        rec.update(what="frames", gpu=gpu, repeats=args.repeats)
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
    for rec in lines[:1] if args.parent else []:
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
