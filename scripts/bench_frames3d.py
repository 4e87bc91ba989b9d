"""What batching 3D frames saves: fc_render3d_frames against a loop of fc_render3d over the same frames, and that the
single-frame path (fc_render3d on bear 1024^3 and prospero 4096^3, bench.py's value) holds against the parent build.
One JSON line per measurement, appended to --out, each carrying the card's name and power limit (read in the same run).

    mkdir -p build/parent && git archive <parent commit> | tar -x -C build/parent && (cd build/parent && ./build.sh)
    python scripts/bench_frames3d.py --parent build/parent --out profiles/frames3d_bench.jsonl

Per workload, `--repeats` times each (median and range reported):
  - device time: both ways enqueued asynchronously into a device tensor, timed with CUDA events on the stream;
  - end to end: host wall time of synchronous calls into pinned host memory.
Workloads: a 64-view bear orbit at 256^3 and 512^3; a 64-frame ShapeVars sphere sweep at 256^3; 16 colonnade views at
512^3; 8 prospero views at 1024^3.  The parent comparison alternates the two builds round by round in one run."""
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


def _orbit(n):
    def rot(a):
        c, s = np.cos(a), np.sin(a)
        return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]], dtype=np.float32)
    return np.stack([rot(2 * np.pi * k / n) for k in range(n)])


def _sphere_var(fb, cuda):
    g = fb.Context()
    x, y, z = g.x(), g.y(), g.z()
    r, _ = g.var()
    td = g.tape(g.sub(g.sqrt(g.add(g.add(g.square(x), g.square(y)), g.square(z))), r))
    slot = [i for i, (k, _) in enumerate(td.vars()) if k == "v"][0]
    return fb.CudaShape(cuda, td), td.n_vars, slot


def workloads(fb, cuda):
    bear = fb.CudaShape.from_vm(cuda, _model("bear.vm"))
    out = [("bear orbit 64 x 256^3", bear, fb.RenderConfig3D(256, 256, 256), dict(world_to_model=_orbit(64))),
           ("bear orbit 64 x 512^3", bear, fb.RenderConfig3D(512, 512, 512), dict(world_to_model=_orbit(64)))]
    shape, nv, slot = _sphere_var(fb, cuda)
    vv = np.zeros((64, nv), dtype=np.float32)
    vv[:, slot] = np.linspace(0.1, 0.95, 64)
    out.append(("sphere var sweep 64 x 256^3", shape, fb.RenderConfig3D(256, 256, 256), dict(var_values=vv)))
    out.append(("colonnade 16 views x 512^3", fb.CudaShape.from_vm(cuda, _model("colonnade.vm")),
                fb.RenderConfig3D(512, 512, 512), dict(world_to_model=_orbit(16))))
    out.append(("prospero 8 views x 1024^3", fb.CudaShape.from_vm(cuda, _model("prospero.vm")),
                fb.RenderConfig3D(1024, 1024, 1024), dict(world_to_model=_orbit(8))))
    return out


def measure(fb, cuda, label, shape, cfg, per_frame, repeats):
    import torch
    table = fb.frame_table_3d(cfg, **per_frame)
    n = len(table)
    singles = [fb.RenderConfig3D(cfg.width, cfg.height, cfg.depth, mat=np.array(f.mat, dtype=np.float32).reshape(4, 4),
                                 var_values=tuple(f.var_values[:f.n_var_values])) for f in table]
    dims = (n, cfg.height, cfg.width, 4)
    dev = torch.empty(dims, dtype=torch.int32, device="cuda")
    pinned = torch.empty(dims, dtype=torch.int32, pin_memory=True)
    stream = torch.cuda.current_stream()
    cuda.set_stream(stream.cuda_stream)

    def batch(out, asynchronous):
        assert fb.render3d_frames(shape, cfg, out=out, asynchronous=asynchronous, **per_frame) is not None

    def loop(out, asynchronous):
        for k, c in enumerate(singles):
            assert fb.render3d(shape, c, out=out[k], asynchronous=asynchronous) is not None

    # the two ways agree bit for bit before anything is timed
    batch(dev, False)
    ref = dev.clone()
    loop(dev, False)
    assert torch.equal(ref, dev)

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


# one fc_render3d of `model` at size^3 into a device tensor, device ms from events (median of `reps` after a warm-up),
# run in `tree` (its own build of the library)
_SINGLE = r"""
import json, os, sys, statistics
sys.path.insert(0, os.getcwd())
import torch, fidget_b200 as fb
model, size, reps = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
cuda = fb.CudaContext(0)
cuda.set_arena_bytes(8 << 30)   # prospero 4096^3, as bench.py renders it
shape = fb.CudaShape.from_vm(cuda, open(os.path.join("models", model)).read())
out = torch.empty((size, size, 4), dtype=torch.int32, device="cuda")
stream = torch.cuda.current_stream()
cuda.set_stream(stream.cuda_stream)
cfg = fb.RenderConfig3D(size, size, size)
for _ in range(3):
    fb.render3d(shape, cfg, out=out, asynchronous=True)
cuda.synchronize()
ms = []
for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fb.render3d(shape, cfg, out=out, asynchronous=True)
    e1.record(stream)
    cuda.synchronize()
    ms.append(e0.elapsed_time(e1))
print(json.dumps({"ms": statistics.median(ms)}))
"""


def single_ms(tree, model, size, reps):
    env = dict(os.environ)
    env.pop("FIDGET_B200_LIB", None)
    r = subprocess.run([sys.executable, "-c", _SINGLE, model, str(size), str(reps)], capture_output=True, text=True,
                       env=env, cwd=tree)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode or not line:
        raise SystemExit(f"render3d timing failed in {tree}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return json.loads(line[-1])["ms"]


def _compare(what, gpu, rounds, fn):
    """alternating rounds of the parent build and this one: medians, the parent's spread and the difference"""
    vals = {"parent": [], "this": []}
    for _ in range(rounds):
        vals["parent"].append(fn("parent"))
        vals["this"].append(fn("this"))
    p, t = statistics.median(vals["parent"]), statistics.median(vals["this"])
    return {"what": what, "gpu": gpu, "rounds": rounds,
            "parent": [round(v, 3) for v in vals["parent"]], "this": [round(v, 3) for v in vals["this"]],
            "parent_spread_pct": round(100 * (max(vals["parent"]) - min(vals["parent"])) / p, 2),
            "this_spread_pct": round(100 * (max(vals["this"]) - min(vals["this"])) / t, 2),
            "this_vs_parent_pct": round(100 * (t / p - 1), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="tree of the parent commit with its library built (./build.sh)")
    ap.add_argument("--rounds", type=int, default=4, help="alternating runs per build")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10, help="fc_render3d calls per single-frame timing")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--skip-frames", action="store_true", help="only the parent comparison")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "frames3d_bench.jsonl"))
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
    if not args.skip_frames:
        import fidget_b200 as fb
        cuda = fb.CudaContext(0)
        cuda.set_arena_bytes(8 << 30)   # rotated prospero views at 1024^3 take more than the default 1 GiB
        for label, shape, cfg, per_frame in workloads(fb, cuda):
            rec = measure(fb, cuda, label, shape, cfg, per_frame, args.repeats)
            rec.update(what="frames3d", gpu=gpu, repeats=args.repeats)
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
