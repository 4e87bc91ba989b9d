"""Cost of cancellation (fc_ctx_set_cancel): overhead without a flag (against the parent build), overhead with a flag
attached but never set, and the latency from setting the flag to the call's return.  One JSON line per measurement,
appended to --out, each carrying the card's name and power limit.

    git worktree add /tmp/parent <parent commit> && (cd /tmp/parent && ./build.sh)
    python scripts/bench_cancel.py --parent /tmp/parent --out profiles/cancel_bench.jsonl

Workloads: bench.py's prospero 2D 4096^2 frame (device image), prospero 3D 4096^3 (device image) and the gyroid-sphere
mesh at depth 9 with cell collapse (fc_mesh_build alone: the mesh stays in HBM).  Every timing is host wall time of
one synchronous call.  The parent and this build run in alternating subprocesses, `--rounds` times each."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = ("2d", "3d", "mesh")


def _workload(fb, ctx, kind):
    """-> fn(token) running one call; True when it completed, False when it was cancelled"""
    import torch
    from fidget_b200 import _lib
    model = "gyroid-sphere.vm" if kind == "mesh" else "prospero.vm"
    with open(os.path.join(ROOT, "models", model)) as f:
        shape = fb.CudaShape.from_vm(ctx, f.read())
    if kind == "2d":
        img = torch.empty((4096, 4096), dtype=torch.float32, device="cuda")

        def run(tok):
            kw = {"cancel": tok} if tok is not None else {}
            return fb.render2d(shape, fb.RenderConfig2D(4096, 4096, **kw), out=img) is not None
        return run
    if kind == "3d":
        img = torch.empty((4096, 4096, 4), dtype=torch.float32, device="cuda")

        def run(tok):
            kw = {"cancel": tok} if tok is not None else {}
            return fb.render3d(shape, fb.RenderConfig3D(4096, 4096, 4096, **kw), out=img) is not None
        return run
    cfg = _lib.FcOctreeCfg()
    cfg.depth = 9
    cfg.flags = _lib.FC_FLAG_MESH_COLLAPSE
    info = _lib.FcMeshInfo()
    lib = shape._lib

    def build():
        return lib.fc_mesh_build(ctx._h, shape._h, C.byref(cfg), C.byref(info))

    def run(tok):
        rc = ctx._cancellable(tok, build) if tok is not None else build()
        assert rc in (0, -6), rc
        return rc == 0
    return run


def worker(args):
    """one process, one library: per workload, median call time without a flag (and with an unset one) or the
    cancel latencies"""
    if args.lib_dir:
        sys.path.insert(0, args.lib_dir)
    else:
        sys.path.insert(0, ROOT)
    import fidget_b200 as fb
    ctx = fb.CudaContext(0)
    ctx.set_arena_bytes(8 << 30)        # as bench.py: prospero 4096^3 needs more than the default 1 GiB
    out = {"lib": os.path.abspath(fb._lib.LIB_PATH)}
    for kind in WORKLOADS:
        run = _workload(fb, ctx, kind)
        for _ in range(2):
            assert run(None)
        modes = ["none"] + (["unset"] if args.mode == "overhead" and hasattr(fb, "CancelToken") else [])

        def timed(tok_fn):
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                assert run(tok_fn())
                ts.append((time.perf_counter() - t0) * 1e3)
            return ts
        if args.mode == "overhead":
            for m in modes:
                ts = timed(lambda: None if m == "none" else fb.CancelToken())
                out[f"{kind}/{m}"] = ts
        else:
            t_full = statistics.median(timed(lambda: None)) / 1e3
            lat = {}
            for frac in (0.1, 0.5, 0.9):
                xs = []
                for _ in range(5):
                    tok = fb.CancelToken()
                    stamp = {}

                    def setter():
                        time.sleep(frac * t_full)
                        stamp["t"] = time.perf_counter()
                        tok.cancel()
                    th = threading.Thread(target=setter)
                    th.start()
                    done = run(tok)
                    t_ret = time.perf_counter()
                    th.join()
                    xs.append({"cancelled": not done, "ms": (t_ret - stamp["t"]) * 1e3})
                lat[str(frac)] = xs
            out[f"{kind}/latency"] = {"t_full_ms": t_full * 1e3, "runs": lat}
    print("RESULT " + json.dumps(out))


def _run_worker(lib_dir, mode, reps):
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--mode", mode, "--reps", str(reps)]
    if lib_dir:
        cmd += ["--lib-dir", lib_dir]
    env = dict(os.environ)
    env.pop("FIDGET_B200_LIB", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
    if r.returncode or not line:
        raise SystemExit(f"worker failed ({lib_dir or 'this build'}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return json.loads(line[0][7:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="checkout of the parent commit with its library built (./build.sh)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "cancel_bench.jsonl"))
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--mode", default="overhead", choices=("overhead", "latency"))
    ap.add_argument("--lib-dir")
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    lines = []
    runs = {"parent": [], "this": []}
    for _ in range(args.rounds):   # alternate the two builds
        if args.parent:
            runs["parent"].append(_run_worker(args.parent, "overhead", args.reps))
        runs["this"].append(_run_worker(None, "overhead", args.reps))
    for kind in WORKLOADS:
        rec = {"what": "overhead", "workload": kind, "gpu": gpu, "rounds": args.rounds, "reps": args.reps}
        for build, modes in (("parent", ("none",)), ("this", ("none", "unset"))):
            for m in modes:
                if not runs[build]:
                    continue
                meds = [statistics.median(r[f"{kind}/{m}"]) for r in runs[build]]
                rec[f"{build}_{m}_ms"] = [round(x, 3) for x in meds]       # median of each round
        base = rec.get("parent_none_ms") or rec["this_none_ms"]
        spread = (max(base) - min(base)) / statistics.median(base)
        rec["parent_spread_pct"] = round(100 * spread, 2)
        for key in ("this_none_ms", "this_unset_ms"):
            rec[key.replace("_ms", "_vs_parent_pct")] = round(
                100 * (statistics.median(rec[key]) / statistics.median(base) - 1), 2)
        lines.append(rec)
    lat = _run_worker(None, "latency", args.reps)
    for kind in ("3d", "mesh"):
        L = lat[f"{kind}/latency"]
        for frac, xs in L["runs"].items():
            ms = [x["ms"] for x in xs]
            lines.append({"what": "cancel_latency", "workload": kind, "gpu": gpu, "t_full_ms": round(L["t_full_ms"], 2),
                          "set_at": float(frac), "n": len(xs), "cancelled": sum(x["cancelled"] for x in xs),
                          "median_ms": round(statistics.median(ms), 3), "max_ms": round(max(ms), 3)})
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
            print(json.dumps(rec))


if __name__ == "__main__":
    main()
