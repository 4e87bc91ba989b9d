"""Where the prospero 4096^2 frame spends its time after the root level, and what a build changes there: stage times
of fc_render2d (CUDA events inside the library, FC_FLAG_TIMING) for the parent build and this one in alternating
rounds, with L2 flushed before every frame as bench.py does and once more without the flush; bench.py's `value` and
its 4096^3 volume for both builds; fc_render3d on bear 1024^3; and the rate of same-address atomics, which is what a
shared work cursor costs per claim.  One JSON line per measurement, appended to --out, each carrying the card's name,
power limit and SM clock (read in the same run).

    mkdir -p build/parent && git archive <parent commit> | tar -x -C build/parent && (cd build/parent && ./build.sh)
    python scripts/bench_levels2d.py --parent build/parent --out profiles/levels2d_bench.jsonl

Each round starts one process per build (FIDGET_B200_LIB selects the library) that renders `--frames` timed frames per
mode, and one bench.py per build."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIZE = 4096
STAGES = {"level0": 0, "level1": 1, "level2": 2, "fills": 8, "leaves": 9, "total": 15}

# W warps, K dependent atomicAdd each: on ONE word (what a shared cursor is), on one word per warp, 128 bytes apart
# (the same instructions without the shared address), and no atomics at all (what the launch itself costs)
ATOMIC_SRC = r"""
#include <cuda_runtime.h>
__global__ void __launch_bounds__(128) k_claims(unsigned* words, unsigned stride, int k) {
    const unsigned gw = blockIdx.x * 4u + (threadIdx.x >> 5);
    if ((threadIdx.x & 31) == 0)
        for (int i = 0; i < k; ++i)
            if (atomicAdd(words + size_t(gw) * stride, 1u) == 0xffffffffu) break;   // (a claim waits for the one before it)
}
extern "C" int claims_ms(int blocks, int k, int reps, float* same_ms, float* apart_ms, float* empty_ms) {
    unsigned* words = nullptr;
    if (cudaMalloc(&words, size_t(blocks) * 4 * 128) != cudaSuccess) return 1;
    cudaMemset(words, 0, size_t(blocks) * 4 * 128);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float* outs[3] = {same_ms, apart_ms, empty_ms};
    const unsigned strides[3] = {0u, 32u, 0u};
    const int ks[3] = {k, k, 0};
    for (int m = 0; m < 3; ++m) {
        k_claims<<<blocks, 128>>>(words, strides[m], ks[m]);   // warm
        cudaEventRecord(e0);
        for (int r = 0; r < reps; ++r) k_claims<<<blocks, 128>>>(words, strides[m], ks[m]);
        cudaEventRecord(e1);
        if (cudaEventSynchronize(e1) != cudaSuccess) return 2;
        cudaEventElapsedTime(outs[m], e0, e1);
        *outs[m] /= float(reps);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(words);
    return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
"""


def _stats(xs):
    return {"median": round(statistics.median(xs), 5), "min": round(min(xs), 5), "max": round(max(xs), 5)}


def gpu_id():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    if not q:
        raise SystemExit("no GPU: this script measures on the device only")
    return q[0]


def atomic_rate(tmp, sm_count):
    """ns per claim of k_pixels_2d's grid shape (8 CTAs of 4 warps per SM) making the ~31 k claims of the leaf kernel"""
    src, lib = os.path.join(tmp, "claims.cu"), os.path.join(tmp, "libclaims.so")
    with open(src, "w") as f:
        f.write(ATOMIC_SRC)
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                           "-shared", "-Xcompiler", "-fPIC", "-o", lib, src])
    dll = ctypes.CDLL(lib)
    blocks, k, reps = sm_count * 8, 7, 50
    ms = [ctypes.c_float() for _ in range(3)]
    rc = dll.claims_ms(blocks, k, reps, *[ctypes.byref(m) for m in ms])
    if rc:
        raise SystemExit(f"claims_ms failed: {rc}")
    same, apart, empty = (m.value for m in ms)
    n = blocks * 4 * k
    return {"what": "same-address atomicAdd", "warps": blocks * 4, "claims_per_warp": k, "claims": n,
            "one_word_ms": round(same, 5), "word_per_warp_ms": round(apart, 5), "no_atomics_ms": round(empty, 5),
            "ns_per_claim_one_word": round((same - empty) * 1e6 / n, 3),
            "ns_per_claim_word_per_warp": round((apart - empty) * 1e6 / n, 3)}


def worker(args):
    """One build (the library FIDGET_B200_LIB names, else this tree's): stage times and 3D times, as one JSON line"""
    import torch
    import fidget_b200 as fb
    dev = torch.device("cuda", 0)
    cuda = fb.CudaContext(0)
    cuda.set_arena_bytes(8 << 30)
    stream = torch.cuda.current_stream()
    cuda.set_stream(stream.cuda_stream)

    def model(name):
        with open(os.path.join(ROOT, "models", name)) as f:
            return fb.CudaShape.from_vm(cuda, f.read())

    shape = model("prospero.vm")
    image = torch.zeros((SIZE, SIZE), dtype=torch.float32, device=dev)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)   # > the 50 MB L2
    tcfg = fb.RenderConfig2D(SIZE, SIZE, timing=True)
    out = {}
    for _ in range(5):
        fb.render2d(shape, tcfg, out=image, stats=True)
    for mode in ("flushed", "unflushed"):
        rows = []
        for i in range(args.frames):
            if mode == "flushed":
                flush.fill_(i & 255)
            _, st = fb.render2d(shape, tcfg, out=image, stats=True)
            rows.append([st["stage_ms"][k] for k in STAGES.values()])
        med = np.median(np.array(rows), axis=0)
        out[mode] = {n: float(med[i]) for i, n in enumerate(STAGES)}
    out["census"] = {k: st[k][:3] for k in ("evaluated", "ambiguous")}

    def device_ms(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()
        cuda.synchronize()
        e0.record(stream)
        for _ in range(n):
            fn()
        e1.record(stream)
        cuda.synchronize()
        return e0.elapsed_time(e1) / n

    # a frame batch (its kernels keep the shared cursor) and the 3D render of another model
    views = np.stack([np.array([[0.85 ** k, 0, 0.01 * k], [0, 0.85 ** k, 0.01 * k], [0, 0, 1]], dtype=np.float32) for k in range(8)])
    batch = torch.zeros((8, SIZE, SIZE), dtype=torch.float32, device=dev)
    out["frames8_ms_per_frame"] = device_ms(
        lambda: fb.render2d_frames(shape, fb.RenderConfig2D(SIZE, SIZE), out=batch, asynchronous=True, world_to_model=views), 5) / 8
    del batch
    bear = model("bear.vm")
    img3 = torch.zeros((1024, 1024, 4), dtype=torch.float32, device=dev)
    cfg3 = fb.RenderConfig3D(1024, 1024, 1024)
    out["bear_1024_3d_ms"] = device_ms(lambda: fb.render3d(bear, cfg3, out=img3, asynchronous=True), 5)
    if args.atomics:
        with tempfile.TemporaryDirectory() as tmp:
            out["atomics"] = atomic_rate(tmp, torch.cuda.get_device_properties(0).multi_processor_count)
    print("RESULT " + json.dumps(out), flush=True)


def run_worker(lib, frames, atomics):
    env = dict(os.environ)
    env.pop("FIDGET_B200_LIB", None)
    if lib:
        env["FIDGET_B200_LIB"] = lib
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--frames", str(frames)] + (["--atomics"] if atomics else [])
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
    if r.returncode or not line:
        raise SystemExit(f"worker failed ({lib}):\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return json.loads(line[-1][7:])


def bench_line(tree, steps, warmup):
    env = dict(os.environ)
    env.pop("FIDGET_B200_LIB", None)
    r = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
                        str(warmup), "--no-cpu-baseline"], capture_output=True, text=True, env=env, cwd=tree)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode or not line:
        raise SystemExit(f"bench.py failed in {tree}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return json.loads(line[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="tree of the parent commit with its library built (./build.sh)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=30, help="timed frames per round and mode")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "levels2d_bench.jsonl"))
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--atomics", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    gpu = gpu_id()
    builds = ([("parent", os.path.abspath(args.parent))] if args.parent else []) + [("this", ROOT)]
    runs = {name: [] for name, _ in builds}
    bench = {name: [] for name, _ in builds}
    atomics = []
    for r in range(args.rounds):
        for name, tree in builds:   # alternate the builds
            lib = os.path.join(tree, "fidget_b200", "libfidget_cuda.so") if name == "parent" else None
            w = run_worker(lib, args.frames, atomics=(name == "this"))
            if "atomics" in w:
                atomics.append(w.pop("atomics"))
            runs[name].append(w)
            bench[name].append(bench_line(tree, args.steps, args.warmup))
            print(name, r, json.dumps(w["flushed"]), round(bench[name][-1]["value"], 1), flush=True)
    lines = []
    common = {"gpu (name, power limit, SM clock, max SM clock)": gpu, "rounds": args.rounds, "frames_per_round": args.frames}
    for mode in ("flushed", "unflushed"):
        rec = {"what": f"prospero 4096^2 stage ms, L2 {mode} before each frame; median of each round's median frame",
               **common, "census": runs["this"][0]["census"]}
        for name in runs:
            rec[name] = {st: _stats([w[mode][st] for w in runs[name]]) for st in STAGES}
        lines.append(rec)
    for key, what in (("frames8_ms_per_frame", "prospero 8 zoom views x 4096^2, fc_render2d_frames, device ms per frame"),
                      ("bear_1024_3d_ms", "bear 1024^3 fc_render3d, device ms")):
        lines.append({"what": what, **common, **{name: _stats([w[key] for w in runs[name]]) for name in runs}})
    vals = {name: [b["value"] for b in bench[name]] for name in bench}
    rec = {"what": "bench.py value (prospero 4096^2, Mvoxels/s)", **common, "steps": args.steps,
           **{name: [round(v, 1) for v in vals[name]] for name in vals},
           "ms_per_step": {name: _stats([b["ms_per_step"] for b in bench[name]]) for name in bench}}
    if args.parent:
        p, t = statistics.median(vals["parent"]), statistics.median(vals["this"])
        rec["parent_spread_pct"] = round(100 * (max(vals["parent"]) - min(vals["parent"])) / p, 2)
        rec["this_vs_parent_pct"] = round(100 * (t / p - 1), 2)
    lines.append(rec)
    lines.append({"what": "bench.py strong_scaling_base: prospero 4096^3 fc_render3d, ms", **common,
                  **{name: _stats([b["strong_scaling_base"]["ms_per_step"] for b in bench[name]]) for name in bench}})
    for a in atomics[:1]:
        a.update(common)
        a["ns_per_claim_one_word_rounds"] = [x["ns_per_claim_one_word"] for x in atomics]
        lines.append(a)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
            print(json.dumps(rec))


if __name__ == "__main__":
    main()
