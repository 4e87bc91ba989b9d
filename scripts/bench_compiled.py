"""Compiled tapes (fc_tape_compile) against the interpreters on the bulk evaluators: n = 2^24 device-resident points
(x, y, z ~ U[-1, 1], numpy.random.default_rng(0)) for the float and gradient kinds, 2^20 boxes for intervals.  The
interpreter side is whatever fc_float_slice_eval / fc_grad_slice_eval pick today (the TMA-fed kernel or the per-thread
one) and fc_interval_eval_batch.  Device time of each call from CUDA events, median of 5 after two warm-up calls, L2
flushed before each (as bench_slices.py).  Algorithmic bytes per point: 4 per input and output for f32, 16 for
gradients, 8 per box input and output plus one choice byte per choice clause and the simplify byte for intervals; their
rate is given as a fraction of the H100 SXM data sheet's 3.35 TB/s.  Each line says whether the compiled and the
interpreted outputs of the timed calls are equal bit for bit, and how many points repay the compile at that rate.
Writes profiles/compiled_bench.jsonl (or the path given).

  python scripts/bench_compiled.py [out.jsonl] [log2_n]
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import fidget_b200 as fb
from scripts.bench_slices import csg_tape

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0
MODELS = ("hi.vm", "quarter.vm", "colonnade.vm", "bear.vm", "gyroid-sphere.vm", "prospero.vm")
REPS, WARMUP = 5, 2


def machine():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def timed(fn, stream, flush):
    for _ in range(WARMUP):
        fn()
    ms = []
    for _ in range(REPS):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "compiled_bench.jsonl")
    lg = int(sys.argv[2]) if len(sys.argv) > 2 else 24
    n, nb = 1 << lg, 1 << (lg - 4)
    dev = torch.device("cuda", 0)
    cuda = fb.CudaContext(0)
    stream = torch.cuda.current_stream()
    cuda.set_stream(stream.cuda_stream)
    rng = np.random.default_rng(0)
    xyz = [torch.from_numpy(rng.uniform(-1, 1, n).astype(np.float32)).to(dev) for _ in range(3)]
    grads = []
    for k in range(3):
        g = torch.zeros((n, 4), dtype=torch.float32, device=dev)
        g[:, 0] = xyz[k]
        g[:, 1 + k] = 1.0
        grads.append(g)
    c = rng.uniform(-1, 1, (nb, 3, 1)).astype(np.float32)
    w = (rng.uniform(0, 1, (nb, 3, 1)) ** 3).astype(np.float32)
    boxes = torch.from_numpy(np.concatenate([c - w, c + w], -1)).to(dev)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    mach = machine()
    tapes = {"csg25": csg_tape()}
    for name in MODELS:
        ctx, root = fb.Context.from_text(open(os.path.join(ROOT, "models", name)).read())
        tapes[name] = ctx.tape(root)
    lines = []
    for name, td in tapes.items():
        shape = fb.CudaShape(cuda, td)
        comp = shape.compile()
        info = comp.info
        nv, nch = shape.n_vars, shape.choice_count
        for k, kind in enumerate(("float", "grad", "interval")):
            if kind == "interval":
                count = nb
                ins = boxes[:, :nv].contiguous()
                bytes_pt = 8 * nv + 8 + nch + 1
                outs = {}
                for side, fn in (("interpreted", shape._lib.fc_interval_eval_batch), ("compiled", comp._lib.fc_compiled_interval_eval_batch)):
                    o = torch.empty((nb, 1, 2), dtype=torch.float32, device=dev)
                    ch = torch.empty((nb, max(nch, 1)), dtype=torch.uint8, device=dev)
                    si = torch.empty(nb, dtype=torch.uint8, device=dev)
                    h = shape._h if side == "interpreted" else comp._h
                    call = (lambda fn=fn, h=h, o=o, ch=ch, si=si:
                            fb.shape._ck(fn(shape._ev(), h, fb.shape._ptr(ins), nb, fb.shape._ptr(o), fb.shape._ptr(ch),
                                            fb.shape._ptr(si))))
                    outs[side] = (timed(call, stream, flush), (o, ch, si))
                same = all(torch.equal(a.view(torch.uint8), b.view(torch.uint8))
                           for a, b in zip(outs["interpreted"][1], outs["compiled"][1]))
            else:
                count = n
                ins = (xyz if kind == "float" else grads)[:nv]
                bytes_pt = (4 * nv + 4) if kind == "float" else (16 * nv + 16)
                outs = {}
                for side, obj in (("interpreted", shape), ("compiled", comp)):
                    o = torch.empty(n if kind == "float" else (n, 4), dtype=torch.float32, device=dev)
                    fn = obj.float_slice_eval if kind == "float" else obj.grad_slice_eval
                    outs[side] = (timed(lambda fn=fn, o=o: fn(ins, out=o), stream, flush), (o,))
                same = torch.equal(outs["interpreted"][1][0].view(torch.int32), outs["compiled"][1][0].view(torch.int32))
            ti, tc = outs["interpreted"][0], outs["compiled"][0]
            saved_ms_per_point = (ti - tc) / count
            line = {"tape": name, "clauses": len(td), "vm_regs": int(shape.info.reg_count), "kind": kind, "n": count,
                    "interpreted_ms": ti, "compiled_ms": tc, "speedup": ti / tc,
                    "compile_ms": info["compile_ms"][k], "regs": info["regs"][k], "local_bytes": info["local_bytes"][k],
                    "nvrtc_version": info["nvrtc_version"], "algorithmic_bytes_per_point": bytes_pt,
                    "interpreted_frac_of_3.35TBps": count * bytes_pt / ti / 1e6 / HBM_GBS,
                    "compiled_frac_of_3.35TBps": count * bytes_pt / tc / 1e6 / HBM_GBS,
                    "break_even_points": (info["compile_ms"][k] / saved_ms_per_point) if saved_ms_per_point > 0 else None,
                    "bitwise_equal": bool(same), **mach}
            print(json.dumps(line), flush=True)
            lines.append(line)
        comp.close()
        shape.close()
    with open(out_path, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
