"""SURVEY 8(d) API micro-bench: fc_float_slice_eval / fc_grad_slice_eval on device-resident SoA inputs,
n = 2^24 points, x, y, z ~ U[-1, 1] (numpy.random.default_rng(0)).  Algorithmic bytes: 16 B per point for
f32 (12 read + 4 written), 64 B per point for gradients (3 x 16 read + 16 written).  Prints one JSON line
per (tape, evaluator, path): the TMA-fed persistent kernel (bulk.cu) and, with FIDGET_B200_NO_TMA=1, the
per-thread kernel it replaces.  Results of the two paths are compared bit for bit.

  python scripts/bench_slices.py [log2_n]
"""
import json, os, sys
os.environ.setdefault("FIDGET_B200_ENV_LIVE", "1")   # the two paths are selected by an environment knob per call
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import fidget_b200 as fb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK = 3350.0   # H100 SXM data sheet (HBM3), unless a measured copy bandwidth is supplied
if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")):
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs", PEAK)


def csg_tape():
    """A 25-clause IEEE-only tape: two spheres, a box, union / intersection (no libm)."""
    ctx = fb.Context()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    s1 = ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), 0.6)
    xs = ctx.sub(x, 0.3)
    s2 = ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(xs), ctx.square(y)), ctx.square(z))), 0.4)
    box = ctx.max(ctx.max(ctx.sub(ctx.abs(x), 0.5), ctx.sub(ctx.abs(y), 0.45)), ctx.sub(ctx.abs(z), 0.4))
    return ctx.tape(ctx.max(ctx.min(s1, s2), ctx.neg(box)))


def main():
    lg = int(sys.argv[1]) if len(sys.argv) > 1 else 24
    n = 1 << lg
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
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    tapes = {"csg25 (IEEE only)": csg_tape()}
    for name in ("gyroid-sphere.vm", "prospero.vm"):
        ctx, root = fb.Context.from_text(open(os.path.join(ROOT, "models", name)).read())
        tapes[name] = ctx.tape(root)
    for name, td in tapes.items():
        shape = fb.CudaShape(cuda, td)
        nv = shape.n_vars
        reps = 3 if name == "prospero.vm" else 10
        for kind in ("f32", "grad"):
            ins = (xyz if kind == "f32" else grads)[:nv]
            out = torch.empty(n if kind == "f32" else (n, 4), dtype=torch.float32, device=dev)
            results = {}
            for path in ("tma", "per-thread"):
                os.environ["FIDGET_B200_NO_TMA"] = "0" if path == "tma" else "1"
                fn = shape.float_slice_eval if kind == "f32" else shape.grad_slice_eval
                for _ in range(2):
                    fn(ins, out=out)
                ms = []
                for _ in range(reps):
                    flush.fill_(1)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    fn(ins, out=out)
                    e1.record(stream)
                    torch.cuda.synchronize()
                    ms.append(e0.elapsed_time(e1))
                t = float(np.median(ms))
                bytes_pt = (4 * nv + 4) if kind == "f32" else (16 * nv + 16)
                results[path] = out.clone()
                print(json.dumps({"tape": name, "clauses": len(td), "regs": int(shape.info.reg_count), "evaluator": kind, "path": path,
                                  "n": n, "ms": t, "Mpoints_per_s": n / t / 1e3, "algorithmic_bytes_per_point": bytes_pt,
                                  "GB_per_s": n * bytes_pt / t / 1e6, "frac_of_measured_hbm": n * bytes_pt / t / 1e6 / PEAK}), flush=True)
            same = torch.equal(results["tma"].view(torch.int32), results["per-thread"].view(torch.int32))
            print(json.dumps({"tape": name, "evaluator": kind, "tma_equals_per_thread_bitwise": bool(same)}), flush=True)
    os.environ["FIDGET_B200_NO_TMA"] = "0"


if __name__ == "__main__":
    main()
