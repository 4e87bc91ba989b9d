"""Times fc_mesh_build with and without cell collapse (FC_FLAG_MESH_COLLAPSE) and prints one JSON line per config.

    python scripts/bench_mesh.py [--iters 5] [--warmup 1]

Models: gyroid-sphere at depth 8 and 9, bear and colonnade at depth 8.  Times are the device times
fc_mesh_build measures with CUDA events: sampler_ms (the octree sampler) and mesh_ms (everything after it:
QEF vertices, and in collapse mode the cell tree, the collapse and the adaptive dual walk), the median over
--iters runs.  The L2 is flushed before every run by a 512 MiB fill, outside the timed regions.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [("gyroid-sphere.vm", 8), ("gyroid-sphere.vm", 9), ("bear.vm", 8), ("colonnade.vm", 8)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    import torch
    import fidget_b200 as fb

    cuda = fb.CudaContext(0)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda:0")
    for name, depth in CONFIGS:
        with open(os.path.join(ROOT, "models", name)) as f:
            shape = fb.CudaShape.from_vm(cuda, f.read())
        for collapse in (False, True):
            runs = []
            for i in range(args.warmup + args.iters):
                flush.fill_(i & 255)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                verts, tris, info = fb.mesh(shape, depth, collapse=collapse)
                wall = (time.perf_counter() - t0) * 1e3
                if i >= args.warmup:
                    runs.append((info["sampler_ms"], info["mesh_ms"], wall))
            s, m, w = (float(np.median([r[k] for r in runs])) for k in range(3))
            line = {"model": name, "depth": depth, "collapse": collapse, "sampler_ms": round(s, 3),
                    "mesh_ms": round(m, 3), "wall_ms": round(w, 3), "surface_leaves": int(info["n_leaves"]),
                    "final_leaves": int(len(fb.mesh_cells(cuda))) if collapse else int(info["n_leaves"]),
                    "vertices": int(info["n_vertices"]), "triangles": int(info["n_triangles"]),
                    "open_edges": int(info["open_edges"]), "iters": args.iters,
                    "device": torch.cuda.get_device_name(0)}
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
