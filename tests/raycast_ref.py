"""Test infrastructure for fc_raycast: the CPU mirror of its descent and the ray families the tests cast.

``oracle_raycast`` runs tests/csrc/raycast_oracle.cc (on the oracle's interval, simplify, float and gradient
evaluators, compiled here once per process) and returns hits in fc_ray_hit's layout (``fidget_b200.RAY_HIT``).
``sample_points`` gives the f32 samples of a ray as the contract defines them, for brute force.  ``ray_families`` builds
the seeded rays: through the cube and missing it, axis-aligned and grazing, starting inside, zero-direction."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from fidget_b200.shape import RAY, RAY_HIT

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_RO = None


def _raycast_lib(orc):
    """tests/csrc/raycast_oracle.cc as a shared library in a temporary directory, linked against liboracle.so"""
    global _RO
    if _RO is None:
        orc.lib()   # (liboracle.so built and loaded: the library below resolves its evaluators there)
        odir = os.path.join(ROOT, "oracle")
        out = os.path.join(tempfile.mkdtemp(prefix="raycast_oracle_"), "libraycast_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([cxx, "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared",
                        "-I", odir, "-o", out, os.path.join(ROOT, "tests", "csrc", "raycast_oracle.cc"),
                        "-L", odir, "-l:liboracle.so", "-Wl,-rpath," + odir], check=True, capture_output=True)
        L = C.CDLL(out)
        L.ro_raycast.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                 C.POINTER(C.c_uint64)]
        L.ro_raycast.restype = C.c_int32
        L.ro_levels.argtypes = [C.c_uint32]
        L.ro_levels.restype = C.c_uint32
        _RO = L
    return _RO


def levels(orc, steps):
    """L of the descent for ``steps`` samples, as the oracle computes it"""
    return int(_raycast_lib(orc).ro_levels(steps))


def make_rays(origins, dirs, t0, dt):
    n = len(origins)
    rays = np.zeros(n, dtype=RAY)
    rays["origin"] = np.asarray(origins, dtype=f32).reshape(n, 3)
    rays["dir"] = np.asarray(dirs, dtype=f32).reshape(n, 3)
    rays["t0"] = np.broadcast_to(np.asarray(t0, dtype=f32).reshape(-1), (n,))
    rays["dt"] = np.broadcast_to(np.asarray(dt, dtype=f32).reshape(-1), (n,))
    return rays


def oracle_raycast(orc, tape, rays, steps, var_values=()):
    """The hits of ``rays`` (a ``RAY`` array) by the CPU descent: a ``RAY_HIT`` array, and the stats dict (segments
    evaluated per level, leaf samples) of the oracle's walk"""
    L = _raycast_lib(orc)
    rays = np.ascontiguousarray(rays)
    hits = np.zeros(len(rays), dtype=RAY_HIT)
    vals = np.ascontiguousarray(np.asarray(var_values, dtype=f32).reshape(-1)) if len(var_values) else np.zeros(1, f32)
    stats = (C.c_uint64 * 9)()
    assert L.ro_raycast(tape._h, rays.ctypes.data, len(rays), steps, vals.ctypes.data, len(var_values),
                        hits.ctypes.data, stats) == 0
    return hits, {"evaluated": list(stats)[:8], "leaf_samples": int(stats[8])}


def sample_points(rays, steps):
    """[n, steps] f32 arrays (t, x, y, z) of every sample: t_k = t0 + k dt, x_k = origin + t_k dir, one rounding per
    operation"""
    k = np.arange(steps, dtype=f32)
    t = (rays["t0"][:, None] + (k[None, :] * rays["dt"][:, None]).astype(f32)).astype(f32)
    xyz = [(rays["origin"][:, a][:, None] + (t * rays["dir"][:, a][:, None]).astype(f32)).astype(f32) for a in range(3)]
    return t, xyz[0], xyz[1], xyz[2]


def first_inside(values):
    """Per row of [n, steps] values: the first index with value < 0, FC_RAY_MISS if none"""
    ins = np.asarray(values) < 0
    k = np.argmax(ins, axis=1).astype(np.uint32)
    return np.where(ins.any(axis=1), k, np.uint32(0xFFFFFFFF))


def ray_families(seed, steps, n=64):
    """Seeded rays of every family, each covering about 3 units of t over ``steps`` samples: ``{name: RAY array}``"""
    rng = np.random.default_rng(seed)
    span = f32(3.0)
    dt = f32(span / f32(max(steps - 1, 1)))

    def unit(v):
        v = np.asarray(v, dtype=np.float64)
        return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(f32)

    fam = {}
    # through the cube: start outside, aim at a random point inside
    o = unit(rng.normal(size=(n, 3))) * f32(1.5)
    target = rng.uniform(-0.6, 0.6, size=(n, 3)).astype(f32)
    fam["through"] = make_rays(o, unit(target - o), 0.0, dt)
    # missing the cube: start outside, aim away from it
    fam["miss"] = make_rays(o, unit(o + rng.normal(scale=0.1, size=(n, 3))), 0.0, dt)
    # axis-aligned: along +-X, +-Y, +-Z from a face
    ax = rng.integers(0, 3, size=n)
    sg = rng.choice([-1.0, 1.0], size=n)
    d = np.zeros((n, 3), dtype=f32)
    d[np.arange(n), ax] = sg
    o = rng.uniform(-0.9, 0.9, size=(n, 3)).astype(f32)
    o[np.arange(n), ax] = -sg * 1.5
    fam["axis"] = make_rays(o, d, 0.0, dt)
    # grazing: tangent-ish to a sphere of radius 0.5..1 around the origin
    p = unit(rng.normal(size=(n, 3))) * rng.uniform(0.5, 1.0, size=(n, 1)).astype(f32)
    tang = unit(np.cross(p, rng.normal(size=(n, 3))))
    fam["grazing"] = make_rays(p - tang * f32(1.5), tang, 0.0, dt)
    # starting inside the cube (maybe inside the shape), and offset t0
    fam["inside"] = make_rays(rng.uniform(-0.3, 0.3, size=(n, 3)).astype(f32), unit(rng.normal(size=(n, 3))),
                              rng.uniform(-0.2, 0.2, size=n).astype(f32), dt)
    # zero direction: every sample is the origin
    fam["zero_dir"] = make_rays(rng.uniform(-1, 1, size=(n, 3)).astype(f32), np.zeros((n, 3), dtype=f32), 0.0, dt)
    return fam
