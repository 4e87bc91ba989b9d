"""Test infrastructure for fc_measure: the cell-centre brute force and the exact derived results.

``centres`` gives the f32 world centres -1 + (2i + 1) 2^-D of one Z range of depth-D cells, ``inside_mask`` classifies
them with any float evaluator after the f32 transform of dev_ops.cuh (``contour_oracle.xform_f32``), and
``brute_sums`` turns the masks into fc_measure's integers with Python ints.  ``derive_exact`` recomputes the float64
results from the integers in exact rational arithmetic (``fractions.Fraction``) and an exact affine map, for comparing
against what the host derives in float64.  ``oracle_measure`` is the CPU mirror of fc_measure's descent
(tests/csrc/measure_oracle.cc, on the oracle's evaluators), compiled here once per process."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from fractions import Fraction

import numpy as np

from contour_oracle import xform_f32

f32 = np.float32
INTS = ("n_inside", "n_proven", "n_undecided", "s1", "s2", "lo", "hi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_MO = None


def _measure_lib(orc):
    """tests/csrc/measure_oracle.cc as a shared library in a temporary directory, linked against liboracle.so"""
    global _MO
    if _MO is None:
        orc.lib()   # (liboracle.so built and loaded: the library below resolves its evaluators there)
        odir = os.path.join(ROOT, "oracle")
        out = os.path.join(tempfile.mkdtemp(prefix="measure_oracle_"), "libmeasure_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([cxx, "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared",
                        "-I", odir, "-o", out, os.path.join(ROOT, "tests", "csrc", "measure_oracle.cc"),
                        "-L", odir, "-l:liboracle.so", "-Wl,-rpath," + odir], check=True, capture_output=True)
        L = C.CDLL(out)
        L.mo_measure.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_uint64),
                                 C.POINTER(C.c_uint32)]
        L.mo_measure.restype = C.c_int32
        L.mo_block.argtypes = [C.c_uint32] * 4 + [C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.mo_block.restype = None
        _MO = L
    return _MO


def _ints_dict(out, box):
    o = [int(v) for v in out]
    b = [int(v) for v in box]
    return {"n_inside": o[0], "n_proven": o[1], "n_undecided": o[2], "s1": o[3:6], "s2": o[6:12], "lo": b[0:3],
            "hi": b[3:6]}


def oracle_measure(orc, tape, depth, world_to_model=None):
    """fc_measure's integers by the same descent on the CPU, for an oracle.Tape: a dict of n_inside, n_proven,
    n_undecided, s1 [3], s2 [6], lo [3], hi [3] (Python ints)"""
    L = _measure_lib(orc)
    m = None
    if world_to_model is not None:
        mm = np.ascontiguousarray(world_to_model, dtype=f32).reshape(16)
        m = mm.ctypes.data_as(C.POINTER(C.c_float))
    out, box = (C.c_uint64 * 12)(), (C.c_uint32 * 6)()
    assert L.mo_measure(tape._h, depth, m, out, box) == 0
    return _ints_dict(out, box)


def oracle_block(orc, x0, y0, z0, T):
    """The closed-form sums of the block of T^3 depth-D cells at (x0, y0, z0), as ``oracle_measure`` returns them"""
    out, box = (C.c_uint64 * 12)(), (C.c_uint32 * 6)()
    _measure_lib(orc).mo_block(x0, y0, z0, T, out, box)
    return _ints_dict(out, box)


def empty_sums():
    return {"n_inside": 0, "s1": [0, 0, 0], "s2": [0] * 6, "lo": [0xFFFFFFFF] * 3, "hi": [0] * 3}


def centres(depth, k0, k1):
    """f32 world coordinates (x, y, z) of the cells with k0 <= k < k1, as [k, j, i] arrays."""
    n = 1 << depth
    inv = f32(1) / f32(n)
    c = ((2 * np.arange(n) + 1).astype(f32) * inv - f32(1)).astype(f32)
    z, y, x = np.meshgrid(c[k0:k1], c, c, indexing="ij")
    return x, y, z


def inside_mask(evaluate, axes, n_vars, depth, k0, k1, world_to_model=None, var_values=()):
    """[k1 - k0, 2^D, 2^D] bool: the value at each cell centre is < 0.  evaluate(list of n_vars f32 arrays) -> values;
    axes: the tape's (x, y, z) input slots."""
    x, y, z = centres(depth, k0, k1)
    shape = x.shape
    x, y, z = x.ravel(), y.ravel(), z.ravel()
    if world_to_model is not None:
        x, y, z = xform_f32(np.asarray(world_to_model, dtype=f32), x, y, z)
    ins = []
    for s in range(n_vars):
        ins.append(x if s == axes[0] else y if s == axes[1] else z if s == axes[2]
                   else np.full_like(x, f32(var_values[s] if s < len(var_values) else 0)))
    return (np.asarray(evaluate(ins)) < 0).reshape(shape)


def add_mask(sums, mask, k0):
    """Adds the inside cells of mask [k, j, i] (k offset by k0) to sums (Python ints throughout)."""
    if not mask.any():
        return sums
    n = mask.shape[1]
    odd = 2 * np.arange(n, dtype=np.int64) + 1
    w = 2 * np.arange(k0, k0 + mask.shape[0], dtype=np.int64) + 1
    m = mask.astype(np.int64)
    cx, cy, cz = m.sum(axis=(0, 1)), m.sum(axis=(0, 2)), m.sum(axis=(1, 2))   # cells per i, per j, per k
    myx, mzx, mzy = m.sum(axis=0), m.sum(axis=1), m.sum(axis=2)               # [j, i], [k, i], [k, j]
    py = lambda v: int(v)   # noqa: E731
    sums["n_inside"] += py(m.sum())
    sums["s1"] = [sums["s1"][0] + py(cx @ odd), sums["s1"][1] + py(cy @ odd), sums["s1"][2] + py(cz @ w)]
    add = [py(cx @ (odd * odd)), py(cy @ (odd * odd)), py(cz @ (w * w)),
           sum(int(v) for v in (odd @ myx) * odd),   # Σuv: rows j weighted by v, then columns i by u
           sum(int(v) for v in (w @ mzx) * odd),
           sum(int(v) for v in (w @ mzy) * odd)]
    sums["s2"] = [a + b for a, b in zip(sums["s2"], add)]
    for a, c, base in ((0, cx, 0), (1, cy, 0), (2, cz, k0)):
        nz = np.nonzero(c)[0]
        sums["lo"][a] = min(sums["lo"][a], int(nz[0]) + base)
        sums["hi"][a] = max(sums["hi"][a], int(nz[-1]) + base)
    return sums


def brute_sums(evaluate, axes, n_vars, depth, world_to_model=None, var_values=(), slab=None):
    """fc_measure's n_inside, s1, s2, lo, hi over every cell centre, Z slab by slab."""
    n = 1 << depth
    slab = slab or max(1, (1 << 21) // (n * n))
    sums = empty_sums()
    for k0 in range(0, n, slab):
        k1 = min(n, k0 + slab)
        add_mask(sums, inside_mask(evaluate, axes, n_vars, depth, k0, k1, world_to_model, var_values), k0)
    return sums


def ints_of(row):
    """The integer fields of a MEASURE_RESULT row (or an oracle dict) as Python ints and lists."""
    out = {}
    for k in INTS:
        v = row[k]
        out[k] = [int(x) for x in v] if np.ndim(v) else int(v)
    return out


def derive_exact(ints, depth, world_to_model=None):
    """The derived results of fidget_cuda.h, exactly: volume, volume_lo, volume_hi, centroid [3], inertia [6],
    bbox_min [3], bbox_max [3] as Fractions (None for the NaN fields of an empty frame).  The matrix entries are the f32
    values the call takes, read exactly."""
    A = [[Fraction(int(i == j)) for j in range(3)] for i in range(3)]
    t = [Fraction(0)] * 3
    if world_to_model is not None:
        m = np.asarray(world_to_model, dtype=f32).reshape(4, 4)
        A = [[Fraction(float(m[i, j])) for j in range(3)] for i in range(3)]
        t = [Fraction(float(m[i, 3])) for i in range(3)]
    det = (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])
           + A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]))
    h = Fraction(2, 1 << depth)
    N = ints["n_inside"]
    out = {"volume_lo": ints["n_proven"] * h ** 3 * abs(det),
           "volume_hi": (ints["n_proven"] + ints["n_undecided"]) * h ** 3 * abs(det)}
    if N == 0:
        out.update(volume=Fraction(0), centroid=None, inertia=None, bbox_min=None, bbox_max=None)
        return out
    vol = N * h ** 3 * abs(det)
    s1, s2 = ints["s1"], ints["s2"]
    c = [Fraction(s1[a], N << depth) - 1 for a in range(3)]
    pairs = ((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2))
    C = [[Fraction(0)] * 3 for _ in range(3)]
    for k, (p, q) in enumerate(pairs):
        C[p][q] = C[q][p] = Fraction(N * s2[k] - s1[p] * s1[q], N * N * 4 ** depth)
    for a in range(3):
        C[a][a] += h * h / 12
    cm = [t[i] + sum(A[i][j] * c[j] for j in range(3)) for i in range(3)]
    Cm = [[sum(A[i][p] * C[p][q] * A[j][q] for p in range(3) for q in range(3)) for j in range(3)] for i in range(3)]
    tr = Cm[0][0] + Cm[1][1] + Cm[2][2]
    inertia = [vol * ((tr if p == q else 0) - Cm[p][q]) for p, q in pairs]
    lo = [ints["lo"][a] * h - 1 for a in range(3)]
    hi = [(ints["hi"][a] + 1) * h - 1 for a in range(3)]
    corners = [[(hi if (k >> a) & 1 else lo)[a] for a in range(3)] for k in range(8)]
    mapped = [[t[i] + sum(A[i][j] * p[j] for j in range(3)) for i in range(3)] for p in corners]
    out.update(volume=vol, centroid=cm, inertia=inertia,
               bbox_min=[min(p[i] for p in mapped) for i in range(3)],
               bbox_max=[max(p[i] for p in mapped) for i in range(3)])
    return out
