"""Test infrastructure for fc_volume_build: the CPU mirror of its descent and the checks every volume must pass.

``oracle_volume`` runs tests/csrc/volume_oracle.cc (compiled here once per process, on the oracle's evaluators) and
returns its bricks, values, gradients and tiles in fc_volume_build's canonical order, in the layout of ``fb.volume``
(bricks [n, 4] (frame, ix, iy, iz), values [n, B, B, B] indexed [z, y, x], tiles [m, 6] (frame, ix, iy, iz, log2_edge,
inside)).  ``check_volume`` checks one frame of a volume against the root tape's value at every cell centre: the
partition, completeness within the band, the tiles' signs and the brick values."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from measure_ref import centres
from contour_oracle import xform_f32

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_VO = None


def _volume_lib(orc):
    """tests/csrc/volume_oracle.cc as a shared library in a temporary directory, linked against liboracle.so"""
    global _VO
    if _VO is None:
        orc.lib()
        odir = os.path.join(ROOT, "oracle")
        out = os.path.join(tempfile.mkdtemp(prefix="volume_oracle_"), "libvolume_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([cxx, "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared",
                        "-I", odir, "-o", out, os.path.join(ROOT, "tests", "csrc", "volume_oracle.cc"),
                        "-L", odir, "-l:liboracle.so", "-Wl,-rpath," + odir], check=True, capture_output=True)
        L = C.CDLL(out)
        L.vo_build.argtypes = [C.c_void_p, C.c_uint32, C.c_float, C.POINTER(C.c_float), C.c_uint32]
        L.vo_build.restype = C.c_void_p
        L.vo_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.vo_counts.restype = None
        L.vo_read.argtypes = [C.c_void_p] + [C.c_void_p] * 4
        L.vo_read.restype = None
        L.vo_free.argtypes = [C.c_void_p]
        L.vo_free.restype = None
        _VO = L
    return _VO


def canonical(bricks, tiles):
    """The orders that sort bricks [n, 4] and tiles [m, 6] by (frame, iz, iy, ix)"""
    ob = np.lexsort((bricks[:, 1], bricks[:, 2], bricks[:, 3], bricks[:, 0])) if len(bricks) else np.zeros(0, np.int64)
    ot = np.lexsort((tiles[:, 1], tiles[:, 2], tiles[:, 3], tiles[:, 0])) if len(tiles) else np.zeros(0, np.int64)
    return ob, ot


def oracle_volume(orc, tape, depth, band=0.0, world_to_model=None, grads=False, frame=0):
    """fc_volume_build's output for one frame by the same descent on the CPU, for an oracle.Tape: a dict of bricks,
    values, grads (or None) and tiles, in canonical order, frame numbers set to ``frame``"""
    L = _volume_lib(orc)
    m = None
    if world_to_model is not None:
        mm = np.ascontiguousarray(world_to_model, dtype=f32).reshape(16)
        m = mm.ctypes.data_as(C.POINTER(C.c_float))
    h = L.vo_build(tape._h, depth, f32(band), m, int(grads))
    assert h
    try:
        nb, nt = C.c_uint64(), C.c_uint64()
        L.vo_counts(h, C.byref(nb), C.byref(nt))
        nb, nt = nb.value, nt.value
        B = 1 << min(depth, 3)
        b = np.zeros((nb, 3), dtype=np.uint32)
        v = np.zeros((nb, B, B, B), dtype=f32)
        g = np.zeros((nb, B, B, B, 3), dtype=f32) if grads else None
        t = np.zeros((nt, 5), dtype=np.uint32)
        L.vo_read(h, b.ctypes.data, v.ctypes.data, g.ctypes.data if grads else None, t.ctypes.data)
    finally:
        L.vo_free(h)
    bricks = np.concatenate([np.full((nb, 1), frame, np.int32), b.astype(np.int32)], 1)
    tiles = np.concatenate([np.full((nt, 1), frame, np.int32), t.astype(np.int32)], 1)
    ob, ot = canonical(bricks, tiles)
    return {"bricks": bricks[ob], "values": v[ob], "grads": None if g is None else g[ob], "tiles": tiles[ot]}


def root_values(evaluate, axes, n_vars, depth, world_to_model=None, var_values=()):
    """[2^D, 2^D, 2^D] f32 ([z, y, x]): the root tape at every mapped cell centre.  evaluate(list of n_vars f32
    arrays) -> values; axes: the tape's (x, y, z) input slots."""
    n = 1 << depth
    out = np.empty((n, n, n), dtype=f32)
    slab = max(1, (1 << 21) // (n * n))
    for k0 in range(0, n, slab):
        k1 = min(n, k0 + slab)
        x, y, z = (a.ravel() for a in centres(depth, k0, k1))
        if world_to_model is not None:
            x, y, z = xform_f32(np.asarray(world_to_model, dtype=f32), x, y, z)
        ins = [x if s == axes[0] else y if s == axes[1] else z if s == axes[2]
               else np.full_like(x, f32(var_values[s] if s < len(var_values) else 0)) for s in range(n_vars)]
        out[k0:k1] = np.asarray(evaluate(ins), dtype=f32).reshape(k1 - k0, n, n)
    return out


def check_volume(bricks, values, tiles, depth, band, v, frame=0, exact_values=True):
    """One frame of a volume (numpy, canonical order) against the root values v [z, y, x] of every cell centre:
    bricks and tiles partition the cube, sit on their own grids and are sorted; |v| <= band only in bricks; inside
    tiles hold v < -band and outside tiles v > band; brick values equal v (bit for bit with exact_values).  Returns
    the number of brick values that differ from v."""
    n, B = 1 << depth, 1 << min(depth, 3)
    b = bricks[bricks[:, 0] == frame]
    vals = values[bricks[:, 0] == frame]
    t = tiles[tiles[:, 0] == frame]
    for rows, key in ((b, b[:, [3, 2, 1]]), (t, t[:, [3, 2, 1]])):
        if len(rows) > 1:
            k = (key[:, 0].astype(np.int64) << 24) | (key[:, 1].astype(np.int64) << 12) | key[:, 2]
            assert np.all(np.diff(k) > 0), "not in canonical order"
    cover = np.zeros((n, n, n), dtype=np.uint8)
    in_brick = np.zeros((n, n, n), dtype=bool)
    dense = np.full((n, n, n), np.nan, dtype=f32)
    for _, ix, iy, iz in b.tolist():
        assert ix % B == 0 and iy % B == 0 and iz % B == 0
        cover[iz:iz + B, iy:iy + B, ix:ix + B] += 1
        in_brick[iz:iz + B, iy:iy + B, ix:ix + B] = True
    for r, (_, ix, iy, iz) in enumerate(b.tolist()):
        dense[iz:iz + B, iy:iy + B, ix:ix + B] = vals[r]
    for _, ix, iy, iz, lg, ins in t.tolist():
        e = 1 << lg
        assert e >= B and ix % e == 0 and iy % e == 0 and iz % e == 0
        cover[iz:iz + e, iy:iy + e, ix:ix + e] += 1
        block = v[iz:iz + e, iy:iy + e, ix:ix + e]
        if ins:
            assert np.all(block < -band), ("inside tile", ix, iy, iz, lg)
        else:
            assert np.all(block > band), ("outside tile", ix, iy, iz, lg)
    assert np.all(cover == 1), "bricks and tiles do not partition the cube"
    assert np.all(in_brick[np.abs(v) <= band]), "a centre within the band is outside every brick"
    same = (dense.view(np.uint32) == v.view(np.uint32))[in_brick]
    if exact_values:
        assert same.all(), "brick values differ from the root tape's"
    return int((~same).sum())
