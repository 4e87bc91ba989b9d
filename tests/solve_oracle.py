"""ctypes face of the solver's CPU oracle, ``oracle/libsolve_oracle.so`` (built by build.sh from oracle/solve.cc on
top of ``oracle/liboracle.so``): fc_solve_batch restated operation for operation, and its Jacobi pseudo-inverse.
Test infrastructure; takes ``oracle.oracle.Tape`` handles."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
SOLVE_RESULT = np.dtype([("status", np.uint32), ("iterations", np.uint32), ("err", np.float32), ("pad", np.uint32)])
_LIB = None


def _build(out):
    """build.sh's recipe, for a tree where only liboracle.so was built"""
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                           "-shared", "-o", out, os.path.join(ORACLE_DIR, "solve.cc"), "-L" + ORACLE_DIR,
                           "-l:liboracle.so", "-Wl,-rpath," + ORACLE_DIR])


def lib() -> C.CDLL:
    global _LIB
    if _LIB is not None:
        return _LIB
    orc.lib()   # liboracle.so first: the solver shares its tapes
    path = os.path.join(ORACLE_DIR, "libsolve_oracle.so")
    if not os.path.exists(path):
        path = os.path.join(tempfile.mkdtemp(prefix="solve_oracle_"), "libsolve_oracle.so")
        _build(path)
    L = C.CDLL(path)
    vp, u32, i32, P = C.c_void_p, C.c_uint32, C.c_int32, C.POINTER
    fp = P(C.c_float)
    L.orc_solve_last_error.restype = C.c_char_p
    L.orc_solve_batch.argtypes = [P(vp), u32, P(P(i32)), u32, u32, u32, fp, C.c_uint64, vp]
    L.orc_solve_batch.restype = i32
    L.orc_sym_pinv_apply.argtypes = [u32, fp, fp, fp]
    L.orc_sym_pinv_apply.restype = None
    _LIB = L
    return L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def solve_batch(tapes, slot_params, n_free, values, max_iters=0):
    """fc_solve_batch on the CPU.  tapes: oracle Tapes; slot_params[k]: parameter index of each input slot of
    tapes[k]; values: [n_problems, n_params] (free parameters first).  Returns (values, results)."""
    vals = np.array(values, dtype=np.float32, order="C", copy=True)
    if vals.ndim == 1:
        vals = vals[None, :]
    n_problems, n_params = vals.shape
    m = len(tapes)
    sps = [np.ascontiguousarray(s, dtype=np.int32) for s in slot_params]
    th = (C.c_void_p * max(m, 1))(*[t._h for t in tapes])
    sp = (C.POINTER(C.c_int32) * max(m, 1))(*[s.ctypes.data_as(C.POINTER(C.c_int32)) for s in sps])
    res = np.zeros(n_problems, dtype=SOLVE_RESULT)
    L = lib()
    if L.orc_solve_batch(th, m, sp, n_params, n_free, max_iters, _fp(vals), n_problems,
                         res.ctypes.data_as(C.c_void_p)) != 0:
        raise RuntimeError(L.orc_solve_last_error().decode())
    return vals, res


def sym_pinv_apply(a, b):
    """pinv(a) @ b for a symmetric float32 matrix, through the solver's Jacobi eigen-solve."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    out = np.zeros(len(b), dtype=np.float32)
    lib().orc_sym_pinv_apply(len(b), _fp(a), _fp(b), _fp(out))
    return out
