"""The host side of fb.mesh_frames: the fc_mesh_frame / fc_mesh_frame_info layouts, the frame table (per-frame
arguments, their lengths, the var limit, the has_transform flag) and the split of a batch's read buffers and STL into
per-frame outputs.  No GPU needed."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_struct(name):
    """(type, field, array length) of a struct of include/fidget_cuda.h, in order"""
    text = open(os.path.join(ROOT, "include", "fidget_cuda.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype, names = decl.split(None, 1)
        for n in names.split(","):
            m = re.match(r"\s*(\w+)(?:\[(\w+)\])?", n)
            out.append((ctype, m.group(1), m.group(2)))
    return out


SIZES = {"uint32_t": 4, "uint64_t": 8, "float": 4}


@pytest.mark.parametrize("name,cls", [("fc_mesh_frame", "FcMeshFrame"), ("fc_mesh_frame_info", "FcMeshFrameInfo")])
def test_structs_match_the_header(name, cls):
    """Sizes and offsets of the ctypes mirrors against a C layout of the header's declaration"""
    st = getattr(_lib, cls)
    off = 0
    fields = _header_struct(name)
    assert [f for f, _ in st._fields_] == [n for _, n, _ in fields]
    for ctype, n, count in fields:
        size = SIZES[ctype]
        off = (off + size - 1) // size * size
        assert getattr(st, n).offset == off, n
        k = 1 if count is None else (getattr(_lib, count) if not count.isdigit() else int(count))
        assert getattr(st, n).size == size * k, n
        off += size * k
    assert C.sizeof(st) == off
    assert C.sizeof(_lib.FcMeshFrame) == 4 + 16 * 4 + 4 + 16 * 4
    assert C.sizeof(_lib.FcMeshFrameInfo) == 5 * 8
    assert "fc_mesh_build_frames" in _lib.CUDA_API


def test_one_default_frame():
    t = fb.mesh_frame_table()
    assert len(t) == 1
    assert t[0].has_transform == 0 and t[0].n_var_values == 0


def test_per_frame_views_and_vars():
    m = np.stack([np.eye(4) * (1 + k) for k in range(5)]).astype(np.float32)
    vv = np.arange(10, dtype=np.float32).reshape(5, 2)
    t = fb.mesh_frame_table(world_to_model=m, var_values=vv)
    assert len(t) == 5
    for k in range(5):
        assert t[k].has_transform == 1 and list(t[k].world_to_model) == m[k].reshape(16).tolist()
        assert t[k].n_var_values == 2 and list(t[k].var_values)[:2] == vv[k].tolist()


def test_a_none_view_is_no_transform():
    t = fb.mesh_frame_table(world_to_model=[None, np.eye(4), None])
    assert [f.has_transform for f in t] == [0, 1, 0]
    assert list(t[1].world_to_model) == np.eye(4, dtype=np.float32).reshape(16).tolist()
    assert list(t[0].world_to_model) == [0.0] * 16


@pytest.mark.parametrize("kw", [dict(world_to_model=[None, None], var_values=np.zeros((3, 1))),
                                dict(var_values=np.zeros((2, 1)), world_to_model=[None]),
                                dict(world_to_model=np.zeros((2, 3, 3))),
                                dict(var_values=np.zeros(3))])
def test_bad_arguments_are_refused(kw):
    with pytest.raises(ValueError):
        fb.mesh_frame_table(**kw)


def test_var_limits():
    t = fb.mesh_frame_table(var_values=np.ones((2, _lib.FC_MAX_VARS)))
    assert t[1].n_var_values == _lib.FC_MAX_VARS
    with pytest.raises(ValueError):
        fb.mesh_frame_table(var_values=np.zeros((2, _lib.FC_MAX_VARS + 1)))


def _per(nv, nt, nc=None):
    return [{"n_vertices": a, "n_triangles": b, "n_cells": 0 if nc is None else nc[k]} for k, (a, b) in enumerate(zip(nv, nt))]


def test_split_gives_each_frame_its_rows():
    nv, nt, nc = [4, 0, 3, 5], [2, 0, 1, 3], [2, 0, 1, 4]
    v = np.arange(sum(nv) * 3, dtype=np.float32).reshape(-1, 3)
    t = np.concatenate([np.array([[0, 1, 2], [3, 2, 1]]), np.zeros((0, 3)), np.array([[0, 2, 1]]),
                        np.array([[4, 3, 0], [1, 2, 3], [0, 4, 2]])]).astype(np.uint32)
    cells = np.zeros(sum(nc), dtype=fb.MESH_CELL)
    cells["ix"] = np.arange(sum(nc))
    out = fb.split_mesh_frames(v, t, _per(nv, nt, nc), cells)
    assert len(out) == 4
    p = q = r = 0
    for k, (fv, ft, fc) in enumerate(out):
        assert np.array_equal(fv, v[p:p + nv[k]]) and np.array_equal(ft, t[q:q + nt[k]])
        assert np.array_equal(fc["ix"], np.arange(r, r + nc[k]))
        assert len(ft) == 0 or ft.max() < len(fv)          # local indices: a complete mesh on its own
        p, q, r = p + nv[k], q + nt[k], r + nc[k]
    assert [len(x) for x in fb.split_mesh_frames(v, t, _per(nv, nt))[0]] == [4, 2]


@pytest.mark.parametrize("nv,nt,nc", [([4, 3], [2, 1], None), ([4, 0, 3, 6], [2, 0, 1, 3], None),
                                      ([4, 0, 3, 5], [2, 0, 1, 3], [2, 0, 1, 5])])
def test_counts_that_do_not_add_up_are_refused(nv, nt, nc):
    v = np.zeros((12, 3), np.float32)
    t = np.zeros((6, 3), np.uint32)
    cells = np.zeros(7, dtype=fb.MESH_CELL) if nc is not None else None
    with pytest.raises(ValueError):
        fb.split_mesh_frames(v, t, _per(nv, nt, nc), cells)


def test_split_stl():
    files = [b"H" * 80 + (2).to_bytes(4, "little") + b"a" * 100, b"H" * 80 + bytes(4),
             b"H" * 80 + (1).to_bytes(4, "little") + b"b" * 50]
    got = fb.split_mesh_stl(b"".join(files), [2, 0, 1])
    assert got == files
    with pytest.raises(ValueError):
        fb.split_mesh_stl(b"".join(files), [2, 0, 2])
