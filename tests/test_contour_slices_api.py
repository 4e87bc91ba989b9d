"""The host side of fb.contour_slices: the fc_contour_slice table (per-slice arguments, their lengths, the var limit,
the has_transform flag) and the split of a stacked contour into per-slice outputs.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib


def test_slice_struct_matches_the_header():
    assert C.sizeof(_lib.FcContourSlice) == 4 + 4 + 9 * 4 + 4 + 16 * 4
    assert "fc_contour_build_slices" in _lib.CUDA_API


def test_one_default_slice():
    t = fb.contour_slice_table()
    assert len(t) == 1
    s = t[0]
    assert s.z == 0.0 and s.has_transform == 0 and s.n_var_values == 0


def test_per_slice_z_values_and_views():
    z = np.linspace(-0.5, 0.5, 5, dtype=np.float32)
    m = np.stack([np.eye(3) * (1 + k) for k in range(5)]).astype(np.float32)
    vv = np.arange(10, dtype=np.float32).reshape(5, 2)
    t = fb.contour_slice_table(z=z, world_to_model=m, var_values=vv)
    assert len(t) == 5
    for k in range(5):
        assert np.float32(t[k].z) == z[k]
        assert t[k].has_transform == 1 and list(t[k].world_to_model) == m[k].reshape(9).tolist()
        assert t[k].n_var_values == 2 and list(t[k].var_values)[:2] == vv[k].tolist()


def test_a_none_view_is_no_transform():
    t = fb.contour_slice_table(world_to_model=[None, np.eye(3), None])
    assert [s.has_transform for s in t] == [0, 1, 0]
    assert list(t[1].world_to_model) == np.eye(3, dtype=np.float32).reshape(9).tolist()


def test_non_finite_z_is_kept():
    t = fb.contour_slice_table(z=[np.inf, -np.inf, np.nan, -0.0])
    assert t[0].z == np.inf and t[1].z == -np.inf and np.isnan(t[2].z)
    assert np.signbit(np.float32(t[3].z))


@pytest.mark.parametrize("kw", [dict(z=[0, 1], var_values=np.zeros((3, 1))),
                                dict(z=[0, 1, 2], world_to_model=np.zeros((2, 3, 3))),
                                dict(var_values=np.zeros((2, 1)), world_to_model=[None])])
def test_lengths_that_disagree_are_refused(kw):
    with pytest.raises(ValueError):
        fb.contour_slice_table(**kw)


def test_var_limits():
    fb.contour_slice_table(var_values=np.zeros((2, _lib.FC_MAX_VARS)))
    with pytest.raises(ValueError):
        fb.contour_slice_table(var_values=np.zeros((2, _lib.FC_MAX_VARS + 1)))
    with pytest.raises(ValueError):
        fb.contour_slice_table(var_values=np.zeros(3))


def test_bad_matrices_are_refused():
    with pytest.raises(ValueError):
        fb.contour_slice_table(world_to_model=np.zeros((2, 4, 4)))


def test_split_rebases_offsets_per_slice():
    # three slices: two polylines, none, one
    v = np.arange(20, dtype=np.float32).reshape(10, 2)
    off = np.array([0, 3, 7, 10], np.uint32)
    closed = np.array([1, 0, 1], np.uint8)
    parts = fb.split_contour_stack(v, off, closed, [2, 0, 1])
    assert len(parts) == 3
    (v0, o0, c0), (v1, o1, c1), (v2, o2, c2) = parts
    assert np.array_equal(v0, v[:7]) and o0.tolist() == [0, 3, 7] and c0.tolist() == [True, False]
    assert v1.shape == (0, 2) and o1.tolist() == [0] and c1.tolist() == [] and o1.dtype == np.uint32
    assert np.array_equal(v2, v[7:]) and o2.tolist() == [0, 3] and c2.tolist() == [True]
    assert c0.dtype == bool


def test_split_of_an_empty_stack():
    parts = fb.split_contour_stack(np.zeros((0, 2), np.float32), np.zeros(1, np.uint32), np.zeros(0, np.uint8), [0, 0])
    assert [p[1].tolist() for p in parts] == [[0], [0]]


def test_split_refuses_counts_that_do_not_add_up():
    with pytest.raises(ValueError):
        fb.split_contour_stack(np.zeros((3, 2), np.float32), np.array([0, 3], np.uint32), np.zeros(1, np.uint8), [2])
