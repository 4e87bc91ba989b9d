"""Loader for the in-tree ``libfidget_cuda.so`` (built by ``build.sh`` /
``__graft_entry__.build()``).  There is no CPU fallback: if the CUDA library is
missing this raises instead of silently routing anywhere else."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# FIDGET_B200_LIB: another build of the same library (A/B measurements of a kernel change on one box)
LIB_PATH = os.environ.get("FIDGET_B200_LIB") or os.path.join(_HERE, "libfidget_cuda.so")
_LIB = None


class BackendMissing(RuntimeError):
    pass


def _default_nvrtc():
    """The library opens NVRTC at its first tape compile (fc_tape_compile); point it at the copy that ships with torch
    (the nvidia-cuda-nvrtc wheel) unless FIDGET_B200_NVRTC already names one."""
    if os.environ.get("FIDGET_B200_NVRTC"):
        return
    import importlib.util
    try:
        spec = importlib.util.find_spec("nvidia.cuda_nvrtc")
    except (ImportError, ValueError):
        return
    for base in (spec.submodule_search_locations or []) if spec else []:
        lib = os.path.join(base, "lib")
        if os.path.isdir(lib):
            os.environ["FIDGET_B200_NVRTC"] = lib
            return


def load() -> C.CDLL:
    global _LIB
    if _LIB is None:
        _default_nvrtc()
        if not os.path.exists(LIB_PATH):
            raise BackendMissing(
                f"{LIB_PATH} not found: build it with ./build.sh (nvcc, sm_90a). "
                "fidget_b200 has no CPU fallback.")
        from .host import bind_host_api
        lib = C.CDLL(LIB_PATH)
        bind_host_api(lib)
        _bind_cuda_api(lib)
        _LIB = lib
    return _LIB


class _Record(C.Structure):
    """A C struct whose fields read back as a dict (arrays as lists)"""

    def as_dict(self):
        return {n: list(v) if isinstance(v, C.Array) else v for n, _ in self._fields_ for v in [getattr(self, n)]}


class FcTapeInfo(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in
                ("n_ops", "ref_len", "choice_count", "reg_count", "mem_count", "n_vars", "n_outputs")]


class FcRender2dCfg(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("mat", C.c_float * 16), ("z", C.c_float),
                ("pixel_perfect", C.c_uint32), ("n_tile_sizes", C.c_uint32), ("tile_sizes", C.c_uint32 * 8),
                ("flags", C.c_uint32), ("root_row_begin", C.c_uint32), ("root_row_end", C.c_uint32),
                ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16),
                ("root_stride", C.c_uint32), ("root_offset", C.c_uint32), ("out_format", C.c_uint32)]


class FcFrame2d(C.Structure):
    _fields_ = [("mat", C.c_float * 16), ("z", C.c_float), ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16)]


class FcFrame3d(C.Structure):
    _fields_ = [("mat", C.c_float * 16), ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16)]


class FcScheduleInfo(_Record):
    _fields_ = [(n, C.c_uint32) for n in ("suitable", "n_clauses", "n_waves", "widest_wave", "n_tail", "n_segments",
                                          "n_chain_clauses", "n_slots")]


class FcRender3dCfg(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("depth", C.c_uint32), ("mat", C.c_float * 16),
                ("n_tile_sizes", C.c_uint32), ("tile_sizes", C.c_uint32 * 8), ("flags", C.c_uint32),
                ("z_begin", C.c_uint32), ("z_end", C.c_uint32), ("n_var_values", C.c_uint32),
                ("var_values", C.c_float * 16), ("root_row_begin", C.c_uint32), ("root_row_end", C.c_uint32),
                ("root_stride", C.c_uint32), ("root_offset", C.c_uint32)]


class FcRenderStats(_Record):
    _fields_ = [(n, C.c_uint64 * 8) for n in
                ("evaluated", "filled_inside", "filled_outside", "ambiguous", "simplified")] + \
               [("pixels", C.c_uint64), ("grads", C.c_uint64), ("arena_bytes_used", C.c_uint64),
                ("kernel_launches", C.c_uint32), ("stage_ms", C.c_float * 16)]


class FcOctreeCfg(C.Structure):
    _fields_ = [("depth", C.c_uint32), ("has_transform", C.c_uint32), ("world_to_model", C.c_float * 16),
                ("flags", C.c_uint32), ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16)]


class FcOctreeStats(_Record):
    _fields_ = [(n, C.c_uint64 * 16) for n in ("evaluated", "full", "empty", "ambiguous")] + \
               [(n, C.c_uint64) for n in ("leaf_empty", "leaf_full", "leaf_surface", "float_points", "grad_points",
                                          "arena_bytes_used")] + \
               [("kernel_launches", C.c_uint32), ("total_ms", C.c_float)]


class FcMeshInfo(_Record):
    _fields_ = [(n, C.c_uint64) for n in ("n_leaves", "n_vertices", "n_triangles", "open_edges")] + \
               [("sampler_ms", C.c_float), ("mesh_ms", C.c_float)]


class FcMeshFrame(C.Structure):
    _fields_ = [("has_transform", C.c_uint32), ("world_to_model", C.c_float * 16), ("n_var_values", C.c_uint32),
                ("var_values", C.c_float * 16)]


class FcMeshFrameInfo(_Record):
    _fields_ = [(n, C.c_uint64) for n in ("n_leaves", "n_vertices", "n_triangles", "open_edges", "n_cells")]


class FcMeasureResult(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_inside", "n_proven", "n_undecided")] + \
               [("s1", C.c_uint64 * 3), ("s2", C.c_uint64 * 6), ("lo", C.c_uint32 * 3), ("hi", C.c_uint32 * 3)] + \
               [(n, C.c_double) for n in ("volume", "volume_lo", "volume_hi")] + \
               [("centroid", C.c_double * 3), ("inertia", C.c_double * 6), ("bbox_min", C.c_double * 3),
                ("bbox_max", C.c_double * 3)]


class FcRay(C.Structure):
    _fields_ = [("origin", C.c_float * 3), ("dir", C.c_float * 3), ("t0", C.c_float), ("dt", C.c_float)]


class FcRayHit(C.Structure):
    _fields_ = [("k", C.c_uint32), ("flags", C.c_uint32), ("t", C.c_float), ("pos", C.c_float * 3), ("value", C.c_float),
                ("grad", C.c_float * 3)]


class FcRaycastCfg(C.Structure):
    _fields_ = [("steps", C.c_uint32), ("flags", C.c_uint32), ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16)]


class FcRaycastInfo(_Record):
    _fields_ = [("n_hits", C.c_uint64), ("n_proven", C.c_uint64), ("evaluated", C.c_uint64 * 8),
                ("leaf_samples", C.c_uint64), ("passes", C.c_uint32), ("device_ms", C.c_float)]


class FcVolumeCfg(C.Structure):
    _fields_ = [("depth", C.c_uint32), ("flags", C.c_uint32), ("band", C.c_float), ("pad", C.c_uint32)]


class FcVolumeBrick(C.Structure):
    _fields_ = [("frame", C.c_uint32), ("ix", C.c_uint16), ("iy", C.c_uint16), ("iz", C.c_uint16), ("pad", C.c_uint16)]


class FcVolumeTile(C.Structure):
    _fields_ = [("frame", C.c_uint32), ("ix", C.c_uint16), ("iy", C.c_uint16), ("iz", C.c_uint16),
                ("log2_edge", C.c_uint8), ("inside", C.c_uint8)]


class FcVolumeInfo(_Record):
    _fields_ = [(n, C.c_uint64) for n in ("n_bricks", "n_tiles", "n_inside_tiles")] + \
               [("evaluated", C.c_uint64 * 16), ("brick_edge", C.c_uint32), ("passes", C.c_uint32),
                ("device_ms", C.c_float), ("level_ms", C.c_float)]


class FcVolumeFrameInfo(_Record):
    _fields_ = [(n, C.c_uint64) for n in ("n_bricks", "n_tiles", "first_brick", "first_tile")]


class FcContourCfg(C.Structure):
    _fields_ = [("depth", C.c_uint32), ("has_transform", C.c_uint32), ("world_to_model", C.c_float * 9), ("z", C.c_float),
                ("flags", C.c_uint32), ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16)]


class FcContourInfo(_Record):
    _fields_ = [(n, C.c_uint64) for n in ("n_leaves", "n_vertices", "n_polylines", "n_closed", "n_open")] + \
               [("sampler_ms", C.c_float), ("contour_ms", C.c_float)]


class FcContourSlice(C.Structure):
    _fields_ = [("z", C.c_float), ("has_transform", C.c_uint32), ("world_to_model", C.c_float * 9),
                ("n_var_values", C.c_uint32), ("var_values", C.c_float * 16)]


class FcSolveCfg(C.Structure):
    _fields_ = [("n_params", C.c_uint32), ("n_free", C.c_uint32), ("max_iters", C.c_uint32)]


class FcSolveResult(C.Structure):
    _fields_ = [("status", C.c_uint32), ("iterations", C.c_uint32), ("err", C.c_float), ("pad", C.c_uint32)]


class FcCompiledInfo(_Record):
    _fields_ = [("kinds", C.c_uint32), ("nvrtc_version", C.c_uint32), ("regs", C.c_uint32 * 3),
                ("local_bytes", C.c_uint32 * 3), ("compile_ms", C.c_float * 3), ("cubin_bytes", C.c_uint64)]


FC_COMPILE_FLOAT, FC_COMPILE_GRAD, FC_COMPILE_INTERVAL = 1, 2, 4
FC_SOLVE_MAX_FREE, FC_SOLVE_MAX_CONSTRAINTS, FC_SOLVE_MAX_PARAMS = 64, 256, 1024
FC_SOLVE_LARGE_MAX_FREE, FC_SOLVE_LARGE_MAX_CONSTRAINTS, FC_SOLVE_LARGE_MAX_PARAMS = 1024, 4096, 16384
FC_SOLVE_ZERO_RESIDUAL = 0
FC_SOLVE_UNCHANGED = 1
FC_SOLVE_ZERO_ERR = 2
FC_SOLVE_ZERO_DAMPING = 3
FC_SOLVE_STALLED = 4
FC_SOLVE_MAX_ITERS = 5
FC_FLAG_ASYNC = 1
FC_FLAG_TIMING = 2
FC_FLAG_NO_CLAMP = 4
FC_FLAG_FUSED_TAIL = 8
FC_FLAG_EXACT_CENSUS = 16
FC_FLAG_FULL_LADDER = 32
FC_FLAG_MESH_COLLAPSE = 64
FC_FLAG_VOLUME_GRADS = 128
FC_OUT_F32, FC_OUT_MASK_U8, FC_OUT_BITMAP_1BIT, FC_OUT_RGBA8 = 0, 1, 2, 3
FC_ERR_CANCELLED = -6
FC_FRAMES_PASS_BYTES = 512 << 20
FC_MAX_VARS = 16
FC_MAX_QUADTREE_DEPTH = 14
FC_MAX_OCTREE_DEPTH = 12
FC_MESH_MAX_PASS_FRAMES = 4096
FC_SCENE_MAX_SHAPES = 1024
FC_SCENE_MAX_DEPTH = 262142
FC_SCENE_MAX_ROOT_TILE = 1022
FC_SCENE_MAX_LEAF_JOBS = 67108863
FC_SCENE2D_NONE = 0xFFFF
FC_RAY_MISS = 0xFFFFFFFF
FC_RAY_PROVEN = 1
FC_RAY_MAX_STEPS = 1 << 24

# name -> (restype, argtypes); mirrors include/fidget_cuda.h one to one
_vp, _u32, _i32, _u64, _u8 = C.c_void_p, C.c_uint32, C.c_int32, C.c_uint64, C.c_uint8
_P = C.POINTER
CUDA_API = {
    "fc_last_error": (C.c_char_p, []),
    "fc_abi_version": (_u32, []),
    "fc_ctx_create": (_i32, [_i32, _P(_vp)]),
    "fc_ctx_destroy": (None, [_vp]),
    "fc_ctx_set_stream": (_i32, [_vp, _vp, _i32]),
    "fc_ctx_synchronize": (_i32, [_vp]),
    "fc_ctx_set_arena_bytes": (_i32, [_vp, _u64]),
    "fc_ctx_set_cancel": (_i32, [_vp, _vp]),
    "fc_tape_create": (_i32, [_vp, _P(_u32), C.c_size_t, _u8, _u32, _u32, _u32, _u32, _P(_vp)]),
    "fc_tape_retain": (_i32, [_vp]),
    "fc_tape_release": (_i32, [_vp]),
    "fc_tape_get_info": (_i32, [_vp, _P(FcTapeInfo)]),
    "fc_tape_set_axes": (_i32, [_vp, _i32, _i32, _i32]),
    "fc_tape_read": (_i32, [_vp, _P(_u32), C.c_size_t, _P(C.c_size_t)]),
    "fc_tape_serialize": (_i32, [_vp, _vp, C.c_size_t, _P(C.c_size_t)]),
    "fc_tape_deserialize": (_i32, [_vp, _vp, C.c_size_t, _P(_vp)]),
    "fc_eval_create": (_i32, [_vp, _P(_vp)]),
    "fc_eval_destroy": (None, [_vp]),
    "fc_interval_eval": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "fc_point_eval": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "fc_interval_eval_batch": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _vp]),
    "fc_float_slice_eval": (_i32, [_vp, _vp, _P(_vp), _P(_vp), _u64]),
    "fc_grad_slice_eval": (_i32, [_vp, _vp, _P(_vp), _P(_vp), _u64]),
    "fc_simplify": (_i32, [_vp, _vp, _vp, C.c_size_t, _P(_vp)]),
    "fc_tape_compile": (_i32, [_vp, _vp, _u32, _P(_vp)]),
    "fc_compiled_get_info": (_i32, [_vp, _P(FcCompiledInfo)]),
    "fc_compiled_release": (_i32, [_vp]),
    "fc_compiled_float_slice_eval": (_i32, [_vp, _vp, _P(_vp), _P(_vp), _u64]),
    "fc_compiled_grad_slice_eval": (_i32, [_vp, _vp, _P(_vp), _P(_vp), _u64]),
    "fc_compiled_interval_eval_batch": (_i32, [_vp, _vp, _vp, _u64, _vp, _vp, _vp]),
    "fc_compile_check": (_i32, [_P(_u32), C.c_size_t, _u8, _u32, _u32, _u32, _u32, C.c_char_p, C.c_size_t,
                                _P(C.c_size_t), _P(FcCompiledInfo)]),
    "fc_render2d": (_i32, [_vp, _vp, _P(FcRender2dCfg), _vp, _P(FcRenderStats)]),
    "fc_render2d_frames": (_i32, [_vp, _vp, _P(FcRender2dCfg), _P(FcFrame2d), _u32, _vp, _P(FcRenderStats)]),
    "fc_render3d": (_i32, [_vp, _vp, _P(FcRender3dCfg), _vp, _P(FcRenderStats)]),
    "fc_render3d_frames": (_i32, [_vp, _vp, _P(FcRender3dCfg), _P(FcFrame3d), _u32, _vp, _P(FcRenderStats)]),
    "fc_render3d_scene": (_i32, [_vp, _P(_vp), _P(FcFrame3d), _u32, _P(FcRender3dCfg), _vp, _vp, _P(FcRenderStats)]),
    "fc_render2d_scene": (_i32, [_vp, _P(_vp), _P(FcFrame2d), _u32, _P(FcRender2dCfg), _vp, _vp, _vp, _P(FcRenderStats)]),
    "fc_merge_slabs": (_i32, [_vp, _P(_vp), _u32, _u32, _u32, _u32, _vp]),
    "fc_tiles_per_rank": (_u32, [_u32, _u32, _u32, _u32]),
    "fc_tiles_pack": (_i32, [_vp, _vp, _u32, _u32, _u32, _u32, _u32, _u32, _vp]),
    "fc_tiles_unpack": (_i32, [_vp, _vp, _u32, _u32, _u32, _u32, _u32, _vp]),
    "fc_octree_sample": (_i32, [_vp, _vp, _P(FcOctreeCfg), _vp, _u64, _P(_u64), _P(FcOctreeStats)]),
    "fc_mesh_build": (_i32, [_vp, _vp, _P(FcOctreeCfg), _P(FcMeshInfo)]),
    "fc_mesh_read": (_i32, [_vp, _vp, _vp]),
    "fc_mesh_read_cells": (_i32, [_vp, _vp, _u64, _P(_u64)]),
    "fc_mesh_write_stl": (_i32, [_vp, _vp, C.c_size_t, _P(C.c_size_t)]),
    "fc_mesh_build_frames": (_i32, [_vp, _vp, _P(FcOctreeCfg), _P(FcMeshFrame), _u32, _P(FcMeshInfo),
                                    _P(FcMeshFrameInfo)]),
    "fc_measure": (_i32, [_vp, _vp, _P(FcOctreeCfg), _P(FcMeshFrame), _u32, _vp, _P(C.c_float)]),
    "fc_volume_build": (_i32, [_vp, _vp, _P(FcVolumeCfg), _P(FcMeshFrame), _u32, _P(FcVolumeInfo),
                               _P(FcVolumeFrameInfo)]),
    "fc_volume_read": (_i32, [_vp, _vp, _vp, _vp, _vp]),
    "fc_raycast": (_i32, [_vp, _vp, _P(FcRaycastCfg), _vp, _u64, _vp, _P(FcRaycastInfo)]),
    "fc_contour_build": (_i32, [_vp, _vp, _P(FcContourCfg), _P(FcContourInfo)]),
    "fc_contour_read": (_i32, [_vp, _vp, _vp, _vp]),
    "fc_contour_build_slices": (_i32, [_vp, _vp, _P(FcContourCfg), _P(FcContourSlice), _u32, _P(FcContourInfo),
                                       _P(FcContourInfo)]),
    "fc_solve_batch": (_i32, [_vp, _P(_vp), _u32, _P(_P(_i32)), _P(FcSolveCfg), _vp, _u64, _vp]),
    "fc_solve_large_batch": (_i32, [_vp, _P(_vp), _u32, _P(_P(_i32)), _P(FcSolveCfg), _vp, _u64, _vp]),
    "fc_schedule_check": (_i32, [_P(_u32), C.c_size_t, _u8, _u32, _u32, _u32, _P(FcScheduleInfo)]),
    "fc_denoise_normals": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "fc_compute_ssao": (_i32, [_vp, _vp, _u32, _u32, _u32, _vp, _u32, _vp, _u32, _vp]),
    "fc_blur_ssao": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "fc_apply_shading": (_i32, [_vp, _vp, _u32, _u32, _u32, _i32, _vp, _u32, _vp, _u32, _vp]),
    "fc_shade_with_occlusion": (_i32, [_vp, _vp, _u32, _u32, _u32, _vp, _vp]),
    "fc_normals_to_color": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "fc_to_rgba_bitmap": (_i32, [_vp, _vp, _u32, _u32, _i32, _vp]),
    "fc_to_debug_bitmap": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "fc_to_rgba_distance": (_i32, [_vp, _vp, _u32, _u32, _vp]),
}


def _bind_cuda_api(lib):
    for name, (res, args) in CUDA_API.items():
        f = getattr(lib, name)  # AttributeError here == header/library mismatch
        f.restype = res
        f.argtypes = args
