"""fidget_b200 -- H100-native (sm_90a CUDA) backend for Fidget's tape
evaluation hot path: interval evaluation + tape simplification over tiles and
bulk f32 / gradient evaluation of the surviving voxels.

Layout
  host.py    host-side tape front end (Context, .vm loader, SSA, register
             allocation, bytecode) -- mirrors fidget-core / fidget-bytecode
  shape.py   CudaShape / evaluators / pixel.render / voxel.render -- mirrors
             the reference's Shape + fidget-raster API on top of the C ABI
  effects.py fidget-raster's post-processing effects (denoise, SSAO, shading, RGBA conversions)
  csrc/      CUDA kernels + the C ABI (include/fidget_cuda.h)
"""
from .host import Context, TapeData, Bytecode, OPCODES  # noqa: F401
from .shape import (  # noqa: F401
    CudaContext, CudaShape, CudaError, CancelToken, RenderConfig2D, RenderConfig3D, GEOMETRY_PIXEL,
    render2d, render2d_frames, frame_table, render3d, render3d_frames, frame_table_3d, render3d_scene, scene_table, render2d_scene, scene_table_2d, scene_colors, octree_sample, mesh, mesh_cells, mesh_frames, mesh_frame_table, measure, MEASURE_RESULT, volume, volume_dense, Volume, raycast, pick, pick_rays, RAY, RAY_HIT, split_mesh_frames, split_mesh_stl, contour, contour_slices, contour_slice_table, split_contour_stack, contours_svg, MESH_CELL, schedule_check, OCTREE_LEAF, pixel_inside, screen_to_world_2d, screen_to_world_3d, pixel_mat, voxel_mat,
    Free, Fixed, solve, solve_batch, solve_large_batch, CompiledShape, compile_check,
)
from ._lib import FC_SCENE2D_NONE  # noqa: F401,E402
from . import effects  # noqa: F401,E402
