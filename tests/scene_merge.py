"""The merge fc_render3d_scene computes in one call, restated in numpy: the fold of fidget-wgpu's effects merge
(merge.wgsl, merge_pixel: `a.depth >= b.depth` keeps a) over per-shape voxel images, each tagged with the index of
the image it came from (PackedVoxel::index)."""
import numpy as np

import fidget_b200 as fb


def clamp_image(img, depth):
    """The final clamp of voxel::render (voxel.rs:535-546) applied to an unclamped image: every pixel at depth >= D - 1
    becomes depth D with normal [0, 0, 1]"""
    out = np.array(img, dtype=fb.GEOMETRY_PIXEL, copy=True)
    zone = out["depth"].astype(np.int64) >= depth - 1
    out["depth"][zone] = depth
    out["normal"][zone] = np.array([0.0, 0.0, 1.0], dtype=np.float32)
    return out


def fold(images):
    """acc = img_0; acc = (acc.depth >= img_k.depth) ? acc : img_k for k = 1 ..; returns (image, index): the greatest
    depth wins, the lowest k on equal depth, and an empty pixel (depth 0 everywhere) keeps index 0"""
    acc = np.array(images[0], dtype=fb.GEOMETRY_PIXEL, copy=True)
    index = np.zeros(acc.shape, dtype=np.uint16)
    for k in range(1, len(images)):
        img = np.asarray(images[k], dtype=fb.GEOMETRY_PIXEL)
        take = ~(acc["depth"] >= img["depth"])
        acc[take] = img[take]
        index[take] = k
    return acc, index
