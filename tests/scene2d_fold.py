"""What fc_render2d_scene computes, restated in numpy: the reference viewer's 2D draw list, where every draw(shape) /
draw_rgb(shape, r, g, b) is rendered with pixel::render, mapped to RGBA (its colour where RawDistancePixel::inside,
[0, 0, 0, 0] elsewhere) and painted over the layers before it with opaque OVER: the last shape inside a pixel wins."""
import numpy as np

import fidget_b200 as fb

NONE = 0xFFFF


def fold_inside(insides):
    """index per pixel: the largest k with insides[k] true there, NONE where no shape is inside"""
    index = np.full(np.shape(insides[0]), NONE, dtype=np.uint16)
    for k, m in enumerate(insides):
        index[np.asarray(m, dtype=bool)] = k
    return index


def fold(images):
    """the index of per-shape fc_render2d f32 images (RawDistancePixel bits), in draw order"""
    return fold_inside([fb.pixel_inside(np.asarray(img, dtype=np.float32)) for img in images])


def rgba(index, colors=None):
    """the FC_OUT_RGBA8 image of an index: shape k's colour (white without a table) with alpha 255, zeros where NONE"""
    n = int(index[index != NONE].max()) + 1 if (index != NONE).any() else 0
    colors = np.full((max(n, 1), 3), 255, dtype=np.uint8) if colors is None else np.asarray(colors, dtype=np.uint8)
    out = np.zeros(index.shape + (4,), dtype=np.uint8)
    hit = index != NONE
    out[hit, :3] = colors[index[hit]]
    out[hit, 3] = 255
    return out


def mask_u8(index):
    return np.where(index != NONE, 255, 0).astype(np.uint8)


def bitmap_1bit(index):
    """FC_OUT_BITMAP_1BIT: rows of (w + 7) // 8 bytes, bit x % 8 (LSB first) of byte x / 8 set = inside"""
    return np.packbits(index != NONE, axis=1, bitorder="little")
