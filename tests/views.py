"""Test infrastructure: a catalogue of ``world_to_model`` views -- rotated, sheared, mirrored, perspective, degenerate
and non-finite -- and a float64 reading of what a renderer must produce under them.

Every consumer of a tape takes a homogeneous matrix and sends it through ``Transformable for f32 / Interval / Grad``
(fidget-core/src/shape/mod.rs:894-948): four rows, then a division by the homogeneous term ``w``.  The reference here
is numpy float64 throughout and shares no code with ``oracle/`` or the device: ``model_points64`` transforms,
``eval64`` evaluates the test shapes (closed forms, or a line-by-line reading of ``.vm`` text), ``expected_heightmap``
and ``expected_normal64`` say what a 3D render may return, ``check_image2d`` what a 2D render may.

The catalogue matrices are computed here from angles and constants; nothing is loaded from a file."""
from __future__ import annotations

import numpy as np

from conftest import model_text

U32 = 2.0 ** -24            # unit roundoff of float32


# ---- the catalogue ---------------------------------------------------------------------------------------------------
def _rot(axis, deg):
    """Rotation about ``axis`` by ``deg`` degrees (Rodrigues), 4x4 float64."""
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    t = np.deg2rad(deg)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    m = np.eye(4)
    m[:3, :3] = np.eye(3) + np.sin(t) * k + (1 - np.cos(t)) * (k @ k)
    return m


def _eye(n=4, **entries):
    """Identity with entries replaced: _eye(m32=0.3) sets [3][2]."""
    m = np.eye(n)
    for key, v in entries.items():
        m[int(key[1]), int(key[2])] = v
    return m


def _diag(*d):
    return np.diag(np.array(d + (1.0,), dtype=np.float64))


def _translate(*t):
    m = np.eye(len(t) + 1)
    m[:-1, -1] = t
    return m


def _f32(m):
    with np.errstate(over="ignore"):
        return np.asarray(m, dtype=np.float64).astype(np.float32)


def _zero_last_row(m):
    m = np.array(m, dtype=np.float64)
    m[-1, :] = 0.0
    return m


# roll 30 deg . pitch 60 deg . scale 1/0.7 . camera with m[3][2] = 0.3: the camera of the reference's voxel benchmark
# (fidget/benches/voxel.rs), composed in float64 and rounded once
BENCH_CAMERA = _rot((0, 0, 1), 30) @ _rot((1, 0, 0), 60) @ _diag(1 / 0.7, 1 / 0.7, 1 / 0.7) @ _eye(m32=0.3)
_TILT = _rot((0, 1, 0), 40) @ _diag(1.2, 1.2, 1.2)

# name -> (matrix, kind).  kind: "affine" | "persp" (w > 0 in the volume) | "strong" (w changes sign or vanishes in the
# volume) | "degenerate" (finite, but the view shows nothing or everything) | "nonfinite"
VIEWS3 = {
    "bench_camera": (BENCH_CAMERA, "persp"),
    "rot_x_25": (_rot((1, 0, 0), 25), "affine"),
    "rot_y_40": (_rot((0, 1, 0), 40), "affine"),
    "rot_z_70": (_rot((0, 0, 1), 70), "affine"),
    "rot_axis_123_50": (_rot((1, 2, 3), 50), "affine"),
    "shear": (_eye(m01=0.4, m12=-0.3), "affine"),
    "scale_xyz": (_diag(1.3, 0.8, 1.7), "affine"),
    "mirror_x": (_diag(-1.0, 1.0, 1.0), "affine"),
    "permute_yzx": (np.array([[0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 1.0]]), "affine"),
    "persp_x": (_eye(m30=0.3), "persp"),
    "persp_y": (_eye(m31=0.3), "persp"),
    "persp_z": (_eye(m32=0.3), "persp"),
    "rot_persp": (_rot((0, 1, 0), 35) @ _eye(m32=0.3), "persp"),
    "persp_strong": (_eye(m32=1.5), "strong"),                       # w = 1.5 z + 1 changes sign at z = -2/3
    "persp_w0_plane": (_eye(m32=1.0, m33=0.0), "strong"),            # w = z: exactly 0 on the voxel plane z = depth / 2
    "zero_last_row": (_zero_last_row(_TILT), "strong"),              # w = 0 everywhere: f32 skips the division
    "zero_z_column": (_eye(m22=0.0), "degenerate"),                  # every voxel of a column at one model point
    "scale_1e-6": (_diag(1e-6, 1e-6, 1e-6), "degenerate"),           # the camera inside the solid
    "scale_1e+6": (_diag(1e6, 1e6, 1e6), "degenerate"),
    "out_of_view": (_translate(5.0, 0.0, 0.0), "degenerate"),
    "nan_entry": (_eye(m01=np.nan), "nonfinite"),
    "inf_entry": (_eye(m13=np.inf), "nonfinite"),
}
VIEWS2 = {
    "rot_33": (np.array([[np.cos(np.deg2rad(33)), -np.sin(np.deg2rad(33)), 0],
                         [np.sin(np.deg2rad(33)), np.cos(np.deg2rad(33)), 0], [0, 0, 1.0]]), "affine"),
    "shear": (_eye(3, m01=0.4), "affine"),
    "scale_xy": (np.diag([1.3, 0.8, 1.0]), "affine"),
    "mirror_x": (np.diag([-1.0, 1.0, 1.0]), "affine"),
    "swap_xy": (np.array([[0, 1, 0], [1, 0, 0], [0, 0, 1.0]]), "affine"),
    "persp_x": (_eye(3, m20=0.3), "persp"),
    "persp_y": (_eye(3, m21=0.3), "persp"),
    "rot_persp": (np.array([[np.cos(0.5), -np.sin(0.5), 0], [np.sin(0.5), np.cos(0.5), 0], [0, 0, 1.0]])
                  @ _eye(3, m21=0.3), "persp"),
    "persp_strong": (_eye(3, m21=1.5), "strong"),
    "persp_w0_line": (_eye(3, m21=1.0, m22=0.0), "strong"),          # w = y: exactly 0 on the pixel row y = 0
    "zero_last_row": (_zero_last_row(np.diag([1.2, 1.1, 1.0]) @ _eye(3, m01=0.2)), "strong"),
    "zero_y_column": (_eye(3, m11=0.0), "degenerate"),
    "scale_1e-6": (np.diag([1e-6, 1e-6, 1.0]), "degenerate"),
    "scale_1e+6": (np.diag([1e6, 1e6, 1.0]), "degenerate"),
    "out_of_view": (_translate(5.0, 0.0), "degenerate"),
    "nan_entry": (_eye(3, m01=np.nan), "nonfinite"),
    "inf_entry": (_eye(3, m12=np.inf), "nonfinite"),
}


def view3(name):
    """float32 4x4 ``world_to_model`` of a catalogue view."""
    return _f32(VIEWS3[name][0])


def view2(name):
    """float32 3x3 ``world_to_model`` of a 2D catalogue view."""
    return _f32(VIEWS2[name][0])


def with_unit_last_row(m):
    """``m`` with its last row replaced by (0, .., 0, 1): what a zero last row must render like, since
    ``transform_point`` divides only by a non-zero ``w``."""
    m = np.array(m, dtype=np.float32)
    m[-1, :] = 0.0
    m[-1, -1] = 1.0
    return m


def names3(*kinds):
    return [n for n, (_, k) in VIEWS3.items() if not kinds or k in kinds]


def names2(*kinds):
    return [n for n, (_, k) in VIEWS2.items() if not kinds or k in kinds]


# ---- float64 transform -----------------------------------------------------------------------------------------------
def model_points64(mat, xs, ys, zs):
    """rows . (x, y, z, 1), divided by ``w`` where ``w != 0``: [n, 3] float64.  ``mat`` is the 4x4 the renderer is
    given (screen to model)."""
    m = np.asarray(mat, dtype=np.float64).reshape(4, 4)
    p = np.stack([np.asarray(xs, np.float64), np.asarray(ys, np.float64), np.asarray(zs, np.float64)], axis=-1)
    r = p @ m[:, :3].T + m[:, 3]
    w = r[:, 3:4]
    with np.errstate(all="ignore"):
        return np.where(w != 0, r[:, :3] / np.where(w != 0, w, 1.0), r[:, :3])


def transform_error64(mat, xs, ys, zs):
    """First-order bound on |f32 transform - model_points64|, per point and coordinate [n, 3].  Three additions and
    four products per row stay within 4 u of the sum of the terms' magnitudes (u = 2^-24); the quotient r / w
    inherits the numerator's error over |w|, the denominator's scaled by |r / w| / |w|, and one rounding of its own."""
    m = np.abs(np.asarray(mat, dtype=np.float64).reshape(4, 4))
    p = np.abs(np.stack([np.asarray(xs, np.float64), np.asarray(ys, np.float64), np.asarray(zs, np.float64)], axis=-1))
    mag = p @ m[:, :3].T + m[:, 3]                     # sum of |terms| per row
    m64 = np.asarray(mat, dtype=np.float64).reshape(4, 4)
    q = np.stack([np.asarray(xs, np.float64), np.asarray(ys, np.float64), np.asarray(zs, np.float64)], axis=-1)
    w = (q @ m64[:, :3].T + m64[:, 3])[:, 3:4]
    pts = np.abs(model_points64(mat, xs, ys, zs))
    with np.errstate(all="ignore"):
        aw = np.where(w != 0, np.abs(w), 1.0)
        err = 4 * U32 * mag[:, :3] / aw + np.where(w != 0, pts * (4 * U32 * mag[:, 3:4] / aw), 0.0) + U32 * pts
    return err


# ---- float64 shapes --------------------------------------------------------------------------------------------------
def _fmin(a, b):      # the VM's rule: NaN if either is NaN
    return np.where(np.isnan(a) | np.isnan(b), np.nan, np.minimum(a, b))


def _fmax(a, b):
    return np.where(np.isnan(a) | np.isnan(b), np.nan, np.maximum(a, b))


_UNARY64 = {
    "neg": lambda a: -a, "abs": np.abs, "sqrt": np.sqrt, "square": lambda a: a * a, "recip": lambda a: 1.0 / a,
    "exp": np.exp, "ln": np.log, "sin": np.sin, "cos": np.cos, "tan": np.tan, "asin": np.arcsin, "acos": np.arccos,
    "atan": np.arctan, "floor": np.floor, "ceil": np.ceil,
}
_BINARY64 = {
    "add": lambda a, b: a + b, "sub": lambda a, b: a - b, "mul": lambda a, b: a * b, "div": lambda a, b: a / b,
    "min": _fmin, "max": _fmax, "atan2": np.arctan2,
}


def eval_vm_text64(text, x, y, z):
    """(value, error bound) of the last node of a ``.vm`` listing, all arithmetic in float64.  The bound is what a
    float32 evaluation of the same listing may differ by, to first order: every arithmetic node rounds once (u of its
    own magnitude) and passes on what its arguments carry, scaled by its partial derivatives; min / max pass on the
    larger of the two; constants round once on entry.  The libm opcodes take 4 u, above the 1-2 ulp CUDA documents."""
    env, err, last = {}, {}, None
    x = np.asarray(x, dtype=np.float64)
    zero = np.zeros_like(x)
    with np.errstate(all="ignore"):
        for line in text.splitlines():
            line = line.split("#", 1)[0].split()
            if not line:
                continue
            name, op, args = line[0], line[1], line[2:]
            if op == "const":
                c = float(args[0])
                v, e = np.full_like(x, c), zero + U32 * abs(c)
            elif op in ("var-x", "var-y", "var-z"):
                v, e = np.asarray({"var-x": x, "var-y": y, "var-z": z}[op], dtype=np.float64), zero
            elif op in _UNARY64:
                a, ea = env[args[0]], err[args[0]]
                v = _UNARY64[op](a)
                slope = {"neg": 1.0, "abs": 1.0, "square": 2 * np.abs(a), "sqrt": 0.5 / np.sqrt(np.abs(a)),
                         "recip": 1.0 / (a * a), "exp": np.abs(v), "ln": 1.0 / np.abs(a), "sin": 1.0, "cos": 1.0,
                         "tan": 1.0 + v * v, "asin": 1.0 / np.sqrt(np.abs(1 - a * a)),
                         "acos": 1.0 / np.sqrt(np.abs(1 - a * a)), "atan": 1.0, "floor": 0.0, "ceil": 0.0}[op]
                own = 0.0 if op in ("neg", "abs") else (U32 if op in ("square", "sqrt", "recip", "floor", "ceil") else 4 * U32)
                e = slope * ea + own * np.abs(v)
            elif op in _BINARY64:
                a, b, ea, eb = env[args[0]], env[args[1]], err[args[0]], err[args[1]]
                v = _BINARY64[op](a, b)
                if op in ("min", "max"):
                    e = np.maximum(ea, eb)
                elif op in ("add", "sub"):
                    e = ea + eb + U32 * np.abs(v)
                elif op == "mul":
                    e = np.abs(b) * ea + np.abs(a) * eb + U32 * np.abs(v)
                elif op == "div":
                    e = ea / np.abs(b) + np.abs(v) * eb / np.abs(b) + U32 * np.abs(v)
                else:
                    e = (ea + eb) / np.maximum(np.hypot(a, b), 1e-300) + 4 * U32 * np.abs(v)
            else:
                raise AssertionError(f"opcode {op} not known to the float64 reader")
            env[name], err[name], last = v, np.nan_to_num(e, nan=np.inf), name
    return env[last], err[last]


class Shape:
    """A test shape: ``tape(Ctx)`` builds it with a Context class (the product's or the oracle's), ``f(x, y, z)`` is its
    float64 value and first-order float32 evaluation error; ``ieee`` when device, oracle and reference agree bit for
    bit on it; ``var_values`` the ShapeVars a render needs."""

    def __init__(self, name, tape, f, ieee=True, var_values=()):
        self.name, self.tape, self.f, self.ieee, self.var_values = name, tape, f, ieee, var_values


def _vm_shape(name, ieee=True):
    text = model_text(name)

    def tape(Ctx):
        ctx, root = Ctx.from_text(text)
        return ctx.tape(root)

    return Shape(name, tape, lambda x, y, z: eval_vm_text64(text, x, y, z), ieee)


def _listing_shape(name, listing, tape, var_values=()):
    """An analytic shape: built node by node with ``tape``, read in float64 from the equivalent listing."""
    return Shape(name, tape, lambda x, y, z: eval_vm_text64(listing, x, y, z), True, var_values)


def _sphere_tape(Ctx):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    return ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), 0.6))


def _box_tape(Ctx):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    return ctx.tape(ctx.max(ctx.max(ctx.sub(ctx.abs(x), 0.5), ctx.sub(ctx.abs(y), 0.35)), ctx.sub(ctx.abs(z), 0.45)))


def _torus_tape(Ctx):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    ring = ctx.sub(ctx.sqrt(ctx.add(ctx.square(x), ctx.square(y))), 0.5)
    return ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.square(ring), ctx.square(z))), 0.2))


def _sphere_var_tape(Ctx):
    ctx = Ctx()
    x, y, z = ctx.x(), ctx.y(), ctx.z()
    r, _ = ctx.var()
    return ctx.tape(ctx.sub(ctx.sqrt(ctx.add(ctx.add(ctx.square(x), ctx.square(y)), ctx.square(z))), r))


_R2 = "x var-x\ny var-y\nz var-z\nxx square x\nyy square y\nzz square z\nxy add xx yy\n"
_SPHERE = _R2 + "r2 add xy zz\nr sqrt r2\nc const {r}\nout sub r c\n"
SHAPES = {
    "sphere": _listing_shape("sphere", _SPHERE.format(r=0.6), _sphere_tape),
    "box": _listing_shape("box", "x var-x\ny var-y\nz var-z\nax abs x\nay abs y\naz abs z\nhx const 0.5\nhy const 0.35\n"
                          "hz const 0.45\ndx sub ax hx\ndy sub ay hy\ndz sub az hz\nm max dx dy\nout max m dz\n", _box_tape),
    "torus": _listing_shape("torus", _R2 + "q sqrt xy\nR const 0.5\nring sub q R\nrr square ring\ns add rr zz\nt sqrt s\n"
                            "c const 0.2\nout sub t c\n", _torus_tape),
    # a radius bound at render time: every ShapeVars slot holds it (the axis slots are ignored)
    "sphere_var": _listing_shape("sphere_var", _SPHERE.format(r=0.55), _sphere_var_tape, var_values=(0.55,) * 4),
    "colonnade.vm": _vm_shape("colonnade.vm"),
    "hi.vm": _vm_shape("hi.vm"),
    "tanglecube.vm": _vm_shape("tanglecube.vm"),
    "prospero.vm": _vm_shape("prospero.vm"),
    "bear.vm": _vm_shape("bear.vm", ieee=False),
}


def eval64(shape, pts):
    """(float64 values, float32 evaluation error bound) of ``SHAPES[shape]`` at ``pts`` [n, 3]."""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    parts = [SHAPES[shape].f(c[:, 0], c[:, 1], c[:, 2]) for c in np.array_split(pts, max(1, len(pts) // 16384))]
    return np.concatenate([v for v, _ in parts]), np.concatenate([e for _, e in parts])   # in pieces: a listing keeps every node


def slope64(vals, pts):
    """Twice the steepest slope |f(a) - f(b)| / |a - b| seen between neighbouring samples of a grid of values
    ``vals`` [..] at model points ``pts`` [.., 3]: what turns a bound on the transform's error into one on the
    value."""
    best = 0.0
    with np.errstate(all="ignore"):
        for ax in range(vals.ndim):
            df = np.abs(np.diff(vals, axis=ax))
            dp = np.linalg.norm(np.diff(pts, axis=ax), axis=-1)
            ok = np.isfinite(df) & np.isfinite(dp) & (dp > 0)
            if ok.any():
                best = max(best, float((df[ok] / dp[ok]).max()))
    return 2.0 * best


def field64(shape, mat, w, h, d=None, z=0.0):
    """(values, band) on the pixel grid [h, w] (at ``z``) or the voxel grid [d, h, w] of a render with matrix ``mat``:
    the float64 value of ``f(T(p))``, and a bound on what a float32 render may differ from it by -- the evaluation
    error of ``eval64`` plus the transform's error through the field's slope.  Outside the band the sign is certain."""
    if d is None:
        ys, xs = np.mgrid[0:h, 0:w]
        zs = np.full(xs.shape, float(z))
    else:
        zs, ys, xs = np.mgrid[0:d, 0:h, 0:w]
    grid = xs.shape
    pts = model_points64(mat, xs.ravel(), ys.ravel(), zs.ravel())
    vals, err = eval64(shape, pts)
    terr = np.linalg.norm(transform_error64(mat, xs.ravel(), ys.ravel(), zs.ravel()), axis=-1)
    vals = vals.reshape(grid)
    with np.errstate(all="ignore"):
        band = err.reshape(grid) + slope64(vals, pts.reshape(grid + (3,))) * terr.reshape(grid)
    return vals, np.nan_to_num(band, nan=np.inf)


# ---- what a render may return ----------------------------------------------------------------------------------------
def expected_heightmap(vals64, band):
    """(lo, hi) per column of a voxel grid [d, h, w]: ``lo`` = highest voxel with value < -band, plus one; ``hi`` =
    highest voxel with value < +band, plus one.  A depth ``e`` is right iff lo <= e <= hi.  A NaN value is outside,
    as ``value < 0`` is for the renderer."""
    d = vals64.shape[0]

    def top(inside):
        return np.where(inside.any(axis=0), d - np.argmax(inside[::-1], axis=0), 0)

    with np.errstate(invalid="ignore"):
        return top(vals64 < -band), top(vals64 < band)


def check_heightmap(depth_img, vals64, band, max_loose=0.05):
    """Asserts every depth of a 3D render within its bracket, and that the bracket is tight (lo == hi) on all but
    ``max_loose`` of the columns.  Returns the mask of tight columns."""
    d = vals64.shape[0]
    lo, hi = expected_heightmap(vals64, band)
    def clamp(e):       # voxel.rs:535-546: a column that reaches the last voxel saturates to the image depth
        return np.where(e >= d - 1, d, e)

    lo, hi, got = clamp(lo), clamp(hi), clamp(np.asarray(depth_img, dtype=np.int64))
    bad = (got < lo) | (got > hi)
    if bad.any():
        y, x = np.argwhere(bad)[0]
        raise AssertionError(f"{int(bad.sum())} depths outside their bracket; first at x={x} y={y}: "
                             f"{got[y, x]} not in [{lo[y, x]}, {hi[y, x]}]")
    tight = lo == hi
    assert (~tight).mean() <= max_loose, f"{(~tight).mean():.3f} of the columns have a loose bracket"
    return tight


def expected_normal64(shape, mat, x, y, z, step=1e-3):
    """Gradient of ``f(T(p))`` with respect to the voxel coordinates at (x, y, z), by float64 central differences of
    ``step`` voxels through ``model_points64``: (gradient [n, 3], smooth [n]).  ``smooth`` is false where the forward
    and backward differences disagree by more than 1e-2 of their size (curvature moves them by 1e-4 or so): a crease of the field (a min / max switching
    branch), where a gradient is whichever side the evaluation falls on."""
    p = [np.asarray(a, dtype=np.float64) for a in (x, y, z)]
    f0 = eval64(shape, model_points64(mat, *p))[0]
    g = np.zeros((len(p[0]), 3))
    smooth = np.ones(len(p[0]), dtype=bool)
    for ax in range(3):
        hi_p = [a + (step if i == ax else 0.0) for i, a in enumerate(p)]
        lo_p = [a - (step if i == ax else 0.0) for i, a in enumerate(p)]
        fh = eval64(shape, model_points64(mat, *hi_p))[0]
        fl = eval64(shape, model_points64(mat, *lo_p))[0]
        g[:, ax] = (fh - fl) / (2 * step)
        fwd, bwd = (fh - f0) / step, (f0 - fl) / step
        with np.errstate(invalid="ignore"):
            smooth &= np.abs(fwd - bwd) <= 1e-2 * np.maximum(np.abs(fwd), np.abs(bwd)) + 1e-12
    return g, smooth


# Angle allowed between a float32 normal and the float64 gradient.  The quotient rule (r' w - r w') / w^2 subtracts
# terms of like size, so a handful of float32 roundings (2^-24 each) are magnified by the ratio of those terms to their
# difference, below 100 in the catalogue; the central difference itself is good to 1e-6 of the gradient.  1e-3 rad leaves
# an order of magnitude above both, and is far below the 0.3 rad a sign error in the quotient rule produces.
NORMAL_TOLERANCE = 1e-3


def check_normals(img, shape, mat, tight, depth, min_checked=20):
    """Device normals against ``expected_normal64`` at the columns whose bracket is tight, away from saturated columns,
    creases and vanishing gradients (``depth``: the volume's).  Returns the number of columns checked."""
    d_img = np.asarray(img["depth"], dtype=np.int64)
    hit = tight & (d_img > 0) & (d_img < depth - 1)
    yy, xx = np.nonzero(hit)
    if len(yy) > 4000:                                  # a spread of columns is as good as all of them
        pick = np.random.default_rng(1).choice(len(yy), 4000, replace=False)
        yy, xx = yy[pick], xx[pick]
    zz = d_img[yy, xx] - 1
    want, smooth = expected_normal64(shape, mat, xx, yy, zz)
    got = np.asarray(img["normal"], dtype=np.float64)[yy, xx]
    nw, ng = np.linalg.norm(want, axis=1), np.linalg.norm(got, axis=1)
    ok = smooth & np.isfinite(nw) & np.isfinite(ng) & (nw > 1e-6 * max(float(np.nanmax(nw, initial=0.0)), 1e-30)) & (ng > 0)
    with np.errstate(all="ignore"):
        cosang = np.einsum("ij,ij->i", want, got) / (nw * ng)
        sinang = np.linalg.norm(np.cross(want, got), axis=1) / (nw * ng)
    angle = np.arctan2(sinang, cosang)
    bad = ok & ~(angle < NORMAL_TOLERANCE)
    if bad.any():
        i = int(np.argmax(bad))
        raise AssertionError(f"{int(bad.sum())} of {int(ok.sum())} normals off by more than {NORMAL_TOLERANCE} rad; first at "
                             f"x={xx[i]} y={yy[i]} z={zz[i]}: {got[i]} vs {want[i]} ({angle[i]:.4f} rad)")
    assert ok.sum() >= min_checked, f"only {int(ok.sum())} normals could be checked"
    return int(ok.sum())


FILL_MASK, FILL_TAG = np.uint32(0xFF << 9), np.uint32(0xF6 << 9)


def is_fill(img):
    """Pixels of a RawDistancePixel image that an interval proof filled (pixel.rs:150-183)."""
    return np.isnan(img) & ((img.view(np.uint32) & FILL_MASK) == FILL_TAG)


def check_image2d(img, vals64, band, max_loose=0.05):
    """A 2D render against the float64 field: the sign of every pixel outside the band, and the value of every shaded
    (not filled) pixel within the band of it.  A NaN value is outside, and shades as NaN."""
    fill = is_fill(img)
    inside = np.where(fill, (img.view(np.uint32) & 1) == 1, img < 0.0)
    with np.errstate(invalid="ignore"):
        sure = np.isnan(vals64) | (np.abs(vals64) > band)
        want = vals64 < 0
        bad = sure & (inside != want)
        shaded = ~fill & np.isfinite(vals64) & np.isfinite(band)
        bad |= shaded & ~(np.abs(img.astype(np.float64) - vals64) <= band + U32 * np.abs(vals64))
    if bad.any():
        y, x = np.argwhere(bad)[0]
        raise AssertionError(f"{int(bad.sum())} pixels disagree with float64; first at x={x} y={y}: "
                             f"{img[y, x]!r} (fill {bool(fill[y, x])}) vs {vals64[y, x]!r} +- {band[y, x]:.3g}")
    assert (~sure).mean() <= max_loose, f"{(~sure).mean():.3f} of the pixels lie within the band"
