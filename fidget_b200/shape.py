"""Python face of the CUDA backend, shaped like the reference's API:

  CudaShape            <-> ``Shape<F>`` for a new ``F = CudaFunction``
                           (fidget-core/src/shape/mod.rs:51, eval/mod.rs:80-208)
  .interval_eval etc.  <-> the four evaluators (eval/tracing.rs, eval/bulk.rs)
  RenderConfig2D/3D    <-> pixel::RenderConfig / voxel::RenderConfig
                           (fidget-raster/src/pixel.rs:27-39, voxel.rs:26-36)
  render2d / render3d  <-> pixel::render / voxel::render (pixel.rs:452, voxel.rs:500)
  CancelToken          <-> fidget_core::render::CancelToken (render/config.rs:59-80)

Everything here calls through the C ABI in include/fidget_cuda.h; there is no
CPU implementation behind it.
"""
from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from .host import Context, TapeData

GEOMETRY_PIXEL = np.dtype([("normal", np.float32, 3), ("depth", np.uint32)])


class CudaError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[fc_status {code}] {msg}")
        self.code = code


def _ck(rc):
    if rc != 0:
        raise CudaError(rc, _lib.load().fc_last_error().decode())


def _ptr(a):
    """Raw address of a numpy array or of anything with ``data_ptr()`` (torch)."""
    if a is None:
        return None
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    return C.c_void_p(a.ctypes.data)


def schedule_check(tape: TapeData) -> dict:
    """Host-only: build and symbolically replay the level-0 schedule (waves, chain runs, slot colouring) of
    ``tape``; raises CudaError if the schedule is inconsistent.  Needs no GPU."""
    lib = _lib.load()
    bc = tape.bytecode()
    info = _lib.FcScheduleInfo()
    _ck(lib.fc_schedule_check(bc.words.ctypes.data_as(C.POINTER(C.c_uint32)), len(bc.words), bc.reg_count, bc.mem_count,
                              tape.n_vars, tape.output_count, C.byref(info)))
    return info.as_dict()


class CancelToken:
    """``CancelToken``: a flag another thread sets to stop a render, ``octree_sample``, ``mesh``, ``contour`` or solve in
    flight (the call then returns ``None``).  One byte, read by the library with an acquire load (``fc_ctx_set_cancel``)."""

    def __init__(self):
        self._flag = C.c_uint8(0)

    def cancel(self):
        self._flag.value = 1

    def is_cancelled(self) -> bool:
        return bool(self._flag.value)

    def _address(self):
        return C.c_void_p(C.addressof(self._flag))


class CudaContext:
    """One GPU: stream + scratch arenas (``fc_ctx``)."""

    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        h = C.c_void_p()
        _ck(self._lib.fc_ctx_create(device, C.byref(h)))
        self._h = h
        self.device = device
        self._stream = None
        # the cancel flag is context-wide: a call attaches its token (or none), runs and detaches it under this lock, so
        # that two threads sharing the context cannot run under each other's token
        self._cancel_lock = threading.Lock()
        self._async_cancel = None      # token of the last asynchronous call, re-attached by synchronize()

    def _cancellable(self, token, fn, asynchronous=False):
        """fn() with ``token``'s flag attached; returns fn's status."""
        with self._cancel_lock:
            _ck(self._lib.fc_ctx_set_cancel(self._h, token._address() if token is not None else None))
            try:
                rc = fn()
            finally:
                self._lib.fc_ctx_set_cancel(self._h, None)
            if asynchronous:
                self._async_cancel = token
            return rc

    def close(self):
        if getattr(self, "_h", None):
            self._lib.fc_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def set_stream(self, cuda_stream: int | None):
        """Run on the given cudaStream_t handle (0 = CUDA default stream); None = the context's own stream."""
        if cuda_stream is None:
            _ck(self._lib.fc_ctx_set_stream(self._h, None, 1))
        else:
            _ck(self._lib.fc_ctx_set_stream(self._h, C.c_void_p(cuda_stream), 0))
        self._stream = cuda_stream

    def on_stream(self, cuda_stream: int):
        """Context manager: enqueue on ``cuda_stream`` (e.g. ``torch.cuda.current_stream().cuda_stream``) inside
        the block, then go back to whatever stream was bound before.  A no-op when already bound to it."""
        ctx = self

        class _Bound:
            def __enter__(self_b):
                self_b.prev = getattr(ctx, "_stream", None)
                self_b.changed = self_b.prev != cuda_stream
                if self_b.changed:
                    ctx.set_stream(cuda_stream)
                return ctx

            def __exit__(self_b, *a):
                if self_b.changed:
                    ctx.set_stream(self_b.prev)
                return False

        return _Bound()

    def synchronize(self):
        """Waits for the enqueued work; raises CudaError (code -6, FC_ERR_CANCELLED) when the token of the last
        ``asynchronous=True`` call cancelled it."""
        with self._cancel_lock:
            token, self._async_cancel = self._async_cancel, None
            _ck(self._lib.fc_ctx_set_cancel(self._h, token._address() if token is not None else None))
            try:
                rc = self._lib.fc_ctx_synchronize(self._h)
            finally:
                self._lib.fc_ctx_set_cancel(self._h, None)
        _ck(rc)

    def set_arena_bytes(self, n: int):
        _ck(self._lib.fc_ctx_set_arena_bytes(self._h, n))


class CudaShape:
    """A tape resident on the GPU plus its evaluators."""

    def __init__(self, cuda: CudaContext, tape: TapeData | None = None, *, _handle=None, _axes=None):
        self._lib = cuda._lib
        self.cuda = cuda
        if _handle is None:
            bc = tape.bytecode()
            h = C.c_void_p()
            _ck(self._lib.fc_tape_create(
                cuda._h, bc.words.ctypes.data_as(C.POINTER(C.c_uint32)), len(bc.words), bc.reg_count,
                bc.mem_count, tape.n_vars, tape.output_count, tape.choice_count, C.byref(h)))
            self._h = h
            self._axes = tape.var_slots()
            _ck(self._lib.fc_tape_set_axes(h, *self._axes))
            # input slot -> ("x" | "y" | "z" | "v", var id): what fb.solve binds parameters by
            self._vars = tape.vars()
        else:
            self._h = _handle
            self._axes = _axes
            self._vars = None
        info = _lib.FcTapeInfo()
        _ck(self._lib.fc_tape_get_info(self._h, C.byref(info)))
        self.info = info
        self._eval = None

    @classmethod
    def from_vm(cls, cuda: CudaContext, text: str, n_regs: int = 255):
        ctx, root = Context.from_text(text)
        return cls(cuda, ctx.tape(root, n_regs))

    @classmethod
    def from_blob(cls, cuda: CudaContext, blob: bytes):
        """Loads a serialized tape (``TapeData.serialize`` / ``CudaShape.serialize``): fc_tape_deserialize."""
        h = C.c_void_p()
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        _ck(cuda._lib.fc_tape_deserialize(cuda._h, buf, len(blob), C.byref(h)))
        ax = np.frombuffer(blob, dtype=np.int32, count=3, offset=28)
        return cls(cuda, _handle=h, _axes=tuple(int(a) for a in ax))

    def serialize(self) -> bytes:
        n = C.c_size_t()
        _ck(self._lib.fc_tape_serialize(self._h, None, 0, C.byref(n)))
        buf = (C.c_uint8 * n.value)()
        _ck(self._lib.fc_tape_serialize(self._h, buf, n.value, C.byref(n)))
        return bytes(buf)

    def close(self):
        """Releases the tape and its evaluator now (a second call does nothing).  Both belong to the CudaContext, so
        they must go before ``CudaContext.close``; the shape cannot be used afterwards.  A shape whose context is already
        closed -- the collector frees a reference cycle holding both in any order -- only drops its handles: releasing
        them would read the destroyed context."""
        cuda = getattr(self, "cuda", None)
        if cuda is not None and getattr(cuda, "_h", None) is None:
            self._eval = None
            self._h = None
            return
        if getattr(self, "_eval", None):
            self._lib.fc_eval_destroy(self._eval)
            self._eval = None
        if getattr(self, "_h", None):
            self._lib.fc_tape_release(self._h)
            self._h = None

    def __del__(self):
        self.close()

    # Function::size / choice_count / vars
    def size(self): return self.info.ref_len
    @property
    def choice_count(self): return self.info.choice_count
    @property
    def n_vars(self): return self.info.n_vars

    def _ev(self):
        if self._eval is None:
            h = C.c_void_p()
            _ck(self._lib.fc_eval_create(self.cuda._h, C.byref(h)))
            self._eval = h
        return self._eval

    def bytecode_words(self):
        n = C.c_size_t()
        _ck(self._lib.fc_tape_read(self._h, None, 0, C.byref(n)))
        w = np.zeros(n.value, dtype=np.uint32)
        _ck(self._lib.fc_tape_read(self._h, w.ctypes.data_as(C.POINTER(C.c_uint32)), n.value, C.byref(n)))
        return w

    def compile(self, kinds=("float", "grad", "interval")) -> "CompiledShape":
        """Compiles the tape to sm_90a kernels for the given evaluator kinds with NVRTC (``fc_tape_compile``): host
        time up front, then the same results as this shape's evaluators from kernels that keep values in registers."""
        return CompiledShape(self, kinds)

    # ---- tracing evaluators ------------------------------------------------
    def interval_eval(self, vars_lo_hi):
        """-> (out [n_out,2], choices uint8[choice_count], simplify flag)"""
        v = np.ascontiguousarray(vars_lo_hi, dtype=np.float32).reshape(-1, 2)
        out = np.zeros((self.info.n_outputs, 2), dtype=np.float32)
        ch = np.zeros(max(self.choice_count, 1), dtype=np.uint8)
        s = np.zeros(1, dtype=np.uint8)
        _ck(self._lib.fc_interval_eval(self._ev(), self._h, _ptr(v), _ptr(out), _ptr(ch), _ptr(s)))
        return out, ch[:self.choice_count], bool(s[0])

    def point_eval(self, vars_):
        v = np.ascontiguousarray(vars_, dtype=np.float32)
        out = np.zeros(self.info.n_outputs, dtype=np.float32)
        ch = np.zeros(max(self.choice_count, 1), dtype=np.uint8)
        s = np.zeros(1, dtype=np.uint8)
        _ck(self._lib.fc_point_eval(self._ev(), self._h, _ptr(v), _ptr(out), _ptr(ch), _ptr(s)))
        return out, ch[:self.choice_count], bool(s[0])

    def interval_eval_batch(self, boxes, want_choices=False):
        """boxes: [n, n_vars, 2] -> out [n, n_out, 2] (+ choices [n, choice_count], simplify [n])"""
        return self._interval_batch(self._lib.fc_interval_eval_batch, self._h, boxes, want_choices)

    def _interval_batch(self, fn, h, boxes, want_choices):
        v = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, max(self.n_vars, 1), 2)
        n = v.shape[0]
        out = np.zeros((n, self.info.n_outputs, 2), dtype=np.float32)
        ch = np.zeros((n, max(self.choice_count, 1)), dtype=np.uint8) if want_choices else None
        s = np.zeros(n, dtype=np.uint8)
        _ck(fn(self._ev(), h, _ptr(v), n, _ptr(out), _ptr(ch), _ptr(s)))
        if want_choices:
            return out, ch[:, :self.choice_count], s.astype(bool)
        return out

    # ---- bulk evaluators ---------------------------------------------------
    def float_slice_eval(self, vars_, out=None):
        """vars_: n_vars arrays (numpy or torch, host or device) of n floats"""
        return self._float_slice(self._lib.fc_float_slice_eval, self._h, vars_, out)

    def _float_slice(self, fn, h, vars_, out):
        n = int(vars_[0].shape[0]) if len(vars_) else 0
        host = not (len(vars_) and hasattr(vars_[0], "data_ptr"))
        if host:
            vars_ = [np.ascontiguousarray(v, dtype=np.float32) for v in vars_]
        if out is None:
            if host:
                outs = [np.zeros(n, dtype=np.float32) for _ in range(self.info.n_outputs)]
            else:
                import torch
                outs = [torch.empty(n, dtype=torch.float32, device=vars_[0].device)
                        for _ in range(self.info.n_outputs)]
        else:
            outs = out if isinstance(out, (list, tuple)) else [out]
        va = (C.c_void_p * max(len(vars_), 1))(*[_ptr(v) for v in vars_])
        oa = (C.c_void_p * len(outs))(*[_ptr(o) for o in outs])
        _ck(fn(self._ev(), h, va, oa, n))
        return outs[0] if self.info.n_outputs == 1 else outs

    def grad_slice_eval(self, vars_, out=None):
        """vars_: n_vars arrays [n,4] = {v,dx,dy,dz}"""
        return self._grad_slice(self._lib.fc_grad_slice_eval, self._h, vars_, out)

    def _grad_slice(self, fn, h, vars_, out):
        n = int(vars_[0].shape[0]) if len(vars_) else 0
        host = not (len(vars_) and hasattr(vars_[0], "data_ptr"))
        if host:
            vars_ = [np.ascontiguousarray(v, dtype=np.float32).reshape(-1, 4) for v in vars_]
        if out is None:
            if host:
                outs = [np.zeros((n, 4), dtype=np.float32) for _ in range(self.info.n_outputs)]
            else:
                import torch
                outs = [torch.empty((n, 4), dtype=torch.float32, device=vars_[0].device)
                        for _ in range(self.info.n_outputs)]
        else:
            outs = out if isinstance(out, (list, tuple)) else [out]
        va = (C.c_void_p * max(len(vars_), 1))(*[_ptr(v) for v in vars_])
        oa = (C.c_void_p * len(outs))(*[_ptr(o) for o in outs])
        _ck(fn(self._ev(), h, va, oa, n))
        return outs[0] if self.info.n_outputs == 1 else outs

    def simplify(self, choices) -> "CudaShape":
        c = np.ascontiguousarray(choices, dtype=np.uint8)
        h = C.c_void_p()
        _ck(self._lib.fc_simplify(self._ev(), self._h, _ptr(c), len(c), C.byref(h)))
        child = CudaShape(self.cuda, _handle=h, _axes=self._axes)
        child._vars = self._vars
        return child

    def slot_keys(self) -> list:
        """The variable behind each tape input slot: "x", "y", "z" or the var id of ``Context.var()``.  A shape
        loaded from a blob knows only its axis slots, so another input raises ValueError."""
        if self._vars is not None:
            return [kind if kind in "xyz" else vid for kind, vid in self._vars]
        keys = []
        for s in range(self.n_vars):
            if s in self._axes:
                keys.append("xyz"[self._axes.index(s)])
            else:
                raise ValueError(f"input slot {s} is not an axis, and a shape loaded from a blob does not know which "
                                 "Var it is; build the shape from its TapeData to solve with it")
        return keys


_COMPILE_KINDS = {"float": _lib.FC_COMPILE_FLOAT, "grad": _lib.FC_COMPILE_GRAD, "interval": _lib.FC_COMPILE_INTERVAL}


def _compile_mask(kinds) -> int:
    if isinstance(kinds, str):
        kinds = (kinds,)
    mask = 0
    for k in kinds:
        if k not in _COMPILE_KINDS:
            raise ValueError(f"unknown kind {k!r}: expected some of {sorted(_COMPILE_KINDS)}")
        mask |= _COMPILE_KINDS[k]
    return mask


class CompiledShape:
    """``JitShape``'s counterpart: a CudaShape's tape compiled to sm_90a kernels for some of the bulk evaluators
    (``fc_tape_compile``).  Same signatures, return types and bits as the CudaShape's evaluators; ``info`` has the
    registers, local memory and compile time per kind."""

    def __init__(self, shape: CudaShape, kinds=("float", "grad", "interval")):
        self.shape = shape
        self._lib = shape._lib
        h = C.c_void_p()
        _ck(self._lib.fc_tape_compile(shape.cuda._h, shape._h, _compile_mask(kinds), C.byref(h)))
        self._h = h
        info = _lib.FcCompiledInfo()
        _ck(self._lib.fc_compiled_get_info(h, C.byref(info)))
        self.info = info.as_dict()

    def float_slice_eval(self, vars_, out=None):
        return self.shape._float_slice(self._lib.fc_compiled_float_slice_eval, self._h, vars_, out)

    def grad_slice_eval(self, vars_, out=None):
        return self.shape._grad_slice(self._lib.fc_compiled_grad_slice_eval, self._h, vars_, out)

    def interval_eval_batch(self, boxes, want_choices=False):
        return self.shape._interval_batch(self._lib.fc_compiled_interval_eval_batch, self._h, boxes, want_choices)

    def close(self):
        """Releases the compiled kernels now (a second call does nothing); like ``CudaShape.close``, a handle whose
        context is already closed is only dropped."""
        cuda = getattr(getattr(self, "shape", None), "cuda", None)
        if cuda is not None and getattr(cuda, "_h", None) is None:
            self._h = None
            return
        if getattr(self, "_h", None):
            self._lib.fc_compiled_release(self._h)
            self._h = None

    def __del__(self):
        self.close()


def compile_check(tape: TapeData, kinds=("float", "grad", "interval")):
    """Host-only (no GPU): generate and compile ``tape`` for ``kinds`` with NVRTC (``fc_compile_check``).
    -> (info dict, generated source)"""
    lib = _lib.load()
    bc = tape.bytecode()
    info = _lib.FcCompiledInfo()
    n = C.c_size_t()
    words = bc.words.ctypes.data_as(C.POINTER(C.c_uint32))
    args = (words, len(bc.words), bc.reg_count, bc.mem_count, tape.n_vars, tape.output_count, _compile_mask(kinds))
    cap = 65536 + 256 * len(bc.words)   # above what the generator writes for any tape: one compile, not two
    buf = C.create_string_buffer(cap)
    _ck(lib.fc_compile_check(*args, buf, cap, C.byref(n), C.byref(info)))
    if n.value >= cap:
        buf = C.create_string_buffer(n.value + 1)
        _ck(lib.fc_compile_check(*args, buf, n.value + 1, C.byref(n), C.byref(info)))
    return info.as_dict(), buf.value.decode()


# ---------------------------------------------------------------------------
# Transforms (f32 arithmetic, same operation order as the reference)
_f = np.float32


def screen_to_world_2d(w: int, h: int) -> np.ndarray:
    """RegionSize<2>::screen_to_world (fidget-core/src/render/region.rs:87-108) as a 4x4."""
    cx, cy = _f(w) / _f(2), _f(h) / _f(2) - _f(1)
    s = _f(2) / _f(min(w, h))
    sy = s * _f(-1)
    m = np.eye(4, dtype=np.float32)
    m[0, 0], m[0, 3] = s, -cx * s
    m[1, 1], m[1, 3] = sy, -cy * sy
    return m


def screen_to_world_3d(w: int, h: int, d: int) -> np.ndarray:
    cx, cy, cz = _f(w) / _f(2), _f(h) / _f(2) - _f(1), _f(d) / _f(2)
    s = _f(2) / _f(min(w, h, d))
    sy = s * _f(-1)
    m = np.eye(4, dtype=np.float32)
    m[0, 0], m[0, 3] = s, -cx * s
    m[1, 1], m[1, 3] = sy, -cy * sy
    m[2, 2], m[2, 3] = s, -cz * s
    return m


def _matmul_f32(a, b):
    n = a.shape[0]
    r = np.zeros((n, n), dtype=np.float32)
    for i in range(n):
        for j in range(n):
            acc = _f(0)
            for k in range(n):
                acc = _f(acc + _f(a[i, k] * b[k, j]))
            r[i, j] = acc
    return r


def pixel_mat(w: int, h: int, world_to_model=None) -> np.ndarray:
    """pixel::RenderConfig::mat embedded as 4x4 with Z preserved (pixel.rs:122-124,283-287)."""
    s = screen_to_world_2d(w, h)
    s3 = np.array([[s[0, 0], s[0, 1], s[0, 3]], [s[1, 0], s[1, 1], s[1, 3]], [0, 0, 1]], dtype=np.float32)
    wm = np.eye(3, dtype=np.float32) if world_to_model is None else \
        np.asarray(world_to_model, dtype=np.float32).reshape(3, 3)
    r = _matmul_f32(wm, s3)
    m = np.zeros((4, 4), dtype=np.float32)
    idx = [0, 1, 3]
    for i in range(3):
        for j in range(3):
            m[idx[i], idx[j]] = r[i, j]
    m[2, 2] = 1.0
    return m


def voxel_mat(w: int, h: int, d: int, world_to_model=None) -> np.ndarray:
    """voxel::RenderConfig::mat (voxel.rs:107-109)."""
    s = screen_to_world_3d(w, h, d)
    if world_to_model is None:
        return s
    return _matmul_f32(np.asarray(world_to_model, dtype=np.float32).reshape(4, 4), s)


@dataclass
class RenderConfig2D:
    width: int
    height: int
    world_to_model: np.ndarray | None = None   # 3x3
    pixel_perfect: bool = False
    z: float = 0.0
    tile_sizes: tuple = ()                      # () => backend default (128, 32, 8)
    mat: np.ndarray | None = None               # full 4x4 override
    root_rows: tuple = (0, 0)                   # band of root-tile rows (multi-GPU)
    timing: bool = False
    var_values: tuple = ()                      # ShapeVars: value per tape input slot (axis slots ignored)
    interleave: tuple = (0, 0)                  # (N, r): only the root tiles rank r of N owns (shard.tile_owner)
    out_format: str = "f32"                     # "f32" | "mask_u8" | "bitmap_1bit" | "rgba8"
    fused_tail: bool = False                    # experimental: levels 1.., leaf pixels, fills as one persistent launch
    cancel: CancelToken | None = None           # EvalConfig::cancel: render2d returns None once it is cancelled

    def matrix(self):
        return self.mat if self.mat is not None else pixel_mat(self.width, self.height, self.world_to_model)


@dataclass
class RenderConfig3D:
    width: int
    height: int
    depth: int
    world_to_model: np.ndarray | None = None   # 4x4
    tile_sizes: tuple = ()
    mat: np.ndarray | None = None
    z_range: tuple = (0, 0)
    root_rows: tuple = (0, 0)                   # band of root-tile rows, full depth (multi-GPU)
    timing: bool = False
    var_values: tuple = ()
    clamp: bool = True                          # False for slab renders (fc_merge_slabs applies it)
    interleave: tuple = (0, 0)                  # (N, r): only the root-tile columns rank r of N owns
    exact_census: bool = False                  # stats = the reference's front-to-back census (voxel.rs:244-357)
    full_ladder: bool = False                   # default tile sizes: evaluate all of (128,64,32,16,8), not the device's (128,32,8)
    cancel: CancelToken | None = None           # EvalConfig::cancel: render3d returns None once it is cancelled

    def matrix(self):
        return self.mat if self.mat is not None else voxel_mat(self.width, self.height, self.depth,
                                                               self.world_to_model)


OUT_FORMATS = {"f32": _lib.FC_OUT_F32, "mask_u8": _lib.FC_OUT_MASK_U8, "bitmap_1bit": _lib.FC_OUT_BITMAP_1BIT,
               "rgba8": _lib.FC_OUT_RGBA8}


def _render2d_cfg(cfg: RenderConfig2D, asynchronous: bool) -> _lib.FcRender2dCfg:
    c = _lib.FcRender2dCfg()
    c.width, c.height = cfg.width, cfg.height
    c.mat[:] = np.ascontiguousarray(cfg.matrix(), dtype=np.float32).reshape(16).tolist()
    c.z = cfg.z
    c.pixel_perfect = int(cfg.pixel_perfect)
    c.n_tile_sizes = len(cfg.tile_sizes)
    for i, t in enumerate(cfg.tile_sizes):
        c.tile_sizes[i] = t
    c.flags = (_lib.FC_FLAG_TIMING if cfg.timing else 0) | (_lib.FC_FLAG_ASYNC if asynchronous else 0) | \
        (_lib.FC_FLAG_FUSED_TAIL if cfg.fused_tail else 0)
    c.root_row_begin, c.root_row_end = cfg.root_rows
    c.root_stride, c.root_offset = cfg.interleave
    c.n_var_values = len(cfg.var_values)
    for i, v in enumerate(cfg.var_values):
        c.var_values[i] = float(v)
    c.out_format = OUT_FORMATS[cfg.out_format]
    return c


def _image_shape_2d(cfg: RenderConfig2D) -> tuple:
    """Shape and dtype of one image of ``cfg.out_format``."""
    if cfg.out_format == "f32":
        return (cfg.height, cfg.width), np.float32
    if cfg.out_format == "mask_u8":
        return (cfg.height, cfg.width), np.uint8
    if cfg.out_format == "bitmap_1bit":
        return (cfg.height, (cfg.width + 7) // 8), np.uint8
    return (cfg.height, cfg.width, 4), np.uint8


def _check_out(out, need: int):
    """A caller-given ``out`` must be one contiguous buffer of at least ``need`` bytes: the library writes that many."""
    if hasattr(out, "data_ptr"):   # torch
        contiguous, nbytes = out.is_contiguous(), out.numel() * out.element_size()
    else:
        contiguous, nbytes = out.flags["C_CONTIGUOUS"], out.nbytes
    if not contiguous:
        raise ValueError("out must be contiguous")
    if nbytes < need:
        raise ValueError(f"out holds {nbytes} bytes, the call writes {need}")


def render2d(shape: CudaShape, cfg: RenderConfig2D, out=None, stats: bool = False, asynchronous: bool = False):
    """pixel::render.  ``out``: None (returns a numpy float32 [h,w] of
    RawDistancePixel bits), a numpy array, or a CUDA torch tensor.  None when ``cfg.cancel`` cancelled it."""
    lib = shape._lib
    c = _render2d_cfg(cfg, asynchronous)
    if out is None:
        dims, dtype = _image_shape_2d(cfg)
        out = np.zeros(dims, dtype=dtype)
    st = _lib.FcRenderStats() if stats else None
    rc = shape.cuda._cancellable(cfg.cancel, lambda: lib.fc_render2d(shape.cuda._h, shape._h, C.byref(c), _ptr(out),
                                                                     C.byref(st) if stats else None), asynchronous)
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, st.as_dict()) if stats else out


def _per_frame(what: str, z=None, var_values=None, mats=(), none_ok: bool = False):
    """The per-frame (per-``what``) arguments of a table builder that are given, checked and converted: ``z`` [n],
    ``var_values`` [n, k] with k <= FC_MAX_VARS, and each ``(name, value, r)`` of ``mats`` an [n, r, r] stack of
    matrices -- with ``none_ok`` a sequence whose entries may also be None.  Returns ``(per, n)``: ``per`` maps each
    given name to its values; lengths that disagree raise ValueError, and with nothing given n is 1."""
    per = {}
    if z is not None:
        per["z"] = np.asarray(z, dtype=np.float32).reshape(-1)
    if var_values is not None:
        vv = np.asarray(var_values, dtype=np.float32)
        if vv.ndim != 2 or vv.shape[1] > _lib.FC_MAX_VARS:
            raise ValueError(f"var_values must be [n, k] with k <= {_lib.FC_MAX_VARS}")
        per["var_values"] = vv
    for name, m, r in mats:
        if m is None:
            continue
        if none_ok:
            m = [None if w is None else np.asarray(w, dtype=np.float32) for w in m]
            if any(w is not None and w.shape != (r, r) for w in m):
                raise ValueError(f"{name} must be [n, {r}, {r}] (an entry may be None: no transform)")
        else:
            m = np.asarray(m, dtype=np.float32)
            if m.ndim != 3 or m.shape[1:] != (r, r):
                raise ValueError(f"{name} must be [n, {r}, {r}]")
        per[name] = m
    lengths = {k: len(v) for k, v in per.items()}
    if len(set(lengths.values())) > 1:
        raise ValueError(f"per-{what} arguments disagree in length: {lengths}")
    return per, next(iter(lengths.values()), 1)


def _set_vars(rec, values):
    """``n_var_values`` and ``var_values`` of a C record"""
    rec.n_var_values = len(values)
    for i, v in enumerate(values):
        rec.var_values[i] = float(v)


def frame_table(cfg: RenderConfig2D, z=None, var_values=None, world_to_model=None, mats=None):
    """The ``fc_frame2d`` table of ``render2d_frames``: frame k's matrix, Z and ShapeVars, each exactly what
    ``render2d`` puts into ``fc_render2d_cfg`` for the config ``cfg`` with that frame's values.  Every argument
    given is per frame (leading dimension n: ``z`` [n], ``var_values`` [n, k], ``world_to_model`` [n, 3, 3],
    ``mats`` [n, 4, 4]); the others come from ``cfg``.  Lengths that disagree raise ValueError; with no per-frame
    argument at all there is one frame.  ``mats`` and ``world_to_model`` are exclusive."""
    if mats is not None and world_to_model is not None:
        raise ValueError("give mats or world_to_model, not both")
    per, n = _per_frame("frame", z=z, var_values=var_values, mats=(("world_to_model", world_to_model, 3),
                                                                    ("mats", mats, 4)))
    table = (_lib.FcFrame2d * n)()
    base = None if ("mats" in per or "world_to_model" in per) else \
        np.ascontiguousarray(cfg.matrix(), dtype=np.float32).reshape(16).tolist()
    for k in range(n):
        f = table[k]
        if "mats" in per:
            f.mat[:] = per["mats"][k].reshape(16).tolist()
        elif "world_to_model" in per:
            f.mat[:] = pixel_mat(cfg.width, cfg.height, per["world_to_model"][k]).reshape(16).tolist()
        else:
            f.mat[:] = base
        f.z = float(per["z"][k]) if "z" in per else cfg.z
        _set_vars(f, per["var_values"][k] if "var_values" in per else cfg.var_values)
    return table


def render2d_frames(shape: CudaShape, cfg: RenderConfig2D, z=None, var_values=None, world_to_model=None, mats=None,
                    out=None, stats: bool = False, asynchronous: bool = False):
    """Many frames of ``shape`` in one call (``fc_render2d_frames``): frame k is bit for bit ``render2d`` of ``cfg``
    with frame k's ``z`` / ``var_values`` / ``world_to_model`` / ``mats`` (see ``frame_table``).  Returns a numpy
    array [n, h, w] (f32, mask_u8), [n, h, (w + 7) // 8] (bitmap_1bit) or [n, h, w, 4] (rgba8), or fills ``out``
    (a numpy array or CUDA tensor of that many bytes).  None when ``cfg.cancel`` cancelled it."""
    lib = shape._lib
    table = frame_table(cfg, z=z, var_values=var_values, world_to_model=world_to_model, mats=mats)
    n = len(table)
    c = _render2d_cfg(cfg, asynchronous)
    dims, dtype = _image_shape_2d(cfg)
    if out is None:
        out = np.zeros((n,) + dims, dtype=dtype)
    else:   # n frames of the format, back to back
        _check_out(out, n * int(np.prod(dims)) * np.dtype(dtype).itemsize)
    st = _lib.FcRenderStats() if stats else None
    rc = shape.cuda._cancellable(cfg.cancel, lambda: lib.fc_render2d_frames(
        shape.cuda._h, shape._h, C.byref(c), table, n, _ptr(out), C.byref(st) if stats else None), asynchronous)
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, st.as_dict()) if stats else out


def _render3d_cfg(cfg: RenderConfig3D, asynchronous: bool) -> _lib.FcRender3dCfg:
    c = _lib.FcRender3dCfg()
    c.width, c.height, c.depth = cfg.width, cfg.height, cfg.depth
    c.mat[:] = np.ascontiguousarray(cfg.matrix(), dtype=np.float32).reshape(16).tolist()
    c.n_tile_sizes = len(cfg.tile_sizes)
    for i, t in enumerate(cfg.tile_sizes):
        c.tile_sizes[i] = t
    c.flags = (_lib.FC_FLAG_TIMING if cfg.timing else 0) | (_lib.FC_FLAG_ASYNC if asynchronous else 0) | \
        (0 if cfg.clamp else _lib.FC_FLAG_NO_CLAMP) | (_lib.FC_FLAG_EXACT_CENSUS if cfg.exact_census else 0) | \
        (_lib.FC_FLAG_FULL_LADDER if cfg.full_ladder else 0)
    c.z_begin, c.z_end = cfg.z_range
    c.root_row_begin, c.root_row_end = cfg.root_rows
    c.root_stride, c.root_offset = cfg.interleave
    c.n_var_values = len(cfg.var_values)
    for i, v in enumerate(cfg.var_values):
        c.var_values[i] = float(v)
    return c


def render3d(shape: CudaShape, cfg: RenderConfig3D, out=None, stats: bool = False, asynchronous: bool = False):
    """voxel::render -> numpy structured array [h,w] of GEOMETRY_PIXEL (or fills ``out``); None when ``cfg.cancel``
    cancelled it."""
    lib = shape._lib
    c = _render3d_cfg(cfg, asynchronous)
    if out is None:
        out = np.zeros((cfg.height, cfg.width), dtype=GEOMETRY_PIXEL)
    st = _lib.FcRenderStats() if stats else None
    rc = shape.cuda._cancellable(cfg.cancel, lambda: lib.fc_render3d(shape.cuda._h, shape._h, C.byref(c), _ptr(out),
                                                                     C.byref(st) if stats else None), asynchronous)
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, st.as_dict()) if stats else out


def frame_table_3d(cfg: RenderConfig3D, var_values=None, world_to_model=None, mats=None):
    """The ``fc_frame3d`` table of ``render3d_frames``: frame k's matrix and ShapeVars, each exactly what ``render3d``
    puts into ``fc_render3d_cfg`` for the config ``cfg`` with that frame's values: ``voxel_mat(w, h, d,
    world_to_model[k])``, or ``mats[k]``, and ``var_values[k]``.  Every argument given is per frame (leading dimension
    n: ``var_values`` [n, k], ``world_to_model`` [n, 4, 4], ``mats`` [n, 4, 4]); the others come from ``cfg``.
    Lengths that disagree raise ValueError; with no per-frame argument at all there is one frame.  ``mats`` and
    ``world_to_model`` are exclusive."""
    if mats is not None and world_to_model is not None:
        raise ValueError("give mats or world_to_model, not both")
    per, n = _per_frame("frame", var_values=var_values, mats=(("world_to_model", world_to_model, 4), ("mats", mats, 4)))
    table = (_lib.FcFrame3d * n)()
    base = None if ("mats" in per or "world_to_model" in per) else \
        np.ascontiguousarray(cfg.matrix(), dtype=np.float32).reshape(16).tolist()
    for k in range(n):
        f = table[k]
        if "mats" in per:
            f.mat[:] = per["mats"][k].reshape(16).tolist()
        elif "world_to_model" in per:
            f.mat[:] = voxel_mat(cfg.width, cfg.height, cfg.depth, per["world_to_model"][k]).reshape(16).tolist()
        else:
            f.mat[:] = base
        _set_vars(f, per["var_values"][k] if "var_values" in per else cfg.var_values)
    return table


def render3d_frames(shape: CudaShape, cfg: RenderConfig3D, var_values=None, world_to_model=None, mats=None, out=None,
                    stats: bool = False, asynchronous: bool = False):
    """Many 3D frames of ``shape`` in one call (``fc_render3d_frames``): frame k is bit for bit ``render3d`` of
    ``cfg`` with frame k's ``var_values`` / ``world_to_model`` / ``mats`` (see ``frame_table_3d``).  Returns a numpy
    structured array [n, h, w] of GEOMETRY_PIXEL, or fills ``out`` (a numpy array or CUDA tensor of that many bytes,
    contiguous).  None when ``cfg.cancel`` cancelled it."""
    lib = shape._lib
    table = frame_table_3d(cfg, var_values=var_values, world_to_model=world_to_model, mats=mats)
    n = len(table)
    c = _render3d_cfg(cfg, asynchronous)
    if out is None:
        out = np.zeros((n, cfg.height, cfg.width), dtype=GEOMETRY_PIXEL)
    else:
        _check_out(out, n * cfg.height * cfg.width * GEOMETRY_PIXEL.itemsize)
    st = _lib.FcRenderStats() if stats else None
    rc = shape.cuda._cancellable(cfg.cancel, lambda: lib.fc_render3d_frames(
        shape.cuda._h, shape._h, C.byref(c), table, n, _ptr(out), C.byref(st) if stats else None), asynchronous)
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, st.as_dict()) if stats else out


def scene_table(cfg: RenderConfig3D, n: int, var_values=None, world_to_model=None, mats=None):
    """The ``fc_frame3d`` placement table of ``render3d_scene`` for ``n`` shapes: entry k is what ``frame_table_3d``
    gives for placement k's values (``world_to_model`` [n, 4, 4], ``mats`` [n, 4, 4], ``var_values`` [n, k]).  What is
    not given per placement comes from ``cfg``, for all n; lengths other than n raise ValueError."""
    return _scene_table(lambda **per: frame_table_3d(cfg, **per), n, var_values=var_values,
                        world_to_model=world_to_model, mats=mats)


def _scene_table(build, n: int, **given):
    """The placement table of a scene of n shapes: ``build(**per)`` (``frame_table`` or ``frame_table_3d`` of the
    scene's config) of the per-placement arguments given, each of length n; with none given, n copies of its one
    frame."""
    per = {name: v for name, v in given.items() if v is not None}
    for name, v in per.items():
        if len(v) != n:
            raise ValueError(f"{name} has {len(v)} entries for {n} shapes")
    if not per:   # every placement is cfg's own view (Z) and vars
        one = build()[0]
        return (type(one) * n)(*[one] * n)
    return build(**per)


def render3d_scene(shapes, cfg: RenderConfig3D, var_values=None, world_to_model=None, mats=None, out=None,
                   index_out=None, stats: bool = False, asynchronous: bool = False):
    """Several shapes rendered into one image (``fc_render3d_scene``): a viewer's draw list, or fidget-wgpu's merge
    of voxel images.  Shape k is ``shapes[k]`` placed by entry k of ``scene_table`` (per-placement ``var_values`` /
    ``world_to_model`` / ``mats``, leading dimension ``len(shapes)``; the rest from ``cfg``).  Each pixel is that of
    the per-shape ``render3d`` image with the greatest depth (after the final clamp), the lowest k on equal depth, bit
    for bit; ``index`` holds that k (0 where every image is empty).  Returns ``(image, index)`` -- GEOMETRY_PIXEL
    [h, w] and uint16 [h, w], or the given ``out`` / ``index_out`` (numpy arrays or CUDA tensors of that many bytes,
    contiguous) -- plus the stats with ``stats=True``; None when ``cfg.cancel`` cancelled it.  Without ``index_out`` the
    index lands next to ``out``: a numpy uint16 array for a host ``out``, an int16 CUDA tensor (the same bits) on
    ``out``'s device for a CUDA ``out``, so that ``asynchronous=True`` stays asynchronous.  All shapes must live on one
    CudaContext."""
    shapes = list(shapes)
    n = len(shapes)
    if n == 0:
        raise ValueError("a scene needs at least one shape")
    lib, cuda = shapes[0]._lib, shapes[0].cuda
    if any(sh.cuda is not cuda for sh in shapes):
        raise ValueError("the shapes of a scene must belong to one CudaContext")
    table = scene_table(cfg, n, var_values=var_values, world_to_model=world_to_model, mats=mats)
    c = _render3d_cfg(cfg, asynchronous)
    if out is None:
        out = np.zeros((cfg.height, cfg.width), dtype=GEOMETRY_PIXEL)
    else:
        _check_out(out, cfg.height * cfg.width * GEOMETRY_PIXEL.itemsize)
    if index_out is None and getattr(out, "is_cuda", False):
        import torch
        index_out = torch.zeros((cfg.height, cfg.width), dtype=torch.int16, device=out.device)
    elif index_out is None:
        index_out = np.zeros((cfg.height, cfg.width), dtype=np.uint16)
    else:
        _check_out(index_out, cfg.height * cfg.width * 2)
    handles = (C.c_void_p * n)(*[sh._h for sh in shapes])
    st = _lib.FcRenderStats() if stats else None
    rc = cuda._cancellable(cfg.cancel, lambda: lib.fc_render3d_scene(
        cuda._h, handles, table, n, C.byref(c), _ptr(out), _ptr(index_out), C.byref(st) if stats else None), asynchronous)
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, index_out, st.as_dict()) if stats else (out, index_out)


def scene_table_2d(cfg: RenderConfig2D, n: int, z=None, var_values=None, world_to_model=None, mats=None):
    """The ``fc_frame2d`` placement table of ``render2d_scene`` for ``n`` shapes: entry k is what ``frame_table`` gives
    for placement k's values (``z`` [n], ``var_values`` [n, k], ``world_to_model`` [n, 3, 3], ``mats`` [n, 4, 4]).  What
    is not given per placement comes from ``cfg``, for all n; lengths other than n raise ValueError."""
    return _scene_table(lambda **per: frame_table(cfg, **per), n, z=z, var_values=var_values,
                        world_to_model=world_to_model, mats=mats)


def scene_colors(colors, n: int) -> np.ndarray:
    """The [n, 3] uint8 colour table of ``render2d_scene``.  uint8 input is taken as is; other numbers are converted
    per channel as the viewer's ``draw_rgb`` does: below 0 -> 0, above 1 -> 255, otherwise ``a * 255`` truncated (in
    f64), NaN -> 0."""
    a = np.asarray(colors)
    if a.shape != (n, 3):
        raise ValueError(f"colors must be [{n}, 3], got {list(a.shape)}")
    if a.dtype == np.uint8:
        return np.ascontiguousarray(a)
    a = a.astype(np.float64)
    with np.errstate(invalid="ignore"):
        out = np.where(a < 0.0, 0.0, np.where(a > 1.0, 255.0, np.trunc(a * 255.0)))
    return np.nan_to_num(out, nan=0.0).astype(np.uint8)


def render2d_scene(shapes, cfg: RenderConfig2D, colors=None, z=None, var_values=None, world_to_model=None, mats=None,
                   out=None, index_out=None, stats: bool = False, asynchronous: bool = False):
    """A 2D draw list in one call (``fc_render2d_scene``): the viewer's 2D mode, each shape painted opaque over the
    ones before it.  Shape k is ``shapes[k]`` placed by entry k of ``scene_table_2d`` (per-placement ``z`` /
    ``var_values`` / ``world_to_model`` / ``mats``, leading dimension ``len(shapes)``; the rest from ``cfg``).
    ``index`` holds, per pixel, the last k whose ``render2d`` is inside there (``FC_SCENE2D_NONE`` where none is), bit
    for bit; the image is ``cfg.out_format`` of that: "rgba8" the colour of shape k (``colors``, see ``scene_colors``;
    None: white) with alpha 255 and zeros elsewhere, "mask_u8" / "bitmap_1bit" the union of the shapes.  "f32" is
    refused.  Returns ``(image, index)`` -- or the given ``out`` / ``index_out`` (numpy arrays or CUDA tensors of that
    many bytes, contiguous) -- plus the stats with ``stats=True``; None when ``cfg.cancel`` cancelled it.  Without
    ``index_out`` the index lands next to ``out``: a numpy uint16 array for a host ``out``, an int16 CUDA tensor (the
    same bits) on ``out``'s device for a CUDA ``out``.  All shapes must live on one CudaContext."""
    shapes = list(shapes)
    n = len(shapes)
    if n == 0:
        raise ValueError("a scene needs at least one shape")
    lib, cuda = shapes[0]._lib, shapes[0].cuda
    if any(sh.cuda is not cuda for sh in shapes):
        raise ValueError("the shapes of a scene must belong to one CudaContext")
    table = scene_table_2d(cfg, n, z=z, var_values=var_values, world_to_model=world_to_model, mats=mats)
    col = scene_colors(colors, n) if colors is not None else None
    c = _render2d_cfg(cfg, asynchronous)
    dims, dtype = _image_shape_2d(cfg)
    if out is None:
        out = np.zeros(dims, dtype=dtype)
    else:
        _check_out(out, int(np.prod(dims)) * np.dtype(dtype).itemsize)
    if index_out is None and getattr(out, "is_cuda", False):
        import torch
        index_out = torch.zeros((cfg.height, cfg.width), dtype=torch.int16, device=out.device)
    elif index_out is None:
        index_out = np.zeros((cfg.height, cfg.width), dtype=np.uint16)
    else:
        _check_out(index_out, cfg.height * cfg.width * 2)
    handles = (C.c_void_p * n)(*[sh._h for sh in shapes])
    st = _lib.FcRenderStats() if stats else None
    rc = cuda._cancellable(cfg.cancel, lambda: lib.fc_render2d_scene(
        cuda._h, handles, table, n, C.byref(c), None if col is None else col.ctypes.data, _ptr(out), _ptr(index_out),
        C.byref(st) if stats else None), asynchronous)
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, index_out, st.as_dict()) if stats else (out, index_out)


OCTREE_LEAF =np.dtype([("ix", np.uint16), ("iy", np.uint16), ("iz", np.uint16), ("mask", np.uint8),
                        ("n_edges", np.uint8), ("present", np.uint16), ("pad", np.uint16),
                        ("pos", np.float32, (12, 3)), ("grad", np.float32, (12, 4))])


def _octree_cfg(depth: int, timing: bool, collapse: bool = False, world_to_model=None, var_values=()):
    """The ``fc_octree_cfg`` of ``octree_sample``, ``mesh``, ``mesh_frames`` and ``measure``"""
    c = _lib.FcOctreeCfg()
    c.depth = depth
    c.flags = (_lib.FC_FLAG_TIMING if timing else 0) | (_lib.FC_FLAG_MESH_COLLAPSE if collapse else 0)
    if world_to_model is not None:
        c.has_transform = 1
        c.world_to_model[:] = np.ascontiguousarray(world_to_model, dtype=np.float32).reshape(16).tolist()
    _set_vars(c, var_values)
    return c


def octree_sample(shape: CudaShape, depth: int, world_to_model=None, capacity: int | None = None,
                  stats: bool = False, timing: bool = False, var_values=(), cancel: CancelToken | None = None):
    """Sampler half of ``fidget_mesh::Octree::build`` (octree.rs:521-808): surface leaves with their
    corner mask and per-edge Hermite data, sorted by (iz, iy, ix).  None when ``cancel`` cancelled it."""
    lib = shape._lib
    c = _octree_cfg(depth, timing, world_to_model=world_to_model, var_values=var_values)
    cap = capacity if capacity is not None else max(1024, min(8 ** depth, 6 * 4 ** depth))
    st = _lib.FcOctreeStats()
    while True:
        out = np.zeros(cap, dtype=OCTREE_LEAF)
        n = C.c_uint64()
        rc = shape.cuda._cancellable(cancel, lambda: lib.fc_octree_sample(shape.cuda._h, shape._h, C.byref(c), _ptr(out),
                                                                          cap, C.byref(n), C.byref(st)))
        if rc == _lib.FC_ERR_CANCELLED:
            return None
        if rc != 0 and n.value > cap and capacity is None:
            cap = int(n.value)          # retry once with the exact count
            continue
        _ck(rc)
        break
    leaves = out[:n.value]
    leaves = leaves[np.lexsort((leaves["ix"], leaves["iy"], leaves["iz"]))]
    return (leaves, st.as_dict()) if stats else leaves


def mesh(shape: CudaShape, depth: int, world_to_model=None, var_values=(), stl: bool = False, collapse: bool = False,
         cancel: CancelToken | None = None):
    """``Octree::build(...).walk_dual()`` (fidget-mesh): returns ``(vertices [n,3] float32, triangles [m,3] uint32,
    info dict)`` -- plus the binary STL bytes (``Mesh::write_stl``) when ``stl``.  Without ``collapse`` the mesh is
    the uniform-depth one (no cell collapse); with it, cells are collapsed as the reference's octree does and the
    dual is walked over leaves of different depths (``mesh_cells`` then lists the final leaves).  None when
    ``cancel`` cancelled the build (the context then holds no mesh)."""
    lib = shape._lib
    c = _octree_cfg(depth, True, collapse, world_to_model=world_to_model, var_values=var_values)
    info = _lib.FcMeshInfo()
    rc = shape.cuda._cancellable(cancel, lambda: lib.fc_mesh_build(shape.cuda._h, shape._h, C.byref(c), C.byref(info)))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    verts, tris, _, buf = _mesh_read(shape.cuda, info, stl=stl)
    return (verts, tris, info.as_dict(), buf) if stl else (verts, tris, info.as_dict())


MESH_CELL = np.dtype([("ix", np.uint16), ("iy", np.uint16), ("iz", np.uint16), ("depth", np.uint8), ("mask", np.uint8),
                      ("vertex", np.float32, 3)])


def _mesh_read(cuda, info, cells: bool = False, stl: bool = False):
    """The context's mesh of ``info``'s counts: ``(vertices [n, 3], triangles [m, 3], final leaves, binary STL bytes)``,
    the leaves (in the library's order) with ``cells`` and the STL with ``stl``, else None"""
    lib = cuda._lib
    verts = np.zeros((info.n_vertices, 3), dtype=np.float32)
    tris = np.zeros((info.n_triangles, 3), dtype=np.uint32)
    _ck(lib.fc_mesh_read(cuda._h, _ptr(verts), _ptr(tris)))
    buf = None
    if stl:
        n = C.c_size_t()
        _ck(lib.fc_mesh_write_stl(cuda._h, None, 0, C.byref(n)))
        buf = np.zeros(n.value, dtype=np.uint8)
        _ck(lib.fc_mesh_write_stl(cuda._h, _ptr(buf), n.value, C.byref(n)))
        buf = buf.tobytes()
    return verts, tris, _read_cells(cuda) if cells else None, buf


def _read_cells(cuda) -> np.ndarray:
    """The final leaves of the context's mesh, in the library's order (frame by frame)"""
    lib = cuda._lib
    n = C.c_uint64()
    _ck(lib.fc_mesh_read_cells(cuda._h, None, 0, C.byref(n)))
    out = np.zeros(n.value, dtype=MESH_CELL)
    _ck(lib.fc_mesh_read_cells(cuda._h, _ptr(out), n.value, C.byref(n)))
    return out


def mesh_cells(cuda) -> np.ndarray:
    """Final leaves of the octree of the context's last ``mesh(..., collapse=True)``: depth, cell coordinates at
    that depth, corner mask and first cell vertex, sorted by (depth, iz, iy, ix).  Empty after a uniform mesh."""
    return _sorted_cells(_read_cells(cuda))


def mesh_frame_table(world_to_model=None, var_values=None):
    """The ``fc_mesh_frame`` table of ``mesh_frames``: frame k's ``world_to_model`` (4x4, world -> model) and ShapeVars,
    each what ``mesh`` puts into ``fc_octree_cfg`` for that frame's values.  Every argument given is per frame (leading
    dimension n: ``world_to_model`` [n, 4, 4], ``var_values`` [n, k]); the other takes ``mesh``'s default (no transform,
    no values).  A ``world_to_model`` entry of None is a frame without a transform, as ``mesh``'s
    ``world_to_model=None``.  Lengths that disagree raise ValueError, as in ``contour_slice_table``; with no per-frame
    argument at all there is one frame."""
    per, n = _per_frame("frame", var_values=var_values, mats=(("world_to_model", world_to_model, 4),), none_ok=True)
    table = (_lib.FcMeshFrame * n)()
    for k in range(n):
        f = table[k]
        if "world_to_model" in per and per["world_to_model"][k] is not None:
            f.has_transform = 1
            f.world_to_model[:] = per["world_to_model"][k].reshape(16).tolist()
        _set_vars(f, per["var_values"][k] if "var_values" in per else ())
    return table


def split_mesh_frames(vertices, triangles, per_frame, cells=None):
    """The per-frame ``(vertices, triangles)`` (and final leaves, with ``cells``) of a batch's read buffers: frame k
    takes the next ``n_vertices`` / ``n_triangles`` / ``n_cells`` rows of ``per_frame[k]``; its triangle indices are
    already local to its vertices.  Counts that do not add up to the buffers' lengths raise ValueError."""
    v = np.asarray(vertices, dtype=np.float32).reshape(-1, 3)
    t = np.asarray(triangles, dtype=np.uint32).reshape(-1, 3)
    out, pv, pt, pc = [], 0, 0, 0
    for p in per_frame:
        nv, nt = int(p["n_vertices"]), int(p["n_triangles"])
        part = [v[pv:pv + nv], t[pt:pt + nt]]
        if cells is not None:
            nc = int(p["n_cells"])
            part.append(cells[pc:pc + nc])
            pc += nc
        out.append(tuple(part))
        pv, pt = pv + nv, pt + nt
    if pv != len(v) or pt != len(t) or (cells is not None and pc != len(cells)):
        raise ValueError("per-frame counts do not add up to the batch's")
    return out


def split_mesh_stl(buf, n_triangles):
    """The per-frame binary STL files of a batch's ``fc_mesh_write_stl`` output: frame k's takes 84 + 50 n_k bytes.
    Counts that do not add up to the buffer's length raise ValueError."""
    b = bytes(buf)
    out, p = [], 0
    for nt in n_triangles:
        size = 84 + 50 * int(nt)
        out.append(b[p:p + size])
        p += size
    if p != len(b):
        raise ValueError("per-frame triangle counts do not add up to the STL's length")
    return out


def _sorted_cells(cells):
    return cells[np.lexsort((cells["ix"], cells["iy"], cells["iz"], cells["depth"]))]


def mesh_frames(shape: CudaShape, depth: int, world_to_model=None, var_values=None, collapse: bool = False,
                stl: bool = False, cells: bool = False, cancel: CancelToken | None = None):
    """Meshes of many frames in one call (``fc_mesh_build_frames``): frame k is ``mesh`` of its own
    ``world_to_model`` / ``var_values`` (see ``mesh_frame_table``), the same vertices bit for bit and the same
    triangles.  Returns ``(frames, info, per_frame)``: ``frames[k] = (vertices, triangles)``, plus frame k's binary STL
    bytes when ``stl`` and its final leaves (sorted as ``mesh_cells`` sorts them) when ``cells``; ``info`` the totals
    (device times summed over passes) and ``per_frame[k]`` frame k's counts.  None when ``cancel`` cancelled the call
    (the context then holds no mesh)."""
    lib = shape._lib
    table = mesh_frame_table(world_to_model=world_to_model, var_values=var_values)
    n = len(table)
    c = _octree_cfg(depth, True, collapse)
    info = _lib.FcMeshInfo()
    per = (_lib.FcMeshFrameInfo * n)()
    rc = shape.cuda._cancellable(cancel, lambda: lib.fc_mesh_build_frames(
        shape.cuda._h, shape._h, C.byref(c), table, n, C.byref(info), per))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    verts, tris, all_cells, buf = _mesh_read(shape.cuda, info, cells=cells, stl=stl)
    per_frame = [p.as_dict() for p in per]
    frames = split_mesh_frames(verts, tris, per_frame, all_cells)
    if cells:
        frames = [(v, t, _sorted_cells(cl)) for v, t, cl in frames]
    if stl:
        files = split_mesh_stl(buf, [p["n_triangles"] for p in per_frame])
        frames = [(f[0], f[1], files[k]) + tuple(f[2:]) for k, f in enumerate(frames)]
    return frames, info.as_dict(), per_frame


# fc_measure_result as a numpy record (one row per frame)
MEASURE_RESULT = np.dtype([("n_inside", np.uint64), ("n_proven", np.uint64), ("n_undecided", np.uint64),
                           ("s1", np.uint64, 3), ("s2", np.uint64, 6), ("lo", np.uint32, 3), ("hi", np.uint32, 3),
                           ("volume", np.float64), ("volume_lo", np.float64), ("volume_hi", np.float64),
                           ("centroid", np.float64, 3), ("inertia", np.float64, 6), ("bbox_min", np.float64, 3),
                           ("bbox_max", np.float64, 3)])


def measure(shape: CudaShape, depth: int, world_to_model=None, var_values=None, cancel: CancelToken | None = None,
            timing: bool = False):
    """Volume, centroid, inertia and bounding box of the shape's voxel solid at ``depth`` (``fc_measure``), per frame:
    ``world_to_model`` / ``var_values`` are per-frame as in ``mesh_frame_table`` (a single 4x4 matrix or a 1-D value
    list is one frame; with neither there is one frame).  Returns a ``MEASURE_RESULT`` array with one row per frame --
    the exact integer sums and counts, and the float64 results in model space -- and with ``timing`` also the device
    time in ms.  None when ``cancel`` cancelled the call."""
    lib = shape._lib
    if world_to_model is not None and not isinstance(world_to_model, (list, tuple)) and \
            np.asarray(world_to_model).shape == (4, 4):
        world_to_model = [world_to_model]
    if var_values is not None and np.asarray(var_values, dtype=np.float32).ndim == 1:
        var_values = [var_values]
    table = mesh_frame_table(world_to_model=world_to_model, var_values=var_values)
    n = len(table)
    c = _octree_cfg(depth, timing)
    out = np.zeros(n, dtype=MEASURE_RESULT)
    ms = C.c_float()
    rc = shape.cuda._cancellable(cancel, lambda: lib.fc_measure(shape.cuda._h, shape._h, C.byref(c), table, n, _ptr(out),
                                                                C.byref(ms)))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return (out, ms.value) if timing else out


class Volume:
    """A sparse narrow-band volume (``fc_volume_build``), in its canonical order:

    - ``bricks``: [n, 4] int32 rows (frame, ix, iy, iz), each brick's first cell;
    - ``values``: [n, B, B, B] float32, indexed [z, y, x] inside the brick; ``grads``: [n, B, B, B, 3] or None;
    - ``tiles``: [m, 6] int32 rows (frame, ix, iy, iz, log2_edge, inside) of the proven tiles;
    - ``per_frame``: dict of [n_frames] int64 arrays n_bricks, n_tiles, first_brick, first_tile; ``info``: a dict.

    numpy arrays, or with ``device=True`` CUDA torch tensors (``per_frame`` and ``info`` stay on the host)."""

    def __init__(self, depth, band, bricks, values, grads, tiles, per_frame, info):
        self.depth, self.band = depth, band
        self.brick_edge = info["brick_edge"]
        self.bricks, self.values, self.grads, self.tiles = bricks, values, grads, tiles
        self.per_frame, self.info = per_frame, info


def _volume_rows(raw, n, words, torch_dev):
    """fc_volume_brick / fc_volume_tile records (12 bytes each, raw bytes) as [n, 4] / [n, 6] int32 rows"""
    if torch_dev is not None:
        import torch
        u16 = raw[:, 4:10].contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
        cols = [raw[:, 0:4].contiguous().view(torch.int32), u16]
        if words == 6:
            cols.append(raw[:, 10:12].to(torch.int32))
        return torch.cat(cols, 1)
    u32 = raw[:, 0:4].copy().view(np.uint32).astype(np.int32)
    u16 = raw[:, 4:10].copy().view(np.uint16).astype(np.int32)
    cols = [u32, u16] + ([raw[:, 10:12].astype(np.int32)] if words == 6 else [])
    return np.concatenate(cols, 1).reshape(n, words)


def volume(shape: CudaShape, depth: int, band: float = 0.0, world_to_model=None, var_values=None, grads: bool = False,
           device: bool = False, cancel: CancelToken | None = None, timing: bool = False):
    """The shape's field at the cell centres of the depth-``depth`` grid of [-1,1]^3, as 8^3 bricks where the interval
    octree cannot rule out |v| <= ``band`` and proven inside / outside tiles everywhere else (``fc_volume_build``).
    ``world_to_model`` / ``var_values`` are per-frame as in ``measure``.  Returns a ``Volume``, None when ``cancel``
    cancelled the call."""
    lib = shape._lib
    if world_to_model is not None and not isinstance(world_to_model, (list, tuple)) and \
            np.asarray(world_to_model).shape == (4, 4):
        world_to_model = [world_to_model]
    if var_values is not None and np.asarray(var_values, dtype=np.float32).ndim == 1:
        var_values = [var_values]
    table = mesh_frame_table(world_to_model=world_to_model, var_values=var_values)
    n = len(table)
    c = _lib.FcVolumeCfg()
    c.depth = depth
    c.band = band
    c.flags = (_lib.FC_FLAG_TIMING if timing else 0) | (_lib.FC_FLAG_VOLUME_GRADS if grads else 0)
    info = _lib.FcVolumeInfo()
    per = (_lib.FcVolumeFrameInfo * max(n, 1))()
    cuda = shape.cuda
    rc = cuda._cancellable(cancel, lambda: lib.fc_volume_build(cuda._h, shape._h, C.byref(c), table, n, C.byref(info),
                                                               per))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    d = info.as_dict()
    B, nb, nt = d["brick_edge"], d["n_bricks"], d["n_tiles"]
    pf = {k: np.array([getattr(per[i], k) for i in range(n)], dtype=np.int64)
          for k in ("n_bricks", "n_tiles", "first_brick", "first_tile")}
    torch_dev = None
    if device:
        import torch
        torch_dev = torch.device("cuda", cuda.device)
        raw_b = torch.empty((nb, 12), dtype=torch.uint8, device=torch_dev)
        vals = torch.empty((nb, B, B, B), dtype=torch.float32, device=torch_dev)
        grd = torch.empty((nb, B, B, B, 3), dtype=torch.float32, device=torch_dev) if grads else None
        raw_t = torch.empty((nt, 12), dtype=torch.uint8, device=torch_dev)
    else:
        raw_b = np.empty((nb, 12), dtype=np.uint8)
        vals = np.empty((nb, B, B, B), dtype=np.float32)
        grd = np.empty((nb, B, B, B, 3), dtype=np.float32) if grads else None
        raw_t = np.empty((nt, 12), dtype=np.uint8)
    _ck(lib.fc_volume_read(cuda._h, _ptr(raw_b) if nb else None, _ptr(vals) if nb else None,
                           _ptr(grd) if grads and nb else None, _ptr(raw_t) if nt else None))
    return Volume(depth, band, _volume_rows(raw_b, nb, 4, torch_dev), vals, grd, _volume_rows(raw_t, nt, 6, torch_dev),
                  pf, d)


def volume_dense(vol: Volume, frame: int = 0, inside: float = -np.inf, outside: float = np.inf):
    """Frame ``frame`` of a ``Volume`` as a dense [2^D, 2^D, 2^D] float32 array indexed [z, y, x]: the brick values,
    ``inside`` in inside tiles and ``outside`` in outside tiles (numpy, or torch on the volume's device).  For small
    depths: the array has 8^D cells."""
    n, B = 1 << vol.depth, vol.brick_edge
    if hasattr(vol.values, "data_ptr"):
        import torch
        out = torch.full((n, n, n), float("nan"), dtype=torch.float32, device=vol.values.device)
        tiles, bricks = vol.tiles.cpu().numpy(), vol.bricks.cpu().numpy()
    else:
        out = np.full((n, n, n), np.nan, dtype=np.float32)
        tiles, bricks = vol.tiles, vol.bricks
    for f, ix, iy, iz, lg, ins in tiles[tiles[:, 0] == frame].tolist():
        e = 1 << lg
        out[iz:iz + e, iy:iy + e, ix:ix + e] = inside if ins else outside
    for r in np.nonzero(bricks[:, 0] == frame)[0].tolist():
        _, ix, iy, iz = bricks[r].tolist()
        out[iz:iz + B, iy:iy + B, ix:ix + B] = vol.values[r]
    return out


# ---------------------------------------------------------------------------
# Ray casts: fc_raycast
RAY = np.dtype([("origin", np.float32, 3), ("dir", np.float32, 3), ("t0", np.float32), ("dt", np.float32)])
RAY_HIT = np.dtype([("k", np.uint32), ("flags", np.uint32), ("t", np.float32), ("pos", np.float32, 3),
                    ("value", np.float32), ("grad", np.float32, 3)])


def _ray_columns(origins, dirs, t0, dt, n, torch_dev):
    """The [n, 8] float32 rows of fc_ray (origin, dir, t0, dt), numpy or on the tensors' device"""
    if torch_dev is not None:
        import torch

        def col(v):
            v = torch.as_tensor(v, dtype=torch.float32, device=torch_dev)
            return (v.reshape(-1) if v.numel() == n else v.reshape(()).expand(n)).reshape(n, 1)
        return torch.cat([origins.reshape(n, 3).float(), dirs.reshape(n, 3).float(), col(t0), col(dt)], 1).contiguous()
    rays = np.zeros(n, dtype=RAY)
    rays["origin"] = np.asarray(origins, dtype=np.float32).reshape(n, 3)
    rays["dir"] = np.asarray(dirs, dtype=np.float32).reshape(n, 3)
    rays["t0"] = np.broadcast_to(np.asarray(t0, dtype=np.float32).reshape(-1), (n,))
    rays["dt"] = np.broadcast_to(np.asarray(dt, dtype=np.float32).reshape(-1), (n,))
    return rays


def raycast(shape: CudaShape, origins, dirs, t0, dt, steps: int, var_values=(), cancel: CancelToken | None = None,
            timing: bool = False):
    """The first inside sample of each ray (``fc_raycast``): ray i samples ``origins[i] + t_k * dirs[i]`` at
    ``t_k = t0 + k * dt``, k < ``steps``, in model space, f32 with one rounding per operation.  ``origins`` and ``dirs``
    are [n, 3]; ``t0`` and ``dt`` scalars or [n].  numpy inputs give numpy outputs; CUDA torch tensors stay on the device
    and give tensors there.  Returns ``(k, t, pos, value, grad, proven, info)``: k (``FC_RAY_MISS`` = 0xFFFFFFFF for a
    miss, as int64 for tensors), t, pos [n, 3], the root tape's value and gradient [n, 3] at pos, proven (the hit is
    the first sample of an interval-proven-inside segment) and the info dict of ``fc_raycast_info``.  ``var_values``
    bind the tape's other inputs (ShapeVars).  None when ``cancel`` cancelled the call."""
    lib = shape._lib
    torch_dev = origins.device if hasattr(origins, "data_ptr") and getattr(origins, "is_cuda", False) else None
    n = int(origins.shape[0]) if hasattr(origins, "shape") else len(origins)
    rays = _ray_columns(origins, dirs, t0, dt, n, torch_dev)
    if torch_dev is not None:
        import torch
        hits = torch.empty((n, 10), dtype=torch.float32, device=torch_dev)
        torch.cuda.synchronize(torch_dev)   # (the rays are built on torch's stream; the call runs on the context's)
    else:
        hits = np.zeros(n, dtype=RAY_HIT)
    c = _lib.FcRaycastCfg()
    c.steps = steps
    c.flags = _lib.FC_FLAG_TIMING if timing else 0
    _set_vars(c, var_values)
    info = _lib.FcRaycastInfo()
    rc = shape.cuda._cancellable(cancel, lambda: lib.fc_raycast(shape.cuda._h, shape._h, C.byref(c), _ptr(rays), n,
                                                                _ptr(hits), C.byref(info)))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    if torch_dev is not None:
        import torch
        words = hits.view(torch.int32)
        k = words[:, 0].to(torch.int64) & 0xFFFFFFFF
        proven = (words[:, 1] & _lib.FC_RAY_PROVEN) != 0
        return k, hits[:, 2], hits[:, 3:6], hits[:, 6], hits[:, 7:10], proven, info.as_dict()
    return (hits["k"], hits["t"], hits["pos"], hits["value"], hits["grad"], (hits["flags"] & _lib.FC_RAY_PROVEN) != 0,
            info.as_dict())


def pick_rays(cfg: RenderConfig3D, pixels):
    """The model-space rays of ``pick``: for screen pixel (x, y), origin = the voxel (x, y, depth - 1) under
    ``cfg.matrix()`` (f32, as the renderer maps voxels: ((m0 x + m1 y) + m2 z) + m3), dir = minus the matrix's Z column,
    t0 = 0, dt = 1, so that sample k lies on voxel (x, y, depth - 1 - k).  Returns ``(origins [n, 3], dirs [n, 3])``;
    ValueError for a projective matrix (last row other than 0 0 0 1)."""
    m = np.asarray(cfg.matrix(), dtype=np.float32).reshape(4, 4)
    if not np.array_equal(m[3], np.array([0, 0, 0, 1], dtype=np.float32)):
        raise ValueError("pick needs an affine view (the matrix's last row 0 0 0 1)")
    px = np.asarray(pixels).reshape(-1, 2)
    x, y = px[:, 0].astype(np.float32), px[:, 1].astype(np.float32)
    z = np.float32(cfg.depth - 1)
    origins = np.stack([((m[i, 0] * x + m[i, 1] * y) + m[i, 2] * z) + m[i, 3] for i in range(3)], 1).astype(np.float32)
    dirs = np.broadcast_to(-m[:3, 2], origins.shape).astype(np.float32)
    return origins, dirs


def pick(shape: CudaShape, cfg: RenderConfig3D, pixels, cancel: CancelToken | None = None):
    """What lies under screen pixels (x, y) of a 3D view (``pixels`` [n, 2]): each pixel's ray runs down its voxel column
    from z = depth - 1 to 0 (``pick_rays``, ``steps`` = depth) through ``fc_raycast``.  Returns ``(depth, pos, normal)``:
    the depth ``fc_render3d`` stores for the pixel (depth - k for a hit at sample k, 0 for a miss, and with
    ``cfg.clamp`` depth for anything at depth - 1 or above, voxel.rs:535-546), the model-space position of the hit and
    the root tape's model-space gradient there (0 for a miss).  Affine views only.  The samples are the renderer's voxel
    positions bit for bit, and the depth equals ``render3d``'s, when every coordinate is exact in f32: an identity
    view (no ``world_to_model``) of power-of-two sizes.  Other views sample the same column up to rounding.  None when
    ``cancel`` cancelled the call."""
    origins, dirs = pick_rays(cfg, pixels)
    r = raycast(shape, origins, dirs, 0.0, 1.0, cfg.depth, var_values=cfg.var_values, cancel=cancel)
    if r is None:
        return None
    k, _, pos, _, grad, _, _ = r
    hit = k != _lib.FC_RAY_MISS
    depth = np.where(hit, np.uint32(cfg.depth) - np.where(hit, k, 0), 0).astype(np.uint32)
    if cfg.clamp:
        depth = np.where(depth >= cfg.depth - 1, cfg.depth, depth).astype(np.uint32)
    return depth, pos, grad


# ---------------------------------------------------------------------------
# 2D contours (libfive's Contours::render): fc_contour_build / fc_contour_read
def contour(shape: CudaShape, depth: int, z: float = 0.0, world_to_model=None, var_values=(),
            cancel: CancelToken | None = None):
    """Contours of the shape's Z slice over the [-1, 1]^2 world square, by dual contouring on a uniform quadtree of
    ``depth`` (fc_contour_build): returns ``(vertices [n,2] float32, offsets [k+1] uint32, closed [k] bool, info dict)``,
    polyline i being ``vertices[offsets[i]:offsets[i + 1]]``.  Inside regions lie on the left of the direction of travel
    (counter-clockwise, y up) in the world square; a mirroring ``world_to_model`` (3x3, world -> model, as the 2D
    renderers take it) reverses it in model space.  The order is canonical, so two builds give the same arrays.  None
    when ``cancel`` cancelled the build (the context then holds no contour)."""
    lib = shape._lib
    c = _lib.FcContourCfg()
    c.depth = depth
    c.z = z
    if world_to_model is not None:
        c.has_transform = 1
        c.world_to_model[:] = np.ascontiguousarray(world_to_model, dtype=np.float32).reshape(9).tolist()
    c.flags = _lib.FC_FLAG_TIMING
    c.n_var_values = len(var_values)          # (more than FC_MAX_VARS is refused by the library)
    for i, v in enumerate(var_values[:_lib.FC_MAX_VARS]):
        c.var_values[i] = float(v)
    info = _lib.FcContourInfo()
    rc = shape.cuda._cancellable(cancel, lambda: lib.fc_contour_build(shape.cuda._h, shape._h, C.byref(c), C.byref(info)))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    return _contour_read(shape.cuda, info) + (info.as_dict(),)


def _contour_read(cuda, info):
    """The context's contour of ``info``'s counts: ``(vertices [n, 2], offsets [k + 1], closed [k] bool)``"""
    verts = np.zeros((info.n_vertices, 2), dtype=np.float32)
    offsets = np.zeros(info.n_polylines + 1, dtype=np.uint32)
    closed = np.zeros(info.n_polylines, dtype=np.uint8)
    _ck(cuda._lib.fc_contour_read(cuda._h, _ptr(verts), _ptr(offsets), _ptr(closed)))
    return verts, offsets, closed.astype(bool)


def contour_slice_table(z=None, world_to_model=None, var_values=None):
    """The ``fc_contour_slice`` table of ``contour_slices``: slice k's Z, ``world_to_model`` (3x3, world -> model) and
    ShapeVars, each what ``contour`` puts into ``fc_contour_cfg`` for that slice's values.  Every argument given is per
    slice (leading dimension n: ``z`` [n], ``world_to_model`` [n, 3, 3], ``var_values`` [n, k]); the others take
    ``contour``'s defaults (z = 0, no transform, no values).  A ``world_to_model`` entry of None is a slice without a
    transform, as ``contour``'s ``world_to_model=None`` (not the same as the identity flagged as a transform: a
    non-finite z then becomes NaN).  Lengths that disagree raise ValueError, as in
    ``frame_table``; with no per-slice argument at all there is one slice."""
    per, n = _per_frame("slice", z=z, var_values=var_values, mats=(("world_to_model", world_to_model, 3),), none_ok=True)
    table = (_lib.FcContourSlice * n)()
    for k in range(n):
        s = table[k]
        s.z = float(per["z"][k]) if "z" in per else 0.0
        if "world_to_model" in per and per["world_to_model"][k] is not None:
            s.has_transform = 1
            s.world_to_model[:] = per["world_to_model"][k].reshape(9).tolist()
        _set_vars(s, per["var_values"][k] if "var_values" in per else ())
    return table


def split_contour_stack(vertices, offsets, closed, n_polylines):
    """The per-slice ``(vertices, offsets, closed)`` of a stacked contour: slice k takes the next ``n_polylines[k]``
    polylines, its offsets rebased to 0 -- each exactly what ``contour`` returns for that slice."""
    v = np.asarray(vertices, dtype=np.float32).reshape(-1, 2)
    off = np.asarray(offsets, dtype=np.uint32)
    cl = np.asarray(closed).astype(bool)
    out, p = [], 0
    for npk in n_polylines:
        npk = int(npk)
        o = off[p:p + npk + 1]
        out.append((v[int(o[0]):int(o[-1])], (o - o[0]).astype(np.uint32), cl[p:p + npk]))
        p += npk
    if p != len(cl) or len(off) != p + 1:
        raise ValueError("per-slice polyline counts do not add up to the stack's")
    return out


def contour_slices(shape: CudaShape, depth: int, z=None, world_to_model=None, var_values=None,
                   cancel: CancelToken | None = None):
    """Contours of many slices in one call (``fc_contour_build_slices``): slice k is bit for bit ``contour`` of its
    own ``z`` / ``world_to_model`` / ``var_values`` (see ``contour_slice_table``).  Returns ``(slices, info,
    per_slice)``: ``slices[k] = (vertices, offsets, closed)`` as ``contour`` returns them, ``info`` the totals (device
    times summed over passes) and ``per_slice[k]`` slice k's counts.  None when ``cancel`` cancelled the call (the
    context then holds no contour)."""
    lib = shape._lib
    table = contour_slice_table(z=z, world_to_model=world_to_model, var_values=var_values)
    n = len(table)
    c = _lib.FcContourCfg()
    c.depth = depth
    c.flags = _lib.FC_FLAG_TIMING
    info = _lib.FcContourInfo()
    per = (_lib.FcContourInfo * n)()
    rc = shape.cuda._cancellable(cancel, lambda: lib.fc_contour_build_slices(
        shape.cuda._h, shape._h, C.byref(c), table, n, C.byref(info), per))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    per_slice = [p.as_dict() for p in per]
    slices = split_contour_stack(*_contour_read(shape.cuda, info), [p["n_polylines"] for p in per_slice])
    return slices, info.as_dict(), per_slice


def contours_svg(vertices, offsets, closed, size: float = 512.0, stroke: str = "black", fill: str = "none",
                 stroke_width: float = 1.0) -> str:
    """An SVG document with one ``<path>`` per polyline of ``contour``'s output, closed ones ending in ``Z``.  The
    view box is the [-1, 1]^2 square (``size`` pixels wide), y flipped to SVG's y-down frame.  Paths use
    ``fill-rule="nonzero"``: the contours' consistent orientation makes a hole wind opposite to its outline."""
    v = np.asarray(vertices, dtype=np.float32).reshape(-1, 2)
    off = np.asarray(offsets, dtype=np.int64)
    cl = np.asarray(closed, dtype=bool)
    out = [f'<svg xmlns="http://www.w3.org/2000/svg" width="{size:g}" height="{size:g}" viewBox="-1 -1 2 2">']
    for k in range(len(off) - 1):
        pts = v[off[k]:off[k + 1]]
        d = " ".join(("M" if i == 0 else "L") + f"{float(x)!r},{-float(y)!r}" for i, (x, y) in enumerate(pts))
        if cl[k]:
            d += " Z"
        out.append(f'<path d="{d}" fill="{fill}" fill-rule="nonzero" stroke="{stroke}" '
                   f'stroke-width="{stroke_width * 2.0 / size:g}"/>')
    out.append("</svg>")
    return "\n".join(out) + "\n"


# ---------------------------------------------------------------------------
# Constraint solver (fidget-solver/src/lib.rs): fc_solve_batch, fc_solve_large_batch
@dataclass(frozen=True)
class Free:
    """``Parameter::Free``: a variable the solver moves, starting at ``value``."""
    value: float


@dataclass(frozen=True)
class Fixed:
    """``Parameter::Fixed``: a variable held at ``value``."""
    value: float


def _solve_call(fn, constraints, free, fixed, values, max_iters, cancel):
    """fc_solve_batch / fc_solve_large_batch (``fn``): the shared staging of solve_batch and solve_large_batch"""
    constraints = list(constraints)
    if not constraints:
        raise ValueError(f"{fn[3:]} needs at least one constraint")
    cuda = constraints[0].cuda
    lib = cuda._lib
    free, fixed = list(free), list(fixed)
    keys = free + fixed
    index = {k: i for i, k in enumerate(keys)}
    if len(index) != len(keys):
        raise ValueError("a variable is listed twice")
    maps = [np.array([index.get(k, -1) for k in c.slot_keys()], dtype=np.int32) for c in constraints]
    device = hasattr(values, "data_ptr") and values.is_cuda
    if device:
        import torch
        vals = values.to(torch.float32).reshape(-1, len(keys)).contiguous().clone()
        res = torch.zeros((vals.shape[0], 4), dtype=torch.int32, device=vals.device)
        torch.cuda.current_stream(vals.device).synchronize()   # the library works on its own stream
    else:
        vals = np.array(values, dtype=np.float32, order="C", copy=True).reshape(-1, len(keys))
        res = np.zeros((vals.shape[0], 4), dtype=np.int32)
    tapes = (C.c_void_p * len(constraints))(*[c._h for c in constraints])
    sp = (C.POINTER(C.c_int32) * len(maps))(*[m.ctypes.data_as(C.POINTER(C.c_int32)) for m in maps])
    cfg = _lib.FcSolveCfg(len(keys), len(free), 0 if max_iters is None else int(max_iters))
    call = getattr(lib, fn)
    rc = cuda._cancellable(cancel, lambda: call(cuda._h, tapes, len(constraints), sp, C.byref(cfg), _ptr(vals),
                                                int(vals.shape[0]), _ptr(res)))
    if rc == _lib.FC_ERR_CANCELLED:
        return None
    _ck(rc)
    if device:
        import torch
        return vals, res[:, 0].clone(), res[:, 1].clone(), res.view(torch.float32)[:, 2].clone()
    return vals, res[:, 0].astype(np.uint32), res[:, 1].astype(np.uint32), res.view(np.float32)[:, 2].copy()


def solve_batch(constraints, free, fixed, values, max_iters=None, cancel: CancelToken | None = None):
    """Levenberg-Marquardt least squares on the constraints' output 0, for many problems at once
    (``fc_solve_batch``).  ``free`` / ``fixed``: the variable keys ("x", "y", "z" or ``Context.var()`` ids); the free
    ones are the Jacobian's columns, in this order.  ``values``: [n_problems, len(free) + len(fixed)] starting values
    of the free variables followed by the fixed ones -- a numpy array, or a CUDA torch tensor (the work and the
    results then stay on the device).  ``max_iters``: step cap (default 1000).
    Returns ``(values, status, iterations, err)``: a copy of ``values`` with the free entries solved, and per problem
    the exit (``FC_SOLVE_*``), the number of steps and the final squared error.  None when ``cancel`` cancelled it."""
    return _solve_call("fc_solve_batch", constraints, free, fixed, values, max_iters, cancel)


def solve_large_batch(constraints, free, fixed, values, max_iters=None, cancel: CancelToken | None = None):
    """``solve_batch`` for problems of up to 1024 free variables, 4096 constraints and 16384 variables in all
    (``fc_solve_large_batch``: one problem per thread-block cluster).  Same arguments and return; on every problem
    ``solve_batch`` accepts, the same bits.  None when ``cancel`` cancelled it."""
    return _solve_call("fc_solve_large_batch", constraints, free, fixed, values, max_iters, cancel)


def solve(constraints, params: dict, max_iters=None, cancel: CancelToken | None = None) -> dict | None:
    """``fidget_solver::solve``: ``params`` maps variable keys ("x", "y", "z" or ``Context.var()`` ids) to
    ``Free(start)`` / ``Fixed(value)``; returns {key: solved value} for the free ones, or None when ``cancel``
    cancelled it.  Problems beyond ``solve_batch``'s limits go to ``solve_large_batch``."""
    for k, p in params.items():
        if not isinstance(p, (Free, Fixed)):
            raise TypeError(f"parameter {k!r} must be Free(..) or Fixed(..), not {p!r}")
    free = [k for k, p in params.items() if isinstance(p, Free)]
    fixed = [k for k, p in params.items() if isinstance(p, Fixed)]
    row = [params[k].value for k in free] + [params[k].value for k in fixed]
    constraints = list(constraints)
    small = (len(free) <= _lib.FC_SOLVE_MAX_FREE and len(constraints) <= _lib.FC_SOLVE_MAX_CONSTRAINTS
             and len(free) + len(fixed) <= _lib.FC_SOLVE_MAX_PARAMS)
    out = (solve_batch if small else solve_large_batch)(constraints, free, fixed, np.array([row], dtype=np.float32),
                                                        max_iters, cancel)
    if out is None:
        return None
    return {k: float(out[0][0, i]) for i, k in enumerate(free)}


def pixel_inside(img: np.ndarray) -> np.ndarray:
    """RawDistancePixel::inside (pixel.rs:177-183)."""
    bits = img.view(np.uint32)
    is_fill = np.isnan(img) & ((bits & np.uint32(0xFF << 9)) == np.uint32(0xF6 << 9))
    return np.where(is_fill, (bits & 1) == 1, img < 0.0)
