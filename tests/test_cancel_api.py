"""Cancellation's C ABI and Python face (fc_ctx_set_cancel, FC_ERR_CANCELLED, fb.CancelToken) on a machine without a
GPU: the header, the ctypes mirror and the Rust binding agree, and the new keywords default to no token."""
import inspect
import os
import re

import fidget_b200 as fb
from fidget_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "fidget_cuda.h")) as f:
        return f.read()


def test_header_declares_cancelled_status():
    m = re.search(r"\bFC_ERR_CANCELLED\s*=\s*(-?\d+)", _header())
    assert m and int(m.group(1)) == -6
    assert _lib.FC_ERR_CANCELLED == -6


def test_set_cancel_is_exported_and_bound():
    assert re.search(r"int32_t\s+fc_ctx_set_cancel\s*\(\s*fc_ctx\s*\*\s*ctx\s*,\s*const\s+uint8_t\s*\*\s*flag\s*\)", _header())
    lib = _lib.load()
    assert hasattr(lib, "fc_ctx_set_cancel")
    assert _lib.CUDA_API["fc_ctx_set_cancel"] == (_lib._i32, [_lib._vp, _lib._vp])
    with open(os.path.join(ROOT, "bindings", "rust", "ffi.rs")) as f:
        rs = f.read()
    assert "pub fn fc_ctx_set_cancel(ctx: *mut fc_ctx, flag: *const u8) -> i32;" in rs
    assert "pub const FC_ERR_CANCELLED: i32 = -6;" in rs


def test_set_cancel_rejects_a_null_context():
    lib = _lib.load()
    assert lib.fc_ctx_set_cancel(None, None) == -1


def test_cancel_token_semantics():
    t = fb.CancelToken()
    assert not t.is_cancelled()
    t.cancel()
    assert t.is_cancelled()
    t.cancel()                                   # idempotent, like AtomicBool::store(true)
    assert t.is_cancelled()
    u = fb.CancelToken()
    assert not u.is_cancelled()                  # tokens do not share their flag
    # the flag is one byte the library reads in place: nonzero once cancelled
    import ctypes as C
    assert C.c_uint8.from_address(t._address().value).value == 1
    assert C.c_uint8.from_address(u._address().value).value == 0


def test_new_keywords_default_to_no_token():
    assert fb.RenderConfig2D(8, 8).cancel is None
    assert fb.RenderConfig3D(8, 8, 8).cancel is None
    assert inspect.signature(fb.octree_sample).parameters["cancel"].default is None
    assert inspect.signature(fb.mesh).parameters["cancel"].default is None
