"""Compiled tapes on the host (fc_compile_check, no GPU): every model and every (opcode, form) generates a source that
NVRTC compiles for sm_90a, each clause calls the dev_ops function its interpreter handler calls, immediates keep their
exact bits, and a missing NVRTC is reported without touching anything else in the library."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import fidget_b200 as fb
import op_reference as R
from conftest import MODELS, model_text

KINDS = ("float", "grad", "interval")
SMALL_MODELS = sorted(f for f in os.listdir(MODELS) if f.endswith(".vm") and f != "prospero.vm")

# The interpreter call behind each (opcode, form) per kind: k_float_slice (float), k_grad_slice (grad) and
# run_interval's handlers (interval)
GRAD_SPECIAL = {("add", f): "gr_add" for f in ("rr", "ri", "ir")}
GRAD_SPECIAL.update({("sub", f): "gr_sub" for f in ("rr", "ri", "ir")})
GRAD_SPECIAL.update({("mul", "rr"): "gr_mul", ("mul", "ri"): "gr_mul_f", ("mul", "ir"): "gr_mul"})
GRAD_SPECIAL.update({("div", f): "gr_div" for f in ("rr", "ri", "ir")})
GRAD_SPECIAL.update({("neg", "r"): "gr_neg", ("square", "r"): "gr_mul"})
IV_SPECIAL = {("add", f): "iv_add" for f in ("rr", "ri", "ir")}
IV_SPECIAL.update({("sub", f): "iv_sub" for f in ("rr", "ri", "ir")})
IV_SPECIAL.update({("mul", "rr"): "iv_mul", ("mul", "ri"): "iv_mul_f", ("mul", "ir"): "iv_mul"})
IV_SPECIAL.update({("neg", "r"): "iv_neg", ("abs", "r"): "iv_abs", ("sqrt", "r"): "iv_sqrt",
                   ("square", "r"): "iv_square"})
CHOICE = {"min", "max", "and", "or"}


def expected_call(kind, op, form):
    unary = form == "r"
    if kind == "float":
        return "f32_unary" if unary else "f32_binary"
    if kind == "grad":
        return GRAD_SPECIAL.get((op, form), "gr_unary" if unary else "gr_binary")
    if op in CHOICE:
        return "iv_choice_op"
    return IV_SPECIAL.get((op, form), "iv_unary" if unary else "iv_binary")


def kernel_body(source, kind):
    name = {"float": "fc_compiled_f32", "grad": "fc_compiled_grad", "interval": "fc_compiled_interval"}[kind]
    i = source.index(name)
    return source[i:source.index("\n}\n", i)]


def _check(info, kinds):
    mask = sum({"float": 1, "grad": 2, "interval": 4}[k] for k in kinds)
    assert info["kinds"] == mask
    assert info["nvrtc_version"] >= 11010 and info["cubin_bytes"] > 0
    for i, k in enumerate(KINDS):
        if k in kinds:
            assert 0 < info["regs"][i] <= 255 and info["compile_ms"][i] > 0, (k, info)
        else:
            assert info["regs"][i] == 0 and info["compile_ms"][i] == 0, (k, info)


@pytest.mark.parametrize("name", SMALL_MODELS)
@pytest.mark.parametrize("n_regs", [255, 24, 12, 6])
def test_every_model_compiles_for_every_kind(name, n_regs):
    ctx, root = fb.Context.from_text(model_text(name))
    td = ctx.tape(root, n_regs)
    info, src = fb.compile_check(td, KINDS)
    _check(info, KINDS)
    if td.bytecode().mem_count:
        assert re.search(r"\bm\d+ = ", src) and re.search(r"= m\d+;", src), "memory slots are locals too"


@pytest.mark.parametrize("kind", KINDS)
def test_prospero_compiles(kind):
    ctx, root = fb.Context.from_text(model_text("prospero.vm"))
    info, src = fb.compile_check(ctx.tape(root), (kind,))
    _check(info, (kind,))
    assert kernel_body(src, kind).count("opq(") > 6000


def test_names_come_from_registers_not_from_the_text():
    """quarter.vm has an SSA value named `out`, colonnade.vm reads Z: neither name reaches the source."""
    for name in ("quarter.vm", "colonnade.vm"):
        text = model_text(name)
        ctx, root = fb.Context.from_text(text)
        td = ctx.tape(root)
        info, src = fb.compile_check(td, KINDS)
        _check(info, KINDS)
        assert td.n_vars == 3 or name != "colonnade.vm"
        for k in KINDS:
            body = kernel_body(src, k)
            declared = set(re.findall(r"\b(?:float|float2|float4) (\w+) = ", body))
            assert declared and all(re.fullmatch(r"[rm]\d+", d) for d in declared), (name, k, declared)
    assert re.search(r"(?m)^_?\w* *out\b|\bout ", model_text("quarter.vm"))


@pytest.mark.parametrize("op", R.UNARY + R.BINARY)
def test_every_opcode_and_form_calls_its_interpreter_function(op):
    forms = ["r"] if op in R.UNARY else ["rr"] + R.FORMS[op]
    for form in forms:
        c = fb.Context()
        if form == "r":
            td = c.tape(c.unary(op, c.x()))
        elif form == "rr":
            td = c.tape(c.binary(op, c.x(), c.y()))
        elif form == "ri":
            td = c.tape(c.binary(op, c.x(), c.constant(0.75)))
        else:
            td = c.tape(c.binary(op, c.constant(0.75), c.x()))
        info, src = fb.compile_check(td, KINDS)
        _check(info, KINDS)
        opname = "OP_" + op.upper()
        for k in KINDS:
            body = kernel_body(src, k)
            fn = expected_call(k, op, form)
            assert re.search(r"opq\(%s\(" % fn, body), (op, form, k, fn)
            takes_op = fn in ("f32_unary", "f32_binary", "gr_unary", "gr_binary", "iv_unary", "iv_binary",
                              "iv_choice_op")
            assert (opname in body) == takes_op, (op, form, k)
            if k == "interval" and op in CHOICE:
                assert "ch[0] = uint8_t(c)" in body


def test_immediates_are_bit_patterns():
    specials = {"-0.0": 0x80000000, "nan payload": 0x7FC01234, "+inf": 0x7F800000, "-inf": 0xFF800000,
                "denormal": 0x00000123}
    c = fb.Context()
    x = c.x()
    roots = []
    for bits in specials.values():
        k = float(np.array([bits], dtype=np.uint32).view(np.float32)[0])
        roots += [c.constant(k), c.binary("mul", x, c.constant(k))]
    info, src = fb.compile_check(c.tape(roots), KINDS)
    _check(info, KINDS)
    table = src[src.index("uint32_t fc_imm["):]
    for label, bits in specials.items():
        assert "0x%08xu" % bits in table, label
    assert not re.search(r"\b(nan|inf|NAN|INFINITY)\b", table.split("};")[0])


def test_multi_output_and_inputless_tapes_compile():
    c = fb.Context()
    x, y, z = c.x(), c.y(), c.z()
    roots = [c.binary("min", x, y), c.binary("max", y, z), c.unary("sqrt", c.binary("add", x, z))]
    info, src = fb.compile_check(c.tape(roots), KINDS)
    _check(info, KINDS)
    for o in range(3):
        assert "out%d[idx] = " % o in kernel_body(src, "float")
        assert "o[%d] = " % (2 * o) in kernel_body(src, "interval")
    c = fb.Context()
    td = c.tape(c.constant(2.5))
    assert td.n_vars == 0
    info, src = fb.compile_check(td, KINDS)
    _check(info, KINDS)


def test_shape_vars_beyond_xyz_compile():
    c = fb.Context()
    v, w = c.var()[0], c.var()[0]
    td = c.tape(c.binary("add", c.binary("mul", c.x(), v), w))
    assert td.n_vars >= 3
    info, src = fb.compile_check(td, KINDS)
    _check(info, KINDS)


def test_bad_kinds_are_refused():
    c = fb.Context()
    td = c.tape(c.x())
    with pytest.raises(ValueError):
        fb.compile_check(td, ("jit",))
    with pytest.raises(fb.CudaError) as e:
        fb.compile_check(td, ())
    assert e.value.code == -1


def test_missing_nvrtc_is_reported_and_changes_nothing_else(tmp_path):
    missing = str(tmp_path / "no" / "libnvrtc.so.12")
    code = f"""
import ctypes as C, sys
sys.path.insert(0, {os.path.dirname(os.path.dirname(os.path.abspath(__file__)))!r})
import fidget_b200 as fb
from fidget_b200 import _lib
lib = _lib.load()
for name in _lib.CUDA_API:
    assert hasattr(lib, name), name
c = fb.Context()
try:
    fb.compile_check(c.tape(c.x()), ("float",))
except fb.CudaError as e:
    print("CODE", e.code)
    print("MSG", str(e))
else:
    print("compiled")
"""
    env = dict(os.environ, FIDGET_B200_NVRTC=missing)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert "CODE -3" in out.stdout, out.stdout
    assert missing in out.stdout
