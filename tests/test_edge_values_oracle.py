"""The CPU oracle on the f32 edge catalogue (edge_values.py), against the float64 numpy reference of op_reference.py:
every opcode in every clause form, edge immediates included.

  float_slice_eval  IEEE opcodes bit for bit with op_reference.f32; libm opcodes within ULP_BOUND of op_reference.f64
  grad_slice_eval   IEEE opcodes bit for bit with op_reference.grad; libm values as above, partials within GRAD_ULPS
  interval_eval     holds the f32 reference value at each box's endpoints and interior samples

The interval check is a property of f32 values: the reference does not round outward, so an interval may miss the real
value by half an ulp, and that is not tested.  These pin the reference side, so that a device mismatch in
test_gpu_edge_values.py points at the device."""
import zlib

import numpy as np
import pytest

import edge_values as E
import op_reference as R

def _seed(op, form, imm):
    return zlib.crc32(f"{op}{form}{imm}".encode())


def _failures(mask, *cols):
    bad = np.flatnonzero(~mask)[:4]
    return [tuple(np.asarray(c)[i].tolist() for c in cols) for i in bad]


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_float_slice_on_the_catalogue(orc, op):
    for form, imm, td in E.op_tapes(orc.Context, op):
        vals, ins, n = E.inputs(td, form)
        got = orc.Tape.from_data(td).float_slice_eval(vals)
        args = E.operands(form, ins, imm)
        ok = E.value_ok(op, got, args)
        assert ok.all(), (op, form, imm, _failures(ok, *args, got))


def test_immediates_survive_folding(orc):
    """Most (op, form, immediate) clauses reach the tape; the ones the host folds away are the identities."""
    for op in R.BINARY:
        tapes = E.op_tapes(orc.Context, op)
        for form in R.FORMS[op][1:]:
            kept = [imm for f, imm, _ in tapes if f == form]
            assert len(kept) >= len(E.IMMEDIATES) - 2, (op, form, kept)
    # a NaN immediate keeps its payload in the tape
    c = orc.Context()
    td = c.tape(c.binary("mix", c.x(), c.constant(float(E.IMMEDIATES[10]))))
    got = orc.Tape.from_data(td).float_slice_eval([E.VALUES])
    assert E.same_bits(got, R.f32("mix", E.VALUES, np.full(len(E.VALUES), E.IMMEDIATES[10]))).all()


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_grad_slice_on_the_catalogue(orc, op):
    for form, imm, td in E.op_tapes(orc.Context, op):
        vx, vy, _ = td.var_slots()
        gin = E.grad_inputs(td, form, _seed(op, form, imm))
        got = orc.Tape.from_data(td).grad_slice_eval(gin)
        args = E.operands(form, E.inputs(td, form)[1], imm)
        ok = E.grad_ok(op, form, got, gin[vx], gin[vy] if form == "rr" else None, imm, args)
        assert ok.all(), (op, form, imm, _failures(ok, gin[vx][:, 0], got))


@pytest.mark.parametrize("op", R.ALL_OPS)
def test_intervals_hold_the_f32_values(orc, op):
    for form, imm, td in E.op_tapes(orc.Context, op):
        vx, vy, _ = td.var_slots()
        b = E.boxes(td.n_vars, 300, _seed(op, form, imm))
        t = orc.Tape.from_data(td)
        out = np.stack([t.interval_eval(box)[0] for box in b])
        ordered = b[:, [vx, vy]] if form == "rr" else b
        ok = E.contains(op, form, ordered, out, imm, _seed(op, form, imm))
        assert ok.all(), (op, form, imm, [(ordered[i].tolist(), out[i].tolist()) for i in np.flatnonzero(~ok)[:4]])
