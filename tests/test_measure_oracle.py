"""fc_measure's CPU mirror (tests/csrc/measure_oracle.cc, on the oracle's evaluators) against a brute force over every
cell centre, its block closed forms against explicit sums, and the ctypes layout of fc_measure_result against the
header.

For tapes made of IEEE operations an interval result never contradicts a point value inside its box, so the mirror's
descent (interval levels down to edge-4 bricks, then the bricks' cell centres) must classify every cell as the brute
force does: the integers are compared exactly."""
import os
import random
import re

import numpy as np
import pytest

from conftest import ROOT, model_text
from measure_ref import brute_sums, oracle_block, oracle_measure
from views import _rot, _translate

IEEE_MODELS = ["prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm"]
ROTATE = (_translate(0.1, -0.05, 0.15) @ _rot((1, 2, 3), 25)).astype(np.float32)


def _depths(name):
    return (0, 1, 2, 3, 5) if name == "prospero.vm" else (0, 1, 2, 3, 4, 6)


@pytest.fixture(scope="module")
def tapes(orc):
    return {name: orc.Tape.from_vm(model_text(name)) for name in IEEE_MODELS}


@pytest.mark.parametrize("view", ["none", "rotate"])
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_oracle_matches_brute_force(orc, tapes, name, view):
    tape = tapes[name]
    m = ROTATE if view == "rotate" else None
    for depth in _depths(name):
        got = oracle_measure(orc, tape, depth, world_to_model=m)
        want = brute_sums(tape.float_slice_eval, tape.data.var_slots(), tape.n_vars, depth, world_to_model=m)
        for k in ("n_inside", "s1", "s2", "lo", "hi"):
            assert got[k] == want[k], (name, view, depth, k)
        n = 1 << depth
        brick = min(4, n)
        assert got["n_proven"] <= got["n_inside"] <= got["n_proven"] + got["n_undecided"]
        assert got["n_undecided"] % brick ** 3 == 0 and got["n_proven"] + got["n_undecided"] <= n ** 3


def _explicit(x0, y0, z0, T):
    u = [2 * i + 1 for i in range(x0, x0 + T)]
    v = [2 * j + 1 for j in range(y0, y0 + T)]
    w = [2 * k + 1 for k in range(z0, z0 + T)]
    su, sv, sw = sum(u), sum(v), sum(w)
    quu, qvv, qww = sum(a * a for a in u), sum(a * a for a in v), sum(a * a for a in w)
    return {"n_inside": T ** 3, "s1": [T * T * su, T * T * sv, T * T * sw],
            "s2": [T * T * quu, T * T * qvv, T * T * qww, T * su * sv, T * su * sw, T * sv * sw],
            "lo": [x0, y0, z0], "hi": [x0 + T - 1, y0 + T - 1, z0 + T - 1]}


def test_block_closed_forms(orc):
    rng = random.Random(12)
    n = 1 << 12
    cases = [(0, 0, 0, n), (0, 0, 0, 1), (n - 1, n - 1, n - 1, 1), (n // 2, 0, n // 2, n // 2)]
    for _ in range(60):
        T = 1 << rng.randrange(0, 11)
        cases.append(tuple(T * rng.randrange(0, n // T) for _ in range(3)) + (T,))
    for x0, y0, z0, T in cases:
        got = oracle_block(orc, x0, y0, z0, T)
        want = _explicit(x0, y0, z0, T)
        for k, v in want.items():
            assert got[k] == v, (x0, y0, z0, T, k)
        assert got["n_proven"] == 0 and got["n_undecided"] == 0


def test_whole_cube_fits_u64(orc):
    got = oracle_block(orc, 0, 0, 0, 1 << 12)
    assert got["n_inside"] == 1 << 36
    assert got["s2"][3] == 1 << 60 and max(got["s2"]) < 1 << 64


def _header_struct(name):
    with open(os.path.join(ROOT, "include", "fidget_cuda.h")) as f:
        text = f.read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype, names = decl.split(None, 1)
        for part in names.split(","):
            mm = re.fullmatch(r"\s*(\w+)\s*(?:\[(\d+)\])?\s*", part)
            fields.append((mm.group(1), ctype, int(mm.group(2) or 1)))
    return fields


def test_result_struct_matches_header():
    import ctypes as C
    from fidget_b200 import _lib
    from fidget_b200.shape import MEASURE_RESULT
    sizes = {"uint64_t": 8, "uint32_t": 4, "double": 8}
    fields = _header_struct("fc_measure_result")
    ct = _lib.FcMeasureResult
    assert [f[0] for f in fields] == [f[0] for f in ct._fields_] == list(MEASURE_RESULT.names)
    offset = 0
    for name, ctype, count in fields:
        size = sizes[ctype]
        offset = (offset + size - 1) // size * size
        assert getattr(ct, name).offset == offset == MEASURE_RESULT.fields[name][1], name
        assert getattr(ct, name).size == size * count == MEASURE_RESULT.fields[name][0].itemsize, name
        offset += size * count
    assert C.sizeof(ct) == offset == MEASURE_RESULT.itemsize == 264
    assert "fc_measure" in _lib.CUDA_API
