"""fc_volume_build's CPU mirror (tests/csrc/volume_oracle.cc, on the oracle's evaluators) against the root tape at every
cell centre, and the ctypes layouts of the fc_volume_* structs against the header.

For tapes made of IEEE operations an interval result never contradicts a point value inside its box, so the mirror's
bricks and tiles must partition the cube with every centre within the band in a brick, every tile's centres on its
side of the band, and every brick value equal to the root tape's, bit for bit."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, model_text
from volume_ref import check_volume, oracle_volume, root_values
from views import _rot, _translate

IEEE_MODELS = ["prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm"]
ROTATE = (_translate(0.1, -0.05, 0.15) @ _rot((1, 2, 3), 25)).astype(np.float32)


def _depths(name):
    return (0, 1, 3, 5) if name == "prospero.vm" else (0, 1, 2, 3, 4, 6)


@pytest.fixture(scope="module")
def tapes(orc):
    return {name: orc.Tape.from_vm(model_text(name)) for name in IEEE_MODELS}


@pytest.mark.parametrize("band", [0.0, 0.05])
@pytest.mark.parametrize("view", ["none", "rotate"])
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_oracle_matches_brute_force(orc, tapes, name, view, band):
    tape = tapes[name]
    m = ROTATE if view == "rotate" else None
    for depth in _depths(name):
        vol = oracle_volume(orc, tape, depth, band=band, world_to_model=m)
        v = root_values(tape.float_slice_eval, tape.data.var_slots(), tape.n_vars, depth, world_to_model=m)
        check_volume(vol["bricks"], vol["values"], vol["tiles"], depth, band, v)


def test_band_grows_the_bricks(orc, tapes):
    tape = tapes["hi.vm"]
    counts = [len(oracle_volume(orc, tape, 6, band=b)["bricks"]) for b in (0.0, 0.02, 0.1, 0.5)]
    assert counts == sorted(counts) and counts[0] < counts[-1]
    # a band wider than any value: no tiles at all, the whole cube in bricks
    vol = oracle_volume(orc, tape, 5, band=1e30)
    assert len(vol["tiles"]) == 0 and len(vol["bricks"]) == (32 // 8) ** 3


def test_oracle_gradients(orc, tapes):
    """Without a transform the gradients are the brick tape's at the world centre: the root tape's there, bit for bit"""
    for name in ("hi.vm", "quarter.vm"):
        tape = tapes[name]
        depth = 5
        vol = oracle_volume(orc, tape, depth, band=0.02, grads=True)
        B = 8
        slots = tape.data.var_slots()
        for r, (_, ix, iy, iz) in enumerate(vol["bricks"].tolist()):
            k, j, i = np.meshgrid(np.arange(iz, iz + B), np.arange(iy, iy + B), np.arange(ix, ix + B), indexing="ij")
            inv = np.float32(1) / np.float32(1 << depth)
            p = [((2 * a + 1).astype(np.float32) * inv - np.float32(1)).ravel() for a in (i, j, k)]
            ins = []
            for s in range(tape.n_vars):
                g = np.zeros((p[0].size, 4), dtype=np.float32)
                axis = slots.index(s)
                g[:, 0] = p[axis]
                g[:, 1 + axis] = 1
                ins.append(g)
            want = tape.grad_slice_eval(ins)
            np.testing.assert_array_equal(vol["values"][r].ravel(), want[:, 0])
            np.testing.assert_array_equal(vol["grads"][r].reshape(-1, 3), want[:, 1:])


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


@pytest.mark.parametrize("name,ct,size", [("fc_volume_cfg", "FcVolumeCfg", 16), ("fc_volume_brick", "FcVolumeBrick", 12),
                                          ("fc_volume_tile", "FcVolumeTile", 12), ("fc_volume_info", "FcVolumeInfo", 168),
                                          ("fc_volume_frame_info", "FcVolumeFrameInfo", 32)])
def test_structs_match_header(name, ct, size):
    import ctypes as C
    from fidget_b200 import _lib
    sizes = {"uint64_t": 8, "uint32_t": 4, "uint16_t": 2, "uint8_t": 1, "float": 4}
    fields = _header_struct(name)
    cls = getattr(_lib, ct)
    assert [f[0] for f in fields] == [f[0] for f in cls._fields_]
    offset = 0
    for fname, ctype, count in fields:
        s = sizes[ctype]
        offset = (offset + s - 1) // s * s
        assert getattr(cls, fname).offset == offset, (name, fname)
        assert getattr(cls, fname).size == s * count, (name, fname)
        offset += s * count
    assert C.sizeof(cls) == size
    assert "fc_volume_build" in _lib.CUDA_API and "fc_volume_read" in _lib.CUDA_API
    assert _lib.FC_FLAG_VOLUME_GRADS == 128
