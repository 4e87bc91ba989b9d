"""The interpreters dispatch through a 256-entry table (first clause byte = opcode * 4 + form -> handler number,
fidget_b200/csrc/cuda/interp.cuh) and their switches treat any other value as unreachable.  The tables are constexpr,
so a host program compiled with nvcc can print them: every entry must be a handler that exists, each handler must sit
at exactly the (opcode, form) bytes it implements, and the interval table must not name the f32-only handlers."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F_RR, F_RI, F_IR, F_ALIAS = 0, 1, 2, 3


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("dop") / "dop_check")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O1",
                    "-I", os.path.join(ROOT, "fidget_b200", "csrc", "cuda"), "-o", exe,
                    os.path.join(ROOT, "tests", "csrc", "dop_table_check.cu")], check=True, capture_output=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines()
    head = out[0].split()
    rows = [tuple(int(v) for v in line.split()) for line in out[1:257]]
    names = dict(kv.split("=") for kv in out[257].split()[1:])
    ops = dict(kv.split("=") for kv in out[258].split()[1:])
    return {"h_count": int(head[1]), "op_count": int(head[3]), "iv": [r[1] for r in rows], "f32": [r[2] for r in rows],
            "H": {k: int(v) for k, v in names.items()}, "OP": {k: int(v) for k, v in ops.items()}}


def test_every_entry_is_an_existing_handler(tables):
    assert len(tables["iv"]) == 256 and len(tables["f32"]) == 256
    assert all(0 <= h < tables["h_count"] for h in tables["iv"] + tables["f32"])
    # bytes beyond the last opcode are never emitted by the bytecode front end; they must fall into the generic path
    assert all(h == 0 for h in tables["iv"][tables["op_count"] * 4:] + tables["f32"][tables["op_count"] * 4:])


def test_handlers_sit_on_their_opcode_and_form(tables):
    H, OP = tables["H"], tables["OP"]
    expect_iv, expect_f32 = {}, {}
    for op, base in (("OP_ADD", "H_ADD_RR"), ("OP_SUB", "H_SUB_RR"), ("OP_MUL", "H_MUL_RR"), ("OP_MIN", "H_MIN_RR"),
                     ("OP_MAX", "H_MAX_RR")):
        for form in (F_RR, F_RI, F_IR):
            expect_iv[OP[op] * 4 + form] = H[base] + form           # H_x_RR, H_x_RI, H_x_IR are consecutive
    for op, h in (("OP_NEG", "H_NEG"), ("OP_ABS", "H_ABS"), ("OP_SQRT", "H_SQRT"), ("OP_SQUARE", "H_SQUARE")):
        expect_iv[OP[op] * 4 + F_RR] = H[h]
    expect_iv[OP["OP_COPY"] * 4 + F_RR] = H["H_COPY_REG"]
    expect_iv[OP["OP_COPY"] * 4 + F_ALIAS] = H["H_COPY_REG"]
    expect_iv[OP["OP_COPY"] * 4 + F_RI] = H["H_COPY_IMM"]
    expect_f32.update(expect_iv)
    for form in (F_RR, F_RI, F_IR):
        expect_f32[OP["OP_DIV"] * 4 + form] = H["H_DIV_RR"] + form
    expect_f32[OP["OP_EXP"] * 4 + F_RR] = H["H_EXP"]
    for byte in range(256):
        assert tables["iv"][byte] == expect_iv.get(byte, H["H_GENERIC"]), byte
        assert tables["f32"][byte] == expect_f32.get(byte, H["H_GENERIC"]), byte


def test_interval_table_has_no_f32_only_handlers(tables):
    H = tables["H"]
    f32_only = set(range(H["H_DIV_RR"], H["H_DIV_RR"] + 3)) | {H["H_EXP"]}
    assert not f32_only & set(tables["iv"])
    assert f32_only <= set(tables["f32"])
