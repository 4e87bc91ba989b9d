"""fc_raycast's CPU mirror (tests/csrc/raycast_oracle.cc, on the oracle's evaluators) against a brute force over every
sample, the descent's level and clipping arithmetic, ``fb.pick``'s rays against the renderer's voxel positions, and the
ctypes layouts of the ray structs against the header.

For tapes made of IEEE operations an interval never contradicts a point value inside its box, and a segment's box
encloses its samples (they are monotone in k), so the mirror's hit must be the first sample whose f32 value is < 0."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import fidget_b200 as fb
from fidget_b200 import _lib
from conftest import ROOT, model_text
from raycast_ref import first_inside, levels, make_rays, oracle_raycast, ray_families, sample_points
from views import _rot, _translate

IEEE_MODELS = ["prospero.vm", "hi.vm", "quarter.vm", "colonnade.vm", "tanglecube.vm"]
STEPS = (1, 31, 32, 33, 1024, 1025, 1 << 24)


@pytest.fixture(scope="module")
def tapes(orc):
    return {name: orc.Tape.from_vm(model_text(name)) for name in IEEE_MODELS}


def _brute(tape, rays, steps):
    t, x, y, z = sample_points(rays, steps)
    xs, ys, zs = tape.data.var_slots()
    cols = [None] * max(tape.n_vars, 1)
    for s, v in ((xs, x), (ys, y), (zs, z)):
        if s >= 0:
            cols[s] = v.ravel()
    cols = [c if c is not None else np.zeros(x.size, np.float32) for c in cols]
    return tape.float_slice_eval(cols).reshape(len(rays), steps)


@pytest.mark.parametrize("steps", [33, 1025])
@pytest.mark.parametrize("name", IEEE_MODELS)
def test_oracle_hit_is_the_first_inside_sample(orc, tapes, name, steps):
    tape = tapes[name]
    n = 8 if name == "prospero.vm" else 24
    for family, rays in ray_families(7, steps, n).items():
        hits, _ = oracle_raycast(orc, tape, rays, steps)
        vals = _brute(tape, rays, steps)
        want = first_inside(vals)
        assert np.array_equal(hits["k"], want), (name, family)
        hit = want != 0xFFFFFFFF
        if hit.any():
            t, x, y, z = sample_points(rays, steps)
            idx = np.nonzero(hit)[0], want[hit].astype(np.int64)
            assert np.array_equal(hits["t"][hit].view(np.uint32), t[idx].view(np.uint32))
            pos = np.stack([x[idx], y[idx], z[idx]], 1)
            assert np.array_equal(hits["pos"][hit].view(np.uint32), pos.view(np.uint32))
            assert np.all(hits["value"][hit] < 0) and np.all(hits["value"][hit] == vals[idx])
        miss = ~hit
        assert np.all(hits["flags"][miss] == 0) and np.all(hits["t"][miss] == 0) and np.all(hits["pos"][miss] == 0)
        assert np.all(hits["flags"] <= _lib.FC_RAY_PROVEN)


@pytest.mark.parametrize("steps", STEPS)
def test_levels_and_clipping(orc, steps):
    """L = max(1, ceil(log2(steps) / 5)); with a field every interval leaves ambiguous and no sample finds inside
    (x - x: intervals [a - b, b - a], points 0), the walk evaluates every segment of every level, clipped to [0, steps),
    and the leaf evaluates every sample once."""
    L = max(1, math.ceil(math.log2(steps) / 5))
    assert levels(orc, steps) == L
    assert 32 ** L >= steps and (L == 1 or 32 ** (L - 1) < steps)
    tape = orc.Tape.from_vm("_0 var-x\n_1 sub _0 _0\n")
    rays = make_rays([[-1.0, 0.0, 0.0]], [[1.0, 0.0, 0.0]], 0.0, np.float32(2.0) / np.float32(max(steps, 2)))
    hits, st = oracle_raycast(orc, tape, rays, steps)
    assert hits["k"][0] == 0xFFFFFFFF
    for l in range(L):
        assert st["evaluated"][l] == -(-steps // 32 ** (L - l)), (steps, l)
    assert st["evaluated"][L:] == [0] * (8 - L)
    assert st["leaf_samples"] == steps


def test_first_sample_and_proven_flag(orc):
    """A ray inside a box from its first sample: k = 0, proven (the whole ray's box is inside)"""
    tape = orc.Tape.from_vm("_0 var-x\n_1 abs _0\n_2 const 0.9\n_3 sub _1 _2\n")
    rays = make_rays([[-0.5, 0, 0], [-2.0, 0, 0]], [[1.0, 0, 0], [1.0, 0, 0]], 0.0, np.float32(1 / 1024))
    hits, _ = oracle_raycast(orc, tape, rays, 1000)
    assert hits["k"][0] == 0 and hits["flags"][0] == _lib.FC_RAY_PROVEN
    # from -2: the first sample with |x| < 0.9 is x > -0.9, k = ceil(1.1 * 1024) = 1127 is past 1000 samples
    assert hits["k"][1] == 0xFFFFFFFF
    hits, _ = oracle_raycast(orc, tape, rays[1:], 2000)
    assert hits["k"][0] == 1127 and hits["value"][0] < 0 and hits["grad"][0][0] == -1.0   # d|x|/dx at x < 0


VIEW = (_translate(0.1, -0.05, 0.15) @ _rot((1, 2, 3), 25)).astype(np.float32)


@pytest.mark.parametrize("dims", [(64, 64, 64), (96, 80, 72), (128, 64, 32)])
@pytest.mark.parametrize("view", ["identity", "rotate"])
def test_pick_rays_follow_the_voxel_columns(dims, view):
    w, h, d = dims
    cfg = fb.RenderConfig3D(w, h, d, world_to_model=None if view == "identity" else VIEW)
    rng = np.random.default_rng(3)
    px = np.stack([rng.integers(0, w, 40), rng.integers(0, h, 40)], 1)
    o, di = fb.pick_rays(cfg, px)
    rays = make_rays(o, di, 0.0, 1.0)
    t, x, y, z = sample_points(rays, d)
    m64 = cfg.matrix().astype(np.float64)
    ks = np.arange(d)
    for i, (pxx, pyy) in enumerate(px):
        vox = np.stack([np.full(d, pxx), np.full(d, pyy), d - 1 - ks, np.ones(d)], 0).astype(np.float64)
        want = (m64 @ vox)[:3]
        got = np.stack([x[i], y[i], z[i]], 0).astype(np.float64)
        assert np.allclose(got, want, rtol=0, atol=1e-5), (dims, view, i)
    pow2 = all(v & (v - 1) == 0 for v in dims)
    if view == "identity" and pow2:
        # every coordinate is dyadic: the samples are the renderer's voxel positions, ((m0 x + m1 y) + m2 z) + m3
        m = cfg.matrix()
        zz = (d - 1 - ks).astype(np.float32)
        for i, (pxx, pyy) in enumerate(px):
            for a, got in enumerate((x[i], y[i], z[i])):
                want = ((m[a, 0] * np.float32(pxx) + m[a, 1] * np.float32(pyy)) + m[a, 2] * zz) + m[a, 3]
                assert np.array_equal(got.view(np.uint32), want.astype(np.float32).view(np.uint32))


def test_pick_refuses_projective_views():
    cfg = fb.RenderConfig3D(16, 16, 16)
    m = cfg.matrix().copy()
    m[3, 2] = 0.1
    cfg.mat = m
    with pytest.raises(ValueError):
        fb.pick_rays(cfg, [[0, 0]])


def test_ray_structs_match_header(tmp_path):
    assert C.sizeof(_lib.FcRay) == 32 and fb.RAY.itemsize == 32
    assert C.sizeof(_lib.FcRayHit) == 40 and fb.RAY_HIT.itemsize == 40
    for name in ("k", "flags", "t", "pos", "value", "grad"):
        assert getattr(_lib.FcRayHit, name).offset == fb.RAY_HIT.fields[name][1], name
    for name in ("origin", "dir", "t0", "dt"):
        assert getattr(_lib.FcRay, name).offset == fb.RAY.fields[name][1], name
    src = tmp_path / "rays.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fidget_cuda.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(fc_ray), sizeof(fc_ray_hit), sizeof(fc_raycast_cfg),\n'
                   '         sizeof(fc_raycast_info), offsetof(fc_ray_hit, value), offsetof(fc_raycast_info, leaf_samples),\n'
                   '         offsetof(fc_raycast_info, device_ms), offsetof(fc_raycast_cfg, var_values));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "rays"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I",
                           os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_lib.FcRay), C.sizeof(_lib.FcRayHit), C.sizeof(_lib.FcRaycastCfg),
                     C.sizeof(_lib.FcRaycastInfo), _lib.FcRayHit.value.offset, _lib.FcRaycastInfo.leaf_samples.offset,
                     _lib.FcRaycastInfo.device_ms.offset, _lib.FcRaycastCfg.var_values.offset]
    assert _lib.FC_RAY_MISS == 0xFFFFFFFF and _lib.FC_RAY_MAX_STEPS == 1 << 24
