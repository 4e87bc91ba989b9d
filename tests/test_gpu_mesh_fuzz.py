"""Random-CSG fuzz of fc_mesh_build in both modes against the oracles, exactly.  The shapes (tests/mesh_shapes.py)
use IEEE-exact opcodes only, so the device sampler's leaves are the oracle's bit for bit and there is no tolerance:

  collapse   final leaf set, cell vertices, vertices, triangles and open_edges against mesh_collapse_oracle's
             Octree::build + walk_dual, then every final leaf's vertex against the float64 QEF solve;
  uniform    vertices, triangles and open_edges against oracle/mesh.py's walk with the device's float32 vertex
             solve, then every cell vertex against the float64 QEF solve.

Seeds run at depths 2-7 (mesh_shapes.fuzz_depth).  The cost is the numpy oracles' CPU time: the file took 67 s of
wall time on an H100 host (it prints its wall time)."""
import time

import pytest

import fidget_b200 as fb
import mesh_compare
import mesh_shapes

pytestmark = pytest.mark.gpu

SEEDS = mesh_shapes.FUZZ_SEEDS


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_gpu_mesh_fuzz.py: {time.perf_counter() - t0:.1f} s wall")


@pytest.mark.parametrize("seed", SEEDS)
def test_random_csg_mesh(orc, cuda, seed):
    depth = mesh_shapes.fuzz_depth(seed)
    dev, o, kind = mesh_shapes.tape_pair(orc, fb, seed, depth)
    g = fb.CudaShape(cuda, dev)
    leaves, _ = orc.octree_sample(o, depth)
    *_, rep_c = mesh_compare.compare_collapse(cuda, g, leaves, depth)
    rep_u = mesh_compare.compare_uniform(g, leaves, depth)
    print(f"seed {seed} ({kind}) depth {depth}: {len(leaves)} leaves; collapse: {rep_c}; uniform: {rep_u}")


def _corner_spheres(ctx, mask):
    shapes = []
    for j in range(8):
        if (mask >> j) & 1:
            x, y, z = ctx.x(), ctx.y(), ctx.z()
            c = (0.5 * (j & 1), 0.5 * ((j >> 1) & 1), 0.5 * ((j >> 2) & 1))
            sq = [ctx.square(ctx.sub(a, v)) for a, v in zip((x, y, z), c)]
            shapes.append(ctx.sub(ctx.sqrt(ctx.add(ctx.add(sq[0], sq[1]), sq[2])), 0.1))
    s = shapes.pop()
    for q in shapes:
        s = ctx.min(s, q)
    return s


def test_all_masks_match_oracles(orc, cuda):
    """test_mesh_manifold_single_thread's 255 shapes (0-8 spheres at the corners of [0, 0.5]^3) at depth 2, both
    modes compared exactly with the oracles"""
    for mask in range(1, 256):
        gc, oc = fb.Context(), orc.Context()
        g = fb.CudaShape(cuda, gc.tape(_corner_spheres(gc, mask)))
        leaves, _ = orc.octree_sample(orc.Tape.from_data(oc.tape(_corner_spheres(oc, mask))), 2)
        mesh_compare.compare_collapse(cuda, g, leaves, 2)
        mesh_compare.compare_uniform(g, leaves, 2)
