"""The mesher's float32 QEF solve (mesh_collapse_oracle.Qef.solve, which the device's qef_vertex / qef_error
match bit for bit) held against QuadraticErrorSolver::solve restated in float64 (tests/qef_f64.py).  CPU only: this is
what vouches for the device's vertex solve on a machine without a GPU.

The bounds (qef_f64.POS_C, DROP_C, ERR_C) were calibrated on test_jacobi_solve_matches_float64's corpus: the largest
normalised deviations it measured are noted beside them, and each bound is four to ten times that (DESIGN.md §5)."""
import numpy as np
import pytest

import mesh_collapse_oracle as mco
import mesh_shapes
import qef_f64
from conftest import model_text

f32 = np.float32


def _qef(points, normals):
    q = mco.Qef()
    for p, n in zip(points, normals):
        q.add_intersection(np.asarray(p, dtype=f32), np.append(np.asarray(n, dtype=f32), f32(0)))
    return q


def _both(q):
    pos32, err32, rank32 = q.solve_rank()
    return pos32, err32, rank32, qef_f64.solve_qef(q)


# ---- the reference's own QEF tests (qef.rs:126-168) ------------------------------------------------------------------
def test_qef_rank2():
    q = mco.Qef()
    q.add_intersection([-0.5, -0.75, -0.75], [0.24, 0.12, 0.0, 0.0])
    q.add_intersection([-0.75, -1.0, -0.6], [0.0, 0.0, 0.31, 0.0])
    q.add_intersection([-0.50, -1.0, -0.6], [0.0, 0.0, 0.31, 0.0])
    s = qef_f64.solve_qef(q)
    assert s.err == qef_f64.ERR_FLOOR and s.rank == 2
    assert q.solve_rank()[2] == 2


def test_qef_near_planar():
    q = mco.Qef()
    q.add_intersection([-0.5, -0.25, 0.4999981], [-0.66666776, -0.33333388, 0.66666526, -1.2516975e-6])
    q.add_intersection([-0.5, -0.25, 0.50], [-0.6666667, -0.33333334, 0.6666667, 0.0])
    q.add_intersection([-0.5, -0.25, 0.50], [-0.6666667, -0.33333334, 0.6666667, 0.0])
    s = qef_f64.solve_qef(q)
    assert s.err == qef_f64.ERR_FLOOR and s.rank == 1
    assert np.linalg.norm(s.pos - [-0.5, -0.25, 0.5]) < 1e-3


# ---- hand cases with closed-form answers -----------------------------------------------------------------------------
def test_one_plane_projects_the_centre():
    n = np.array([1.0, 2.0, 2.0]) / 3
    pts = [[0.1, 0.2, -0.05], [0.3, -0.1, 0.0], [-0.2, 0.05, 0.15]]
    pts = [np.asarray(p) + n * (0.25 - n @ p) for p in pts]            # on the plane n . p = 0.25
    q = _qef(pts, [n] * 3)
    pos32, err32, rank32, s = _both(q)
    c = np.mean(np.asarray(pts, dtype=f32).astype(np.float64), axis=0)
    want = c + n * (0.25 - n @ c)
    assert s.rank == rank32 == 1
    assert np.abs(s.pos - want).max() < 1e-6 and np.abs(pos32 - want).max() < 1e-6
    assert s.dropped.shape == (3, 2) and np.abs(s.dropped.T @ n).max() < 1e-6


def test_two_planes_meet_on_the_line_nearest_the_centre():
    n1, n2 = np.array([1.0, 0, 0]), np.array([0, 0.6, 0.8])
    pts = [[0.3, 0.1, 0.4], [0.3, -0.2, 0.0], [0.0, 0.3, 0.5 - 0.75 * 0.3], [0.2, -0.3, 0.5 + 0.75 * 0.3]]
    q = _qef(pts, [n1, n1, n2, n2])                                    # planes x = 0.3 and 0.6 y + 0.8 z = 0.4
    pos32, err32, rank32, s = _both(q)
    c = np.mean(np.asarray(pts, dtype=f32).astype(np.float64), axis=0)
    d = np.cross(n1, n2)
    base = np.linalg.lstsq(np.array([n1, n2]), np.array([0.3, 0.4]), rcond=None)[0]
    want = base + d * (d @ (c - base))
    assert s.rank == rank32 == 2
    assert np.abs(s.pos - want).max() < 1e-6 and np.abs(pos32 - want).max() < 1e-6
    assert abs(s.dropped[:, 0] @ d) > 1 - 1e-6


def test_three_planes_meet_at_the_corner():
    corner = np.array([0.25, -0.375, 0.125])
    rot = np.linalg.qr(np.array([[1.0, 0.3, -0.2], [0.1, 1.0, 0.4], [-0.3, 0.2, 1.0]]))[0]
    ns = list(rot.T)
    pts = [corner + 0.1 * ns[(k + 1) % 3] - 0.05 * ns[(k + 2) % 3] for k in range(3)]
    q = _qef(pts, ns)
    pos32, err32, rank32, s = _both(q)
    assert s.rank == rank32 == 3
    assert np.abs(s.pos - corner).max() < 1e-6 and np.abs(pos32 - corner).max() < 2e-6
    assert err32 == f32(1e-6) and s.err == qef_f64.ERR_FLOOR


@pytest.mark.parametrize("ratio,rank", [(1.05e-3, 2), (0.95e-3, 1)])
def test_dihedral_angle_at_the_cutoff(ratio, rank):
    """Two planes at dihedral angle theta: A^T A has eigenvalues 1 +- cos(theta), so w_1 / w_0 = tan^2(theta / 2).
    Just above the 1e-3 cutoff the vertex is on their line; just below it is the centre moved onto the mean plane."""
    half = np.arctan(np.sqrt(ratio))
    n1 = np.array([np.cos(half), np.sin(half), 0.0])
    n2 = np.array([np.cos(half), -np.sin(half), 0.0])
    pts = [[0.1, 0.3, 0.2], [0.1, -0.2, -0.1]]
    pts = [np.asarray(p) - n * (n @ p) for p, n in zip(pts, (n1, n2))]   # both planes through the z axis
    q = _qef(pts, [n1, n2])
    pos32, err32, rank32, s = _both(q)
    assert abs(s.ratios[1] / ratio - 1) < 1e-3 and s.ratios[2] < 1e-9
    assert s.rank == rank32 == rank and not s.ambiguous
    c = s.center
    if rank == 2:
        want = np.array([0.0, 0.0, c[2]])                             # on the z axis, level with the centre
    else:
        want = c * [0.0, 1.0, 1.0]                                    # the centre moved onto the mean plane x = 0
    assert np.abs(s.pos - want).max() < 1e-5
    assert np.abs(pos32 - s.pos).max() < 1e-5


# ---- the float32 Jacobi solve against float64 on every QEF the collapse oracle solves ------------------------------
CPU_SEEDS = list(range(24))
MODELS = [("colonnade.vm", 6), ("bear.vm", 6), ("gyroid-sphere.vm", 5)]


def _corpus(orc):
    for seed in CPU_SEEDS:
        depth = mesh_shapes.fuzz_depth(seed)
        _, tape, kind = mesh_shapes.tape_pair(orc, None, seed, depth)
        yield f"seed {seed} ({kind}) depth {depth}", mco.build(orc, tape, depth)
    for name, depth in MODELS:
        yield f"{name} depth {depth}", mco.build(orc, orc.Tape.from_vm(model_text(name)), depth)


def octree_qefs(octree):
    """(cell key, group or None for a merged QEF, Qef) of every QEF the octree solved"""
    for key, q in octree.qefs.items():
        if isinstance(q, list):
            for g, qq in enumerate(q):
                if qq is not None:
                    yield key, g, qq
        else:
            yield key, None, q


def _err_key(octree, key):
    """(key, group) of the QEF whose error is the cell's LeafHermiteData::qef_err: a surface leaf's last group (the last
    writer), a collapsed leaf's merged QEF; None for an Empty / Full cell or a forced last group"""
    q = octree.qefs.get(key)
    if isinstance(q, list):
        return (key, len(q) - 1) if q[-1] is not None else None
    return (key, None) if q is not None and octree.cells[key]["kind"] == "L" else None


def test_jacobi_solve_matches_float64(orc):
    """Every leaf-group QEF and every merged QEF of the corpus: the same rank, the vertex within
    qef_f64.position_bound, nothing along a dropped eigenvector, the error term within rounding.  Rank-ambiguous
    QEFs are counted, not checked; so are the collapse decisions (err < 2 x children's error) that float64 decides
    the other way, which the reference's float32 decision allows."""
    stats = {"n": 0, "ambiguous": 0, "flipped": 0, "decisions": 0}
    worst = {}                                   # class -> (|pos32 - pos64| in cells, where)
    failures = []
    for where, octree in _corpus(orc):
        f64 = {}
        for key, g, q in octree_qefs(octree):
            pos32, err32, rank32 = q.solve_rank()
            s = qef_f64.solve_qef(q)
            f64[(key, g)] = s
            stats["n"] += 1
            if s.ambiguous:
                stats["ambiguous"] += 1
                continue
            tag = f"{where} cell {key} group {g}"
            if rank32 != s.rank:
                failures.append(f"{tag}: rank {rank32} vs {s.rank}, ratios {s.ratios}")
                continue
            dev = float(np.abs(pos32 - s.pos).max()) / (2.0 / 2 ** key[0])
            cls = f"rank {s.rank}, smallest kept ratio {'>=' if s.min_kept_ratio >= 1e-2 else '<'} 1e-2"
            if dev >= worst.get(cls, (0.0, ""))[0]:
                worst[cls] = (dev, tag)
            failures += [f"{tag}: {m}" for m in qef_f64.check_vertex(pos32, s, err32)]
        for key, child_err in octree.child_err.items():
            d, x, y, z = key
            kids = [(d + 1, 2 * x + (c & 1), 2 * y + ((c >> 1) & 1), 2 * z + ((c >> 2) & 1)) for c in range(8)]
            kid64 = [f64[k].err for k in (_err_key(octree, k) for k in kids) if k is not None]
            if not kid64:
                continue
            stats["decisions"] += 1
            v32 = not (octree.qefs[key].solve()[1] >= child_err * 2)
            v64 = f64[(key, None)].err < 2 * min(kid64)
            stats["flipped"] += v32 != v64
    print(f"\n{stats['n']} QEFs, {stats['ambiguous']} rank-ambiguous (a ratio within 1 % of 1e-3); "
          f"{stats['flipped']} of {stats['decisions']} collapse decisions flip in float64")
    for cls, (dev, tag) in sorted(worst.items()):
        print(f"  {cls}: max |pos32 - pos64| = {dev:.3g} cells ({tag})")
    assert not failures, "\n".join(failures[:20]) + f"\n... {len(failures)} in all"
