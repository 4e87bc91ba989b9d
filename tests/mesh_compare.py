"""Test infrastructure: exact comparison of fc_mesh_build's output with the oracles, and of its vertices with the
float64 QEF solve (tests/qef_f64.py), for both mesh modes.

Device vertices are written in atomic order, so meshes are compared as multisets: the vertices bit for bit, and the
triangles as triples of vertex positions (bit for bit, rotation-normalised, winding kept).  That needs no matching by
distance and stays exact when two vertices share a position (a forced vertex sits on an intersection)."""
from __future__ import annotations

import numpy as np

import fidget_b200 as fb
import mesh_collapse_oracle as mco
import qef_f64
from oracle import mesh as om

f32 = np.float32


def _vert_rows(verts):
    v = np.ascontiguousarray(verts, dtype=f32).reshape(-1, 3).view(np.uint32)
    return sorted(map(bytes, v))


def _tri_rows(verts, tris):
    v = np.ascontiguousarray(verts, dtype=f32).reshape(-1, 3).view(np.uint32)
    t = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    p = v[t]                                         # [m, 3 corners, 3 coordinates]
    rot = [np.ascontiguousarray(np.roll(p, -r, axis=1)).reshape(len(t), 9) for r in range(3)]
    return sorted(min(bytes(a), bytes(b), bytes(c)) for a, b, c in zip(*rot))


def assert_same_mesh(verts, tris, o_verts, o_tris):
    assert len(verts) == len(o_verts) and len(tris) == len(o_tris), (len(verts), len(o_verts), len(tris), len(o_tris))
    assert _vert_rows(verts) == _vert_rows(o_verts), "vertices differ"
    assert _tri_rows(verts, tris) == _tri_rows(o_verts, o_tris), "triangles differ"


def leaf_set(cells):
    return sorted(zip(cells["depth"].tolist(), cells["ix"].tolist(), cells["iy"].tolist(), cells["iz"].tolist(),
                      cells["mask"].tolist()))


def _intersections(leaf):
    return {bytes(leaf["pos"][e].astype(f32).view(np.uint32)) for e in range(12) if (int(leaf["present"]) >> e) & 1}


class Report:
    """What a comparison covered: vertices checked against float64, rank-ambiguous ones skipped, forced ones."""

    def __init__(self):
        self.checked = self.ambiguous = self.forced = 0
        self.worst = 0.0                             # max |pos - pos64| / position_bound

    def vertex(self, pos, q, leaf, where):
        """pos: a float32 cell vertex solved from Qef q, or forced (q None) to one of leaf's intersections"""
        if q is None:
            self.forced += 1
            assert bytes(np.asarray(pos, dtype=f32).view(np.uint32)) in _intersections(leaf), f"{where}: forced vertex"
            return
        s = qef_f64.solve_qef(q)
        if s.ambiguous:
            self.ambiguous += 1
            return
        self.checked += 1
        self.worst = max(self.worst, float(np.abs(np.asarray(pos, np.float64) - s.pos).max()) / qef_f64.position_bound(s))
        bad = qef_f64.check_vertex(pos, s)
        assert not bad, f"{where}: {bad}"

    def __str__(self):
        return (f"{self.checked} vertices within the float64 bound (worst {self.worst:.2f} of it), "
                f"{self.ambiguous} rank-ambiguous, {self.forced} forced")


def compare_collapse(cuda, g, leaves, depth):
    """fb.mesh(g, depth, collapse=True) against mco.Octree(leaves, depth).walk_dual(), exactly: final leaves, cell
    vertices, vertices, triangles, open_edges; then every final leaf's vertex against the float64 solve of the QEF
    the oracle solved for that cell.  Returns (vertices, triangles, info, octree, Report)."""
    verts, tris, info = fb.mesh(g, depth, collapse=True)
    cells = fb.mesh_cells(cuda)
    octree = mco.Octree(leaves, depth)
    o_verts, o_tris, o_open = octree.walk_dual()
    final = octree.final_leaves()
    assert leaf_set(cells) == [tuple(int(v) for v in c) for c in final], "final leaves differ"
    assert info["n_triangles"] == len(tris) and info["n_vertices"] == len(verts)
    assert info["open_edges"] == o_open, (info["open_edges"], o_open)
    assert_same_mesh(verts, tris, o_verts, o_tris)
    rep = Report()
    for cell in cells:
        key = (int(cell["depth"]), int(cell["ix"]), int(cell["iy"]), int(cell["iz"]))
        want = octree.cells[key]["verts"][0]
        assert np.array_equal(cell["vertex"].view(np.uint32), np.asarray(want, dtype=f32).view(np.uint32)), \
            f"cell {key}: vertex {cell['vertex']} vs the oracle's {want}"
        q = octree.qefs[key]
        rep.vertex(cell["vertex"], q[0] if isinstance(q, list) else q, octree.leaves.get(key), f"cell {key}")
    return verts, tris, info, octree, rep


class _F32Vertex:
    """oracle/mesh.py's vertex callback with the device's float32 solve (mco.Qef, k_mesh_vertices' order); keeps
    each call's QEF (None when a NaN gradient forced the vertex onto that intersection)"""

    def __init__(self):
        self.calls = []

    def __call__(self, pts, grs):
        q = mco.Qef()
        for p, g in zip(pts, grs):
            if np.isnan(g).any():
                self.calls.append(None)
                return np.asarray(p, dtype=f32)
            q.add_intersection(p, g)
        self.calls.append(q)
        return q.solve()[0]


def compare_uniform(g, leaves, depth):
    """fb.mesh(g, depth) against oracle/mesh.py's walk over the same leaves, exactly, with the device's float32 vertex
    solve; then every cell vertex the mesh uses against the float64 solve of its QEF.  Returns a Report."""
    verts, tris, info = fb.mesh(g, depth)
    solve = _F32Vertex()
    o_verts, o_tris, o_open, slots = om.build_indexed(leaves, vertex=solve)
    assert info["n_leaves"] == len(leaves)
    assert info["open_edges"] == o_open, (info["open_edges"], o_open)
    assert info["n_triangles"] == len(tris) and info["n_vertices"] == len(verts)
    assert_same_mesh(verts, tris, o_verts, o_tris)
    qefs, k = {}, 0
    for i, leaf in enumerate(leaves):
        for grp in range(om.corner_groups(int(leaf["mask"]))[1]):
            qefs[(i, grp)] = solve.calls[k]
            k += 1
    rep = Report()
    for pos, (kind, i, j) in zip(o_verts, slots):
        if kind == "v":
            rep.vertex(pos, qefs[(i, j)], leaves[i], f"leaf {i} group {j}")
    return rep
