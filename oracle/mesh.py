"""ORACLE -- test infrastructure, not product code.

numpy restatement of the meshing back half of fidget-mesh for leaves of equal depth (the part
``fc_mesh_build`` runs on the device), on top of the oracle's sampler output (``oracle.octree_sample``):

  cell vertices   CELL_TO_VERT_TO_EDGES' rule (fidget-mesh/build.rs:25-130: one vertex per connected group of
                  inside corners, owning the transitions that start at its corners) + QuadraticErrorSolver
                  (fidget-mesh/src/qef.rs:44-168) with numpy's SVD standing in for nalgebra's
  triangles       dc_edge for four leaves of equal depth (fidget-mesh/src/dc.rs:104-213)
  STL             Mesh::write_stl (fidget-mesh/src/output.rs:7-38)

  model space     Octree::build's last step (fidget-mesh/src/octree.rs:58-65): the vertices of an octree sampled through
                  ``world_to_model`` go back through that matrix (``to_model``)

Cell collapse (octree.rs:252-440) is out of scope on both sides.  Only tests/ may import this module.
"""
from __future__ import annotations

import struct

import numpy as np

X, Y, Z = 1, 2, 4


def next_axis(a):
    return {X: Y, Y: Z, Z: X}[a]


def corner_groups(mask: int):
    """Connected groups of inside corners (cube-edge adjacency), ordered by lowest corner."""
    label = list(range(8))
    changed = True
    while changed:
        changed = False
        for c in range(8):
            if not (mask >> c) & 1:
                continue
            for ax in (X, Y, Z):
                g = c ^ ax
                if (mask >> g) & 1 and label[c] != label[g]:
                    lo = min(label[c], label[g])
                    label[c] = label[g] = lo
                    changed = True
    roots = sorted({label[c] for c in range(8) if (mask >> c) & 1})
    return {c: roots.index(label[c]) for c in range(8) if (mask >> c) & 1}, len(roots)


def edge_index(start: int, t: int) -> int:
    u = next_axis(t)
    v = next_axis(u)
    return {X: 0, Y: 1, Z: 2}[t] * 4 + (1 if start & u else 0) + (2 if start & v else 0)


def qef_vertex(points, grads):
    """QuadraticErrorSolver::add_intersection + solve (qef.rs:44-168), float32 accumulation like the reference."""
    f = np.float32
    ata = np.zeros((3, 3), dtype=f)
    atb = np.zeros(3, dtype=f)
    mp = np.zeros(4, dtype=f)
    for p, g in zip(points, grads):
        if np.isnan(g).any():
            return p.astype(f)                          # octree.rs:793-801: snap to the intersection
        mp += np.array([p[0], p[1], p[2], 1.0], dtype=f)
        n = (g[:3] / f(np.sqrt(f(np.dot(g[:3], g[:3]))))).astype(f)
        ata += np.outer(n, n).astype(f)
        atb += (n * f(np.dot(n, p))).astype(f)
    center = (mp[:3] / mp[3]).astype(f)
    b = (atb - ata @ center).astype(f)
    u, s, vt = np.linalg.svd(ata.astype(np.float64))
    cutoff = abs(s[0]) * 1e-3
    rank = next((i for i in range(3) if abs(s[i]) < cutoff), 3)
    eps = s[rank] if rank < 3 else 0.0
    sol = np.zeros(3)
    for i in range(3):
        if s[i] > eps:
            sol += vt[i] * (np.dot(u[:, i], b) / s[i])
    pos = (sol + center).astype(f)
    return pos if not np.isnan(pos).any() else center


def to_model(verts, world_to_model):
    """Matrix4::transform_point on every row of ``verts`` [n,3], in float32 and nalgebra's order: ((m0 x + m1 y) + m2 z)
    + m3 per row, divided by the homogeneous term where that is not zero.  Octree::build applies it to every octree
    vertex unless the matrix is the identity (octree.rs:58-65); None stands for the identity here."""
    v = np.asarray(verts, dtype=np.float32).reshape(-1, 3)
    if world_to_model is None or np.array_equal(np.asarray(world_to_model, dtype=np.float32).reshape(4, 4),
                                                np.eye(4, dtype=np.float32)):
        return v
    m = np.asarray(world_to_model, dtype=np.float32).reshape(4, 4)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    with np.errstate(all="ignore"):
        r = [((m[i, 0] * x + m[i, 1] * y) + m[i, 2] * z) + m[i, 3] for i in range(4)]
        out = np.stack([np.where(r[3] != 0, r[i] / np.where(r[3] != 0, r[3], np.float32(1)), r[i]) for i in range(3)], axis=-1)
    return out.astype(np.float32)


def build(leaves):
    """leaves: the structured array of ``oracle.octree_sample``.  Returns (cell_vertices dict (leaf, group) -> pos,
    triangles as a list of three positions each, open edge count)."""
    verts, tri_slots, open_edges = _walk(leaves, qef_vertex)
    tris = [tuple(_slot_pos(leaves, verts, k) for k in t) for t in tri_slots]
    return verts, tris, open_edges


def build_indexed(leaves, vertex=qef_vertex, world_to_model=None):
    """build() indexed the way fc_mesh_build returns the mesh: one vertex per slot the triangles use (MeshBuilder's
    dedup), ``(vertices [n,3] float32, triangles [m,3] int64, open edge count, slots)``, where a slot is
    ('v', leaf, group) for a cell vertex or ('i', leaf, edge) for an intersection.  ``vertex(points, grads)``
    places a cell vertex (qef_vertex by default); the triangles do not depend on it.  ``leaves`` sampled through
    ``world_to_model``: the vertices are returned in model space (``to_model``)."""
    verts, tri_slots, open_edges = _walk(leaves, vertex)
    index = {}
    for t in tri_slots:
        for k in t:
            index.setdefault(k, len(index))
    pos = to_model(np.array([_slot_pos(leaves, verts, k) for k in index], dtype=np.float32), world_to_model)
    tris = np.array([[index[k] for k in t] for t in tri_slots], dtype=np.int64).reshape(-1, 3)
    return pos, tris, open_edges, list(index)


def _slot_pos(leaves, verts, slot):
    kind, i, j = slot
    return verts[(i, j)] if kind == "v" else leaves[i]["pos"][j].astype(np.float32)


def _walk(leaves, vertex):
    index = {(int(l["ix"]), int(l["iy"]), int(l["iz"])): i for i, l in enumerate(leaves)}
    groups = []
    verts = {}
    for i, l in enumerate(leaves):
        mask = int(l["mask"])
        g_of, n = corner_groups(mask)
        groups.append(g_of)
        for g in range(n):
            pts, grs = [], []
            for s in range(8):
                if g_of.get(s) != g:
                    continue
                for t in (X, Y, Z):
                    if (mask >> (s ^ t)) & 1:
                        continue
                    e = edge_index(s, t)
                    pts.append(l["pos"][e].astype(np.float32))
                    grs.append(l["grad"][e].astype(np.float32))
            verts[(i, g)] = vertex(pts, grs)
    tris = []
    open_edges = 0
    for ci, l in enumerate(leaves):
        mask = int(l["mask"])
        for ti, t in enumerate((X, Y, Z)):
            if (mask & 1) == ((mask >> t) & 1):
                continue
            u = next_axis(t)
            v = next_axis(u)
            c = np.array([int(l["ix"]), int(l["iy"]), int(l["iz"])])
            du = np.array([1 if u & X else 0, 1 if u & Y else 0, 1 if u & Z else 0])
            dv = np.array([1 if v & X else 0, 1 if v & Y else 0, 1 if v & Z else 0])
            cells = [tuple(c - du - dv), tuple(c - dv), tuple(c), tuple(c - du)]       # a, b, c, d
            if any(k not in index for k in cells):
                open_edges += 1
                continue
            ids = [index[k] for k in cells]
            edges = [ti * 4 + 3, ti * 4 + 2, ti * 4 + 0, ti * 4 + 1]
            vs = []
            for k in range(4):
                e = edges[k]
                start = (u if e & 1 else 0) | (v if e & 2 else 0)
                mk = int(leaves[ids[k]]["mask"])
                inside = start if (mk >> start) & 1 else start | t
                vs.append(("v", ids[k], groups[ids[k]][inside]))
            iv = ("i", ids[3], edges[3])                                            # the deepest (= last) cell's intersection
            start_d = (u if edges[3] & 1 else 0) | (v if edges[3] & 2 else 0)
            winding = 1 if (int(leaves[ids[3]]["mask"]) >> start_d) & 1 else 3
            for j in range(4):
                tris.append((vs[j], vs[(j + winding) % 4], iv))
    return verts, tris, open_edges


def write_stl(tris) -> bytes:
    """Mesh::write_stl (output.rs:7-38) for a list of (a, b, c) position triples."""
    hdr = b"This is a binary STL file exported by Fidget"
    out = [hdr + bytes(80 - len(hdr)), struct.pack("<I", len(tris))]
    f = np.float32
    for a, b, c in tris:
        ab, ac = (b - a).astype(f), (c - a).astype(f)
        n = np.array([f(ab[1] * ac[2]) - f(ab[2] * ac[1]), f(ab[2] * ac[0]) - f(ab[0] * ac[2]),
                      f(ab[0] * ac[1]) - f(ab[1] * ac[0])], dtype=f)
        out.append(n.tobytes() + a.astype(f).tobytes() + b.astype(f).tobytes() + c.astype(f).tobytes() + b"\x00\x00")
    return b"".join(out)
