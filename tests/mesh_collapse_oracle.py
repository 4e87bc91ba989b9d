"""ORACLE -- test infrastructure, not product code.

numpy restatement of the adaptive half of fidget-mesh's Manifold Dual Contouring, on top of the oracle's sampler
output (``oracle.octree_sample``: the surface leaves at the maximum depth with their Hermite data):

  Octree::build      recurse -> leaf -> check_done -> try_collapse -> collapsible (fidget-mesh/src/octree.rs:252-583)
                     with LeafHermiteData::{merge, solve} (octree.rs:912-1033) and QuadraticErrorSolver's error term
                     (qef.rs:111-115); the result is the reference's cell table: Empty / Full / Leaf / Branch per cell
  walk_dual          dc_cell / dc_face / dc_edge (fidget-mesh/src/dc.rs) with MeshBuilder's vertex dedup (builder.rs)

A cell the sampler left no surface leaf in is Empty or Full as a whole; the reference learns which from an interval
evaluation, here it is the sample at the parent's centre, which every child of that parent shares (``sign_at``
decides it for a tree without any surface leaf).  Everything is float32 like the reference; the eigen-solve inside
QuadraticErrorSolver::solve is the device's float32 Jacobi (``jacobi3``), operation for operation, where the reference
calls nalgebra's SVD.  So agreement with the device proves only that the two agree: tests/qef_f64.py solves the same
QEFs in float64, and tests/test_qef_f64.py holds this solve against it (``Octree.qefs`` keeps every QEF solved).
"""
from __future__ import annotations

import numpy as np

from oracle import mesh as om

f32 = np.float32
X, Y, Z = 1, 2, 4
QEF_ERR_EMPTY = f32(-1.0)      # octree.rs:895-899
QEF_ERR_INVALID = f32(-2.0)


def nxt(a):
    return om.next_axis(a)


def axis_index(a):
    return {X: 0, Y: 1, Z: 2}[a]


class Qef:
    """QuadraticErrorSolver (qef.rs): A^T A, A^T b, b^T b and the mass point, accumulated in float32."""

    def __init__(self):
        self.ata = np.zeros((3, 3), dtype=f32)
        self.atb = np.zeros(3, dtype=f32)
        self.btb = f32(0)
        self.mp = np.zeros(4, dtype=f32)

    def copy(self):
        q = Qef()
        q.ata, q.atb, q.btb, q.mp = self.ata.copy(), self.atb.copy(), f32(self.btb), self.mp.copy()
        return q

    def __iadd__(self, o):
        self.ata = (self.ata + o.ata).astype(f32)
        self.atb = (self.atb + o.atb).astype(f32)
        self.btb = f32(self.btb + o.btb)
        self.mp = (self.mp + o.mp).astype(f32)
        return self

    def add_intersection(self, p, g):
        p = np.asarray(p, dtype=f32)
        g = np.asarray(g, dtype=f32)
        self.mp = (self.mp + np.array([p[0], p[1], p[2], 1.0], dtype=f32)).astype(f32)
        nl = f32(np.sqrt(f32(f32(g[0] * g[0] + g[1] * g[1]) + g[2] * g[2])))
        n = np.array([g[0] / nl, g[1] / nl, g[2] / nl], dtype=f32)
        d = f32(f32(n[0] * p[0] + n[1] * p[1]) + n[2] * p[2])
        self.ata = (self.ata + np.outer(n, n).astype(f32)).astype(f32)
        self.atb = (self.atb + (n * d).astype(f32)).astype(f32)
        self.btb = f32(self.btb + f32(d * d))

    def solve(self):
        """QuadraticErrorSolver::solve: (vertex, error clamped to >= 1e-6)."""
        pos, err, _ = self.solve_rank()
        return pos, err

    def solve_rank(self):
        """solve's (vertex, clamped error, rank of the truncated pseudo-inverse).  The truncated pseudo-inverse is the
        float32 Jacobi eigen-solve of the device, operation for operation (see jacobi3): the error term cancels
        down to the size of its rounding where the surface is flat, so a collapse decision near the 2x threshold
        depends on the last bit of the vertex."""
        with np.errstate(all="ignore"):
            a = [[f32(self.ata[r, c]) for c in range(3)] for r in range(3)]
            mp = [f32(v) for v in self.mp]
            center = [mp[0] / mp[3], mp[1] / mp[3], mp[2] / mp[3]]
            b = [f32(self.atb[r]) - ((a[r][0] * center[0] + a[r][1] * center[1]) + a[r][2] * center[2]) for r in range(3)]
            w, V = jacobi3([row[:] for row in a])
            order = [0, 1, 2]
            for x in range(2):
                for y in range(x + 1, 3):
                    if abs(w[order[y]]) > abs(w[order[x]]):
                        order[x], order[y] = order[y], order[x]
            cutoff = abs(w[order[0]]) * f32(1e-3)
            rank = next((k for k in range(3) if abs(w[order[k]]) < cutoff), 3)
            eps = abs(w[order[rank]]) if rank < 3 else f32(0)
            sol = [f32(0), f32(0), f32(0)]
            for k in range(3):
                j = order[k]
                if not abs(w[j]) > eps:
                    continue
                coef = ((V[0][j] * b[0] + V[1][j] * b[1]) + V[2][j] * b[2]) / w[j]
                sol = [sol[r] + coef * V[r][j] for r in range(3)]
            pos = np.array([sol[r] + center[r] for r in range(3)], dtype=f32)
            if np.isnan(pos).any():
                pos = np.array(center, dtype=f32)
            p = pos
            row = [f32(f32(f32(p[0] * a[0][c]) + f32(p[1] * a[1][c])) + f32(p[2] * a[2][c])) for c in range(3)]
            quad = f32(f32(row[0] * p[0] + row[1] * p[1]) + row[2] * p[2])
            lin = f32(f32(f32(2 * p[0]) * self.atb[0] + f32(2 * p[1]) * self.atb[1]) + f32(2 * p[2]) * self.atb[2])
            err = f32(f32(quad - lin) + self.btb)
        return pos, (err if err > f32(1e-6) else f32(1e-6)), rank


def jacobi3(a):
    """Symmetric 3x3 eigen-decomposition by cyclic Jacobi rotations in float32, in the order mesh.cu's jacobi3
    performs them (nalgebra's SVD is a third-party algorithm): returns (eigenvalues, eigenvectors as columns)."""
    one, zero = f32(1), f32(0)
    v = [[one if i == j else zero for j in range(3)] for i in range(3)]
    for _ in range(12):
        off = (abs(a[0][1]) + abs(a[0][2])) + abs(a[1][2])
        if off < f32(1e-30):
            break
        for p in range(2):
            for q in range(p + 1, 3):
                if abs(a[p][q]) < f32(1e-37):
                    continue
                theta = (a[q][q] - a[p][p]) / (f32(2) * a[p][q])
                t = (one if theta >= zero else -one) / (abs(theta) + np.sqrt(theta * theta + one))
                c = one / np.sqrt(t * t + one)
                s = t * c
                for k in range(3):
                    akp, akq = a[k][p], a[k][q]
                    a[k][p] = c * akp - s * akq
                    a[k][q] = s * akp + c * akq
                for k in range(3):
                    apk, aqk = a[p][k], a[q][k]
                    a[p][k] = c * apk - s * aqk
                    a[q][k] = s * apk + c * aqk
                for k in range(3):
                    vkp, vkq = v[k][p], v[k][q]
                    v[k][p] = c * vkp - s * vkq
                    v[k][q] = s * vkp + c * vkq
    return [a[i][i] for i in range(3)], v


class Hermite:
    """LeafHermiteData: 12 intersections (pos.w = 1 when present), 6 face QEFs, the centre QEF, qef_err."""

    def __init__(self):
        self.inter = [None] * 12          # (pos[3], grad[4]) or None
        self.face = [Qef() for _ in range(6)]
        self.center = Qef()
        self.err = QEF_ERR_EMPTY

    def qef_of(self, e):                  # From<LeafIntersection> for QuadraticErrorSolver
        q = Qef()
        if self.inter[e] is not None:
            q.add_intersection(*self.inter[e])
        return q

    @staticmethod
    def merge(ch):
        """LeafHermiteData::merge (octree.rs:917-1021), as written: in the face and centre loops `v` is
        `t.next()` like `u`, and the `u` edges are indexed with edge_index_v."""
        if any(h.err == QEF_ERR_INVALID for h in ch):
            return None
        out = Hermite()
        for t in (X, Y, Z):
            u = nxt(t)
            v = nxt(u)
            for edge in range(4):
                start = (u if edge & 1 else 0) | (v if edge & 2 else 0)
                end = start | t
                e = axis_index(t) * 4 + edge
                a, b = ch[start].inter[e], ch[end].inter[e]
                assert not (a is not None and b is not None), "duplicate intersection"
                out.inter[e] = a if a is not None else b
        for t in (X, Y, Z):
            u = nxt(t)
            v = nxt(t)
            for face in range(2):
                a = t if face == 1 else 0
                b, c, d = a | u, a | v, a | u | v
                f = axis_index(t) * 2 + face
                for q in (a, b, c, d):
                    out.face[f] += ch[q].face[f]
                ev = axis_index(v) * 4 + face * 2 + 1
                out.face[f] += ch[a].qef_of(ev)
                out.face[f] += ch[b].qef_of(ev)
                eu = axis_index(v) * 4 + face * 2 + 1
                out.face[f] += ch[a].qef_of(eu)
                out.face[f] += ch[c].qef_of(eu)
        for t in (X, Y, Z):
            u = nxt(t)
            v = nxt(t)
            a = 0
            b, c, d = a | u, a | v, a | u | v
            for q in (a, b, c, d):
                out.center += ch[q].face[axis_index(t) * 2 + 1]
            out.center += ch[a].qef_of(axis_index(u) * 4 + 3)
            out.center += ch[b].qef_of(axis_index(u) * 4 + 3)
        for h in ch:
            out.center += h.center
        out.err = f32(np.inf)
        for h in ch:
            if h.err >= 0:
                out.err = min(out.err, h.err)
        return out

    def qef(self):                         # the QEF LeafHermiteData::solve solves
        q = self.center.copy()
        for e in range(12):
            q += self.qef_of(e)
        for f in self.face:
            q += f
        return q

    def solve(self):
        return self.qef().solve()


def groups_of(mask):
    """CELL_TO_VERT_TO_EDGES' vertex count and corner -> vertex map (0 vertices without a sign change)."""
    if mask in (0, 255):
        return {}, 0
    return om.corner_groups(mask)


class Octree:
    """Octree::build over the sampler leaves.  ``cells`` maps (depth, x, y, z) to a dict with ``kind`` in
    'E' / 'F' / 'L' / 'B' (plus ``mask``, ``groups`` and the vertices ``verts`` {slot: pos} of a leaf: slots 0-3
    are cell vertices, 4 + e the intersection on undirected edge e).

    ``qefs`` keeps the QEFs that were solved, by cell key: a surface leaf's list with one per vertex group (None for a
    group forced to an intersection by a NaN gradient), and the merged QEF of every cell whose children were merged
    (it became a Leaf or stayed a Branch); ``child_err`` holds the children's error that merged QEF was held
    against.  They are records only: nothing reads them here."""

    def __init__(self, leaves, depth, sign_at=None):
        self.depth = depth
        self.qefs = {}
        self.child_err = {}
        self.leaves = {(depth, int(l["ix"]), int(l["iy"]), int(l["iz"])): l for l in leaves}
        self.anc = set()
        for (d, x, y, z) in self.leaves:
            for k in range(d + 1):
                self.anc.add((d - k, x >> k, y >> k, z >> k))
        self.cells = {}
        root = (0, 0, 0, 0)
        if root in self.anc:
            self._recurse(root)
        else:
            inside = bool(sign_at((-1.0, -1.0, -1.0))) if sign_at else False
            self.cells[root] = {"kind": "F" if inside else "E"}

    # OctreeBuilder::recurse, children first; Empty / Full children take the sign at their parent's centre
    def _recurse(self, key):
        d, x, y, z = key
        if d == self.depth:
            return self._leaf(key)
        kids = [(d + 1, 2 * x + (c & 1), 2 * y + ((c >> 1) & 1), 2 * z + ((c >> 2) & 1)) for c in range(8)]
        herm = [None] * 8
        for c, k in enumerate(kids):
            if k in self.anc:
                herm[c] = self._recurse(k)
        centre = None
        for c, k in enumerate(kids):
            if herm[c] is not None and centre is None:
                centre = self.corner(k, 7 ^ c)
        for c, k in enumerate(kids):
            if herm[c] is None:
                self.cells[k] = {"kind": "F" if centre else "E"}
                herm[c] = Hermite()
        return self._check_done(key, kids, herm)

    def corner(self, key, c):             # Cell::corner; a branch's corner is its child's at that corner
        cell = self.cells[key]
        if cell["kind"] == "L":
            return bool((cell["mask"] >> c) & 1)
        if cell["kind"] == "B":
            return self.corner(self.child(key, c), c)
        return cell["kind"] == "F"

    def _leaf(self, key):
        l = self.leaves[key]
        mask = int(l["mask"])
        g_of, n = groups_of(mask)
        h = Hermite()
        verts = {}
        self.qefs[key] = [None] * n
        for e in range(12):
            if (int(l["present"]) >> e) & 1:
                h.inter[e] = (l["pos"][e].astype(f32), l["grad"][e].astype(f32))
                verts[4 + e] = l["pos"][e].astype(f32)
        for g in range(n):
            q = Qef()
            invalid = False
            for s in range(8):
                if g_of.get(s) != g or invalid:
                    continue
                for t in (X, Y, Z):
                    if (mask >> (s ^ t)) & 1:
                        continue
                    e = om.edge_index(s, t)
                    if np.isnan(l["grad"][e]).any():      # octree.rs:819-827
                        invalid = True
                        verts[g] = l["pos"][e].astype(f32)
                        break
                    q.add_intersection(l["pos"][e], l["grad"][e])
            if invalid:
                h.err = QEF_ERR_INVALID
                continue
            self.qefs[key][g] = q
            verts[g], h.err = q.solve()                 # last writer wins (octree.rs:846-849)
        self.cells[key] = {"kind": "L", "mask": mask, "groups": g_of, "n_groups": n, "verts": verts}
        return h

    def _check_done(self, key, kids, herm):
        kinds = [self.cells[k]["kind"] for k in kids]
        if "B" in kinds:
            self.cells[key] = {"kind": "B"}
            return Hermite()
        if all(k == "F" for k in kinds):
            self.cells[key] = {"kind": "F"}
            return Hermite()
        if all(k == "E" for k in kinds):
            self.cells[key] = {"kind": "E"}
            return Hermite()
        mask = self.collapsible(kids)
        merged = Hermite.merge(herm) if mask is not None else None
        if merged is not None:
            q = merged.qef()
            self.qefs[key], self.child_err[key] = q, merged.err
            pos, err = q.solve()
            if not (err >= merged.err * 2) and self.contains(key, pos):
                merged.err = err
                verts = {0: pos}
                g_of, _ = groups_of(mask)
                for s in g_of:
                    for t in (X, Y, Z):
                        if not (mask >> (s ^ t)) & 1:
                            e = om.edge_index(s, t)
                            verts[4 + e] = merged.inter[e][0]
                self.cells[key] = {"kind": "L", "mask": mask, "groups": g_of, "n_groups": 1, "verts": verts}
                return merged
        self.cells[key] = {"kind": "B"}
        return merged if merged is not None else Hermite()

    @staticmethod
    def contains(key, pos):               # CellBounds::contains: closed intervals
        d, *xyz = key
        size = f32(2.0) / f32(2 ** d)
        for a in range(3):
            lo = f32(-1.0) + f32(xyz[a]) * size
            if not (pos[a] >= lo and pos[a] <= f32(lo + size)):
                return False
        return True

    def collapsible(self, kids):
        """Octree::collapsible (octree.rs:360-440): the corner mask, or None."""
        mask = 0
        for i, k in enumerate(kids):
            cell = self.cells[k]
            if cell["kind"] == "B":
                return None
            if cell["kind"] == "L" and cell["n_groups"] > 1:
                return None
            mask |= int(self.corner(k, i)) << i
        for t, u, v in ((X, Y, Z), (Y, Z, X), (Z, X, Y)):
            for i in range(4):
                a = (u if i & 1 else 0) | (v if i & 2 else 0)
                b = a | t
                center = self.corner(kids[a], b)
                if all(bool((mask >> w) & 1) != center for w in (a, b)):
                    return None
            for i in range(2):
                a = t if (i & 1) == 0 else 0
                b, c, d = a | u, a | v, a | u | v
                center = self.corner(kids[a], d)
                if all(bool((mask >> w) & 1) != center for w in (a, b, c, d)):
                    return None
            center = self.corner(kids[0], t | u | v)
            if all(bool((mask >> w) & 1) != center for w in range(8)):
                return None
        return mask if groups_of(mask)[1] == 1 else None

    # ---- queries -------------------------------------------------------------------------------------------------
    @property
    def root(self):
        return self.cells[(0, 0, 0, 0)]

    def final_leaves(self):
        """(depth, x, y, z, mask) of every Leaf reachable from the root, sorted."""
        out = []
        todo = [(0, 0, 0, 0)]
        while todo:
            k = todo.pop()
            cell = self.cells[k]
            if cell["kind"] == "L":
                out.append((*k, cell["mask"]))
            elif cell["kind"] == "B":
                d, x, y, z = k
                todo += [(d + 1, 2 * x + (c & 1), 2 * y + ((c >> 1) & 1), 2 * z + ((c >> 2) & 1)) for c in range(8)]
        return sorted(out)

    def n_octree_verts(self):
        return sum(len(c["verts"]) for c in self.cells.values() if c["kind"] == "L")

    def is_leaf(self, k):
        return self.cells[k]["kind"] != "B"

    def child(self, k, c):                # Octree::child
        if self.is_leaf(k):
            return k
        d, x, y, z = k
        return (d + 1, 2 * x + (c & 1), 2 * y + ((c >> 1) & 1), 2 * z + ((c >> 2) & 1))

    def walk_dual(self):
        """Octree::walk_dual: (vertices [n,3] float32, triangles [m,3] int64, open edge count)."""
        w = _Walk(self)
        w.cell((0, 0, 0, 0))
        verts = np.array(w.verts, dtype=f32).reshape(-1, 3)
        return verts, np.array(w.tris, dtype=np.int64).reshape(-1, 3), self.open_edges()

    def open_edges(self):
        """Sign-changing edges of final leaves on the boundary of the [-1,1]^3 domain that no dc_edge call reaches:
        one per edge segment, counted at its deepest in-domain leaf (the last of [a, b, c, d] at that depth)."""
        n = 0
        for (d, x, y, z, mask) in self.final_leaves():
            side = 1 << d
            for e in range(12):
                ti, j = divmod(e, 4)
                t = 1 << ti
                u = nxt(t)
                v = nxt(u)
                start = (u if j & 1 else 0) | (v if j & 2 else 0)
                if ((mask >> start) & 1) == ((mask >> (start | t)) & 1):
                    continue
                me = {3: 0, 2: 1, 0: 2, 1: 3}[j]
                du = np.array([u & 1, (u >> 1) & 1, (u >> 2) & 1])
                dv = np.array([v & 1, (v >> 1) & 1, (v >> 2) & 1])
                offu, offv = [0, 1, 1, 0], [0, 0, 1, 1]
                p = np.array([x, y, z])
                pos = [p + (offu[k] - offu[me]) * du + (offv[k] - offv[me]) * dv for k in range(4)]
                inside = [bool(((q >= 0) & (q < side)).all()) for q in pos]
                if all(inside):
                    continue
                depths, skip = [], False
                for k in range(4):
                    if not inside[k]:
                        depths.append(-1)
                        continue
                    r = self._cover(d, pos[k])
                    if r == "branch":
                        skip = True
                    depths.append(r[0] if isinstance(r, tuple) else -1)
                if skip:
                    continue
                if max(k for k in range(4) if depths[k] == d) == me:
                    n += 1
        return n

    def _cover(self, d, p):
        """The final leaf covering cell (d, p): (depth, key); "branch" when smaller leaves own it (a Branch at depth
        d, reachable from the root or not); "empty" for an Empty / Full cell."""
        for k in range(d + 1):
            key = (d - k, int(p[0]) >> k, int(p[1]) >> k, int(p[2]) >> k)
            cell = self.cells.get(key)
            if cell is None:
                continue
            if cell["kind"] == "B":
                return "branch" if k == 0 else "empty"
            if not self._is_final(key):
                continue
            return (d - k, key) if cell["kind"] == "L" else "empty"
        return "empty"

    def _is_final(self, key):
        d, x, y, z = key
        while d > 0:
            d, x, y, z = d - 1, x >> 1, y >> 1, z >> 1
            if self.cells[(d, x, y, z)]["kind"] != "B":
                return False
        return True


class _Walk:
    """MeshBuilder + dc_cell / dc_face / dc_edge (dc.rs)."""

    FRAMES = {X: (X, Y, Z), Y: (Y, Z, X), Z: (Z, X, Y)}

    def __init__(self, octree):
        self.o = octree
        self.map = {}
        self.verts = []
        self.tris = []

    def vertex(self, key):                # MeshBuilder::vertex
        if key not in self.map:
            self.map[key] = len(self.verts)
            self.verts.append(self.o.cells[key[0]]["verts"][key[1]])
        return self.map[key]

    def cell(self, k):
        o = self.o
        if o.cells[k]["kind"] != "B":
            return
        for i in range(8):
            self.cell(o.child(k, i))
        for t in (X, Y, Z):
            _, u, v = self.FRAMES[t]
            for c in (0, u, v, u | v):
                self.face(t, o.child(k, c), o.child(k, c | t))
        for i in (False, True):
            xi, yi, zi = X * i, Y * i, Z * i
            self.edge(X, o.child(k, xi), o.child(k, xi | Y), o.child(k, xi | Y | Z), o.child(k, xi | Z))
            self.edge(Y, o.child(k, yi), o.child(k, yi | Z), o.child(k, yi | X | Z), o.child(k, yi | X))
            self.edge(Z, o.child(k, zi), o.child(k, zi | X), o.child(k, zi | X | Y), o.child(k, zi | Y))

    def face(self, t, lo, hi):
        o = self.o
        if o.is_leaf(lo) and o.is_leaf(hi):
            return
        _, u, v = self.FRAMES[t]
        self.face(t, o.child(lo, t), o.child(hi, 0))
        self.face(t, o.child(lo, t | u), o.child(hi, u))
        self.face(t, o.child(lo, t | v), o.child(hi, v))
        self.face(t, o.child(lo, t | u | v), o.child(hi, u | v))
        for i in (False, True):
            ui, vi = u * i, v * i
            self.edge(u, o.child(lo, ui | t), o.child(lo, ui | v | t), o.child(hi, ui | v), o.child(hi, ui))
            self.edge(v, o.child(lo, vi | t), o.child(hi, vi), o.child(hi, vi | u), o.child(lo, vi | u | t))

    def edge(self, t, a, b, c, d):
        o = self.o
        cs = [a, b, c, d]
        _, u, v = self.FRAMES[t]
        if not all(o.is_leaf(k) for k in cs):
            for i in (False, True):
                ti = t * i
                self.edge(t, o.child(a, ti | u | v), o.child(b, ti | v), o.child(c, ti), o.child(d, ti | u))
            return
        cells = [o.cells[k] for k in cs]
        if any(cell["kind"] != "L" for cell in cells):
            return
        depths = [k[0] for k in cs]
        deepest = max(i for i in range(4) if depths[i] == max(depths))   # Iterator::max_by_key: the last maximum
        ti = axis_index(t)
        edges = [ti * 4 + 3, ti * 4 + 2, ti * 4 + 0, ti * 4 + 1]

        def corners(e):
            s = (u if e & 1 else 0) | (v if e & 2 else 0)
            return s, s | t

        s, en = corners(edges[deepest])
        m = cells[deepest]["mask"]
        start_sign = not (m >> s) & 1
        if start_sign == (not (m >> en) & 1):
            return
        slots = []
        for i in range(4):
            cell = cells[i]
            if depths[i] == depths[deepest]:
                s, en = corners(edges[i])
                inside = s if (cell["mask"] >> s) & 1 else en
                slots.append(cell["groups"][inside])
            else:
                assert cell["n_groups"] == 1, "invalid leaf vertex"
                slots.append(0)
        iv = self.vertex((cs[deepest], 4 + edges[deepest]))
        vs = [self.vertex((cs[i], slots[i])) for i in range(4)]
        winding = 3 if start_sign else 1
        for j in range(4):
            if cs[j] != cs[(j + winding) % 4]:
                self.tris.append((vs[j], vs[(j + winding) % 4], iv))


def build(orc, tape, depth, sign_at=None):
    """Octree::build over ``orc.octree_sample(tape, depth)``."""
    leaves, _ = orc.octree_sample(tape, depth)
    return Octree(leaves, depth, sign_at)


def check_for_vertex_dupes(verts):
    """octree.rs:1561-1570: no two output vertices are bitwise equal."""
    v = np.ascontiguousarray(verts, dtype=f32)
    return len(np.unique(v.view(np.uint32).reshape(-1, 3), axis=0)) == len(v)


def check_for_edge_matching(tris):
    """octree.rs:1572-1594: no degenerate triangle, every directed edge once, each with its reverse."""
    t = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    if ((t[:, 0] == t[:, 1]) | (t[:, 1] == t[:, 2]) | (t[:, 0] == t[:, 2])).any():
        return False
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    keys = e[:, 0] * (1 << 32) + e[:, 1]
    rev = e[:, 1] * (1 << 32) + e[:, 0]
    return len(np.unique(keys)) == len(keys) and bool(np.isin(keys, rev).all())
