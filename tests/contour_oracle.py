"""ORACLE -- test infrastructure, not product code.

numpy restatement of fc_contour_build's definition (include/fidget_cuda.h, DESIGN.md section 10), sharing no code with
the device path:

  sampling   brute force over the full (2^D + 1)^2 corner grid with the oracle's root tape (Tape.float_slice_eval); a
             cell is a surface leaf when its corner mask is not 0 or 15.  Interval results enclose the function and a
             simplified tape returns the root tape's bits inside its box, so this leaf set is the one the device's
             pruned descent keeps;
  edges      the octree sampler's rule: four rounds of 16-ary search from the inside corner to the outside one in u16
             fractions, the bracket midpoint, and the gradient there (Tape.grad_slice_eval), seeded and transformed
             like the device's;
  vertices   one per connected group of inside corners, by the 2D QEF in float32, operation for operation as
             contour.cu's qef2_vertex (tests/qef_f64.py's solve2 is the independent float64 answer);
  polylines  one segment per interior sign-changing edge, inside on the left, linked and put in canonical order.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

f32 = np.float32
ONE = f32(1)


def embed(w2m):
    """The row-major 3x3 world_to_model as the 4x4 the device applies to (x, y, z, 1)."""
    w = np.asarray(w2m, dtype=f32).reshape(3, 3)
    m = np.zeros((4, 4), dtype=f32)
    idx = (0, 1, 3)
    for i in range(3):
        for j in range(3):
            m[idx[i], idx[j]] = w[i, j]
    m[2, 2] = 1
    return m


def xform_f32(M, x, y, z):
    """dev_ops.cuh xform_f32 on arrays: ((m0 x + m1 y) + m2 z) + m3, divided by the homogeneous term where it is not 0."""
    m = M.reshape(16)
    with np.errstate(all="ignore"):
        n = ((m[12] * x + m[13] * y) + m[14] * z) + m[15]
        r = [((m[4 * i] * x + m[4 * i + 1] * y) + m[4 * i + 2] * z) + m[4 * i + 3] for i in range(3)]
        nz = n != 0
        r = [np.where(nz, ri / np.where(nz, n, ONE), ri).astype(f32) for ri in r]
    return r


def _gr_div(a, b):
    d = b[:, 0] * b[:, 0]
    return np.stack([a[:, 0] / b[:, 0]] + [(b[:, 0] * a[:, k] - a[:, 0] * b[:, k]) / d for k in (1, 2, 3)], axis=1).astype(f32)


def xform_gr(M, gx, gy, gz):
    """dev_ops.cuh xform_gr on (n, 4) arrays (value, dx, dy, dz)."""
    m = M.reshape(16)
    with np.errstate(all="ignore"):
        o = []
        for i in range(4):
            r = m[4 * i:4 * i + 4]
            c = np.zeros_like(gx)
            c[:, 0] = r[3]
            o.append((((gx * r[0]) + (gy * r[1])) + (gz * r[2])) + c)
        return [_gr_div(o[k], o[3]) for k in range(3)]


def _lerp_u16(lo, hi, p):
    frac = np.asarray(p, dtype=np.int64).astype(f32) / f32(65535)
    return (lo * (ONE - frac) + hi * frac).astype(f32)


# corner groups: 2 bits per corner, as contour.cu's corner_groups2
def corner_groups(mask):
    if mask == 6:
        return {1: 0, 2: 1}, 2
    if mask == 9:
        return {0: 0, 3: 1}, 2
    return {c: 0 for c in range(4) if (mask >> c) & 1}, 1


def edge_of(s, t):
    """Edge index of corner s's edge along axis bit t (1: X, 2: Y)."""
    return ((s >> 1) & 1) if t == 1 else 2 + (s & 1)


def edge_corners(e):
    t, sv = e >> 1, e & 1
    c0 = sv << (1 - t)
    return c0, c0 | (1 << t)


@dataclass
class Qef2:
    """QuadraticErrorSolver restricted to the plane, accumulated in float32."""
    ata: list = field(default_factory=lambda: [f32(0)] * 3)      # xx xy yy
    atb: list = field(default_factory=lambda: [f32(0)] * 2)
    btb: np.float32 = f32(0)
    mp: list = field(default_factory=lambda: [f32(0)] * 3)       # x, y, count

    def add_intersection(self, p, g):
        self.mp = [self.mp[0] + p[0], self.mp[1] + p[1], self.mp[2] + ONE]
        nl = np.sqrt(g[0] * g[0] + g[1] * g[1])
        n = (g[0] / nl, g[1] / nl)
        d = n[0] * p[0] + n[1] * p[1]
        self.ata = [self.ata[0] + n[0] * n[0], self.ata[1] + n[0] * n[1], self.ata[2] + n[1] * n[1]]
        self.atb = [self.atb[0] + n[0] * d, self.atb[1] + n[1] * d]
        self.btb = self.btb + d * d

    def vertex(self):
        with np.errstate(all="ignore"):
            a, b_, c = self.ata
            center = (self.mp[0] / self.mp[2], self.mp[1] / self.mp[2])
            ata = ((a, b_), (b_, c))
            b = [self.atb[r] - (ata[r][0] * center[0] + ata[r][1] * center[1]) for r in range(2)]
            w, V = eigen2(a, b_, c)
            order = [1, 0] if abs(w[1]) > abs(w[0]) else [0, 1]
            cutoff = abs(w[order[0]]) * f32(1e-3)
            rank = next((k for k in range(2) if abs(w[order[k]]) < cutoff), 2)
            eps = abs(w[order[rank]]) if rank < 2 else f32(0)
            sol = [f32(0), f32(0)]
            for k in range(2):
                j = order[k]
                if not abs(w[j]) > eps:
                    continue
                coef = (V[0][j] * b[0] + V[1][j] * b[1]) / w[j]
                sol = [sol[0] + coef * V[0][j], sol[1] + coef * V[1][j]]
            pos = [sol[0] + center[0], sol[1] + center[1]]
            if np.isnan(pos[0]) or np.isnan(pos[1]):
                pos = list(center)
        return np.array(pos, dtype=f32)


def eigen2(a, b, c):
    """contour.cu's eigen2: one Jacobi rotation of [[a, b], [b, c]] -> (eigenvalues, eigenvectors as columns)."""
    if abs(b) < f32(1e-37):
        return [a, c], [[ONE, f32(0)], [f32(0), ONE]]
    theta = (c - a) / (f32(2) * b)
    t = (ONE if theta >= 0 else -ONE) / (abs(theta) + np.sqrt(theta * theta + ONE))
    cs = ONE / np.sqrt(t * t + ONE)
    s = t * cs
    return [a - t * b, c + t * b], [[cs, s], [-s, cs]]


@dataclass
class Contour:
    vertices: np.ndarray        # (n, 2) float32, polyline order (model space when transformed)
    offsets: np.ndarray         # (k + 1,) uint32
    closed: np.ndarray          # (k,) bool
    n_leaves: int
    n_open: int
    cells: np.ndarray           # (n, 3) per output vertex: iy, ix, group
    qefs: list                  # every Qef2 solved (for the float64 check)


def contour(tape, depth, z=0.0, world_to_model=None, var_values=()) -> Contour:
    n = 1 << depth
    h = f32(2) / f32(n)
    z = f32(z)
    M = None if world_to_model is None else embed(world_to_model)
    slots = tape.data.var_slots()
    n_vars = tape.n_vars

    def values(x, y):
        x = np.asarray(x, dtype=f32)
        y = np.asarray(y, dtype=f32)
        zz = np.full_like(x, z)
        if M is not None:
            x, y, zz = xform_f32(M, x, y, zz)
        ins = []
        for s in range(n_vars):
            ins.append(x if s == slots[0] else y if s == slots[1] else zz if s == slots[2]
                       else np.full_like(x, f32(var_values[s])))
        return tape.float_slice_eval(ins)

    coords = (np.arange(n + 1).astype(f32) * h - ONE).astype(f32)
    gx, gy = np.meshgrid(coords, coords)           # [iy, ix]
    inside = (values(gx.ravel(), gy.ravel()) < 0).reshape(n + 1, n + 1)
    mask = (inside[:-1, :-1].astype(np.int64) | (inside[:-1, 1:] << 1) | (inside[1:, :-1] << 2) | (inside[1:, 1:] << 3))
    iy, ix = np.nonzero((mask != 0) & (mask != 15))     # row-major: sorted by key (iy, ix)
    masks = mask[iy, ix]
    nl = len(iy)
    lo = np.stack([coords[ix], coords[iy]], axis=1)
    hi = np.stack([coords[ix + 1], coords[iy + 1]], axis=1)
    # edge searches of every active edge at once
    recs = []       # (leaf, edge)
    S, E = [], []
    for k in range(nl):
        for e in range(4):
            c0, c1 = edge_corners(e)
            in0, in1 = (masks[k] >> c0) & 1, (masks[k] >> c1) & 1
            if in0 == in1:
                continue
            t, sv = e >> 1, e & 1
            s_ = [0, 0]
            e_ = [0, 0]
            s_[1 - t] = e_[1 - t] = 65535 if sv else 0
            s_[t], e_[t] = (0, 65535) if in0 else (65535, 0)
            recs.append((k, e))
            S.append(s_)
            E.append(e_)
    pos = np.zeros((nl, 4, 2), dtype=f32)
    grad = np.zeros((nl, 4, 3), dtype=f32)
    if recs:
        S = np.array(S, dtype=np.int64)
        E = np.array(E, dtype=np.int64)
        leaf = np.array([r[0] for r in recs])
        edge = np.array([r[1] for r in recs])
        jj = np.arange(16, dtype=np.int64)
        L0, H0 = lo[leaf], hi[leaf]
        for _ in range(4):
            q = (S[:, None, :] * (15 - jj)[None, :, None] + E[:, None, :] * jj[None, :, None]) // 15
            px = _lerp_u16(L0[:, None, 0], H0[:, None, 0], q[:, :, 0])
            py = _lerp_u16(L0[:, None, 1], H0[:, None, 1], q[:, :, 1])
            v = values(px.ravel(), py.ravel()).reshape(-1, 16)
            outside = v >= 0
            frac = np.where(outside.any(axis=1), np.argmax(outside, axis=1), 15)
            frac = np.maximum(frac, 1)[:, None]
            na = (S * (16 - frac) + E * (frac - 1)) // 15
            nb = (S * (15 - frac) + E * frac) // 15
            S, E = na & 0xffff, nb & 0xffff
        mid = ((S + E) // 2) & 0xffff
        p = np.stack([_lerp_u16(L0[:, 0], H0[:, 0], mid[:, 0]), _lerp_u16(L0[:, 1], H0[:, 1], mid[:, 1])], axis=1)
        pos[leaf, edge] = p
        m = len(p)
        g = [np.zeros((m, 4), dtype=f32) for _ in range(3)]
        g[0][:, 0], g[0][:, 1] = p[:, 0], 1
        g[1][:, 0], g[1][:, 2] = p[:, 1], 1
        g[2][:, 0], g[2][:, 3] = z, 1
        if M is not None:
            g = xform_gr(M, *g)
        ins = []
        for s in range(n_vars):
            if s in slots[:3]:
                ins.append(g[slots.index(s)])
            else:
                c = np.zeros((m, 4), dtype=f32)
                c[:, 0] = var_values[s]
                ins.append(c)
        r = tape.grad_slice_eval(ins)
        grad[leaf, edge] = np.stack([r[:, 1], r[:, 2], r[:, 0]], axis=1)
    # vertices, in key order
    groups = [corner_groups(int(mk)) for mk in masks]
    vbase = np.concatenate([[0], np.cumsum([g[1] for g in groups])]).astype(np.int64)
    nv = int(vbase[-1])
    vpos = np.zeros((nv, 2), dtype=f32)
    vcell = np.zeros((nv, 3), dtype=np.int64)
    qefs = []
    for k in range(nl):
        gof, ng = groups[k]
        mk = int(masks[k])
        for g in range(ng):
            q = Qef2()
            forced = None
            for s in range(4):
                if forced is not None:
                    break
                if not (mk >> s) & 1 or gof[s] != g:
                    continue
                for t in (1, 2):
                    if (mk >> (s ^ t)) & 1:
                        continue
                    e = edge_of(s, t)
                    pp, gg = pos[k, e], grad[k, e]
                    if np.isnan(gg).any():
                        forced = pp.copy()
                        break
                    q.add_intersection((pp[0], pp[1]), (gg[0], gg[1], gg[2]))
            if forced is None:
                vpos[vbase[k] + g] = q.vertex()
                qefs.append(q)
            else:
                vpos[vbase[k] + g] = forced
            vcell[vbase[k] + g] = (iy[k], ix[k], g)
    # segments
    index = {(int(a), int(b)): k for k, (a, b) in enumerate(zip(iy, ix))}
    nxt = np.full(nv, -1, dtype=np.int64)
    prv = np.full(nv, -1, dtype=np.int64)
    n_open = 0
    bit = lambda mk, c: (int(mk) >> c) & 1     # noqa: E731
    for k in range(nl):
        mk, x, y = masks[k], int(ix[k]), int(iy[k])
        gof = groups[k][0]
        if x == n - 1 and bit(mk, 1) != bit(mk, 3):
            n_open += 1
        if y == n - 1 and bit(mk, 2) != bit(mk, 3):
            n_open += 1
        for d, (a0, a1), (b0, b1) in ((0, (0, 2), (1, 3)), (1, (0, 1), (2, 3))):
            if bit(mk, a0) == bit(mk, a1):
                continue
            if (x if d == 0 else y) == 0:
                n_open += 1
                continue
            j = index.get((y, x - 1) if d == 0 else (y - 1, x))
            if j is None or bit(masks[j], b0) != bit(mk, a0) or bit(masks[j], b1) != bit(mk, a1):
                n_open += 1
                continue
            up = bit(mk, a1) if d == 0 else bit(mk, a0)
            ka, kb = ((a1, b1) if d == 0 else (a0, b0)) if up else ((a0, b0) if d == 0 else (a1, b1))
            va = vbase[k] + gof[ka]
            vb = vbase[j] + groups[j][0][kb]
            frm, to = (vb, va) if up else (va, vb)
            assert nxt[frm] < 0 and prv[to] < 0
            nxt[frm], prv[to] = to, frm
    # polylines in canonical order
    seen = np.zeros(nv, dtype=bool)
    heads = []

    def walk(v):
        u = v
        while u >= 0 and not seen[u]:
            seen[u] = True
            u = nxt[u]

    for v in np.nonzero(prv < 0)[0]:
        heads.append((int(v), False))
        walk(v)
    for v in range(nv):           # what is left lies on cycles: the first vertex met in id order is its cycle's minimum
        if not seen[v]:
            heads.append((v, True))
            walk(v)
    heads.sort()
    order, offsets, closed = [], [0], []
    for hv, cyc in heads:
        u = hv
        while True:
            order.append(u)
            u = nxt[u]
            if u < 0 or u == hv:
                break
        offsets.append(len(order))
        closed.append(cyc)
    assert len(order) == nv
    verts = vpos[order] if nv else np.zeros((0, 2), dtype=f32)
    if M is not None and not np.array_equal(np.asarray(world_to_model, dtype=f32).reshape(3, 3), np.eye(3, dtype=f32)):
        x, y, _ = xform_f32(M, verts[:, 0].copy(), verts[:, 1].copy(), np.full(nv, z, dtype=f32))
        verts = np.stack([x, y], axis=1).astype(f32)
    return Contour(np.ascontiguousarray(verts, dtype=f32).reshape(-1, 2), np.array(offsets, dtype=np.uint32),
                   np.array(closed, dtype=bool), nl, n_open, vcell[order] if nv else np.zeros((0, 3), np.int64), qefs)
