// 2D contours (fc_contour_build): dual contouring on a uniform quadtree of the [-1,1]^2 world square, linked into
// polylines on the device.  The pipeline restricts the mesher's to two dimensions:
//
//   descent    k_tree_level<2, *> (octree.cu): the octree sampler's interval levels with Z fixed (level_job's TREE
//              mode), one launch per depth, four children per cell;
//   leaves     k_contour_leaf: one warp per leaf, four corners, then the samplers' 16-ary edge search (edge_search) --
//              four edges x 16 probes, two points per lane, in one pass; k_contour_grads: (dx, dy, v) at the
//              intersections (grad_at), one lane per edge, with the tape the leaf was sampled with;
//   order      the surface leaves sorted by key (iy, ix): vertex ids come from a scan of the group counts in that
//              order, so vertex id order is key order (iy, ix, group) and the sorted key list is the cell lookup;
//   vertices   k_contour_vertices: one per connected group of inside corners, by the 2D QEF (qef2_vertex);
//   segments   k_contour_segments: every interior sign-changing edge links the vertices owning it in its two cells,
//              inside on the left.  Every vertex owns exactly two sign-changing edges, so it has at most one successor
//              and one predecessor: next[] / prev[] are written directly, without a counting pass;
//   linking    list ranking by pointer jumping over prev[]: pass 1 finds the smallest vertex of every cycle, pass 2
//              cuts each cycle there and ranks every vertex from its polyline's head;
//   emit       one scan over the heads in vertex order gives each polyline's place, and every vertex is scattered to
//              head offset + rank.
//
// A slice stack (fc_contour_build_slices) runs the same pipeline over the slices of a pass at once: slice k owns the cell
// rows [k * 2^depth, (k + 1) * 2^depth) of one tall quadtree grid, level 0 evaluates one root cell per slice, and the
// sort key is (slice, iy, ix), so vertex ids are slice-major, no search or segment leaves its slice, and every slice's
// polylines come out in its own canonical order.  fc_contour_build is the stack of one slice; kernels with STACK = false
// read that slice from their launch parameters, as the one-slice passes of a stack do.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>

#include "capi_internal.h"
#include "level_job.cuh"
#include "pass_plan.h"

namespace fdev {

constexpr uint32_t NONE = ~0u;

// One surface leaf of the quadtree.  Edge e: axis t = e >> 1 (0: along X, 1: along Y) at bit e & 1 of the other axis,
// from corner c0 = (e & 1) << (1 - t) to c0 | 1 << t: edge 0 = corners 0-1, 1 = 2-3, 2 = 0-2, 3 = 1-3.
struct ContourLeaf {
    uint16_t ix, iy;         // cell of its slice
    uint8_t mask, present;   // corner mask; bit e = edge e carries an intersection
    uint16_t slice;          // slice within the pass
    float pos[4][2];
    float grad[4][3];        // dx, dy, v
};

struct ContourLeafParams {
    const TileJob* jobs;
    uint32_t cap_jobs;
    Counters* ctr;
    int list, cursor;
    float cell_h, z;
    uint32_t has_transform;
    Mat4 mat;
    VarBind vb;
    ContourLeaf* out;
    TapeRef* out_tapes;
    uint32_t cap_out;
    uint32_t* n_out;
    CancelRef cancel;
    const ContourSlice* slices;   // STACK: the pass's slice table, `rows` cell rows per slice
    uint32_t rows;
};

__device__ __forceinline__ bool edge_setup2(uint32_t e, uint32_t mask, EdgeState& st) {
    const uint32_t t = e >> 1, u = 1u - t, sv = e & 1u;
    const uint32_t c0 = sv << u, c1 = c0 | (1u << t);
    const bool in0 = (mask >> c0) & 1u, in1 = (mask >> c1) & 1u;
    st.s[2] = st.e[2] = 0u;
    if (in0 == in1) {
        st.s[0] = st.e[0] = st.s[1] = st.e[1] = 0u;
        return false;
    }
    st.s[u] = st.e[u] = sv ? 65535u : 0u;
    st.s[t] = in0 ? 0u : 65535u;   // the search runs inside -> outside
    st.e[t] = in0 ? 65535u : 0u;
    return true;
}

// One warp per leaf job: corner mask, then the four edges' searches in one pass of edge_search (lanes 0-15 follow edges
// 0 and 2, lanes 16-31 edges 1 and 3, one probe each)
template <bool STACK>
__global__ void __launch_bounds__(128) k_contour_leaf(const __grid_constant__ ContourLeafParams p) {
    const int lane = threadIdx.x & 31;
    float2 slots[REG_SLOTS];
    const uint32_t n_jobs = min(p.ctr->n_jobs[p.list], p.cap_jobs);
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_CONTOUR_LEAF, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        const TileJob* job = p.jobs + j;
        // (STACK: the slice of the job's row supplies Z, matrix and vars, and cy is the row within the slice)
        const uint32_t s = STACK ? job->y / p.rows : 0u;
        const uint32_t cx = job->x, cy = STACK ? job->y - s * p.rows : job->y;
        const TapeRef tr = job->tape;
        const float h = p.cell_h;
        const float lo[2] = {float(cx) * h - 1.0f, float(cy) * h - 1.0f};
        const float hi[2] = {float(cx + 1u) * h - 1.0f, float(cy + 1u) * h - 1.0f};
        auto eval2 = [&](float x0, float y0, float x1, float y1) -> float2 {
            float z0 = STACK ? p.slices[s].z : p.z, z1 = z0;
            if (STACK ? p.slices[s].has_transform : p.has_transform) {
                xform_f32(STACK ? p.slices[s].mat : p.mat, x0, y0, z0, x0, y0, z0);
                xform_f32(STACK ? p.slices[s].mat : p.mat, x1, y1, z1, x1, y1, z1);
            }
            const float2 X = make_float2(x0, x1), Y = make_float2(y0, y1), Z = make_float2(z0, z1);
            return run_f32x2(tr.ptr, tr.n_ops, slots, [&](uint32_t i) {
                return pick_input(STACK ? p.slices[s].vb : p.vb, i, X, Y, Z, [](float f) { return make_float2(f, f); });
            });
        };
        const int c = lane & 3;
        const float2 cv = eval2((c & 1) ? hi[0] : lo[0], (c & 2) ? hi[1] : lo[1], lo[0], lo[1]);
        const uint32_t mask = __ballot_sync(FULL, cv.x < 0.0f) & 0xfu;
        if (mask == 0u || mask == 15u) continue;
        uint32_t slot = 0;
        if (lane == 0) slot = atomicAdd(p.n_out, 1u);
        slot = __shfl_sync(FULL, slot, 0);
        if (slot >= p.cap_out) continue;   // counted: the host retries with the exact count
        ContourLeaf* L = p.out + slot;
        const int half = lane >> 4;
        EdgeState s0, s1;
        const bool v0 = edge_setup2(uint32_t(half), mask, s0), v1 = edge_setup2(uint32_t(half) + 2u, mask, s1);
        uint32_t present = 0;
        for (uint32_t e = 0; e < 4u; ++e) {
            EdgeState tmp;
            if (edge_setup2(e, mask, tmp)) present |= 1u << e;
        }
        if (lane == 0) {
            p.out_tapes[slot] = tr;
            L->ix = uint16_t(cx); L->iy = uint16_t(cy);
            L->mask = uint8_t(mask); L->present = uint8_t(present); L->slice = uint16_t(s);
        }
        edge_search<2>(s0, s1, lo, hi, eval2, L->pos, v0, uint32_t(half), v1, uint32_t(half) + 2u);
    }
}

// Gradients at the intersections (grad_at, Z at the slice's): one warp per leaf, one lane per edge
template <bool STACK>
__global__ void __launch_bounds__(128) k_contour_grads(const __grid_constant__ ContourLeafParams p) {
    grd slots[REG_SLOTS];
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t n = min(*p.n_out, p.cap_out);
    for (uint32_t i = warp; i < n; i += n_warps) {
        if (cancel_poll(p.cancel, CS_CONTOUR_GRADS, i)) break;   // (uniform over the warp)
        ContourLeaf* L = p.out + i;
        const TapeRef tr = p.out_tapes[i];
        const uint32_t active = L->present;
        const bool mine = lane < 4 && ((active >> lane) & 1u);
        const int e = mine ? lane : (__ffs(active) - 1);
        const ContourSlice* sl = STACK ? p.slices + L->slice : nullptr;   // (STACK: the leaf's slice)
        const grd r = grad_at(tr, slots, L->pos[e][0], L->pos[e][1], STACK ? sl->z : p.z,
                              STACK ? sl->has_transform : p.has_transform, STACK ? sl->mat : p.mat, STACK ? sl->vb : p.vb);
        if (mine) { L->grad[e][0] = r.y; L->grad[e][1] = r.z; L->grad[e][2] = r.x; }
    }
}

// ---- QEF in 2D (QuadraticErrorSolver restricted to the plane) ---------------------------------------------------
struct Qef2 { float ata[3], atb[2], btb, mp[3]; };   // ata = xx xy yy; mp = x, y, count

__device__ inline void qef2_add_intersection(Qef2& q, const float p[2], const float g[3]) {
    q.mp[0] += p[0]; q.mp[1] += p[1]; q.mp[2] += 1.0f;
    const float nl = sqrtf(g[0] * g[0] + g[1] * g[1]);
    const float n[2] = {g[0] / nl, g[1] / nl};
    const float d = n[0] * p[0] + n[1] * p[1];
    q.ata[0] += n[0] * n[0]; q.ata[1] += n[0] * n[1]; q.ata[2] += n[1] * n[1];
    q.atb[0] += n[0] * d; q.atb[1] += n[1] * d;
    q.btb += d * d;
}

// Symmetric 2x2 eigen-decomposition [[a, b], [b, c]] = V diag(w) V^T: one Jacobi rotation diagonalises it (the
// rotation jacobi3 would apply to the pair, with the classic a - t b / c + t b update)
__device__ inline void eigen2(float a, float b, float c, float w[2], float V[2][2]) {
    if (fabsf(b) < 1e-37f) {
        w[0] = a; w[1] = c;
        V[0][0] = 1.0f; V[0][1] = 0.0f; V[1][0] = 0.0f; V[1][1] = 1.0f;
        return;
    }
    const float theta = (c - a) / (2.0f * b);
    const float t = (theta >= 0.0f ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
    const float cs = 1.0f / sqrtf(t * t + 1.0f), s = t * cs;
    w[0] = a - t * b;
    w[1] = c + t * b;
    V[0][0] = cs; V[0][1] = s; V[1][0] = -s; V[1][1] = cs;
}

// QuadraticErrorSolver::solve in 2D: truncated pseudo-inverse about the mass point (relative cut-off 1e-3), the mass
// point when the solve gives NaN
__device__ inline void qef2_vertex(const Qef2& q, float pos[2]) {
    const float ata[2][2] = {{q.ata[0], q.ata[1]}, {q.ata[1], q.ata[2]}};
    const float center[2] = {q.mp[0] / q.mp[2], q.mp[1] / q.mp[2]};
    float b[2];
    for (int r = 0; r < 2; ++r) b[r] = q.atb[r] - (ata[r][0] * center[0] + ata[r][1] * center[1]);
    float w[2], V[2][2];
    eigen2(q.ata[0], q.ata[1], q.ata[2], w, V);
    int order[2] = {0, 1};
    if (fabsf(w[1]) > fabsf(w[0])) { order[0] = 1; order[1] = 0; }
    const float cutoff = fabsf(w[order[0]]) * 1e-3f;
    int rank = 2;
    for (int k = 0; k < 2; ++k) if (fabsf(w[order[k]]) < cutoff) { rank = k; break; }
    const float eps = rank < 2 ? fabsf(w[order[rank]]) : 0.0f;
    float sol[2] = {0, 0};
    for (int k = 0; k < 2; ++k) {
        const int j = order[k];
        if (!(fabsf(w[j]) > eps)) continue;
        const float coef = (V[0][j] * b[0] + V[1][j] * b[1]) / w[j];
        sol[0] += coef * V[0][j]; sol[1] += coef * V[1][j];
    }
    for (int r = 0; r < 2; ++r) pos[r] = sol[r] + center[r];
    if (!(pos[0] == pos[0] && pos[1] == pos[1])) { pos[0] = center[0]; pos[1] = center[1]; }
}

// Connected groups of a 4-bit mask's inside corners along cell edges, numbered by their lowest corner: 2 bits per
// corner, the group count in bits 8.. (two groups only for the diagonal masks 6 and 9)
__device__ __forceinline__ uint32_t corner_groups2(uint32_t mask) {
    if (mask == 6u) return (1u << 4) | (2u << 8);          // corners 1, 2
    if (mask == 9u) return (1u << 6) | (2u << 8);          // corners 0, 3
    return (mask == 0u ? 0u : 1u) << 8;
}
__device__ __forceinline__ uint32_t group_of(uint32_t packed, uint32_t corner) { return (packed >> (2u * corner)) & 3u; }

// Sort key (slice, iy, ix): 2 * depth bits of cell, the slice above them
__device__ __forceinline__ unsigned long long leaf_key(const ContourLeaf& L, uint32_t depth) {
    return ((unsigned long long)L.slice << (2u * depth)) | ((unsigned long long)L.iy << depth) | L.ix;
}

// Per slice of the pass (ContourScratch::per_slice, PS_WORDS words each): one past its last sorted leaf and its last
// vertex (0: no leaves), its polylines, closed polylines and open edges
enum { PS_LEAF_END, PS_VERT_END, PS_POLYS, PS_CLOSED, PS_OPEN, PS_WORDS };

struct ContourScratch {
    const ContourLeaf* leaves;
    uint32_t n_leaves, side, depth;  // side: cells per axis
    const unsigned long long* keys;  // sorted leaf keys
    const uint32_t* order;           // leaf index of each sorted position
    uint32_t* packed;                // per sorted position: corner groups (corner_groups2)
    uint32_t* n_groups;
    const uint32_t* vbase;           // exclusive scan of n_groups: first vertex of each sorted position
    float2* vpos;                    // [vertex] world position
    uint32_t* vslice;                // [vertex] its slice
    uint32_t* next;
    uint32_t* prev;
    uint32_t* counts;                // [0] vertices [1] polylines, then the per-slice words
    uint32_t* per_slice;
    CancelRef cancel;
};

__global__ void k_contour_keys(const ContourLeaf* leaves, uint32_t n, uint32_t depth, unsigned long long* keys, uint32_t* idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = leaf_key(leaves[i], depth);
    idx[i] = i;
}

__global__ void k_contour_groups(ContourScratch m) {
    if (cancel_poll(m.cancel, CS_CONTOUR_VERTICES, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const uint32_t packed = corner_groups2(m.leaves[m.order[i]].mask);
    m.packed[i] = packed;
    m.n_groups[i] = packed >> 8;
}

// One thread per sorted leaf: a QEF vertex per group; intersections enter in corner order, X-neighbour then Y
__global__ void __launch_bounds__(128) k_contour_vertices(ContourScratch m) {
    if (cancel_poll(m.cancel, CS_CONTOUR_VERTICES, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const ContourLeaf& L = m.leaves[m.order[i]];
    const uint32_t mask = L.mask, packed = m.packed[i], ng = packed >> 8, base = m.vbase[i];
    const uint32_t s = uint32_t(m.keys[i] >> (2u * m.depth));
    if (i == m.n_leaves - 1u) m.counts[0] = base + ng;
    if (i == m.n_leaves - 1u || uint32_t(m.keys[i + 1u] >> (2u * m.depth)) != s) {   // the slice's last leaf
        m.per_slice[PS_WORDS * s + PS_LEAF_END] = i + 1u;
        m.per_slice[PS_WORDS * s + PS_VERT_END] = base + ng;
    }
    for (uint32_t g = 0; g < ng; ++g) {
        m.vslice[base + g] = s;
        Qef2 q{};
        bool forced = false;
        float pos[2];
        for (uint32_t s = 0; s < 4 && !forced; ++s) {
            if (!((mask >> s) & 1u) || group_of(packed, s) != g) continue;
            for (uint32_t t = 1; t < 4; t <<= 1) {
                if ((mask >> (s ^ t)) & 1u) continue;   // not a transition
                const uint32_t e = t == 1u ? ((s >> 1) & 1u) : 2u + (s & 1u);
                const float p[2] = {L.pos[e][0], L.pos[e][1]};
                const float gr3[3] = {L.grad[e][0], L.grad[e][1], L.grad[e][2]};
                if (gr3[0] != gr3[0] || gr3[1] != gr3[1] || gr3[2] != gr3[2]) {   // a NaN gradient snaps to the intersection
                    forced = true;
                    pos[0] = p[0]; pos[1] = p[1];
                    break;
                }
                qef2_add_intersection(q, p, gr3);
            }
        }
        if (!forced) qef2_vertex(q, pos);
        m.vpos[base + g] = make_float2(pos[0], pos[1]);
    }
}

__device__ __forceinline__ uint32_t find_leaf(const ContourScratch& m, unsigned long long key) {
    uint32_t lo = 0, hi = m.n_leaves;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (m.keys[mid] < key) lo = mid + 1u; else hi = mid;
    }
    return lo < m.n_leaves && m.keys[lo] == key ? lo : NONE;
}

// One thread per sorted leaf: its boundary edges are counted, its -X and -Y edges linked to the neighbours' vertices
__global__ void __launch_bounds__(128) k_contour_segments(ContourScratch m) {
    if (cancel_poll(m.cancel, CS_CONTOUR_SEGMENTS, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const ContourLeaf& L = m.leaves[m.order[i]];
    const uint32_t mask = L.mask, x = L.ix, y = L.iy, packed = m.packed[i], base = m.vbase[i];
    const unsigned long long key = m.keys[i];   // (the -X neighbour's key is key - 1, the -Y one's key - side)
    auto in = [](uint32_t mk, uint32_t c) { return (mk >> c) & 1u; };
    uint32_t open = 0;
    if (x + 1u == m.side && in(mask, 1) != in(mask, 3)) ++open;
    if (y + 1u == m.side && in(mask, 2) != in(mask, 3)) ++open;
    // a: this cell's corners on the shared edge (low, high), b: the neighbour's; the neighbour is -X (d = 0) or -Y (d = 1)
    const uint32_t ca[2][2] = {{0u, 2u}, {0u, 1u}}, cb[2][2] = {{1u, 3u}, {2u, 3u}};
    for (uint32_t d = 0; d < 2; ++d) {
        const uint32_t a0 = ca[d][0], a1 = ca[d][1];
        if (in(mask, a0) == in(mask, a1)) continue;
        if ((d == 0 ? x : y) == 0u) { ++open; continue; }
        const uint32_t j = find_leaf(m, d == 0 ? key - 1u : key - m.side);
        const uint32_t mj = j == NONE ? 0u : m.leaves[m.order[j]].mask;
        if (j == NONE || in(mj, cb[d][0]) != in(mask, a0) || in(mj, cb[d][1]) != in(mask, a1)) { ++open; continue; }
        // inside on the left: across a -X edge the path runs +X when the upper corner is inside; across a -Y edge it
        // runs +Y when the left corner is inside
        const bool up = d == 0 ? in(mask, a1) != 0u : in(mask, a0) != 0u;
        const uint32_t ka = up ? (d == 0 ? a1 : a0) : (d == 0 ? a0 : a1);
        const uint32_t kb = up ? (d == 0 ? cb[d][1] : cb[d][0]) : (d == 0 ? cb[d][0] : cb[d][1]);
        const uint32_t va = base + group_of(packed, ka), vb = m.vbase[j] + group_of(m.packed[j], kb);
        const uint32_t from = up ? vb : va, to = up ? va : vb;
        m.next[from] = to;
        m.prev[to] = from;
    }
    if (open) atomicAdd(&m.per_slice[PS_WORDS * uint32_t(key >> (2u * m.depth)) + PS_OPEN], open);
}

// List ranking by pointer jumping, one launch per round (ping-pong buffers).  After k rounds of pass 1, P[v] is the
// vertex 2^k steps back (NONE past an open start) and A[v] the smallest vertex among the 2^k before and including v:
// once 2^k reaches the vertex count, vertices with P[v] != NONE lie on cycles and A[v] is their cycle's minimum.  Pass 2
// runs on prev[] with every cycle cut at that minimum: A[v] becomes the head 2^k - 1 steps back (or the polyline's
// start) and R[v] the distance to it, capped at 2^k.
struct LinkBufs { uint32_t *P[2], *A[2], *R[2]; uint8_t* closed; uint32_t* len; unsigned long long* scan; };

template <int PASS>
__global__ void k_link_init(ContourScratch m, LinkBufs b) {
    if (cancel_poll(m.cancel, CS_CONTOUR_LINK, blockIdx.x)) return;
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.counts[0]) return;
    if (PASS == 1) {
        b.P[0][v] = m.prev[v];
        b.A[0][v] = v;
    } else {   // (reads pass 1's final buffers, index 0 or 1 as the host passes them in P[1] / A[1])
        const bool cyc = b.P[1][v] != NONE;
        const uint32_t p = cyc && b.A[1][v] == v ? NONE : m.prev[v];
        b.closed[v] = cyc;
        b.P[0][v] = p;
        b.A[0][v] = v;
        b.R[0][v] = p != NONE;
    }
}
template <int PASS>
__global__ void k_link_round(ContourScratch m, LinkBufs b) {
    if (cancel_poll(m.cancel, CS_CONTOUR_LINK, blockIdx.x)) return;
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.counts[0]) return;
    const uint32_t p = b.P[0][v];
    if (p == NONE) {
        b.P[1][v] = NONE;
        b.A[1][v] = b.A[0][v];
        if (PASS == 2) b.R[1][v] = b.R[0][v];
        return;
    }
    b.P[1][v] = b.P[0][p];
    if (PASS == 1) b.A[1][v] = min(b.A[0][v], b.A[0][p]);
    else {
        b.A[1][v] = b.A[0][p];
        b.R[1][v] = b.R[0][v] + b.R[0][p];
    }
}
// The last vertex of each polyline (no successor, or its head) writes the polyline's length at the head
__global__ void k_link_lengths(ContourScratch m, LinkBufs b) {
    if (cancel_poll(m.cancel, CS_CONTOUR_LINK, blockIdx.x)) return;
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.counts[0]) return;
    const uint32_t h = b.A[0][v], n = m.next[v];
    if (n == NONE || n == h) b.len[h] = b.R[0][v] + 1u;
}
__global__ void k_link_heads(ContourScratch m, LinkBufs b, uint32_t cap) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= cap) return;
    b.scan[v] = v < m.counts[0] && b.A[0][v] == v ? (1ull << 32) | b.len[v] : 0ull;
}

// Where a pass's polylines go: its first vertex and polyline in the stack's output (v, off, closed point there), and
// the map to model space -- to_model / M / z of the one slice, or (STACK) each vertex's slice's
struct EmitOut {
    float2* v;
    uint32_t* off;
    uint8_t* closed;
    uint32_t v0;            // vertices of the stack before this pass: added to every offset
    bool to_model;
    Mat4 M;
    float z;
    const ContourSlice* slices;
};

// Every vertex to its place (head's offset + rank), in model space when its slice asks; heads write their polyline's
// record and count it for their slice
template <bool STACK>
__global__ void k_contour_emit(ContourScratch m, LinkBufs b, const unsigned long long* scan, const __grid_constant__ EmitOut o) {
    if (cancel_poll(m.cancel, CS_CONTOUR_EMIT, blockIdx.x)) return;
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t nv = m.counts[0];
    if (v >= nv) return;
    const uint32_t h = b.A[0][v], s = m.vslice[v];
    float2 q = m.vpos[v];
    const bool to_model = STACK ? o.slices[s].to_model != 0u : o.to_model;
    if (to_model) {
        float zz = STACK ? o.slices[s].z : o.z;
        xform_f32(STACK ? o.slices[s].mat : o.M, q.x, q.y, zz, q.x, q.y, zz);
    }
    o.v[uint32_t(scan[h]) + b.R[0][v]] = q;
    if (h == v) {
        const uint32_t k = uint32_t(scan[v] >> 32);
        o.off[k] = o.v0 + uint32_t(scan[v]);
        o.closed[k] = b.closed[v];
        atomicAdd(&m.per_slice[PS_WORDS * s + PS_POLYS], 1u);
        if (b.closed[v]) atomicAdd(&m.per_slice[PS_WORDS * s + PS_CLOSED], 1u);
    }
    if (v == nv - 1u) {
        const uint32_t n_poly = uint32_t(scan[v] >> 32) + (h == v ? 1u : 0u);
        m.counts[1] = n_poly;
        o.off[n_poly] = o.v0 + nv;
    }
}

}  // namespace fdev


namespace {
using fdev::ContourSlice;

// Device bytes per surface leaf of a pass, for sizing passes: the leaf and its tape, the sort and group words of
// contour_finish, and per vertex (at most two) its position, slice, links, list-ranking buffers, scans and output
constexpr uint64_t CONTOUR_LEAF_BYTES = sizeof(fdev::ContourLeaf) + sizeof(fdev::TapeRef) + 7 * 4 + 12 +
                                        2 * (8 + 4 + 2 * 4 + 6 * 4 + 1 + 4 + 2 * 8 + 8 + 4 + 1);
}  // namespace

int32_t grow_keep(fc_ctx* c, DevBuf& b, size_t need, size_t keep) {
    if (need <= b.cap) return FC_OK;
    const size_t cap = std::max(need, b.cap + b.cap / 2);
    void* p = nullptr;
    CU(cudaMalloc(&p, cap));
    keep = std::min(keep, b.cap);
    if (keep) CU(cudaMemcpyAsync(p, b.p, keep, cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    b.release();
    b.p = p;
    b.cap = cap;
    return FC_OK;
}

// The quadtree sampler over the n slices sl[0..n) (host; with n > 1 also d_sl on the device): interval levels, then the
// leaf and gradient kernels.  *n_out = surface leaves found (nothing beyond cap written), ctr = the pass's counters.
static int32_t contour_sample(fc_ctx* c, const fc_tape* tape, uint32_t D, const ContourSlice* sl, uint32_t n,
                              const ContourSlice* d_sl, fdev::ContourLeaf* dout, uint64_t cap, uint32_t* n_out_p,
                              fdev::Counters& ctr, const CallCancel& cc) {
    using namespace fdev;
    const int L = int(D) + 1;
    const bool stack = n > 1;
    cudaStream_t s = c->stream;
    TreeScratch t;
    if (int32_t trc = tree_scratch(c, tape, D, 2, n, cap, t)) return trc;
    uint32_t* d_n_out = reinterpret_cast<uint32_t*>(c->counters.as<char>() + sizeof(Counters));
    for (int l = 0; l < L; ++l) {
        LevelParams p = tree_level(c, tape, t, l, sl[0], cc);
        p.z2d = sl[0].z;
        launch_tree_level(p, 2, stack ? d_sl : nullptr, t.blocks(l), s);
    }
    ContourLeafParams q{};
    q.jobs = c->jobs[L].as<TileJob>();
    q.cap_jobs = uint32_t(t.level_cap[L]);
    q.ctr = c->counters.as<Counters>();
    q.list = L; q.cursor = L;
    q.cell_h = 2.0f / float(1u << D);
    q.z = sl[0].z;
    q.has_transform = sl[0].has_transform;
    q.mat = sl[0].mat;
    q.vb = sl[0].vb;
    q.out = dout;
    q.out_tapes = c->leaf_tapes.as<TapeRef>();
    q.cap_out = uint32_t(cap);
    q.n_out = d_n_out;
    q.cancel = cc.ref;
    q.slices = stack ? d_sl : nullptr;
    q.rows = 1u << D;
    if (stack) {
        k_contour_leaf<true><<<c->sm_count * 8, 128, 0, s>>>(q);
        k_contour_grads<true><<<c->sm_count * 8, 128, 0, s>>>(q);
    } else {
        k_contour_leaf<false><<<c->sm_count * 8, 128, 0, s>>>(q);
        k_contour_grads<false><<<c->sm_count * 8, 128, 0, s>>>(q);
    }
    CU(cudaGetLastError());
    uint32_t n_out = 0;
    if (int32_t wrc = wait_read(c, s, cc, &n_out, d_n_out, 4)) return wrc;
    *n_out_p = n_out;
    CU(cudaMemcpy(&ctr, c->counters.p, sizeof ctr, cudaMemcpyDeviceToHost));
    return FC_OK;
}

// Vertices, segments, linking and the polylines of one pass, from its n surface leaves in contour_leaves: appended to
// the stack's output after its v0 vertices and p0 polylines.  cnt receives the pass's vertex and polyline counts, then
// PS_WORDS words per slice.
static int32_t contour_finish(fc_ctx* c, uint32_t n, uint32_t D, const ContourSlice* sl, uint32_t n_sl,
                              const ContourSlice* d_sl, uint64_t v0, uint64_t p0, std::vector<uint32_t>& cnt,
                              float* ms, const CallCancel& cc) {
    using namespace fdev;
    cudaStream_t s = c->stream;
    const uint32_t V = 2u * n;   // at most two vertices per leaf
    ContourScratch m{};
    m.leaves = c->contour_leaves.as<ContourLeaf>();
    m.n_leaves = n;
    m.side = 1u << D;
    m.depth = D;
    m.cancel = cc.ref;
    LinkBufs b{};
    unsigned long long *keys_in, *keys;
    uint32_t *idx_in, *order, *vbase;
    unsigned long long* scan_out;
    int key_bits = int(2 * D);   // (cell, then the slice's bits)
    for (uint32_t k = n_sl - 1; k; k >>= 1) ++key_bits;
    key_bits = std::max(key_bits, 1);
    size_t t_sort = 0, t_scan32 = 0, t_scan64 = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                       (uint32_t*)nullptr, (uint32_t*)nullptr, int(n), 0, key_bits, s));
    CU(cub::DeviceScan::ExclusiveSum(nullptr, t_scan32, (uint32_t*)nullptr, (uint32_t*)nullptr, int(n), s));
    CU(cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (unsigned long long*)nullptr, (unsigned long long*)nullptr, int(V), s));
    const size_t t_cub = std::max(t_sort, std::max(t_scan32, t_scan64));
    void* cub_tmp;
    const size_t w = size_t(n) * 4, wv = size_t(V) * 4;
    const size_t cnt_bytes = (2 + size_t(PS_WORDS) * n_sl) * 4;
    CU(carve(c->contour_scratch, [&](Carve& cv) {
        cv.take(keys_in, 2 * w); cv.take(idx_in, w); cv.take(keys, 2 * w); cv.take(order, w);
        cv.take(m.packed, w); cv.take(m.n_groups, w); cv.take(vbase, w);
        cv.take(m.vpos, size_t(V) * sizeof(float2)); cv.take(m.vslice, wv);
        cv.take(m.next, wv); cv.take(m.prev, wv);
        for (int k = 0; k < 2; ++k) { cv.take(b.P[k], wv); cv.take(b.A[k], wv); cv.take(b.R[k], wv); }
        cv.take(b.closed, V); cv.take(b.len, wv);
        cv.take(b.scan, size_t(V) * 8); cv.take(scan_out, size_t(V) * 8);
        cv.take(m.counts, cnt_bytes);
        cv.take(cub_tmp, t_cub);
    }));
    m.per_slice = m.counts + 2;
    if (int32_t rc = grow_keep(c, c->contour_out, size_t(v0 + V) * sizeof(float2), size_t(v0) * sizeof(float2))) return rc;
    if (int32_t rc = grow_keep(c, c->contour_offs, size_t(p0 + V + 1) * 4, size_t(p0 + 1) * 4)) return rc;
    if (int32_t rc = grow_keep(c, c->contour_flags, size_t(p0 + V), size_t(p0))) return rc;
    EmitOut o{};
    o.v = c->contour_out.as<float2>() + v0;
    o.off = c->contour_offs.as<uint32_t>() + p0;
    o.closed = c->contour_flags.as<uint8_t>() + p0;
    o.v0 = uint32_t(v0);
    o.to_model = sl[0].to_model != 0u;
    o.M = sl[0].mat;
    o.z = sl[0].z;
    o.slices = n_sl > 1 ? d_sl : nullptr;
    m.keys = keys;
    m.order = order;
    m.vbase = vbase;
    CU(cudaEventRecord(get_event(c, 2), s));
    CU(cudaMemsetAsync(m.counts, 0, cnt_bytes, s));
    CU(cudaMemsetAsync(m.next, 0xff, wv, s));
    CU(cudaMemsetAsync(m.prev, 0xff, wv, s));
    const unsigned bl = (n + 127) / 128, bv = (V + 127) / 128;
    k_contour_keys<<<bl, 128, 0, s>>>(m.leaves, n, D, keys_in, idx_in);
    size_t t = t_cub;
    CU(cub::DeviceRadixSort::SortPairs(cub_tmp, t, keys_in, keys, idx_in, order, int(n), 0, key_bits, s));
    k_contour_groups<<<bl, 128, 0, s>>>(m);
    t = t_cub;
    CU(cub::DeviceScan::ExclusiveSum(cub_tmp, t, m.n_groups, vbase, int(n), s));
    k_contour_vertices<<<bl, 128, 0, s>>>(m);
    k_contour_segments<<<bl, 128, 0, s>>>(m);
    // rounds: 2^K >= V covers every cycle and every distance to an open start
    int K = 1;
    while ((1ull << K) < V) ++K;
    auto flip = [](LinkBufs x) { std::swap(x.P[0], x.P[1]); std::swap(x.A[0], x.A[1]); std::swap(x.R[0], x.R[1]); return x; };
    k_link_init<1><<<bv, 128, 0, s>>>(m, b);
    for (int r = 0; r < K; ++r) { k_link_round<1><<<bv, 128, 0, s>>>(m, b); b = flip(b); }
    b = flip(b);   // pass 1's result, now in [1], is what k_link_init<2> reads; it writes [0]
    k_link_init<2><<<bv, 128, 0, s>>>(m, b);
    for (int r = 0; r < K; ++r) { k_link_round<2><<<bv, 128, 0, s>>>(m, b); b = flip(b); }
    k_link_lengths<<<bv, 128, 0, s>>>(m, b);
    k_link_heads<<<bv, 128, 0, s>>>(m, b, V);
    t = t_cub;
    CU(cub::DeviceScan::ExclusiveSum(cub_tmp, t, b.scan, scan_out, int(V), s));
    if (n_sl > 1) k_contour_emit<true><<<bv, 128, 0, s>>>(m, b, scan_out, o);
    else k_contour_emit<false><<<bv, 128, 0, s>>>(m, b, scan_out, o);
    cudaEvent_t e3 = get_event(c, 3);
    CU(cudaEventRecord(e3, s));
    CU(cudaGetLastError());
    cnt.assign(cnt_bytes / 4, 0u);
    if (int32_t wrc = wait_read(c, s, cc, cnt.data(), m.counts, cnt_bytes)) return wrc;
    if (ms) cudaEventElapsedTime(ms, get_event(c, 2), e3);
    return FC_OK;
}

// The passes of a checked stack: every slice's polylines appended to the output in slice order, the per-slice counts
// into per (when given) and their sums into info.  The caller holds the context's lock.
static int32_t contour_stack(fc_ctx* c, const fc_tape* tape, uint32_t D, bool timing, const std::vector<ContourSlice>& sl,
                             fc_contour_info* info, fc_contour_info* per, const CallCancel& cc) {
    using namespace fdev;
    const uint32_t N = uint32_t(sl.size());
    // Passes as the 3D batches' (pass_plan.h), the measured quantity being surface leaves (with their link scratch)
    // within FC_FRAMES_PASS_BYTES.  A pass's slice index is 16 bits in its leaves, and its cell rows must fit 32 bits.
    PassPlan plan = tree_passes(c, N, uint32_t(std::min<uint64_t>({N, 0xffffu, (1ull << (32 - D)) - 1})), D, 2, int(D) + 1,
                                double(CONTOUR_LEAF_BYTES));
    uint64_t n_verts = 0, n_polys = 0;   // the stack's output so far
    std::vector<uint32_t> cnt;
    while (plan.more()) {
        const PassPlan::Range r = plan.take();
        const ContourSlice* ps = sl.data() + r.f0;
        ContourSlice* d_sl = nullptr;
        if (r.n > 1) {
            CU(c->contour_slices.ensure(size_t(r.n) * sizeof(ContourSlice)));
            d_sl = c->contour_slices.as<ContourSlice>();
            CU(cudaMemcpyAsync(d_sl, ps, size_t(r.n) * sizeof(ContourSlice), cudaMemcpyHostToDevice, c->stream));
        }
        // leaves: sized as fc_mesh_build sizes its own (the buffer of the last build, else the perimeter of the square
        // in cells per slice, or the most per slice seen so far), and once more with the exact count
        uint64_t cap = c->contour_leaves.cap / sizeof(ContourLeaf);
        if (cap < 1024) cap = std::max<uint64_t>(1024, r.n * std::min<uint64_t>(1ull << (2 * D), 8ull << D));
        if (plan.use_extra > 0) cap = std::max<uint64_t>(cap, uint64_t(std::ceil(plan.use_extra * 1.25 * r.n)));
        cap = std::min<uint64_t>(cap, 0x7fffffffu);   // (cub's item counts are int)
        uint32_t n = 0;
        Counters ctr;
        for (int attempt = 0; attempt < 2; ++attempt) {
            CU(c->contour_leaves.ensure(cap * sizeof(ContourLeaf)));
            if (timing) CU(cudaEventRecord(get_event(c, 0), c->stream));
            if (int32_t rc = contour_sample(c, tape, D, ps, r.n, d_sl, c->contour_leaves.as<ContourLeaf>(), cap, &n, ctr, cc))
                return rc;
            if (n <= cap || ctr.error) break;
            cap = n;
        }
        bool split = false;
        if (!plan.observe(ctr, n, r, split)) return device_error(ctr.error);
        if (split) continue;
        if (n > cap) return fail(FC_ERR_INVALID, "contour leaf buffer too small: " + std::to_string(n) + " surface leaves");
        if (timing) {
            float ms = 0;
            CU(cudaEventRecord(get_event(c, 1), c->stream));
            CU(cudaEventSynchronize(get_event(c, 1)));
            cudaEventElapsedTime(&ms, get_event(c, 0), get_event(c, 1));
            info->sampler_ms += ms;
        }
        if (!n) continue;
        float ms = 0;
        if (int32_t rc = contour_finish(c, n, D, ps, r.n, d_sl, n_verts, n_polys, cnt, timing ? &ms : nullptr, cc)) return rc;
        info->contour_ms += ms;
        uint32_t leaf_end = 0, vert_end = 0;
        for (uint32_t k = 0; k < r.n; ++k) {
            const uint32_t* wk = cnt.data() + 2 + PS_WORDS * k;
            fc_contour_info si{};
            if (wk[PS_LEAF_END]) {
                si.n_leaves = wk[PS_LEAF_END] - leaf_end;
                si.n_vertices = wk[PS_VERT_END] - vert_end;
                leaf_end = wk[PS_LEAF_END];
                vert_end = wk[PS_VERT_END];
            }
            si.n_polylines = wk[PS_POLYS];
            si.n_closed = wk[PS_CLOSED];
            si.n_open = wk[PS_OPEN];
            if (per) per[r.f0 + k] = si;
            info->n_leaves += si.n_leaves;
            info->n_vertices += si.n_vertices;
            info->n_polylines += si.n_polylines;
            info->n_closed += si.n_closed;
            info->n_open += si.n_open;
        }
        n_verts += cnt[0];
        n_polys += cnt[1];
        if (n_verts > 0xffffffffull)
            return fail(FC_ERR_UNSUPPORTED, "contour stack has more vertices than 32-bit offsets can address");
    }
    c->contour_n_verts = uint32_t(n_verts);
    c->contour_n_polys = uint32_t(n_polys);
    c->contour_offsets = c->contour_offs.as<uint32_t>();
    c->contour_closed = c->contour_flags.as<uint8_t>();
    return FC_OK;
}

// fc_contour_build and fc_contour_build_slices: the checks of every slice, then the stack
static int32_t contour_build(fc_ctx* c, const fc_tape* tape, const fc_contour_cfg* cfg, const fc_contour_slice* slices,
                             uint32_t n_slices, fc_contour_info* info, fc_contour_info* per) {
    memset(info, 0, sizeof *info);
    if (per && n_slices) memset(per, 0, size_t(n_slices) * sizeof *per);
    if (int32_t rc = check_tree_call(tape, 2, cfg->depth, slices, n_slices, "the contour sampler")) return rc;
    std::vector<ContourSlice> sl(n_slices);
    for (uint32_t k = 0; k < n_slices; ++k) {
        const fc_contour_slice& in = slices[k];
        // the 3x3 embedded as the 2D renderers embed it: (x, y, z, 1) -> (m0 x + m1 y + m2, m3 x + m4 y + m5, z, m6 x + m7 y + m8)
        float m[16] = {};
        const int idx[3] = {0, 1, 3};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) m[4 * idx[i] + idx[j]] = in.world_to_model[3 * i + j];
        m[10] = 1.0f;
        if (int32_t vrc = bind_frame(tape, in.has_transform, m, in.z, in.var_values, in.n_var_values, sl[k])) return vrc;
    }
    CallCancel cc;
    auto no_contour = [&](int32_t rc) {   // a failed or cancelled build leaves no contour
        std::lock_guard<std::mutex> guard(c->mu);
        c->contour_n_verts = c->contour_n_polys = 0;
        memset(info, 0, sizeof *info);
        if (per && n_slices) memset(per, 0, size_t(n_slices) * sizeof *per);
        return rc;
    };
    if (int32_t crc = begin_call(c, cc)) return crc == FC_ERR_CANCELLED ? no_contour(crc) : crc;
    std::unique_lock<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    c->contour_n_verts = c->contour_n_polys = 0;
    const int32_t rc = n_slices ? contour_stack(c, tape, cfg->depth, cfg->flags & FC_FLAG_TIMING, sl, info, per, cc) : FC_OK;
    guard.unlock();
    return rc == FC_OK ? rc : no_contour(rc);
}

extern "C" {

int32_t fc_contour_build(fc_ctx* c, const fc_tape* tape, const fc_contour_cfg* cfg, fc_contour_info* info) {
    if (!c || !tape || !cfg || !info) return fail(FC_ERR_INVALID, "null argument");
    fc_contour_slice one{};
    one.z = cfg->z;
    one.has_transform = cfg->has_transform;
    memcpy(one.world_to_model, cfg->world_to_model, sizeof one.world_to_model);
    one.n_var_values = cfg->n_var_values;
    memcpy(one.var_values, cfg->var_values, sizeof one.var_values);
    return contour_build(c, tape, cfg, &one, 1, info, nullptr);
}

int32_t fc_contour_build_slices(fc_ctx* c, const fc_tape* tape, const fc_contour_cfg* cfg, const fc_contour_slice* slices,
                                uint32_t n_slices, fc_contour_info* info, fc_contour_info* per_slice) {
    if (!c || !tape || !cfg || !info) return fail(FC_ERR_INVALID, "null argument");
    return contour_build(c, tape, cfg, slices, n_slices, info, per_slice);
}

int32_t fc_contour_read(fc_ctx* c, float* vertices, uint32_t* offsets, uint8_t* closed) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const uint32_t nv = c->contour_n_verts, np = c->contour_n_polys;
    static const uint32_t zero = 0;
    if (vertices && nv) CU(cudaMemcpyAsync(vertices, c->contour_out.p, size_t(nv) * 8, cudaMemcpyDefault, c->stream));
    if (offsets) CU(cudaMemcpyAsync(offsets, np ? c->contour_offsets : &zero, size_t(np + 1) * 4, cudaMemcpyDefault, c->stream));
    if (closed && np) CU(cudaMemcpyAsync(closed, c->contour_closed, np, cudaMemcpyDefault, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

}  // extern "C"
