// Meshing back half on the device (SURVEY.md section 8f.2): the Hermite data fc_octree_sample leaves in HBM is
// turned into a triangle mesh without going back to the host.
//
//   vertices   one per connected group of inside corners of every surface leaf (the rule behind
//              CELL_TO_VERT_TO_EDGES, fidget-mesh/build.rs:25-130), positioned by the quadratic error
//              function of the group's edge intersections: QuadraticErrorSolver::add_intersection / solve
//              (fidget-mesh/src/qef.rs:44-168) -- mass point, A^T A, truncated pseudo-inverse with the
//              relative eigenvalue cut-off 1e-3; a NaN gradient snaps to the intersection (octree.rs:793-801);
//   triangles  dc_edge (fidget-mesh/src/dc.rs:104-213) for leaves of equal depth: every sign-changing cell edge is
//              shared by four leaves [a, b, c, d] = [0, U, U|V, V] around +T; the four cell vertices form a fan
//              around the edge's intersection vertex (taken from cell d), winding 3 or 1 by the sign at the
//              edge's start;
//   STL        Mesh::write_stl (fidget-mesh/src/output.rs:7-38).
//   collapse   with FC_FLAG_MESH_COLLAPSE only (the default stays the uniform-depth mesh): Octree::check_done /
//              collapsible / try_collapse (octree.rs:252-440) merge the eight children of a cell into one leaf when
//              the topology stays manifold and the merged QEF error (LeafHermiteData::merge / solve,
//              octree.rs:912-1033) is below twice the children's; one launch per depth, bottom-up, over a tree of
//              the surface leaves' ancestors keyed by (depth, x, y, z); the dual is then walked over leaves of
//              different depths (k_tree_faces: dc_cell / dc_face / dc_edge's result, one thread per leaf edge).
//
// The 3x3 symmetric eigen-problem is solved with cyclic Jacobi rotations in f32 (the reference calls nalgebra's
// SVD, a third-party algorithm not under /root/reference); positions agree to ~1e-5 of a cell, not bit for bit.
#include <cstddef>

#include "capi_internal.h"

namespace fdev {

__host__ __device__ inline uint32_t next_axis(uint32_t a) { return a == 1u ? 2u : (a == 2u ? 4u : 1u); }   // X -> Y -> Z -> X

struct MeshScratch {
    const OctreeLeaf* leaves;
    uint32_t n_leaves;
    unsigned long long* hkeys;   // open-addressing table: packed cell coordinates -> leaf index
    uint32_t* hvals;
    uint32_t hmask;
    float3* cell_verts;          // [n_leaves][4]
    uint32_t* corner_vert;       // [n_leaves]: 2 bits per corner = vertex (group) of an inside corner
    uint32_t* remap;             // [n_leaves][16]: slot (4 cell vertices, 12 edge vertices) -> output vertex, or ~0
    uint32_t* counts;            // [0] vertices, [1] triangles, [2] triangle cursor, [3] edges without four leaves
    float3* out_verts;
    uint32_t cap_verts;
    uint3* out_tris;
    uint32_t cap_tris;
    CancelRef cancel;            // polled at block entry of every kernel (item = block index)
};

__device__ __forceinline__ unsigned long long cell_key(uint32_t x, uint32_t y, uint32_t z) {
    return (unsigned long long)x | ((unsigned long long)y << 16) | ((unsigned long long)z << 32);
}
__device__ __forceinline__ uint32_t hash_key(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return uint32_t(k);
}
__global__ void k_mesh_hash(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_MESH_HASH, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const OctreeLeaf& L = m.leaves[i];
    const unsigned long long key = cell_key(L.ix, L.iy, L.iz);
    uint32_t h = hash_key(key) & m.hmask;
    for (;;) {
        const unsigned long long old = atomicCAS(&m.hkeys[h], ~0ull, key);
        if (old == ~0ull || old == key) { m.hvals[h] = i; return; }
        h = (h + 1u) & m.hmask;
    }
}
__device__ __forceinline__ uint32_t find_leaf(const MeshScratch& m, uint32_t x, uint32_t y, uint32_t z) {
    const unsigned long long key = cell_key(x, y, z);
    uint32_t h = hash_key(key) & m.hmask;
    for (;;) {
        const unsigned long long k = m.hkeys[h];
        if (k == key) return m.hvals[h];
        if (k == ~0ull) return ~0u;
        h = (h + 1u) & m.hmask;
    }
}

// Symmetric 3x3 eigen-decomposition by cyclic Jacobi rotations: a = V diag(w) V^T
__device__ inline void jacobi3(float a[3][3], float w[3], float v[3][3]) {
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) v[i][j] = i == j ? 1.0f : 0.0f;
    for (int sweep = 0; sweep < 12; ++sweep) {
        const float off = fabsf(a[0][1]) + fabsf(a[0][2]) + fabsf(a[1][2]);
        if (off < 1e-30f) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (fabsf(a[p][q]) < 1e-37f) continue;
                const float theta = (a[q][q] - a[p][p]) / (2.0f * a[p][q]);
                const float t = (theta >= 0.0f ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
                const float c = 1.0f / sqrtf(t * t + 1.0f), s = t * c;
                for (int k = 0; k < 3; ++k) {   // A <- A J
                    const float akp = a[k][p], akq = a[k][q];
                    a[k][p] = c * akp - s * akq;
                    a[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {   // A <- J^T A
                    const float apk = a[p][k], aqk = a[q][k];
                    a[p][k] = c * apk - s * aqk;
                    a[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const float vkp = v[k][p], vkq = v[k][q];
                    v[k][p] = c * vkp - s * vkq;
                    v[k][q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < 3; ++i) w[i] = a[i][i];
}

// One thread per leaf: groups of inside corners, one QEF vertex per group
__global__ void __launch_bounds__(128) k_mesh_vertices(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_MESH_VERTICES, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const OctreeLeaf& L = m.leaves[i];
    const uint32_t mask = L.mask;
    // connected groups of inside corners along cube edges (label = lowest corner of the group)
    uint32_t label[8];
    for (uint32_t c = 0; c < 8; ++c) label[c] = c;
    for (int it = 0; it < 8; ++it) {
        bool changed = false;
        for (uint32_t c = 0; c < 8; ++c) {
            if (!((mask >> c) & 1u)) continue;
            for (uint32_t ax = 1; ax < 8; ax <<= 1) {
                const uint32_t g = c ^ ax;
                if (!((mask >> g) & 1u)) continue;
                const uint32_t lo = min(label[c], label[g]);
                changed |= (label[c] != lo) | (label[g] != lo);
                label[c] = lo;
                label[g] = lo;
            }
        }
        if (!changed) break;
    }
    uint32_t n_groups = 0, group_of[8], packed = 0;
    for (uint32_t c = 0; c < 8; ++c) {
        group_of[c] = 0;
        if (!((mask >> c) & 1u)) continue;
        if (label[c] == c) group_of[c] = n_groups++;
        else group_of[c] = group_of[label[c]];   // label[c] < c: already numbered
        packed |= (group_of[c] & 3u) << (2u * c);
    }
    m.corner_vert[i] = packed | (n_groups << 16);
    for (uint32_t g = 0; g < n_groups && g < 4u; ++g) {
        // QuadraticErrorSolver (qef.rs:44-61)
        float ata[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, atb[3] = {0, 0, 0}, mp[4] = {0, 0, 0, 0};
        bool forced = false;
        float3 force_pos = make_float3(0, 0, 0);
        for (uint32_t s = 0; s < 8 && !forced; ++s) {
            if (!((mask >> s) & 1u) || group_of[s] != g) continue;
            for (uint32_t t = 1; t < 8 && !forced; t <<= 1) {
                const uint32_t e_end = s ^ t;
                if ((mask >> e_end) & 1u) continue;   // not a transition
                const uint32_t u = next_axis(t), v = next_axis(u);
                const uint32_t ti = t == 1u ? 0u : (t == 2u ? 1u : 2u);
                const uint32_t e = ti * 4u + ((s & u) ? 1u : 0u) + ((s & v) ? 2u : 0u);
                const float px = L.pos[e][0], py = L.pos[e][1], pz = L.pos[e][2];
                const float gx = L.grad[e][0], gy = L.grad[e][1], gz = L.grad[e][2], gw = L.grad[e][3];
                if (gx != gx || gy != gy || gz != gz || gw != gw) {   // octree.rs:793-801
                    forced = true;
                    force_pos = make_float3(px, py, pz);
                    break;
                }
                mp[0] += px; mp[1] += py; mp[2] += pz; mp[3] += 1.0f;
                const float nl = sqrtf(gx * gx + gy * gy + gz * gz);
                const float n[3] = {gx / nl, gy / nl, gz / nl};
                const float d = n[0] * px + n[1] * py + n[2] * pz;
                for (int r = 0; r < 3; ++r) {
                    for (int c2 = 0; c2 < 3; ++c2) ata[r][c2] += n[r] * n[c2];
                    atb[r] += n[r] * d;
                }
            }
        }
        float3 pos;
        if (forced) {
            pos = force_pos;
        } else {
            // QuadraticErrorSolver::solve (qef.rs:67-168)
            const float center[3] = {mp[0] / mp[3], mp[1] / mp[3], mp[2] / mp[3]};
            float b[3];
            for (int r = 0; r < 3; ++r) b[r] = atb[r] - (ata[r][0] * center[0] + ata[r][1] * center[1] + ata[r][2] * center[2]);
            float w[3], V[3][3], a2[3][3];
            for (int r = 0; r < 3; ++r) for (int c2 = 0; c2 < 3; ++c2) a2[r][c2] = ata[r][c2];
            jacobi3(a2, w, V);
            // singular values of a symmetric matrix = |eigenvalues|, sorted descending
            int order[3] = {0, 1, 2};
            for (int x = 0; x < 2; ++x) for (int y = x + 1; y < 3; ++y)
                if (fabsf(w[order[y]]) > fabsf(w[order[x]])) { const int tmp = order[x]; order[x] = order[y]; order[y] = tmp; }
            const float cutoff = fabsf(w[order[0]]) * 1e-3f;
            int rank = 3;
            for (int k = 0; k < 3; ++k) if (fabsf(w[order[k]]) < cutoff) { rank = k; break; }
            const float eps = rank < 3 ? fabsf(w[order[rank]]) : 0.0f;
            float sol[3] = {0, 0, 0};
            for (int k = 0; k < 3; ++k) {
                const int j = order[k];
                if (!(fabsf(w[j]) > eps)) continue;   // svd.solve: singular values <= eps are dropped
                const float coef = (V[0][j] * b[0] + V[1][j] * b[1] + V[2][j] * b[2]) / w[j];
                sol[0] += coef * V[0][j]; sol[1] += coef * V[1][j]; sol[2] += coef * V[2][j];
            }
            pos = make_float3(sol[0] + center[0], sol[1] + center[1], sol[2] + center[2]);
            if (!(pos.x == pos.x && pos.y == pos.y && pos.z == pos.z)) pos = make_float3(center[0], center[1], center[2]);
        }
        m.cell_verts[size_t(i) * 4 + g] = pos;
    }
}

// The four leaves around the +T edge at corner 0 of leaf `c` (dc.rs:104-119), or false at the domain boundary
struct EdgeCells { uint32_t leaf[4]; };
__device__ __forceinline__ bool edge_cells(const MeshScratch& m, uint32_t ci, uint32_t t, EdgeCells& ec) {
    const OctreeLeaf& C = m.leaves[ci];
    const uint32_t u = next_axis(t), v = next_axis(u);
    const uint32_t x = C.ix, y = C.iy, z = C.iz;
    const uint32_t du[3] = {(u & 1u) ? 1u : 0u, (u & 2u) ? 1u : 0u, (u & 4u) ? 1u : 0u};
    const uint32_t dv[3] = {(v & 1u) ? 1u : 0u, (v & 2u) ? 1u : 0u, (v & 4u) ? 1u : 0u};
    if ((du[0] + dv[0]) > x || (du[1] + dv[1]) > y || (du[2] + dv[2]) > z) return false;
    ec.leaf[2] = ci;                                                                   // c = a + U + V
    ec.leaf[0] = find_leaf(m, x - du[0] - dv[0], y - du[1] - dv[1], z - du[2] - dv[2]);  // a
    ec.leaf[1] = find_leaf(m, x - dv[0], y - dv[1], z - dv[2]);                          // b = a + U
    ec.leaf[3] = find_leaf(m, x - du[0], y - du[1], z - du[2]);                          // d = a + V
    return ec.leaf[0] != ~0u && ec.leaf[1] != ~0u && ec.leaf[3] != ~0u;
}

// pass 0: mark the vertex slots in use and count triangles; pass 1: emit
template <int PASS>
__global__ void __launch_bounds__(128) k_mesh_faces(MeshScratch m) {
    if (cancel_poll(m.cancel, PASS == 0 ? CS_MESH_FACES0 : CS_MESH_FACES1, blockIdx.x)) return;
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= m.n_leaves * 3u) return;
    const uint32_t ci = gid / 3u, ti = gid % 3u, t = 1u << ti;
    const OctreeLeaf& C = m.leaves[ci];
    const uint32_t in0 = C.mask & 1u, in1 = (C.mask >> t) & 1u;
    if (in0 == in1) return;
    EdgeCells ec;
    if (!edge_cells(m, ci, t, ec)) {
        if (PASS == 0) atomicAdd(&m.counts[3], 1u);
        return;
    }
    const uint32_t u = next_axis(t), v = next_axis(u);
    const uint32_t edge_of[4] = {ti * 4u + 3u, ti * 4u + 2u, ti * 4u + 0u, ti * 4u + 1u};   // a, b, c, d
    uint32_t slot[4];
    for (int k = 0; k < 4; ++k) {
        const uint32_t e = edge_of[k];
        const uint32_t start = ((e & 1u) ? u : 0u) | ((e & 2u) ? v : 0u), end = start | t;
        const uint32_t mk = m.leaves[ec.leaf[k]].mask;
        const uint32_t inside_corner = ((mk >> start) & 1u) ? start : end;
        if ((((mk >> start) & 1u) == ((mk >> end) & 1u))) {   // the neighbour does not see the sign change: skip
            if (PASS == 0) atomicAdd(&m.counts[3], 1u);
            return;
        }
        slot[k] = ec.leaf[k] * 16u + ((m.corner_vert[ec.leaf[k]] >> (2u * inside_corner)) & 3u);
    }
    const uint32_t islot = ec.leaf[3] * 16u + 4u + edge_of[3];   // intersection vertex: cell d's copy
    if (PASS == 0) {
        for (int k = 0; k < 4; ++k) m.remap[slot[k]] = 1u;
        m.remap[islot] = 1u;
        atomicAdd(&m.counts[1], 4u);
        return;
    }
    // winding (dc.rs:188-196): 3 when the edge's start corner is outside, else 1
    const uint32_t md = m.leaves[ec.leaf[3]].mask;
    const uint32_t start_d = ((edge_of[3] & 1u) ? u : 0u) | ((edge_of[3] & 2u) ? v : 0u);
    const uint32_t winding = ((md >> start_d) & 1u) ? 1u : 3u;
    const uint32_t base = atomicAdd(&m.counts[2], 4u);
    const uint32_t iv = m.remap[islot];
    for (uint32_t j = 0; j < 4u; ++j)
        if (base + j < m.cap_tris) m.out_tris[base + j] = make_uint3(m.remap[slot[j]], m.remap[slot[(j + winding) & 3u]], iv);
}

// compaction of the used vertex slots
__global__ void k_mesh_assign(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_MESH_ASSIGN, blockIdx.x)) return;
    const uint64_t s = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (s >= uint64_t(m.n_leaves) * 16u) return;
    if (m.remap[s] != 1u) { m.remap[s] = ~0u; return; }
    const uint32_t id = atomicAdd(&m.counts[0], 1u);
    m.remap[s] = id;
    if (id >= m.cap_verts) return;
    const uint32_t leaf = uint32_t(s / 16u), k = uint32_t(s % 16u);
    if (k < 4u) m.out_verts[id] = m.cell_verts[size_t(leaf) * 4 + k];
    else {
        const OctreeLeaf& L = m.leaves[leaf];
        m.out_verts[id] = make_float3(L.pos[k - 4u][0], L.pos[k - 4u][1], L.pos[k - 4u][2]);
    }
}

// Octree::build's last step (octree.rs:58-65): every vertex goes from the [-1,1]^3 cube the octree was built in back to
// model space, through Matrix4::transform_point.  `pos` is the first of *count (at most cap) float triples `stride`
// bytes apart: the vertex buffer, or the vertex field of the final-leaf list.
__global__ void k_mesh_to_model(char* pos, size_t stride, const uint32_t* count, uint32_t cap, Mat4 M) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(*count, cap)) return;
    float* p = reinterpret_cast<float*>(pos + size_t(i) * stride);
    xform_f32(M, p[0], p[1], p[2], p[0], p[1], p[2]);
}

// Mesh::write_stl (output.rs:7-38): 80-byte header, u32 count, 50 bytes per triangle
__global__ void k_mesh_stl(const float3* verts, const uint3* tris, uint32_t n_tris, uint8_t* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        const char hdr[] = "This is a binary STL file exported by Fidget";
        for (int k = 0; k < 80; ++k) out[k] = k < int(sizeof(hdr) - 1) ? uint8_t(hdr[k]) : 0;
        for (int k = 0; k < 4; ++k) out[80 + k] = uint8_t(n_tris >> (8 * k));
    }
    if (i >= n_tris) return;
    const uint3 t = tris[i];
    const float3 a = verts[t.x], b = verts[t.y], c = verts[t.z];
    const float3 ab = make_float3(b.x - a.x, b.y - a.y, b.z - a.z), ac = make_float3(c.x - a.x, c.y - a.y, c.z - a.z);
    const float rec[12] = {ab.y * ac.z - ab.z * ac.y, ab.z * ac.x - ab.x * ac.z, ab.x * ac.y - ab.y * ac.x,
                           a.x, a.y, a.z, b.x, b.y, b.z, c.x, c.y, c.z};
    uint16_t* dst = reinterpret_cast<uint16_t*>(out + 84 + size_t(i) * 50);   // 84 + 50 i is even
    for (int k = 0; k < 12; ++k) {
        const uint32_t bits = __float_as_uint(rec[k]);
        dst[2 * k] = uint16_t(bits & 0xffffu);
        dst[2 * k + 1] = uint16_t(bits >> 16);
    }
    dst[24] = 0;
}

// ---- cell collapse and the adaptive dual walk (FC_FLAG_MESH_COLLAPSE) ---------------------------------------------
// The tree: node ids [0, n_leaves) are the sampler's surface leaves (depth D); the ids after them are their ancestors,
// built level by level bottom-up, so every depth is one contiguous id range.  A cell that is not a node is Empty or
// Full as a whole (it holds no surface leaf, and neighbouring cells share their corner samples); its sign is the sign
// at its parent's centre, which every child of that parent shares and a node child knows from its corner mask.
constexpr float QEF_ERR_EMPTY = -1.0f, QEF_ERR_INVALID = -2.0f;   // octree.rs:895-899
enum : uint8_t { NODE_LEAF = 1, NODE_BRANCH = 2, NODE_FINAL = 4 };

struct Qef { float ata[6], atb[3], btb, mp[4]; };   // QuadraticErrorSolver; ata = xx xy xz yy yz zz
struct Hermite { float ipos[12][4], igrad[12][4]; Qef face[6], center; };   // LeafHermiteData (qef_err: node_err)

struct TreeScratch {
    const OctreeLeaf* leaves;
    uint32_t n_leaves, depth;
    unsigned long long* hkeys;   // (depth, x, y, z) -> node id
    uint32_t* hvals;
    uint32_t hmask;
    unsigned long long* node_key;
    uint32_t* node_mask;         // corner mask (leaves: CellMask; branches: the signs at their eight corners)
    uint8_t* node_state;
    float* node_err;             // LeafHermiteData::qef_err
    float3* node_vert;           // vertex of a collapsed leaf
    Hermite* herm;               // [node - n_leaves]
    const float3* cell_verts;    // k_mesh_vertices' output for the surface leaves
    const uint32_t* corner_vert;
    uint32_t n_nodes;
    uint32_t* remap;             // [n_nodes][16] as MeshScratch::remap
    uint32_t* counts;            // [0] vertices [1] triangles [2] triangle cursor [3] open edges [4] nodes [5] final leaves
    float3* out_verts;
    uint32_t cap_verts;
    uint3* out_tris;
    uint32_t cap_tris;
    fc_mesh_cell* out_cells;
    CancelRef cancel;            // as MeshScratch::cancel
};

__host__ __device__ __forceinline__ unsigned long long tree_key(uint32_t d, uint32_t x, uint32_t y, uint32_t z) {
    return (unsigned long long)x | ((unsigned long long)y << 16) | ((unsigned long long)z << 32) | ((unsigned long long)d << 48);
}
__device__ __forceinline__ uint32_t key_x(unsigned long long k, int a) { return uint32_t(k >> (16 * a)) & 0xffffu; }
__device__ __forceinline__ uint32_t key_depth(unsigned long long k) { return uint32_t(k >> 48); }
__device__ __forceinline__ uint32_t tree_find(const TreeScratch& m, unsigned long long key) {
    uint32_t h = hash_key(key) & m.hmask;
    for (;;) {
        const unsigned long long k = m.hkeys[h];
        if (k == key) return m.hvals[h];
        if (k == ~0ull) return ~0u;
        h = (h + 1u) & m.hmask;
    }
}
// returns true when `key` was new; the caller owns hvals[slot] then
__device__ __forceinline__ bool tree_insert(const TreeScratch& m, unsigned long long key, uint32_t& slot) {
    uint32_t h = hash_key(key) & m.hmask;
    for (;;) {
        const unsigned long long old = atomicCAS(&m.hkeys[h], ~0ull, key);
        if (old == ~0ull) { slot = h; return true; }
        if (old == key) return false;
        h = (h + 1u) & m.hmask;
    }
}

__device__ inline void qef_zero(Qef& q) {
    for (int k = 0; k < 6; ++k) q.ata[k] = 0.0f;
    for (int k = 0; k < 3; ++k) q.atb[k] = 0.0f;
    q.btb = 0.0f;
    for (int k = 0; k < 4; ++k) q.mp[k] = 0.0f;
}
__device__ inline void qef_add(Qef& q, const Qef& r) {   // AddAssign (qef.rs:19-26)
    for (int k = 0; k < 6; ++k) q.ata[k] += r.ata[k];
    for (int k = 0; k < 3; ++k) q.atb[k] += r.atb[k];
    q.btb += r.btb;
    for (int k = 0; k < 4; ++k) q.mp[k] += r.mp[k];
}
__device__ inline void qef_add_intersection(Qef& q, const float p[3], const float g[4]) {   // qef.rs:48-59
    q.mp[0] += p[0]; q.mp[1] += p[1]; q.mp[2] += p[2]; q.mp[3] += 1.0f;
    const float nl = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
    const float n[3] = {g[0] / nl, g[1] / nl, g[2] / nl};
    const float d = n[0] * p[0] + n[1] * p[1] + n[2] * p[2];
    q.ata[0] += n[0] * n[0]; q.ata[1] += n[0] * n[1]; q.ata[2] += n[0] * n[2];
    q.ata[3] += n[1] * n[1]; q.ata[4] += n[1] * n[2]; q.ata[5] += n[2] * n[2];
    for (int r = 0; r < 3; ++r) q.atb[r] += n[r] * d;
    q.btb += d * d;
}
// QuadraticErrorSolver::solve (qef.rs:67-118): the vertex as k_mesh_vertices places it, and the clamped error
__device__ inline float qef_solve(const Qef& q, float pos[3]) {
    const float ata[3][3] = {{q.ata[0], q.ata[1], q.ata[2]}, {q.ata[1], q.ata[3], q.ata[4]}, {q.ata[2], q.ata[4], q.ata[5]}};
    const float center[3] = {q.mp[0] / q.mp[3], q.mp[1] / q.mp[3], q.mp[2] / q.mp[3]};
    float b[3];
    for (int r = 0; r < 3; ++r) b[r] = q.atb[r] - (ata[r][0] * center[0] + ata[r][1] * center[1] + ata[r][2] * center[2]);
    float w[3], V[3][3], a2[3][3];
    for (int r = 0; r < 3; ++r) for (int c2 = 0; c2 < 3; ++c2) a2[r][c2] = ata[r][c2];
    jacobi3(a2, w, V);
    int order[3] = {0, 1, 2};
    for (int x = 0; x < 2; ++x) for (int y = x + 1; y < 3; ++y)
        if (fabsf(w[order[y]]) > fabsf(w[order[x]])) { const int tmp = order[x]; order[x] = order[y]; order[y] = tmp; }
    const float cutoff = fabsf(w[order[0]]) * 1e-3f;
    int rank = 3;
    for (int k = 0; k < 3; ++k) if (fabsf(w[order[k]]) < cutoff) { rank = k; break; }
    const float eps = rank < 3 ? fabsf(w[order[rank]]) : 0.0f;
    float sol[3] = {0, 0, 0};
    for (int k = 0; k < 3; ++k) {
        const int j = order[k];
        if (!(fabsf(w[j]) > eps)) continue;
        const float coef = (V[0][j] * b[0] + V[1][j] * b[1] + V[2][j] * b[2]) / w[j];
        sol[0] += coef * V[0][j]; sol[1] += coef * V[1][j]; sol[2] += coef * V[2][j];
    }
    for (int r = 0; r < 3; ++r) pos[r] = sol[r] + center[r];
    if (!(pos[0] == pos[0] && pos[1] == pos[1] && pos[2] == pos[2])) for (int r = 0; r < 3; ++r) pos[r] = center[r];
    // pos^T A^T A pos - 2 pos^T A^T b + b^T b, clamped to >= 1e-6 (qef.rs:111-115)
    float row[3];
    for (int c2 = 0; c2 < 3; ++c2) row[c2] = pos[0] * ata[0][c2] + pos[1] * ata[1][c2] + pos[2] * ata[2][c2];
    const float quad = row[0] * pos[0] + row[1] * pos[1] + row[2] * pos[2];
    const float lin = (2.0f * pos[0]) * q.atb[0] + (2.0f * pos[1]) * q.atb[1] + (2.0f * pos[2]) * q.atb[2];
    const float err = (quad - lin) + q.btb;
    return err > 1e-6f ? err : 1e-6f;   // f32::max: a NaN error becomes 1e-6
}

// Surface leaves enter the tree at depth D
__global__ void k_tree_leaves(TreeScratch m) {
    if (cancel_poll(m.cancel, CS_TREE_LEAVES, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const OctreeLeaf& L = m.leaves[i];
    const unsigned long long key = tree_key(m.depth, L.ix, L.iy, L.iz);
    uint32_t slot;
    if (tree_insert(m, key, slot)) m.hvals[slot] = i;
    m.node_key[i] = key;
    m.node_mask[i] = L.mask;
    m.node_state[i] = NODE_LEAF;
}
// The parents of the nodes [lo, hi) (one depth), appended as new nodes
__global__ void k_tree_parents(TreeScratch m, uint32_t lo, uint32_t hi) {
    if (cancel_poll(m.cancel, CS_TREE_PARENTS, blockIdx.x)) return;
    const uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    const unsigned long long k = m.node_key[i];
    const unsigned long long pk = tree_key(key_depth(k) - 1u, key_x(k, 0) >> 1, key_x(k, 1) >> 1, key_x(k, 2) >> 1);
    uint32_t slot;
    if (!tree_insert(m, pk, slot)) return;
    const uint32_t id = atomicAdd(&m.counts[4], 1u);
    m.hvals[slot] = id;
    m.node_key[id] = pk;
}

// LeafHermiteData::qef_err of every surface leaf (OctreeBuilder::leaf, octree.rs:810-851): one QEF per vertex group,
// the last group's error wins; a NaN gradient marks the group QEF_ERR_INVALID
__global__ void __launch_bounds__(128) k_tree_leaf_err(TreeScratch m) {
    if (cancel_poll(m.cancel, CS_TREE_LEAF_ERR, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const OctreeLeaf& L = m.leaves[i];
    const uint32_t mask = L.mask, cv = m.corner_vert[i], n_groups = cv >> 16;
    float err = QEF_ERR_EMPTY;
    for (uint32_t g = 0; g < n_groups && g < 4u; ++g) {
        Qef q;
        qef_zero(q);
        bool invalid = false;
        for (uint32_t s = 0; s < 8 && !invalid; ++s) {
            if (!((mask >> s) & 1u) || ((cv >> (2u * s)) & 3u) != g) continue;
            for (uint32_t t = 1; t < 8; t <<= 1) {
                if ((mask >> (s ^ t)) & 1u) continue;
                const uint32_t u = next_axis(t), v = next_axis(u);
                const uint32_t ti = t == 1u ? 0u : (t == 2u ? 1u : 2u);
                const uint32_t e = ti * 4u + ((s & u) ? 1u : 0u) + ((s & v) ? 2u : 0u);
                const float p[3] = {L.pos[e][0], L.pos[e][1], L.pos[e][2]};
                const float gr[4] = {L.grad[e][0], L.grad[e][1], L.grad[e][2], L.grad[e][3]};
                if (gr[0] != gr[0] || gr[1] != gr[1] || gr[2] != gr[2] || gr[3] != gr[3]) { invalid = true; break; }
                qef_add_intersection(q, p, gr);
            }
        }
        if (invalid) { err = QEF_ERR_INVALID; continue; }
        float pos[3];
        err = qef_solve(q, pos);
    }
    m.node_err[i] = err;
}

// Hermite data of one child, as LeafHermiteData::merge reads it: a surface leaf's intersections, a collapsed leaf's
// merged record, or the default record of an Empty / Full cell (no intersections, zero QEFs)
__device__ __forceinline__ bool child_inter(const TreeScratch& m, uint32_t ch, uint32_t e, float p[3], float g[4]) {
    if (ch == ~0u) return false;
    if (ch < m.n_leaves) {
        const OctreeLeaf& L = m.leaves[ch];
        if (!((L.present >> e) & 1u)) return false;
        for (int k = 0; k < 3; ++k) p[k] = L.pos[e][k];
        for (int k = 0; k < 4; ++k) g[k] = L.grad[e][k];
        return true;
    }
    const Hermite& H = m.herm[ch - m.n_leaves];
    if (!(H.ipos[e][3] != 0.0f)) return false;
    for (int k = 0; k < 3; ++k) p[k] = H.ipos[e][k];
    for (int k = 0; k < 4; ++k) g[k] = H.igrad[e][k];
    return true;
}
__device__ __forceinline__ void add_child_inter(const TreeScratch& m, uint32_t ch, uint32_t e, Qef& q) {   // From<LeafIntersection>
    float p[3], g[4];
    if (child_inter(m, ch, e, p, g)) qef_add_intersection(q, p, g);
}
__device__ __forceinline__ void add_child_face(const TreeScratch& m, uint32_t ch, uint32_t f, Qef& q) {
    if (ch != ~0u && ch >= m.n_leaves) qef_add(q, m.herm[ch - m.n_leaves].face[f]);
}
__device__ __forceinline__ uint32_t axis_index(uint32_t a) { return a == 1u ? 0u : (a == 2u ? 1u : 2u); }

// One thread per node of one depth: Octree::check_done / collapsible / try_collapse (octree.rs:252-440) with
// LeafHermiteData::merge / solve (octree.rs:917-1033)
__global__ void __launch_bounds__(128) k_tree_collapse(TreeScratch m, uint32_t lo, uint32_t hi) {
    if (cancel_poll(m.cancel, CS_TREE_COLLAPSE, blockIdx.x)) return;
    const uint32_t id = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= hi) return;
    const unsigned long long key = m.node_key[id];
    const uint32_t d = key_depth(key), x = key_x(key, 0), y = key_x(key, 1), z = key_x(key, 2);
    uint32_t ch[8];
    for (uint32_t c = 0; c < 8; ++c)
        ch[c] = tree_find(m, tree_key(d + 1u, 2u * x + (c & 1u), 2u * y + ((c >> 1) & 1u), 2u * z + ((c >> 2) & 1u)));
    uint32_t centre = 0;   // sign at this cell's centre: corner 7 ^ c of child c
    for (uint32_t c = 0; c < 8; ++c)
        if (ch[c] != ~0u) { centre = (m.node_mask[ch[c]] >> (7u ^ c)) & 1u; break; }
    uint32_t cmask = 0, cm[8];   // cm[c]: corner mask of child c (Empty / Full: all corners alike)
    bool branch = false, multi = false;
    for (uint32_t c = 0; c < 8; ++c) {
        if (ch[c] == ~0u) { cm[c] = centre ? 0xffu : 0u; }
        else {
            cm[c] = m.node_mask[ch[c]];
            branch |= (m.node_state[ch[c]] & NODE_BRANCH) != 0;
            multi |= ch[c] < m.n_leaves && (m.corner_vert[ch[c]] >> 16) > 1u;   // CELL_TO_VERT_TO_EDGES[mask].len() > 1
        }
        cmask |= ((cm[c] >> c) & 1u) << c;
    }
    m.node_mask[id] = cmask;
    m.node_state[id] = NODE_BRANCH;
    if (branch || multi) return;
    // collapsible: the three predicates of Ju et al. 2002, section 4.1
    const uint32_t frames[3][3] = {{1u, 2u, 4u}, {2u, 4u, 1u}, {4u, 1u, 2u}};
    for (int f = 0; f < 3; ++f) {
        const uint32_t t = frames[f][0], u = frames[f][1], v = frames[f][2];
        for (uint32_t i = 0; i < 4; ++i) {
            const uint32_t a = ((i & 1u) ? u : 0u) | ((i & 2u) ? v : 0u), b = a | t;
            const uint32_t mid = (cm[a] >> b) & 1u;
            if (((cmask >> a) & 1u) != mid && ((cmask >> b) & 1u) != mid) return;
        }
        for (uint32_t i = 0; i < 2; ++i) {
            const uint32_t a = (i & 1u) == 0 ? t : 0u, q[4] = {a, a | u, a | v, a | u | v};
            const uint32_t mid = (cm[a] >> (a | u | v)) & 1u;
            bool agree = false;
            for (int k = 0; k < 4; ++k) agree |= ((cmask >> q[k]) & 1u) == mid;
            if (!agree) return;
        }
        const uint32_t mid = (cm[0] >> (t | u | v)) & 1u;
        bool agree = false;
        for (uint32_t k = 0; k < 8; ++k) agree |= ((cmask >> k) & 1u) == mid;
        if (!agree) return;
    }
    if (cmask == 0u || cmask == 0xffu) return;
    {   // one vertex group (the collapsed cell is manifold)
        uint32_t label[8];
        for (uint32_t c = 0; c < 8; ++c) label[c] = c;
        for (int it = 0; it < 8; ++it)
            for (uint32_t c = 0; c < 8; ++c)
                for (uint32_t ax = 1; ax < 8; ax <<= 1) {
                    const uint32_t g = c ^ ax;
                    if (((cmask >> c) & 1u) && ((cmask >> g) & 1u)) { const uint32_t lo2 = min(label[c], label[g]); label[c] = label[g] = lo2; }
                }
        for (uint32_t c = 0; c < 8; ++c) if (((cmask >> c) & 1u) && label[c] != label[__ffs(cmask) - 1]) return;
    }
    // merge: any invalid child QEF stops the collapse
    float child_err = INFINITY;
    for (uint32_t c = 0; c < 8; ++c) {
        const float e = ch[c] == ~0u ? QEF_ERR_EMPTY : m.node_err[ch[c]];
        if (e == QEF_ERR_INVALID) return;
        if (e >= 0.0f) child_err = fminf(child_err, e);
    }
    Hermite& out = m.herm[id - m.n_leaves];
    for (uint32_t ti = 0; ti < 3; ++ti) {   // intersections along the coarse edges
        const uint32_t t = 1u << ti, u = next_axis(t), v = next_axis(u);
        for (uint32_t edge = 0; edge < 4; ++edge) {
            const uint32_t start = ((edge & 1u) ? u : 0u) | ((edge & 2u) ? v : 0u), end = start | t, e = ti * 4u + edge;
            float p[3], g[4];
            bool have = child_inter(m, ch[start], e, p, g);
            if (!have) have = child_inter(m, ch[end], e, p, g);
            for (int k = 0; k < 3; ++k) out.ipos[e][k] = have ? p[k] : 0.0f;
            out.ipos[e][3] = have ? 1.0f : 0.0f;
            for (int k = 0; k < 4; ++k) out.igrad[e][k] = have ? g[k] : 0.0f;
        }
    }
    // face QEFs, as written in the reference: `v` is `t.next()` like `u`, and the "u" edges use edge_index_v
    for (uint32_t ti = 0; ti < 3; ++ti) {
        const uint32_t t = 1u << ti, u = next_axis(t), v = u;
        for (uint32_t face = 0; face < 2; ++face) {
            const uint32_t a = face == 1 ? t : 0u, b = a | u, c = a | v, dd = a | u | v, f = ti * 2u + face;
            Qef q;
            qef_zero(q);
            add_child_face(m, ch[a], f, q); add_child_face(m, ch[b], f, q); add_child_face(m, ch[c], f, q); add_child_face(m, ch[dd], f, q);
            const uint32_t ev = axis_index(v) * 4u + face * 2u + 1u;
            add_child_inter(m, ch[a], ev, q); add_child_inter(m, ch[b], ev, q);
            add_child_inter(m, ch[a], ev, q); add_child_inter(m, ch[c], ev, q);
            out.face[f] = q;
        }
    }
    {   // centre QEF
        Qef q;
        qef_zero(q);
        for (uint32_t ti = 0; ti < 3; ++ti) {
            const uint32_t t = 1u << ti, u = next_axis(t), v = u;
            const uint32_t a = 0u, b = a | u, c = a | v, dd = a | u | v;
            add_child_face(m, ch[a], ti * 2u + 1u, q); add_child_face(m, ch[b], ti * 2u + 1u, q);
            add_child_face(m, ch[c], ti * 2u + 1u, q); add_child_face(m, ch[dd], ti * 2u + 1u, q);
            add_child_inter(m, ch[a], axis_index(u) * 4u + 3u, q);
            add_child_inter(m, ch[b], axis_index(u) * 4u + 3u, q);
        }
        for (uint32_t c = 0; c < 8; ++c)
            if (ch[c] != ~0u && ch[c] >= m.n_leaves) qef_add(q, m.herm[ch[c] - m.n_leaves].center);
        out.center = q;
    }
    // LeafHermiteData::solve
    Qef q = out.center;
    for (uint32_t e = 0; e < 12; ++e)
        if (out.ipos[e][3] != 0.0f) {
            const float p[3] = {out.ipos[e][0], out.ipos[e][1], out.ipos[e][2]}, g[4] = {out.igrad[e][0], out.igrad[e][1], out.igrad[e][2], out.igrad[e][3]};
            qef_add_intersection(q, p, g);
        }
    for (int f = 0; f < 6; ++f) qef_add(q, out.face[f]);
    float pos[3];
    const float err = qef_solve(q, pos);
    // CellBounds::contains: closed intervals of the cell's bounds
    const float size = 2.0f / float(1u << d), lo3[3] = {-1.0f + float(x) * size, -1.0f + float(y) * size, -1.0f + float(z) * size};
    bool inside = true;
    for (int k = 0; k < 3; ++k) inside &= pos[k] >= lo3[k] && pos[k] <= lo3[k] + size;
    if (err >= child_err * 2.0f || !inside) return;
    m.node_err[id] = err;
    m.node_vert[id] = make_float3(pos[0], pos[1], pos[2]);
    m.node_state[id] = NODE_LEAF;
}

// Final leaves: leaves whose parent stayed a branch (or the root); listed for fc_mesh_read_cells
__global__ void k_tree_final(TreeScratch m) {
    if (cancel_poll(m.cancel, CS_TREE_FINAL, blockIdx.x)) return;
    const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= m.n_nodes || !(m.node_state[id] & NODE_LEAF)) return;
    const unsigned long long k = m.node_key[id];
    const uint32_t d = key_depth(k);
    if (d > 0) {
        const uint32_t p = tree_find(m, tree_key(d - 1u, key_x(k, 0) >> 1, key_x(k, 1) >> 1, key_x(k, 2) >> 1));
        if (!(m.node_state[p] & NODE_BRANCH)) return;
    }
    m.node_state[id] = NODE_LEAF | NODE_FINAL;
    const uint32_t slot = atomicAdd(&m.counts[5], 1u);
    fc_mesh_cell cell;
    cell.ix = uint16_t(key_x(k, 0)); cell.iy = uint16_t(key_x(k, 1)); cell.iz = uint16_t(key_x(k, 2));
    cell.depth = uint8_t(d);
    cell.mask = uint8_t(m.node_mask[id]);
    const float3 v = id < m.n_leaves ? m.cell_verts[size_t(id) * 4] : m.node_vert[id];
    cell.vertex[0] = v.x; cell.vertex[1] = v.y; cell.vertex[2] = v.z;
    m.out_cells[slot] = cell;
}

// The final leaf covering cell (d, p) of the domain: 0 = found (id, depth), 1 = smaller leaves own this spot (a branch
// at depth d), 2 = an Empty / Full cell
__device__ inline int tree_cover(const TreeScratch& m, uint32_t d, const uint32_t p[3], uint32_t& id, uint32_t& depth) {
    for (uint32_t k = 0; k <= d; ++k) {
        const uint32_t dk = d - k, n = tree_find(m, tree_key(dk, p[0] >> k, p[1] >> k, p[2] >> k));
        if (n == ~0u) continue;
        const uint8_t st = m.node_state[n];
        if (st & NODE_FINAL) { id = n; depth = dk; return 0; }
        if (st & NODE_BRANCH) return k == 0 ? 1 : 2;
    }
    return 2;
}

// dc_edge over the adaptive tree (dc.rs:104-213): one thread per (final leaf, edge).  The four cells around the edge
// segment are looked up at the leaf's depth; the quad is emitted by the deepest of them (the last such in [a, b, c, d],
// as Iterator::max_by_key picks), with the vertex of every shallower leaf being its single one, the intersection
// vertex from the emitting leaf, and no triangle between two corners that are the same cell.
template <int PASS>
__global__ void __launch_bounds__(128) k_tree_faces(TreeScratch m) {
    if (cancel_poll(m.cancel, PASS == 0 ? CS_TREE_FACES0 : CS_TREE_FACES1, blockIdx.x)) return;
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= m.n_nodes * 12u) return;
    const uint32_t id = gid / 12u, e = gid % 12u;
    if (!(m.node_state[id] & NODE_FINAL)) return;
    const uint32_t mask = m.node_mask[id], ti = e / 4u, j = e % 4u, t = 1u << ti, u = next_axis(t), v = next_axis(u);
    const uint32_t start = ((j & 1u) ? u : 0u) | ((j & 2u) ? v : 0u);
    if (((mask >> start) & 1u) == ((mask >> (start | t)) & 1u)) return;
    const unsigned long long key = m.node_key[id];
    const uint32_t d = key_depth(key), side = 1u << d;
    const uint32_t self = j == 3u ? 0u : (j == 2u ? 1u : (j == 0u ? 2u : 3u));   // position in [a, b, c, d]
    int pos[4][3];
    const int du[3] = {(u & 1u) ? 1 : 0, (u & 2u) ? 1 : 0, (u & 4u) ? 1 : 0}, dv[3] = {(v & 1u) ? 1 : 0, (v & 2u) ? 1 : 0, (v & 4u) ? 1 : 0};
    const int offu[4] = {0, 1, 1, 0}, offv[4] = {0, 0, 1, 1};
    bool boundary = false;
    for (int k = 0; k < 4; ++k)
        for (int a = 0; a < 3; ++a) {
            pos[k][a] = int(key_x(key, a)) + (offu[k] - offu[self]) * du[a] + (offv[k] - offv[self]) * dv[a];
            boundary |= pos[k][a] < 0 || pos[k][a] >= int(side);
        }
    uint32_t node[4], depth[4];
    bool in_domain[4], empty = false;
    for (int k = 0; k < 4; ++k) {
        in_domain[k] = pos[k][0] >= 0 && pos[k][0] < int(side) && pos[k][1] >= 0 && pos[k][1] < int(side) && pos[k][2] >= 0 && pos[k][2] < int(side);
        if (!in_domain[k]) { node[k] = ~0u; depth[k] = 0; continue; }
        if (uint32_t(k) == self) { node[k] = id; depth[k] = d; continue; }
        const uint32_t p[3] = {uint32_t(pos[k][0]), uint32_t(pos[k][1]), uint32_t(pos[k][2])};
        const int r = tree_cover(m, d, p, node[k], depth[k]);
        if (r == 1) return;
        if (r == 2) { empty = true; node[k] = ~0u; depth[k] = 0; }
    }
    uint32_t deepest = self;
    for (uint32_t k = 0; k < 4; ++k) if (node[k] != ~0u && depth[k] == d) deepest = k;
    if (deepest != self) return;
    if (boundary) {
        if (PASS == 0) atomicAdd(&m.counts[3], 1u);
        return;
    }
    if (empty) return;
    const uint32_t edge_of[4] = {ti * 4u + 3u, ti * 4u + 2u, ti * 4u + 0u, ti * 4u + 1u};
    uint32_t slot[4];
    for (int k = 0; k < 4; ++k) {
        uint32_t g = 0;
        if (depth[k] == d && node[k] < m.n_leaves) {
            const uint32_t ek = edge_of[k], s = ((ek & 1u) ? u : 0u) | ((ek & 2u) ? v : 0u), mk = m.node_mask[node[k]];
            const uint32_t inside_corner = ((mk >> s) & 1u) ? s : (s | t);
            g = (m.corner_vert[node[k]] >> (2u * inside_corner)) & 3u;
        }
        slot[k] = node[k] * 16u + g;
    }
    const uint32_t islot = id * 16u + 4u + e;
    const uint32_t winding = ((mask >> start) & 1u) ? 1u : 3u;
    if (PASS == 0) {   // MeshBuilder::vertex is called for all five vertices, whichever triangles are dropped
        uint32_t n_tris = 0;
        for (uint32_t k = 0; k < 4u; ++k) {
            m.remap[slot[k]] = 1u;
            n_tris += node[k] != node[(k + winding) & 3u];
        }
        m.remap[islot] = 1u;
        atomicAdd(&m.counts[1], n_tris);
        return;
    }
    uint32_t n_tris = 0;
    for (uint32_t k = 0; k < 4u; ++k) n_tris += node[k] != node[(k + winding) & 3u];
    const uint32_t base = atomicAdd(&m.counts[2], n_tris), iv = m.remap[islot];
    uint32_t o = 0;
    for (uint32_t k = 0; k < 4u; ++k)
        if (node[k] != node[(k + winding) & 3u]) {
            if (base + o < m.cap_tris) m.out_tris[base + o] = make_uint3(m.remap[slot[k]], m.remap[slot[(k + winding) & 3u]], iv);
            ++o;
        }
}

// compaction of the used vertex slots (MeshBuilder::vertex: one output vertex per octree vertex)
__global__ void k_tree_assign(TreeScratch m) {
    if (cancel_poll(m.cancel, CS_TREE_ASSIGN, blockIdx.x)) return;
    const uint64_t s = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (s >= uint64_t(m.n_nodes) * 16u) return;
    if (m.remap[s] != 1u) { m.remap[s] = ~0u; return; }
    const uint32_t id = atomicAdd(&m.counts[0], 1u);
    m.remap[s] = id;
    if (id >= m.cap_verts) return;
    const uint32_t node = uint32_t(s / 16u), k = uint32_t(s % 16u);
    if (k < 4u) {
        m.out_verts[id] = node < m.n_leaves ? m.cell_verts[size_t(node) * 4 + k] : m.node_vert[node];
    } else if (node < m.n_leaves) {
        const OctreeLeaf& L = m.leaves[node];
        m.out_verts[id] = make_float3(L.pos[k - 4u][0], L.pos[k - 4u][1], L.pos[k - 4u][2]);
    } else {
        const Hermite& H = m.herm[node - m.n_leaves];
        m.out_verts[id] = make_float3(H.ipos[k - 4u][0], H.ipos[k - 4u][1], H.ipos[k - 4u][2]);
    }
}

}  // namespace fdev

// fc_octree_sample's device half (octree_capi.cu)
int32_t octree_sample_device(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, OctreeLeaf* dout, uint64_t cap,
                             uint32_t* n_out, fc_octree_stats* stats, const CallCancel& cc);

// fc_mesh_build with FC_FLAG_MESH_COLLAPSE, after the sampler (n > 0 surface leaves in c->mesh_leaves; c->mu held)
static int32_t mesh_build_collapse(fc_ctx* c, uint32_t n, uint32_t depth, const fdev::Mat4* to_model, fc_mesh_info* info,
                                   const CallCancel& cc) {
    using namespace fdev;
    cudaStream_t s = c->stream;
    // nodes: the leaves plus at most min(n, 8^d) ancestors at every depth d < D
    uint64_t cap_nodes = n;
    for (uint32_t d = 0; d < depth; ++d) cap_nodes += std::min<uint64_t>(n, 1ull << (3 * d));
    if (cap_nodes * 16 >= (1ull << 32)) return fail(FC_ERR_INVALID, "mesh too large for cell collapse");
    uint64_t hsize = 1024;
    while (hsize < 2 * cap_nodes) hsize <<= 1;
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t b_keys = hsize * 8, b_vals = hsize * 4, b_nkey = cap_nodes * 8, b_nmask = cap_nodes * 4, b_nstate = cap_nodes,
                 b_nerr = cap_nodes * 4, b_nvert = cap_nodes * sizeof(float3), b_cv = size_t(n) * 4 * sizeof(float3), b_cn = size_t(n) * 4;
    CU(c->mesh_tree.ensure(al(b_keys) + al(b_vals) + al(b_nkey) + al(b_nmask) + al(b_nstate) + al(b_nerr) + al(b_nvert) + al(b_cv) +
                           al(b_cn) + 256));
    TreeScratch m{};
    char* q = c->mesh_tree.as<char>();
    m.hkeys = reinterpret_cast<unsigned long long*>(q); q += al(b_keys);
    m.hvals = reinterpret_cast<uint32_t*>(q); q += al(b_vals);
    m.node_key = reinterpret_cast<unsigned long long*>(q); q += al(b_nkey);
    m.node_mask = reinterpret_cast<uint32_t*>(q); q += al(b_nmask);
    m.node_state = reinterpret_cast<uint8_t*>(q); q += al(b_nstate);
    m.node_err = reinterpret_cast<float*>(q); q += al(b_nerr);
    m.node_vert = reinterpret_cast<float3*>(q); q += al(b_nvert);
    float3* cell_verts = reinterpret_cast<float3*>(q); q += al(b_cv);
    uint32_t* corner_vert = reinterpret_cast<uint32_t*>(q); q += al(b_cn);
    m.counts = reinterpret_cast<uint32_t*>(q);
    m.leaves = c->mesh_leaves.as<OctreeLeaf>();
    m.n_leaves = n;
    m.depth = depth;
    m.hmask = uint32_t(hsize - 1);
    m.cell_verts = cell_verts;
    m.corner_vert = corner_vert;
    m.cancel = cc.ref;
    MeshScratch ms{};   // k_mesh_vertices: the surface leaves' vertices, exactly as the uniform mesh places them
    ms.leaves = m.leaves;
    ms.n_leaves = n;
    ms.cell_verts = cell_verts;
    ms.corner_vert = corner_vert;
    ms.cancel = cc.ref;

    cudaEvent_t e0 = get_event(c, 0), e1 = get_event(c, 1);
    CU(cudaEventRecord(e0, s));
    CU(cudaMemsetAsync(m.hkeys, 0xff, b_keys, s));
    CU(cudaMemsetAsync(m.node_state, 0, b_nstate, s));
    CU(cudaMemsetAsync(m.counts, 0, 64, s));
    const uint32_t first_branch = n;
    CU(cudaMemcpyAsync(m.counts + 4, &first_branch, 4, cudaMemcpyHostToDevice, s));
    const unsigned bl = (n + 127) / 128;
    k_mesh_vertices<<<bl, 128, 0, s>>>(ms);
    k_tree_leaves<<<bl, 128, 0, s>>>(m);
    // ancestors, one depth at a time: range[d] = ids of depth d
    uint32_t range_lo[FC_MAX_OCTREE_DEPTH + 1], range_hi[FC_MAX_OCTREE_DEPTH + 1];
    range_lo[depth] = 0;
    range_hi[depth] = n;
    for (int d = int(depth) - 1; d >= 0; --d) {
        const uint32_t lo = range_lo[d + 1], hi = range_hi[d + 1];
        k_tree_parents<<<(hi - lo + 127) / 128, 128, 0, s>>>(m, lo, hi);
        uint32_t count = 0;
        if (int32_t wrc = wait_read(c, s, cc, &count, m.counts + 4, 4)) return wrc;
        range_lo[d] = hi;
        range_hi[d] = count;
    }
    const uint32_t n_nodes = range_hi[0];
    m.n_nodes = n_nodes;
    const size_t b_herm = std::max<size_t>(n_nodes - n, 1) * sizeof(Hermite), b_remap = size_t(n_nodes) * 16 * 4;
    CU(c->mesh_herm.ensure(al(b_herm) + al(b_remap)));
    m.herm = c->mesh_herm.as<Hermite>();
    m.remap = reinterpret_cast<uint32_t*>(c->mesh_herm.as<char>() + al(b_herm));
    CU(c->mesh_cells.ensure(size_t(n_nodes) * sizeof(fc_mesh_cell)));
    m.out_cells = c->mesh_cells.as<fc_mesh_cell>();
    CU(cudaMemsetAsync(m.remap, 0, b_remap, s));
    k_tree_leaf_err<<<bl, 128, 0, s>>>(m);
    for (int d = int(depth) - 1; d >= 0; --d)
        k_tree_collapse<<<(range_hi[d] - range_lo[d] + 127) / 128, 128, 0, s>>>(m, range_lo[d], range_hi[d]);
    k_tree_final<<<(n_nodes + 127) / 128, 128, 0, s>>>(m);
    k_tree_faces<0><<<(n_nodes * 12u + 127) / 128, 128, 0, s>>>(m);
    CU(cudaGetLastError());
    uint32_t cnt[6];
    if (int32_t wrc = wait_read(c, s, cc, cnt, m.counts, sizeof cnt)) return wrc;
    const uint32_t n_tris = cnt[1];
    const uint64_t v_cap = std::min<uint64_t>(uint64_t(n_nodes) * 16, uint64_t(n_tris) * 5 + 16);
    CU(c->mesh_verts.ensure(std::max<uint64_t>(v_cap, 1) * sizeof(float3)));
    CU(c->mesh_tris.ensure(std::max<uint64_t>(n_tris, 1) * sizeof(uint3)));
    m.out_verts = c->mesh_verts.as<float3>();
    m.cap_verts = uint32_t(v_cap);
    m.out_tris = c->mesh_tris.as<uint3>();
    m.cap_tris = n_tris;
    k_tree_assign<<<unsigned((uint64_t(n_nodes) * 16 + 255) / 256), 256, 0, s>>>(m);
    k_tree_faces<1><<<(n_nodes * 12u + 127) / 128, 128, 0, s>>>(m);
    if (to_model) {
        k_mesh_to_model<<<unsigned((v_cap + 255) / 256), 256, 0, s>>>(reinterpret_cast<char*>(m.out_verts), sizeof(float3), m.counts,
                                                                     m.cap_verts, *to_model);
        k_mesh_to_model<<<(n_nodes + 255) / 256, 256, 0, s>>>(reinterpret_cast<char*>(m.out_cells) + offsetof(fc_mesh_cell, vertex),
                                                             sizeof(fc_mesh_cell), m.counts + 5, n_nodes, *to_model);
    }
    CU(cudaEventRecord(e1, s));
    CU(cudaGetLastError());
    if (int32_t wrc = wait_read(c, s, cc, cnt, m.counts, sizeof cnt)) return wrc;
    if (cnt[0] > v_cap) return fail(FC_ERR_CUDA, "mesh vertex buffer overflow");
    c->mesh_n_verts = cnt[0];
    c->mesh_n_tris = n_tris;
    c->mesh_n_cells = cnt[5];
    info->n_vertices = cnt[0];
    info->n_triangles = n_tris;
    info->open_edges = cnt[3];
    cudaEventElapsedTime(&info->mesh_ms, e0, e1);
    return FC_OK;
}

extern "C" {

int32_t fc_mesh_build(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, fc_mesh_info* info) {
    if (!c || !tape || !cfg || !info) return fail(FC_ERR_INVALID, "null argument");
    memset(info, 0, sizeof *info);
    CallCancel cc;
    auto no_mesh = [&](int32_t rc) {   // a cancelled build leaves no mesh (a failed one keeps the previous)
        std::lock_guard<std::mutex> guard(c->mu);
        c->mesh_n_verts = c->mesh_n_tris = c->mesh_n_cells = 0;
        memset(info, 0, sizeof *info);
        return rc;
    };
    if (int32_t crc = begin_call(c, cc)) return crc == FC_ERR_CANCELLED ? no_mesh(crc) : crc;
    // ---- sampler: leaves stay in HBM ----
    uint64_t cap = c->mesh_leaves.cap / sizeof(OctreeLeaf);
    if (cap < 1024) cap = std::max<uint64_t>(1024, std::min<uint64_t>(1ull << (3 * cfg->depth), 6ull << (2 * cfg->depth)));
    uint32_t n = 0;
    fc_octree_stats ost;
    for (int attempt = 0; attempt < 2; ++attempt) {
        CU(cudaSetDevice(c->device));
        CU(c->mesh_leaves.ensure(cap * sizeof(OctreeLeaf)));
        int32_t rc = octree_sample_device(c, tape, cfg, c->mesh_leaves.as<OctreeLeaf>(), cap, &n, &ost, cc);
        if (rc == FC_OK) break;
        if (rc == FC_ERR_CANCELLED) return no_mesh(rc);
        if (n > cap && attempt == 0) { cap = n; continue; }   // retry once with the exact count
        return rc;
    }
    std::unique_lock<std::mutex> guard(c->mu);
    auto cancelled = [&](int32_t rc) {
        guard.unlock();
        return rc == FC_ERR_CANCELLED ? no_mesh(rc) : rc;
    };
    cudaStream_t s = c->stream;
    MeshScratch m{};
    m.leaves = c->mesh_leaves.as<OctreeLeaf>();
    m.n_leaves = n;
    info->n_leaves = n;
    info->sampler_ms = ost.total_ms;
    c->mesh_n_verts = c->mesh_n_tris = c->mesh_n_cells = 0;
    if (n == 0) return FC_OK;
    // Octree::build maps the vertices through Settings::world_to_model unless that is the identity (octree.rs:58-65)
    fdev::Mat4 view;
    memcpy(view.m, cfg->world_to_model, sizeof view.m);
    bool to_model = false;
    for (int i = 0; i < 16 && cfg->has_transform; ++i) to_model |= view.m[i] != (i % 5 == 0 ? 1.0f : 0.0f);
    if (cfg->flags & FC_FLAG_MESH_COLLAPSE)
        return cancelled(mesh_build_collapse(c, n, cfg->depth, to_model ? &view : nullptr, info, cc));
    uint32_t hsize = 1024;
    while (hsize < 2u * n) hsize <<= 1;
    const size_t b_keys = size_t(hsize) * 8, b_vals = size_t(hsize) * 4, b_cv = size_t(n) * 4 * sizeof(float3), b_cn = size_t(n) * 4,
                 b_remap = size_t(n) * 16 * 4;
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    CU(c->mesh_scratch.ensure(al(b_keys) + al(b_vals) + al(b_cv) + al(b_cn) + al(b_remap) + 256));
    char* q = c->mesh_scratch.as<char>();
    m.hkeys = reinterpret_cast<unsigned long long*>(q); q += al(b_keys);
    m.hvals = reinterpret_cast<uint32_t*>(q); q += al(b_vals);
    m.cell_verts = reinterpret_cast<float3*>(q); q += al(b_cv);
    m.corner_vert = reinterpret_cast<uint32_t*>(q); q += al(b_cn);
    m.remap = reinterpret_cast<uint32_t*>(q); q += al(b_remap);
    m.counts = reinterpret_cast<uint32_t*>(q);
    m.hmask = hsize - 1;
    m.cancel = cc.ref;
    cudaEvent_t e0 = get_event(c, 0), e1 = get_event(c, 1);
    CU(cudaEventRecord(e0, s));
    CU(cudaMemsetAsync(m.hkeys, 0xff, b_keys, s));
    CU(cudaMemsetAsync(m.remap, 0, b_remap, s));
    CU(cudaMemsetAsync(m.counts, 0, 64, s));
    const unsigned bl = (n + 127) / 128;
    k_mesh_hash<<<bl, 128, 0, s>>>(m);
    k_mesh_vertices<<<bl, 128, 0, s>>>(m);
    k_mesh_faces<0><<<(n * 3u + 127) / 128, 128, 0, s>>>(m);
    uint32_t cnt[4];
    if (int32_t wrc = wait_read(c, s, cc, cnt, m.counts, sizeof cnt)) return cancelled(wrc);
    const uint32_t n_tris = cnt[1];
    // every used slot becomes a vertex: count them on the device, sized by the worst case (5 slots per triangle fan)
    const uint64_t v_cap = std::min<uint64_t>(uint64_t(n) * 16, uint64_t(n_tris) * 5 / 4 + 16);
    CU(c->mesh_verts.ensure(std::max<uint64_t>(v_cap, 1) * sizeof(float3)));
    CU(c->mesh_tris.ensure(std::max<uint64_t>(n_tris, 1) * sizeof(uint3)));
    m.out_verts = c->mesh_verts.as<float3>();
    m.cap_verts = uint32_t(v_cap);
    m.out_tris = c->mesh_tris.as<uint3>();
    m.cap_tris = n_tris;
    k_mesh_assign<<<unsigned((uint64_t(n) * 16 + 255) / 256), 256, 0, s>>>(m);
    k_mesh_faces<1><<<(n * 3u + 127) / 128, 128, 0, s>>>(m);
    if (to_model)
        k_mesh_to_model<<<unsigned((v_cap + 255) / 256), 256, 0, s>>>(reinterpret_cast<char*>(m.out_verts), sizeof(float3), m.counts,
                                                                     m.cap_verts, view);
    CU(cudaEventRecord(e1, s));
    CU(cudaGetLastError());
    if (int32_t wrc = wait_read(c, s, cc, cnt, m.counts, sizeof cnt)) return cancelled(wrc);
    if (cnt[0] > v_cap) return fail(FC_ERR_CUDA, "mesh vertex buffer overflow");
    c->mesh_n_verts = cnt[0];
    c->mesh_n_tris = n_tris;
    info->n_vertices = cnt[0];
    info->n_triangles = n_tris;
    info->open_edges = cnt[3];
    cudaEventElapsedTime(&info->mesh_ms, e0, e1);
    return FC_OK;
}

int32_t fc_mesh_read(fc_ctx* c, float* vertices, uint32_t* triangles) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    if (vertices && c->mesh_n_verts)
        CU(cudaMemcpyAsync(vertices, c->mesh_verts.p, size_t(c->mesh_n_verts) * 12, cudaMemcpyDefault, c->stream));
    if (triangles && c->mesh_n_tris)
        CU(cudaMemcpyAsync(triangles, c->mesh_tris.p, size_t(c->mesh_n_tris) * 12, cudaMemcpyDefault, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

int32_t fc_mesh_read_cells(fc_ctx* c, fc_mesh_cell* out, uint64_t cap, uint64_t* n) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    std::lock_guard<std::mutex> guard(c->mu);
    if (n) *n = c->mesh_n_cells;
    if (!out) return FC_OK;
    if (cap < c->mesh_n_cells) return fail(FC_ERR_INVALID, "buffer too small");
    CU(cudaSetDevice(c->device));
    if (c->mesh_n_cells)
        CU(cudaMemcpyAsync(out, c->mesh_cells.p, size_t(c->mesh_n_cells) * sizeof(fc_mesh_cell), cudaMemcpyDefault, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

int32_t fc_mesh_write_stl(fc_ctx* c, uint8_t* buf, size_t cap, size_t* n_bytes) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const size_t need = 84 + size_t(c->mesh_n_tris) * 50;
    if (n_bytes) *n_bytes = need;
    if (!buf) return FC_OK;
    if (cap < need) return fail(FC_ERR_INVALID, "buffer too small");
    const bool dev = is_device_ptr(buf);
    uint8_t* d = buf;
    if (!dev) {
        CU(c->fx_out.ensure(need));
        d = c->fx_out.as<uint8_t>();
    }
    k_mesh_stl<<<unsigned((std::max<uint32_t>(c->mesh_n_tris, 1) + 127) / 128), 128, 0, c->stream>>>(
        c->mesh_verts.as<float3>(), c->mesh_tris.as<uint3>(), c->mesh_n_tris, d);
    CU(cudaGetLastError());
    if (!dev) CU(cudaMemcpyAsync(buf, d, need, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

}  // extern "C"
