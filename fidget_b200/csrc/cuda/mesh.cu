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
//              the surface leaves' ancestors; the dual is then walked over leaves of different depths (k_tree_faces:
//              dc_cell / dc_face / dc_edge's result, one thread per leaf edge).
//
// Both modes share one scratch layout (MeshScratch), one cell table keyed by (frame, depth, x, y, z), the surface leaves'
// vertices (k_mesh_vertices, which also gives the collapse its leaf errors), the vertex compaction (k_mesh_assign) and
// the host steps after pass 0 of their face kernels (mesh_finish).  Only the face kernels differ: k_mesh_faces looks
// up the three equal-depth neighbours directly, k_tree_faces finds the final leaves covering them.
//
// A frame batch (fc_mesh_build_frames) meshes the frames of a pass together: the sampler's stacked octree gives every
// leaf its frame (OctreeLeaf::pad) and frame-local coordinates, the frame is part of every cell key, so no lookup leaves
// its frame and coordinate 0 stays the domain boundary, and one launch of each kernel covers every frame.  Counts and
// output cursors are per frame (MeshScratch::per_frame): frame k's vertices, triangles and final leaves come out
// contiguous, in frame order, with triangle indices local to the frame.  fc_mesh_build is the batch of one frame.
//
// The 3x3 symmetric eigen-problem is solved with cyclic Jacobi rotations in f32 (the reference calls nalgebra's
// SVD, a third-party algorithm not under /root/reference); positions agree to ~1e-5 of a cell, not bit for bit.
#include <cmath>
#include <cstddef>
#include <vector>

#include "capi_internal.h"
#include "pass_plan.h"

namespace fdev {

__host__ __device__ inline uint32_t next_axis(uint32_t a) { return a == 1u ? 2u : (a == 2u ? 4u : 1u); }   // X -> Y -> Z -> X
__device__ __forceinline__ uint32_t axis_index(uint32_t a) { return a == 1u ? 0u : (a == 2u ? 1u : 2u); }

// The tree of the collapse: node ids [0, n_leaves) are the sampler's surface leaves (depth D); the ids after them are
// their ancestors, built level by level bottom-up, so every depth is one contiguous id range.  A cell that is not a node
// is Empty or Full as a whole (it holds no surface leaf, and neighbouring cells share their corner samples); its sign is
// the sign at its parent's centre, which every child of that parent shares and a node child knows from its corner mask.
constexpr float QEF_ERR_EMPTY = -1.0f, QEF_ERR_INVALID = -2.0f;   // octree.rs:895-899
enum : uint8_t { NODE_LEAF = 1, NODE_BRANCH = 2, NODE_FINAL = 4 };

struct Qef { float ata[6], atb[3], btb, mp[4]; };   // QuadraticErrorSolver; ata = xx xy xz yy yz zz
struct Hermite { float ipos[12][4], igrad[12][4]; Qef face[6], center; };   // LeafHermiteData (qef_err: node_err)

// Per frame of a pass (MeshScratch::per_frame, PF_WORDS words each): its surface leaves, used vertex slots (counted
// before the compaction in passes of several frames), triangles, final leaves and open edges; the first output row of
// its vertices, triangles and final leaves in the pass (set by the host); and the cursors its outputs are written at
enum { PF_LEAVES, PF_VERTS, PF_TRIS, PF_CELLS, PF_OPEN, PF_VBASE, PF_TBASE, PF_CBASE, PF_VCUR, PF_TCUR, PF_CCUR, PF_WORDS };

// The uniform mesh has no nodes beyond the leaves (n_nodes == n_leaves) and leaves the tree's fields (node_*, herm,
// out_cells) null.
struct MeshScratch {
    const OctreeLeaf* leaves;
    uint32_t n_leaves, depth, n_nodes;
    unsigned long long* hkeys;   // open-addressing table: tree_key(frame, depth, x, y, z) -> node id
    uint32_t* hvals;
    uint32_t hmask;
    float3* cell_verts;          // [n_leaves][4]
    uint32_t* corner_vert;       // [n_leaves]: 2 bits per corner = vertex (group) of an inside corner; group count << 16
    unsigned long long* node_key;
    uint32_t* node_mask;         // corner mask (leaves: CellMask; branches: the signs at their eight corners)
    uint8_t* node_state;
    float* node_err;             // LeafHermiteData::qef_err
    float3* node_vert;           // vertex of a collapsed leaf
    Hermite* herm;               // [node - n_leaves]
    uint32_t* remap;             // [n_nodes][16]: slot (4 cell vertices, 12 edge vertices) -> output vertex, or ~0
    uint32_t* counts;            // [4] nodes
    uint32_t* per_frame;         // [n_frames][PF_WORDS]
    const MeshFrame* frames;     // the pass's frames (to_model, mat: the way back to model space)
    uint32_t n_frames;
    float3* out_verts;
    uint32_t cap_verts;
    uint3* out_tris;
    uint32_t cap_tris;
    fc_mesh_cell* out_cells;
    CancelRef cancel;            // polled at block entry of every kernel (item = block index)
};

// A cell key: x, y, z (16 bits each, local to the frame), depth (4 bits: at most FC_MAX_OCTREE_DEPTH), the frame of the
// pass above them (12 bits: MESH_MAX_PASS_FRAMES).  No key is ~0 (the empty slot): depth 15 never occurs.
constexpr uint32_t MESH_MAX_PASS_FRAMES = FC_MESH_MAX_PASS_FRAMES;
static_assert(MESH_MAX_PASS_FRAMES <= 4096, "cell keys hold the frame in 12 bits");
static_assert(FC_MAX_OCTREE_DEPTH < 15, "cell keys hold the depth in 4 bits");
__host__ __device__ __forceinline__ unsigned long long tree_key(uint32_t f, uint32_t d, uint32_t x, uint32_t y, uint32_t z) {
    return (unsigned long long)x | ((unsigned long long)y << 16) | ((unsigned long long)z << 32) |
           ((unsigned long long)d << 48) | ((unsigned long long)f << 52);
}
__device__ __forceinline__ uint32_t key_x(unsigned long long k, int a) { return uint32_t(k >> (16 * a)) & 0xffffu; }
// FRAMES is a compile-time switch, as in the samplers: the kernels of a single fc_mesh_build (FRAMES = false) have frame
// 0 in every key, count into MeshScratch::counts and leave the way back to model space to k_mesh_to_model, exactly as
// before frame batches existed; with FRAMES (fc_mesh_build_frames) they read the frame from the leaf or the key, count
// and place their outputs per frame, and map each vertex through its own frame's matrix where they write it.
template <bool FRAMES> __device__ __forceinline__ uint32_t key_depth(unsigned long long k) {
    return FRAMES ? uint32_t(k >> 48) & 0xfu : uint32_t(k >> 48);
}
template <bool FRAMES> __device__ __forceinline__ uint32_t key_frame(unsigned long long k) {
    return FRAMES ? uint32_t(k >> 52) : 0u;
}
// the frame of node `id` (a surface leaf records it; a tree node's key holds it)
__device__ __forceinline__ uint32_t node_frame(const MeshScratch& m, uint32_t id) {
    return id < m.n_leaves ? m.leaves[id].pad : key_frame<true>(m.node_key[id]);
}
// atomicAdd(p, v) (v <= 4) over the active lanes of a warp: one atomic per distinct address and warp, each lane getting
// the old value its own atomicAdd would have seen in some order.  nvcc aggregates an atomic per warp on its own only
// where it can prove the address warp-uniform, as it can for the single build's counters but not for per-frame ones.
__device__ __forceinline__ uint32_t warp_add(uint32_t* p, uint32_t v) {
    const uint32_t act = __activemask(), lane = threadIdx.x & 31u;
    const uint32_t peers = __match_any_sync(act, reinterpret_cast<unsigned long long>(p)), lt = peers & ((1u << lane) - 1u);
    uint32_t below = 0, total = 0;
    for (uint32_t k = 1; k <= 4u; ++k) {
        const uint32_t b = __ballot_sync(act, v >= k) & peers;
        below += __popc(b & lt);
        total += __popc(b);
    }
    const uint32_t leader = uint32_t(__ffs(peers) - 1);
    uint32_t base = 0;
    if (lane == leader && total) base = atomicAdd(p, total);
    return __shfl_sync(peers, base, leader) + below;
}
// Adds v to a counter or cursor: frame f's word `pf_word` (FRAMES) or the single build's counts[single]
template <bool FRAMES>
__device__ __forceinline__ uint32_t count_add(const MeshScratch& m, uint32_t f, int pf_word, int single, uint32_t v) {
    if (FRAMES) return warp_add(&m.per_frame[PF_WORDS * f + pf_word], v);
    return atomicAdd(&m.counts[single], v);
}
// frame f's first output row of a kind in the pass (FRAMES; 0 for the single build)
template <bool FRAMES> __device__ __forceinline__ uint32_t frame_base(const MeshScratch& m, uint32_t f, int pf_word) {
    return FRAMES ? m.per_frame[PF_WORDS * f + pf_word] : 0u;
}
// Octree::build's last step (octree.rs:58-65) in a frame batch: a vertex goes from the [-1,1]^3 cube the octree was
// built in back to model space through its frame's Matrix4::transform_point, unless that frame has no transform or the
// identity (the single build does this in k_mesh_to_model)
template <bool FRAMES> __device__ __forceinline__ float3 to_model(const MeshScratch& m, uint32_t f, float3 v) {
    if (FRAMES && m.frames[f].to_model) xform_f32(m.frames[f].mat, v.x, v.y, v.z, v.x, v.y, v.z);
    return v;
}
__device__ __forceinline__ uint32_t hash_key(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return uint32_t(k);
}
__device__ __forceinline__ uint32_t hash_find(const MeshScratch& m, unsigned long long key) {
    uint32_t h = hash_key(key) & m.hmask;
    for (;;) {
        const unsigned long long k = m.hkeys[h];
        if (k == key) return m.hvals[h];
        if (k == ~0ull) return ~0u;
        h = (h + 1u) & m.hmask;
    }
}
// returns true when `key` was new; the caller owns hvals[slot] then
__device__ __forceinline__ bool hash_insert(const MeshScratch& m, unsigned long long key, uint32_t& slot) {
    uint32_t h = hash_key(key) & m.hmask;
    for (;;) {
        const unsigned long long old = atomicCAS(&m.hkeys[h], ~0ull, key);
        if (old == ~0ull) { slot = h; return true; }
        if (old == key) return false;
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
// QuadraticErrorSolver::solve (qef.rs:67-118): the vertex, or the mass point when the solve gives NaN
__device__ inline void qef_vertex(const Qef& q, float pos[3]) {
    const float ata[3][3] = {{q.ata[0], q.ata[1], q.ata[2]}, {q.ata[1], q.ata[3], q.ata[4]}, {q.ata[2], q.ata[4], q.ata[5]}};
    const float center[3] = {q.mp[0] / q.mp[3], q.mp[1] / q.mp[3], q.mp[2] / q.mp[3]};
    float b[3];
    for (int r = 0; r < 3; ++r) b[r] = q.atb[r] - (ata[r][0] * center[0] + ata[r][1] * center[1] + ata[r][2] * center[2]);
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
    for (int r = 0; r < 3; ++r) pos[r] = sol[r] + center[r];
    if (!(pos[0] == pos[0] && pos[1] == pos[1] && pos[2] == pos[2])) for (int r = 0; r < 3; ++r) pos[r] = center[r];
}
// The error at the vertex qef_vertex placed: pos^T A^T A pos - 2 pos^T A^T b + b^T b, clamped to >= 1e-6 (qef.rs:111-115)
__device__ inline float qef_error(const Qef& q, const float pos[3]) {
    const float ata[3][3] = {{q.ata[0], q.ata[1], q.ata[2]}, {q.ata[1], q.ata[3], q.ata[4]}, {q.ata[2], q.ata[4], q.ata[5]}};
    float row[3];
    for (int c2 = 0; c2 < 3; ++c2) row[c2] = pos[0] * ata[0][c2] + pos[1] * ata[1][c2] + pos[2] * ata[2][c2];
    const float quad = row[0] * pos[0] + row[1] * pos[1] + row[2] * pos[2];
    const float lin = (2.0f * pos[0]) * q.atb[0] + (2.0f * pos[1]) * q.atb[1] + (2.0f * pos[2]) * q.atb[2];
    const float err = (quad - lin) + q.btb;
    return err > 1e-6f ? err : 1e-6f;   // f32::max: a NaN error becomes 1e-6
}

// Connected groups of a mask's inside corners along cube edges: returns their count and each inside corner's group,
// numbered in the order of their lowest corners (0 for outside corners)
__device__ inline uint32_t corner_groups(uint32_t mask, uint32_t group_of[8]) {
    uint32_t label[8];   // lowest corner of the group
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
    uint32_t n_groups = 0;
    for (uint32_t c = 0; c < 8; ++c) {
        group_of[c] = 0;
        if (!((mask >> c) & 1u)) continue;
        if (label[c] == c) group_of[c] = n_groups++;
        else group_of[c] = group_of[label[c]];   // label[c] < c: already numbered
    }
    return n_groups;
}

// Surface leaves enter the table at depth D and, when collapsing, the tree as its first nodes
template <bool FRAMES>
__global__ void k_mesh_hash(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_MESH_HASH, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const OctreeLeaf& L = m.leaves[i];
    const uint32_t f = FRAMES ? L.pad : 0u;
    if (FRAMES) warp_add(&m.per_frame[PF_WORDS * f + PF_LEAVES], 1u);
    const unsigned long long key = tree_key(f, m.depth, L.ix, L.iy, L.iz);
    uint32_t slot;
    if (hash_insert(m, key, slot)) m.hvals[slot] = i;
    if (!m.node_key) return;
    m.node_key[i] = key;
    m.node_mask[i] = L.mask;
    m.node_state[i] = NODE_LEAF;
}

// One thread per leaf: groups of inside corners, one QEF vertex per group.  LEAF_ERR (collapse): also the leaf's
// LeafHermiteData::qef_err (OctreeBuilder::leaf, octree.rs:810-851): the last group's error wins; a NaN gradient marks
// the group QEF_ERR_INVALID.  A template argument, not a branch: keeping the QEF live through the solve for its error
// takes registers the uniform mesh need not pay for.
template <bool LEAF_ERR>
__global__ void __launch_bounds__(128) k_mesh_vertices(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_MESH_VERTICES, blockIdx.x)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.n_leaves) return;
    const OctreeLeaf& L = m.leaves[i];
    const uint32_t mask = L.mask;
    uint32_t group_of[8], packed = 0;
    const uint32_t n_groups = corner_groups(mask, group_of);
    for (uint32_t c = 0; c < 8; ++c)
        if ((mask >> c) & 1u) packed |= (group_of[c] & 3u) << (2u * c);
    m.corner_vert[i] = packed | (n_groups << 16);
    float err = QEF_ERR_EMPTY;
    for (uint32_t g = 0; g < n_groups && g < 4u; ++g) {
        Qef q;
        qef_zero(q);
        bool forced = false;
        float pos[3];
        for (uint32_t s = 0; s < 8 && !forced; ++s) {
            if (!((mask >> s) & 1u) || group_of[s] != g) continue;
            for (uint32_t t = 1; t < 8; t <<= 1) {
                if ((mask >> (s ^ t)) & 1u) continue;   // not a transition
                const uint32_t u = next_axis(t), v = next_axis(u);
                const uint32_t e = axis_index(t) * 4u + ((s & u) ? 1u : 0u) + ((s & v) ? 2u : 0u);
                const float p[3] = {L.pos[e][0], L.pos[e][1], L.pos[e][2]};
                const float gr[4] = {L.grad[e][0], L.grad[e][1], L.grad[e][2], L.grad[e][3]};
                if (gr[0] != gr[0] || gr[1] != gr[1] || gr[2] != gr[2] || gr[3] != gr[3]) {   // octree.rs:793-801
                    forced = true;
                    for (int k = 0; k < 3; ++k) pos[k] = p[k];
                    break;
                }
                qef_add_intersection(q, p, gr);
            }
        }
        if (forced) {
            err = QEF_ERR_INVALID;
        } else {
            qef_vertex(q, pos);
            if (LEAF_ERR) err = qef_error(q, pos);
        }
        m.cell_verts[size_t(i) * 4 + g] = make_float3(pos[0], pos[1], pos[2]);
    }
    if (LEAF_ERR) m.node_err[i] = err;
}

// The four leaves around the +T edge at corner 0 of leaf `c` (dc.rs:104-119), or false at the domain boundary
struct EdgeCells { uint32_t leaf[4]; };
template <bool FRAMES>
__device__ __forceinline__ bool edge_cells(const MeshScratch& m, uint32_t ci, uint32_t t, EdgeCells& ec) {
    const OctreeLeaf& C = m.leaves[ci];
    const uint32_t u = next_axis(t), v = next_axis(u);
    const uint32_t x = C.ix, y = C.iy, z = C.iz, D = m.depth, f = FRAMES ? C.pad : 0u;
    const uint32_t du[3] = {(u & 1u) ? 1u : 0u, (u & 2u) ? 1u : 0u, (u & 4u) ? 1u : 0u};
    const uint32_t dv[3] = {(v & 1u) ? 1u : 0u, (v & 2u) ? 1u : 0u, (v & 4u) ? 1u : 0u};
    if ((du[0] + dv[0]) > x || (du[1] + dv[1]) > y || (du[2] + dv[2]) > z) return false;
    ec.leaf[2] = ci;                                                                              // c = a + U + V
    ec.leaf[0] = hash_find(m, tree_key(f, D, x - du[0] - dv[0], y - du[1] - dv[1], z - du[2] - dv[2]));  // a
    ec.leaf[1] = hash_find(m, tree_key(f, D, x - dv[0], y - dv[1], z - dv[2]));                          // b = a + U
    ec.leaf[3] = hash_find(m, tree_key(f, D, x - du[0], y - du[1], z - du[2]));                          // d = a + V
    return ec.leaf[0] != ~0u && ec.leaf[1] != ~0u && ec.leaf[3] != ~0u;
}

// pass 0: mark the vertex slots in use and count triangles; pass 1: emit
template <int PASS, bool FRAMES>
__global__ void __launch_bounds__(128) k_mesh_faces(MeshScratch m) {
    if (cancel_poll(m.cancel, PASS == 0 ? CS_MESH_FACES0 : CS_MESH_FACES1, blockIdx.x)) return;
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= m.n_leaves * 3u) return;
    const uint32_t ci = gid / 3u, ti = gid % 3u, t = 1u << ti;
    const OctreeLeaf& C = m.leaves[ci];
    const uint32_t in0 = C.mask & 1u, in1 = (C.mask >> t) & 1u;
    if (in0 == in1) return;
    const uint32_t f = FRAMES ? C.pad : 0u;
    EdgeCells ec;
    if (!edge_cells<FRAMES>(m, ci, t, ec)) {
        if (PASS == 0) count_add<FRAMES>(m, f, PF_OPEN, 3, 1u);
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
            if (PASS == 0) count_add<FRAMES>(m, f, PF_OPEN, 3, 1u);
            return;
        }
        slot[k] = ec.leaf[k] * 16u + ((m.corner_vert[ec.leaf[k]] >> (2u * inside_corner)) & 3u);
    }
    const uint32_t islot = ec.leaf[3] * 16u + 4u + edge_of[3];   // intersection vertex: cell d's copy
    if (PASS == 0) {
        for (int k = 0; k < 4; ++k) m.remap[slot[k]] = 1u;
        m.remap[islot] = 1u;
        count_add<FRAMES>(m, f, PF_TRIS, 1, 4u);
        return;
    }
    // winding (dc.rs:188-196): 3 when the edge's start corner is outside, else 1
    const uint32_t md = m.leaves[ec.leaf[3]].mask;
    const uint32_t start_d = ((edge_of[3] & 1u) ? u : 0u) | ((edge_of[3] & 2u) ? v : 0u);
    const uint32_t winding = ((md >> start_d) & 1u) ? 1u : 3u;
    const uint32_t base = frame_base<FRAMES>(m, f, PF_TBASE) + count_add<FRAMES>(m, f, PF_TCUR, 2, 4u);
    const uint32_t iv = m.remap[islot];
    for (uint32_t j = 0; j < 4u; ++j)
        if (base + j < m.cap_tris) m.out_tris[base + j] = make_uint3(m.remap[slot[j]], m.remap[slot[(j + winding) & 3u]], iv);
}

// Compaction of the used vertex slots (MeshBuilder::vertex: one output vertex per octree vertex); FRAMES: each frame's
// at its cursor, in model space.  PASS 0 (passes of several frames) only counts each frame's used slots, so that the
// host can place the frames' vertices one after another; the slot keeps the frame-local vertex id for the face kernels.
template <int PASS, bool FRAMES>
__global__ void k_mesh_assign(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_MESH_ASSIGN, blockIdx.x)) return;
    const uint64_t s = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (s >= uint64_t(m.n_nodes) * 16u) return;
    const uint32_t node = uint32_t(s / 16u), k = uint32_t(s % 16u);
    if (PASS == 0) {
        if (m.remap[s] == 1u) warp_add(&m.per_frame[PF_WORDS * node_frame(m, node) + PF_VERTS], 1u);
        return;
    }
    if (m.remap[s] != 1u) { m.remap[s] = ~0u; return; }
    const uint32_t f = FRAMES ? node_frame(m, node) : 0u;
    const uint32_t id = count_add<FRAMES>(m, f, PF_VCUR, 0, 1u), at = frame_base<FRAMES>(m, f, PF_VBASE) + id;
    m.remap[s] = id;
    if (at >= m.cap_verts) return;
    float3 v;
    if (k < 4u) {
        v = node < m.n_leaves ? m.cell_verts[size_t(node) * 4 + k] : m.node_vert[node];
    } else if (node < m.n_leaves) {
        const OctreeLeaf& L = m.leaves[node];
        v = make_float3(L.pos[k - 4u][0], L.pos[k - 4u][1], L.pos[k - 4u][2]);
    } else {
        const Hermite& H = m.herm[node - m.n_leaves];
        v = make_float3(H.ipos[k - 4u][0], H.ipos[k - 4u][1], H.ipos[k - 4u][2]);
    }
    m.out_verts[at] = to_model<FRAMES>(m, f, v);
}

// The single build's way back to model space (Octree::build's last step, octree.rs:58-65): every vertex goes from the
// [-1,1]^3 cube the octree was built in through Matrix4::transform_point.  `pos` is the first of *count (at most cap)
// float triples `stride` bytes apart: the vertex buffer, or the vertex field of the final-leaf list.
__global__ void k_mesh_to_model(char* pos, size_t stride, const uint32_t* count, uint32_t cap, Mat4 M) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(*count, cap)) return;
    float* p = reinterpret_cast<float*>(pos + size_t(i) * stride);
    xform_f32(M, p[0], p[1], p[2], p[0], p[1], p[2]);
}

// Mesh::write_stl (output.rs:7-38), one complete file per frame, back to back: frame k's 80-byte header and u32 count,
// then 50 bytes per triangle.  ranges (null: one frame) holds each frame's first vertex and first triangle; the frames'
// triangles are contiguous and their indices local, so triangle i of frame k sits at 84 (k + 1) + 50 i.
__global__ void k_mesh_stl(const float3* verts, const uint3* tris, uint32_t n_tris, const uint2* ranges, uint32_t n_frames,
                           uint8_t* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_frames) {
        const uint32_t t0 = ranges ? ranges[i].y : 0u, t1 = i + 1 < n_frames ? ranges[i + 1].y : n_tris;
        uint8_t* const o = out + 84 * size_t(i) + 50 * size_t(t0);
        const char hdr[] = "This is a binary STL file exported by Fidget";
        for (int k = 0; k < 80; ++k) o[k] = k < int(sizeof(hdr) - 1) ? uint8_t(hdr[k]) : 0;
        for (int k = 0; k < 4; ++k) o[80 + k] = uint8_t((t1 - t0) >> (8 * k));
    }
    if (i >= n_tris) return;
    uint32_t f = 0;   // the last frame whose first triangle is at most i
    for (uint32_t lo = 1, hi = ranges ? n_frames : 1u; lo < hi;) {
        const uint32_t mid = (lo + hi) / 2;
        if (ranges[mid].y <= i) { f = mid; lo = mid + 1; } else hi = mid;
    }
    const uint32_t v0 = ranges ? ranges[f].x : 0u;
    const uint3 t = tris[i];
    const float3 a = verts[v0 + t.x], b = verts[v0 + t.y], c = verts[v0 + t.z];
    const float3 ab = make_float3(b.x - a.x, b.y - a.y, b.z - a.z), ac = make_float3(c.x - a.x, c.y - a.y, c.z - a.z);
    const float rec[12] = {ab.y * ac.z - ab.z * ac.y, ab.z * ac.x - ab.x * ac.z, ab.x * ac.y - ab.y * ac.x,
                           a.x, a.y, a.z, b.x, b.y, b.z, c.x, c.y, c.z};
    uint16_t* dst = reinterpret_cast<uint16_t*>(out + 84 * size_t(f + 1) + size_t(i) * 50);   // even
    for (int k = 0; k < 12; ++k) {
        const uint32_t bits = __float_as_uint(rec[k]);
        dst[2 * k] = uint16_t(bits & 0xffffu);
        dst[2 * k + 1] = uint16_t(bits >> 16);
    }
    dst[24] = 0;
}

// ---- cell collapse and the adaptive dual walk (FC_FLAG_MESH_COLLAPSE) ---------------------------------------------
// The parents of the nodes [lo, hi) (one depth), appended as new nodes
template <bool FRAMES>
__global__ void k_tree_parents(MeshScratch m, uint32_t lo, uint32_t hi) {
    if (cancel_poll(m.cancel, CS_TREE_PARENTS, blockIdx.x)) return;
    const uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    const unsigned long long k = m.node_key[i];
    const unsigned long long pk = tree_key(key_frame<FRAMES>(k), key_depth<FRAMES>(k) - 1u, key_x(k, 0) >> 1, key_x(k, 1) >> 1, key_x(k, 2) >> 1);
    uint32_t slot;
    if (!hash_insert(m, pk, slot)) return;
    const uint32_t id = atomicAdd(&m.counts[4], 1u);
    m.hvals[slot] = id;
    m.node_key[id] = pk;
}

// Hermite data of one child, as LeafHermiteData::merge reads it: a surface leaf's intersections, a collapsed leaf's
// merged record, or the default record of an Empty / Full cell (no intersections, zero QEFs)
__device__ __forceinline__ bool child_inter(const MeshScratch& m, uint32_t ch, uint32_t e, float p[3], float g[4]) {
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
__device__ __forceinline__ void add_child_inter(const MeshScratch& m, uint32_t ch, uint32_t e, Qef& q) {   // From<LeafIntersection>
    float p[3], g[4];
    if (child_inter(m, ch, e, p, g)) qef_add_intersection(q, p, g);
}
__device__ __forceinline__ void add_child_face(const MeshScratch& m, uint32_t ch, uint32_t f, Qef& q) {
    if (ch != ~0u && ch >= m.n_leaves) qef_add(q, m.herm[ch - m.n_leaves].face[f]);
}

// One thread per node of one depth: Octree::check_done / collapsible / try_collapse (octree.rs:252-440) with
// LeafHermiteData::merge / solve (octree.rs:917-1033)
template <bool FRAMES>
__global__ void __launch_bounds__(128) k_tree_collapse(MeshScratch m, uint32_t lo, uint32_t hi) {
    if (cancel_poll(m.cancel, CS_TREE_COLLAPSE, blockIdx.x)) return;
    const uint32_t id = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= hi) return;
    const unsigned long long key = m.node_key[id];
    const uint32_t d = key_depth<FRAMES>(key), x = key_x(key, 0), y = key_x(key, 1), z = key_x(key, 2),
                   fr = key_frame<FRAMES>(key);
    uint32_t ch[8];
    for (uint32_t c = 0; c < 8; ++c)
        ch[c] = hash_find(m, tree_key(fr, d + 1u, 2u * x + (c & 1u), 2u * y + ((c >> 1) & 1u), 2u * z + ((c >> 2) & 1u)));
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
    uint32_t group_of[8];
    if (corner_groups(cmask, group_of) != 1u) return;   // the collapsed cell must be manifold: one vertex group
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
    qef_vertex(q, pos);
    const float err = qef_error(q, pos);
    // CellBounds::contains: closed intervals of the cell's bounds
    const float size = 2.0f / float(1u << d), lo3[3] = {-1.0f + float(x) * size, -1.0f + float(y) * size, -1.0f + float(z) * size};
    bool inside = true;
    for (int k = 0; k < 3; ++k) inside &= pos[k] >= lo3[k] && pos[k] <= lo3[k] + size;
    if (err >= child_err * 2.0f || !inside) return;
    m.node_err[id] = err;
    m.node_vert[id] = make_float3(pos[0], pos[1], pos[2]);
    m.node_state[id] = NODE_LEAF;
}

// Final leaves: leaves whose parent stayed a branch (or the root), marked; with COUNT counted per frame (FRAMES), with
// EMIT listed for fc_mesh_read_cells at their frame's cursor.  A single build and a pass of one frame do both in one
// launch (their cells start at 0); a pass of several counts first, so that the host can place the frames' cells one
// after another.
template <bool FRAMES, bool COUNT, bool EMIT>
__global__ void k_tree_final(MeshScratch m) {
    if (cancel_poll(m.cancel, CS_TREE_FINAL, blockIdx.x)) return;
    const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= m.n_nodes || !(m.node_state[id] & NODE_LEAF)) return;
    const unsigned long long k = m.node_key[id];
    const uint32_t d = key_depth<FRAMES>(k), f = key_frame<FRAMES>(k);
    if (d > 0) {
        const uint32_t p = hash_find(m, tree_key(f, d - 1u, key_x(k, 0) >> 1, key_x(k, 1) >> 1, key_x(k, 2) >> 1));
        if (!(m.node_state[p] & NODE_BRANCH)) return;
    }
    m.node_state[id] = NODE_LEAF | NODE_FINAL;
    if (FRAMES && COUNT) warp_add(&m.per_frame[PF_WORDS * f + PF_CELLS], 1u);
    if (!EMIT) return;
    const uint32_t slot = frame_base<FRAMES>(m, f, PF_CBASE) + count_add<FRAMES>(m, f, PF_CCUR, 5, 1u);
    fc_mesh_cell cell;
    cell.ix = uint16_t(key_x(k, 0)); cell.iy = uint16_t(key_x(k, 1)); cell.iz = uint16_t(key_x(k, 2));
    cell.depth = uint8_t(d);
    cell.mask = uint8_t(m.node_mask[id]);
    const float3 v = to_model<FRAMES>(m, f, id < m.n_leaves ? m.cell_verts[size_t(id) * 4] : m.node_vert[id]);
    cell.vertex[0] = v.x; cell.vertex[1] = v.y; cell.vertex[2] = v.z;
    m.out_cells[slot] = cell;
}

// The final leaf covering cell (d, p) of the domain: 0 = found (id, depth), 1 = smaller leaves own this spot (a branch
// at depth d), 2 = an Empty / Full cell
template <bool FRAMES>
__device__ inline int tree_cover(const MeshScratch& m, uint32_t f, uint32_t d, const uint32_t p[3], uint32_t& id,
                                 uint32_t& depth) {
    for (uint32_t k = 0; k <= d; ++k) {
        const uint32_t dk = d - k, n = hash_find(m, tree_key(f, dk, p[0] >> k, p[1] >> k, p[2] >> k));
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
template <int PASS, bool FRAMES>
__global__ void __launch_bounds__(128) k_tree_faces(MeshScratch m) {
    if (cancel_poll(m.cancel, PASS == 0 ? CS_TREE_FACES0 : CS_TREE_FACES1, blockIdx.x)) return;
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= m.n_nodes * 12u) return;
    const uint32_t id = gid / 12u, e = gid % 12u;
    if (!(m.node_state[id] & NODE_FINAL)) return;
    const uint32_t mask = m.node_mask[id], ti = e / 4u, j = e % 4u, t = 1u << ti, u = next_axis(t), v = next_axis(u);
    const uint32_t start = ((j & 1u) ? u : 0u) | ((j & 2u) ? v : 0u);
    if (((mask >> start) & 1u) == ((mask >> (start | t)) & 1u)) return;
    const unsigned long long key = m.node_key[id];
    const uint32_t d = key_depth<FRAMES>(key), side = 1u << d, f = key_frame<FRAMES>(key);
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
        const int r = tree_cover<FRAMES>(m, f, d, p, node[k], depth[k]);
        if (r == 1) return;
        if (r == 2) { empty = true; node[k] = ~0u; depth[k] = 0; }
    }
    uint32_t deepest = self;
    for (uint32_t k = 0; k < 4; ++k) if (node[k] != ~0u && depth[k] == d) deepest = k;
    if (deepest != self) return;
    if (boundary) {
        if (PASS == 0) count_add<FRAMES>(m, f, PF_OPEN, 3, 1u);
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
        count_add<FRAMES>(m, f, PF_TRIS, 1, n_tris);
        return;
    }
    uint32_t n_tris = 0;
    for (uint32_t k = 0; k < 4u; ++k) n_tris += node[k] != node[(k + winding) & 3u];
    const uint32_t base = frame_base<FRAMES>(m, f, PF_TBASE) + count_add<FRAMES>(m, f, PF_TCUR, 2, n_tris),
                   iv = m.remap[islot];
    uint32_t o = 0;
    for (uint32_t k = 0; k < 4u; ++k)
        if (node[k] != node[(k + winding) & 3u]) {
            if (base + o < m.cap_tris) m.out_tris[base + o] = make_uint3(m.remap[slot[k]], m.remap[slot[(k + winding) & 3u]], iv);
            ++o;
        }
}

}  // namespace fdev

namespace {

// Device bytes per surface leaf of a pass, for sizing passes: the leaf and its tape, the cell table (at most four slots
// per leaf), the cell vertices, corner words and vertex slots, and the outputs (about four vertices and four triangles
// per leaf); collapsing adds per tree node (at most about two per leaf) its key, mask, state, error, vertex, slots and
// table entries, and a Hermite record per branch (about one per two leaves)
constexpr uint64_t MESH_LEAF_BYTES = sizeof(OctreeLeaf) + sizeof(TapeRef) + 4 * 12 + 4 * sizeof(float3) + 4 + 16 * 4 +
                                     4 * sizeof(float3) + 4 * sizeof(uint3);
constexpr uint64_t MESH_NODE_BYTES = 8 + 4 + 1 + 4 + sizeof(float3) + 16 * 4 + 2 * 12;
constexpr uint64_t MESH_COLLAPSE_LEAF_BYTES = MESH_LEAF_BYTES + 2 * MESH_NODE_BYTES + sizeof(fdev::Hermite) / 2;

// The tree nodes of a collapse over n surface leaves of `frames` frames at depth D: the leaves plus at most
// min(n, frames * 8^d) ancestors at every depth d < D
uint64_t tree_cap_nodes(uint64_t n, uint32_t D, uint32_t frames) {
    uint64_t cap = n;
    for (uint32_t d = 0; d < D; ++d) cap += std::min<uint64_t>(n, uint64_t(frames) << (3 * d));
    return cap;
}

}  // namespace

// The uniform mesh up to pass 0 of its face kernel (m: the surface leaves; m.frames set: a pass of a frame batch)
static int32_t mesh_enqueue_uniform(fc_ctx* c, fdev::MeshScratch& m) {
    using namespace fdev;
    cudaStream_t s = c->stream;
    const uint32_t n = m.n_leaves;
    const bool frames = m.frames != nullptr;
    uint32_t hsize = 1024;
    while (hsize < 2u * n) hsize <<= 1;
    const size_t b_keys = size_t(hsize) * 8, b_remap = size_t(n) * 16 * 4, b_pf = frames ? size_t(m.n_frames) * PF_WORDS * 4 : 0;
    CU(carve(c->mesh_scratch, [&](Carve& cv) {
        cv.take(m.hkeys, b_keys);
        cv.take(m.hvals, size_t(hsize) * 4);
        cv.take(m.cell_verts, size_t(n) * 4 * sizeof(float3));
        cv.take(m.corner_vert, size_t(n) * 4);
        cv.take(m.remap, b_remap);
        cv.take(m.counts, 64);
        cv.take(m.per_frame, b_pf);
    }));
    m.hmask = hsize - 1;
    CU(cudaEventRecord(get_event(c, 0), s));
    CU(cudaMemsetAsync(m.hkeys, 0xff, b_keys, s));
    CU(cudaMemsetAsync(m.remap, 0, b_remap, s));
    CU(cudaMemsetAsync(m.counts, 0, 64, s));
    if (frames) CU(cudaMemsetAsync(m.per_frame, 0, b_pf, s));
    const unsigned bl = (n + 127) / 128;
    if (frames) k_mesh_hash<true><<<bl, 128, 0, s>>>(m);
    else k_mesh_hash<false><<<bl, 128, 0, s>>>(m);
    k_mesh_vertices<false><<<bl, 128, 0, s>>>(m);
    if (frames) k_mesh_faces<0, true><<<(n * 3u + 127) / 128, 128, 0, s>>>(m);
    else k_mesh_faces<0, false><<<(n * 3u + 127) / 128, 128, 0, s>>>(m);
    return FC_OK;
}

// The collapsing mesh up to pass 0 of its face kernel: the tree of the surface leaves' ancestors (one tree for all frames
// of the pass: the keys keep them apart), the collapse one depth at a time bottom-up, and the final leaves (a single
// build's or a lone frame's listed at once, the latter after the batch's c0 earlier ones)
static int32_t mesh_enqueue_collapse(fc_ctx* c, fdev::MeshScratch& m, uint64_t c0, const CallCancel& cc) {
    using namespace fdev;
    cudaStream_t s = c->stream;
    const uint32_t n = m.n_leaves, depth = m.depth;
    const bool frames = m.frames != nullptr;
    const uint64_t cap_nodes = tree_cap_nodes(n, depth, m.n_frames);
    if (cap_nodes * 16 >= (1ull << 32)) return fail(FC_ERR_INVALID, "mesh too large for cell collapse");
    uint64_t hsize = 1024;
    while (hsize < 2 * cap_nodes) hsize <<= 1;
    const size_t b_keys = hsize * 8, b_nstate = cap_nodes, b_pf = frames ? size_t(m.n_frames) * PF_WORDS * 4 : 0;
    CU(carve(c->mesh_tree, [&](Carve& cv) {
        cv.take(m.hkeys, b_keys);
        cv.take(m.hvals, hsize * 4);
        cv.take(m.node_key, cap_nodes * 8);
        cv.take(m.node_mask, cap_nodes * 4);
        cv.take(m.node_state, b_nstate);
        cv.take(m.node_err, cap_nodes * 4);
        cv.take(m.node_vert, cap_nodes * sizeof(float3));
        cv.take(m.cell_verts, size_t(n) * 4 * sizeof(float3));
        cv.take(m.corner_vert, size_t(n) * 4);
        cv.take(m.counts, 64);
        cv.take(m.per_frame, b_pf);
    }));
    m.hmask = uint32_t(hsize - 1);
    CU(cudaEventRecord(get_event(c, 0), s));
    CU(cudaMemsetAsync(m.hkeys, 0xff, b_keys, s));
    CU(cudaMemsetAsync(m.node_state, 0, b_nstate, s));
    CU(cudaMemsetAsync(m.counts, 0, 64, s));
    if (frames) CU(cudaMemsetAsync(m.per_frame, 0, b_pf, s));
    const uint32_t first_branch = n;
    CU(cudaMemcpyAsync(m.counts + 4, &first_branch, 4, cudaMemcpyHostToDevice, s));
    const unsigned bl = (n + 127) / 128;
    if (frames) k_mesh_hash<true><<<bl, 128, 0, s>>>(m);
    else k_mesh_hash<false><<<bl, 128, 0, s>>>(m);
    k_mesh_vertices<true><<<bl, 128, 0, s>>>(m);
    // ancestors, one depth at a time: range[d] = ids of depth d
    uint32_t range_lo[FC_MAX_OCTREE_DEPTH + 1], range_hi[FC_MAX_OCTREE_DEPTH + 1];
    range_lo[depth] = 0;
    range_hi[depth] = n;
    for (int d = int(depth) - 1; d >= 0; --d) {
        const uint32_t lo = range_lo[d + 1], hi = range_hi[d + 1];
        if (frames) k_tree_parents<true><<<(hi - lo + 127) / 128, 128, 0, s>>>(m, lo, hi);
        else k_tree_parents<false><<<(hi - lo + 127) / 128, 128, 0, s>>>(m, lo, hi);
        uint32_t count = 0;
        if (int32_t wrc = wait_read(c, s, cc, &count, m.counts + 4, 4)) return wrc;
        range_lo[d] = hi;
        range_hi[d] = count;
    }
    const uint32_t n_nodes = range_hi[0];
    m.n_nodes = n_nodes;
    const size_t b_remap = size_t(n_nodes) * 16 * 4;
    CU(carve(c->mesh_herm, [&](Carve& cv) {
        cv.take(m.herm, std::max<size_t>(n_nodes - n, 1) * sizeof(Hermite));
        cv.take(m.remap, b_remap);
    }));
    if (frames) {
        if (int32_t rc = grow_keep(c, c->mesh_cells, size_t(c0 + n_nodes) * sizeof(fc_mesh_cell), size_t(c0) * sizeof(fc_mesh_cell)))
            return rc;
    } else {
        CU(c->mesh_cells.ensure(size_t(n_nodes) * sizeof(fc_mesh_cell)));
    }
    m.out_cells = c->mesh_cells.as<fc_mesh_cell>() + c0;
    CU(cudaMemsetAsync(m.remap, 0, b_remap, s));
    const unsigned bn = (n_nodes + 127) / 128, bf = (n_nodes * 12u + 127) / 128;
    for (int d = int(depth) - 1; d >= 0; --d) {
        const unsigned bd = (range_hi[d] - range_lo[d] + 127) / 128;
        if (frames) k_tree_collapse<true><<<bd, 128, 0, s>>>(m, range_lo[d], range_hi[d]);
        else k_tree_collapse<false><<<bd, 128, 0, s>>>(m, range_lo[d], range_hi[d]);
    }
    if (!frames) {
        k_tree_final<false, true, true><<<bn, 128, 0, s>>>(m);
        k_tree_faces<0, false><<<bf, 128, 0, s>>>(m);
        return FC_OK;
    }
    if (m.n_frames > 1) k_tree_final<true, true, false><<<bn, 128, 0, s>>>(m);   // listed in mesh_finish_frames
    else k_tree_final<true, true, true><<<bn, 128, 0, s>>>(m);
    k_tree_faces<0, true><<<bf, 128, 0, s>>>(m);
    return FC_OK;
}

// The single build in both modes after pass 0 of its face kernel: size the outputs by the triangle count, compact the
// used vertex slots, emit the triangles, map to model space and publish the counts
static int32_t mesh_finish(fc_ctx* c, fdev::MeshScratch& m, bool collapse, const fdev::Mat4* to_model, fc_mesh_info* info,
                           const CallCancel& cc) {
    using namespace fdev;
    cudaStream_t s = c->stream;
    CU(cudaGetLastError());
    uint32_t cnt[6];
    if (int32_t wrc = wait_read(c, s, cc, cnt, m.counts, sizeof cnt)) return wrc;
    const uint32_t n_tris = cnt[1];
    // every used slot becomes a vertex: count them on the device, sized by the worst case (5 slots per triangle fan,
    // which keeps all 4 triangles in the uniform mesh and may keep only one in the adaptive walk)
    const uint64_t fan_slots = collapse ? uint64_t(n_tris) * 5 : uint64_t(n_tris) * 5 / 4;
    const uint64_t v_cap = std::min<uint64_t>(uint64_t(m.n_nodes) * 16, fan_slots + 16);
    CU(c->mesh_verts.ensure(std::max<uint64_t>(v_cap, 1) * sizeof(float3)));
    CU(c->mesh_tris.ensure(std::max<uint64_t>(n_tris, 1) * sizeof(uint3)));
    m.out_verts = c->mesh_verts.as<float3>();
    m.cap_verts = uint32_t(v_cap);
    m.out_tris = c->mesh_tris.as<uint3>();
    m.cap_tris = n_tris;
    k_mesh_assign<1, false><<<unsigned((uint64_t(m.n_nodes) * 16 + 255) / 256), 256, 0, s>>>(m);
    if (collapse) k_tree_faces<1, false><<<(m.n_nodes * 12u + 127) / 128, 128, 0, s>>>(m);
    else k_mesh_faces<1, false><<<(m.n_nodes * 3u + 127) / 128, 128, 0, s>>>(m);
    if (to_model) {
        k_mesh_to_model<<<unsigned((v_cap + 255) / 256), 256, 0, s>>>(reinterpret_cast<char*>(m.out_verts), sizeof(float3), m.counts,
                                                                     m.cap_verts, *to_model);
        if (collapse)
            k_mesh_to_model<<<(m.n_nodes + 255) / 256, 256, 0, s>>>(reinterpret_cast<char*>(m.out_cells) + offsetof(fc_mesh_cell, vertex),
                                                                   sizeof(fc_mesh_cell), m.counts + 5, m.n_nodes, *to_model);
    }
    cudaEvent_t e1 = get_event(c, 1);
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
    cudaEventElapsedTime(&info->mesh_ms, get_event(c, 0), e1);
    return FC_OK;
}

// A pass of a frame batch in both modes after pass 0 of its face kernel: place each frame's outputs (after the batch's
// v0 vertices and t0 triangles), compact the used vertex slots, emit the triangles (and, in passes of several frames,
// the final leaves) and read the per-frame words into pf (PF_WORDS per frame of the pass).  A pass of one frame sizes
// its vertices by the triangle count; a pass of several counts every frame's used slots first.
static int32_t mesh_finish_frames(fc_ctx* c, fdev::MeshScratch& m, bool collapse, uint64_t v0, uint64_t t0,
                           std::vector<uint32_t>& pf, float* ms, const CallCancel& cc) {
    using namespace fdev;
    cudaStream_t s = c->stream;
    const bool several = m.n_frames > 1;
    const unsigned b_slots = unsigned((uint64_t(m.n_nodes) * 16 + 255) / 256);
    if (several) k_mesh_assign<0, true><<<b_slots, 256, 0, s>>>(m);
    CU(cudaGetLastError());
    const size_t b_pf = size_t(m.n_frames) * PF_WORDS * 4;
    pf.assign(size_t(m.n_frames) * PF_WORDS, 0u);
    if (int32_t wrc = wait_read(c, s, cc, pf.data(), m.per_frame, b_pf)) return wrc;
    uint64_t nv = 0, nt = 0, nc = 0;
    for (uint32_t f = 0; f < m.n_frames; ++f) {
        uint32_t* w = pf.data() + size_t(f) * PF_WORDS;
        w[PF_VBASE] = uint32_t(nv);
        w[PF_TBASE] = uint32_t(nt);
        w[PF_CBASE] = uint32_t(nc);
        nv += w[PF_VERTS];
        nt += w[PF_TRIS];
        nc += w[PF_CELLS];
    }
    if (t0 + nt > 0xffffffffull || v0 + nv > 0xffffffffull)
        return fail(FC_ERR_UNSUPPORTED, "mesh has more triangles or vertices than 32-bit indices can address");
    if (several) CU(cudaMemcpyAsync(m.per_frame, pf.data(), b_pf, cudaMemcpyHostToDevice, s));
    const uint32_t n_tris = uint32_t(nt);
    // one frame: every used slot becomes a vertex, sized by the worst case (5 slots per triangle fan, which keeps all 4
    // triangles in the uniform mesh and may keep only one in the adaptive walk)
    const uint64_t fan_slots = collapse ? uint64_t(n_tris) * 5 : uint64_t(n_tris) * 5 / 4;
    const uint64_t v_cap = several ? nv : std::min<uint64_t>(uint64_t(m.n_nodes) * 16, fan_slots + 16);
    if (int32_t rc = grow_keep(c, c->mesh_verts, size_t(v0 + std::max<uint64_t>(v_cap, 1)) * sizeof(float3),
                               size_t(v0) * sizeof(float3)))
        return rc;
    if (int32_t rc = grow_keep(c, c->mesh_tris, size_t(t0 + std::max<uint64_t>(n_tris, 1)) * sizeof(uint3),
                               size_t(t0) * sizeof(uint3)))
        return rc;
    m.out_verts = c->mesh_verts.as<float3>() + v0;
    m.cap_verts = uint32_t(std::min<uint64_t>(v_cap, 0xffffffffull));
    m.out_tris = c->mesh_tris.as<uint3>() + t0;
    m.cap_tris = n_tris;
    k_mesh_assign<1, true><<<b_slots, 256, 0, s>>>(m);
    if (collapse) {
        if (several) k_tree_final<true, false, true><<<(m.n_nodes + 127) / 128, 128, 0, s>>>(m);
        k_tree_faces<1, true><<<(m.n_nodes * 12u + 127) / 128, 128, 0, s>>>(m);
    } else {
        k_mesh_faces<1, true><<<(m.n_nodes * 3u + 127) / 128, 128, 0, s>>>(m);
    }
    cudaEvent_t e1 = get_event(c, 1);
    CU(cudaEventRecord(e1, s));
    CU(cudaGetLastError());
    if (int32_t wrc = wait_read(c, s, cc, pf.data(), m.per_frame, b_pf)) return wrc;
    uint64_t used = 0;
    for (uint32_t f = 0; f < m.n_frames; ++f) used += pf[size_t(f) * PF_WORDS + PF_VCUR];
    if (used > v_cap) return fail(FC_ERR_CUDA, "mesh vertex buffer overflow");
    cudaEventElapsedTime(ms, get_event(c, 0), e1);
    return FC_OK;
}

// The sampler of one pass into c->mesh_leaves (cap leaves): *n_out surface leaves (beyond cap too), ctr its counters,
// *ms its device time (when timing)
static int32_t mesh_sample(fc_ctx* c, const fc_tape* tape, uint32_t D, const MeshFrame* fr, uint32_t n,
                           const MeshFrame* d_fr, uint64_t cap, uint32_t* n_out, Counters& ctr, float* ms,
                           const CallCancel& cc) {
    cudaStream_t s = c->stream;
    CU(c->mesh_leaves.ensure(cap * sizeof(OctreeLeaf)));
    if (int32_t rc = octree_enqueue(c, tape, D, fr, n, n > 1 ? d_fr : nullptr, c->mesh_leaves.as<OctreeLeaf>(), cap, false,
                                    ms ? get_event(c, 2) : nullptr, cc, nullptr))
        return rc;
    if (ms) CU(cudaEventRecord(get_event(c, 3), s));
    const uint32_t* d_n_out = reinterpret_cast<const uint32_t*>(c->counters.as<char>() + sizeof(Counters));
    if (int32_t wrc = wait_read(c, s, cc, n_out, d_n_out, 4)) return wrc;
    CU(cudaMemcpy(&ctr, c->counters.p, sizeof ctr, cudaMemcpyDeviceToHost));
    if (ms) cudaEventElapsedTime(ms, get_event(c, 2), get_event(c, 3));
    return FC_OK;
}

static void mesh_clear(fc_ctx* c) {
    c->mesh_n_verts = c->mesh_n_tris = c->mesh_n_cells = 0;
    c->mesh_n_frames = 1;
}

// The passes of a checked batch: every frame's mesh appended to the outputs in frame order, the per-frame counts into
// per (when given) and their sums into info.  The caller holds the context's lock.  The outputs of an earlier build are
// dropped once the first pass has sampled.
static int32_t mesh_passes(fc_ctx* c, const fc_tape* tape, uint32_t D, uint32_t flags, const std::vector<MeshFrame>& fr,
                           fc_mesh_info* info, fc_mesh_frame_info* per, const CallCancel& cc) {
    using namespace fdev;
    const uint32_t N = uint32_t(fr.size());
    const bool collapse = (flags & FC_FLAG_MESH_COLLAPSE) != 0, timing = (flags & FC_FLAG_TIMING) != 0;
    // Passes as the 3D batches' (pass_plan.h), the measured quantity being surface leaves (with their mesh scratch)
    // within FC_FRAMES_PASS_BYTES.  A pass's frame index is 12 bits in the cell keys, and its cell rows must fit 32 bits.
    const double leaf_bytes = double(collapse ? MESH_COLLAPSE_LEAF_BYTES : MESH_LEAF_BYTES);
    PassPlan plan = tree_passes(c, N, uint32_t(std::min<uint64_t>({N, MESH_MAX_PASS_FRAMES, 0xffffffffull >> D})), D, 3,
                                int(D) + 1, leaf_bytes);
    const uint64_t first_guess = std::min<uint64_t>(1ull << (3 * D), 6ull << (2 * D));   // leaves of one frame
    uint64_t v0 = 0, t0 = 0, c0 = 0;   // the batch's output so far
    std::vector<uint2> ranges(N);
    std::vector<uint32_t> pf;
    bool cleared = false;
    while (plan.more()) {
        const PassPlan::Range r = plan.take();
        const MeshFrame* ps = fr.data() + r.f0;
        CU(c->mesh_frames.ensure(size_t(r.n) * sizeof(MeshFrame)));
        MeshFrame* d_fr = c->mesh_frames.as<MeshFrame>();
        CU(cudaMemcpyAsync(d_fr, ps, size_t(r.n) * sizeof(MeshFrame), cudaMemcpyHostToDevice, c->stream));
        // leaves: the buffer of the last build, else fc_mesh_build's first guess per frame (within the pass budget), or
        // the most per frame seen so far; once more with the exact count
        uint64_t cap = c->mesh_leaves.cap / sizeof(OctreeLeaf);
        if (cap < 1024)
            cap = std::max<uint64_t>(1024, std::min<uint64_t>(r.n * first_guess,
                                                              std::max<uint64_t>(first_guess, FC_FRAMES_PASS_BYTES / sizeof(OctreeLeaf))));
        if (plan.use_extra > 0) cap = std::max<uint64_t>(cap, uint64_t(std::ceil(plan.use_extra * 1.25 * r.n)));
        cap = std::min<uint64_t>(cap, 0xfffffff0ull);
        uint32_t n = 0;
        Counters ctr;
        float sampler_ms = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            if (int32_t rc = mesh_sample(c, tape, D, ps, r.n, d_fr, cap, &n, ctr, timing ? &sampler_ms : nullptr, cc))
                return rc;
            // more leaves than the buffer holds: once more with the exact count -- unless a pass of several frames would
            // then break the pass budget; the leaf kernel's overflow bit has it run again in halves (plan.observe)
            if (n <= cap || (r.n > 1 && double(n) * leaf_bytes > double(FC_FRAMES_PASS_BYTES))) break;
            cap = n;
        }
        if (n > cap && (r.n == 1 || !ctr.error))
            return fail(FC_ERR_INVALID, "leaf buffer too small: " + std::to_string(n) + " surface leaves");
        bool split = false;
        if (!plan.observe(ctr, n, r, split)) return device_error(ctr.error);
        if (split) continue;
        if (collapse && r.n > 1 && tree_cap_nodes(n, D, r.n) * 16 >= (1ull << 32)) {   // the tree's slots: in halves
            const uint32_t h = r.n / 2;
            plan.redo.push_back(PassPlan::Range{r.f0 + h, r.n - h});
            plan.redo.push_back(PassPlan::Range{r.f0, h});
            continue;
        }
        info->sampler_ms += sampler_ms;
        if (!cleared) {
            mesh_clear(c);
            cleared = true;
        }
        for (uint32_t k = 0; k < r.n; ++k) ranges[r.f0 + k] = make_uint2(uint32_t(v0), uint32_t(t0));
        if (n == 0) continue;
        MeshScratch m{};
        m.leaves = c->mesh_leaves.as<OctreeLeaf>();
        m.n_leaves = m.n_nodes = n;
        m.depth = D;
        m.cancel = cc.ref;
        m.frames = d_fr;
        m.n_frames = r.n;
        int32_t rc = collapse ? mesh_enqueue_collapse(c, m, c0, cc) : mesh_enqueue_uniform(c, m);
        float mesh_ms = 0;
        if (rc == FC_OK) rc = mesh_finish_frames(c, m, collapse, v0, t0, pf, &mesh_ms, cc);
        if (rc) return rc;
        info->mesh_ms += mesh_ms;
        uint64_t nv = 0, nt = 0, nc = 0;
        for (uint32_t k = 0; k < r.n; ++k) {
            const uint32_t* w = pf.data() + size_t(k) * PF_WORDS;
            fc_mesh_frame_info fi{};
            fi.n_leaves = w[PF_LEAVES];
            fi.n_vertices = w[PF_VCUR];
            fi.n_triangles = w[PF_TRIS];
            fi.open_edges = w[PF_OPEN];
            fi.n_cells = collapse ? w[PF_CCUR] : 0;
            ranges[r.f0 + k] = make_uint2(uint32_t(v0 + w[PF_VBASE]), uint32_t(t0 + w[PF_TBASE]));
            if (per) per[r.f0 + k] = fi;
            info->n_leaves += fi.n_leaves;
            info->n_vertices += fi.n_vertices;
            info->n_triangles += fi.n_triangles;
            info->open_edges += fi.open_edges;
            nv += fi.n_vertices;
            nt += fi.n_triangles;
            nc += fi.n_cells;
        }
        v0 += nv;
        t0 += nt;
        c0 += nc;
    }
    if (N > 1) {
        CU(c->mesh_ranges.ensure(size_t(N) * sizeof(uint2)));
        CU(cudaMemcpy(c->mesh_ranges.p, ranges.data(), size_t(N) * sizeof(uint2), cudaMemcpyHostToDevice));
    }
    c->mesh_n_verts = uint32_t(v0);
    c->mesh_n_tris = uint32_t(t0);
    c->mesh_n_cells = uint32_t(c0);
    c->mesh_n_frames = N;
    return FC_OK;
}

// fc_mesh_build_frames: the checks of every frame, then the passes.  A failed, cancelled or empty call leaves no mesh.
static int32_t mesh_build_frames(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, const fc_mesh_frame* frames,
                                 uint32_t n_frames, fc_mesh_info* info, fc_mesh_frame_info* per) {
    memset(info, 0, sizeof *info);
    if (per && n_frames) memset(per, 0, size_t(n_frames) * sizeof *per);
    auto no_mesh = [&](int32_t rc) {
        std::lock_guard<std::mutex> guard(c->mu);
        mesh_clear(c);
        memset(info, 0, sizeof *info);
        if (per && n_frames) memset(per, 0, size_t(n_frames) * sizeof *per);
        return rc;
    };
    if (int32_t rc = check_tree_call(tape, 3, cfg->depth, frames, n_frames, "the octree sampler")) return no_mesh(rc);
    std::vector<MeshFrame> fr(n_frames);
    for (uint32_t k = 0; k < n_frames; ++k) {
        const fc_mesh_frame& in = frames[k];
        if (int32_t vrc = bind_frame(tape, in.has_transform, in.world_to_model, 0.0f, in.var_values, in.n_var_values, fr[k]))
            return no_mesh(vrc);
    }
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return no_mesh(crc);
    std::unique_lock<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    if (!n_frames) mesh_clear(c);
    const int32_t rc = n_frames ? mesh_passes(c, tape, cfg->depth, cfg->flags, fr, info, per, cc) : FC_OK;
    guard.unlock();
    return rc == FC_OK ? rc : no_mesh(rc);
}

// fc_octree_sample's device half (octree_capi.cu)
int32_t octree_sample_device(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, OctreeLeaf* dout, uint64_t cap,
                             uint32_t* n_out, fc_octree_stats* stats, const CallCancel& cc);

extern "C" {

// The single build keeps a host path of its own, with the FRAMES = false kernels: run through the batch's driver as a
// batch of one frame, its back half (mesh_ms) took 10-40 % longer on an H100 (per-frame counters, cursors and
// model-space lookups; scripts/bench_mesh.py against the parent build, alternating).
int32_t fc_mesh_build(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, fc_mesh_info* info) {
    if (!c || !tape || !cfg || !info) return fail(FC_ERR_INVALID, "null argument");
    memset(info, 0, sizeof *info);
    CallCancel cc;
    auto no_mesh = [&](int32_t rc) {   // a cancelled build leaves no mesh (a failed one keeps the previous)
        std::lock_guard<std::mutex> guard(c->mu);
        mesh_clear(c);
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
    MeshFrame view;   // the frame octree_sample_device bound, for its to_model
    if (int32_t vrc = bind_frame(tape, cfg->has_transform, cfg->world_to_model, 0.0f, cfg->var_values, cfg->n_var_values,
                                 view))
        return vrc;
    std::unique_lock<std::mutex> guard(c->mu);
    info->n_leaves = n;
    info->sampler_ms = ost.total_ms;
    mesh_clear(c);
    if (n == 0) return FC_OK;
    fdev::MeshScratch m{};
    m.leaves = c->mesh_leaves.as<OctreeLeaf>();
    m.n_leaves = m.n_nodes = n;
    m.depth = cfg->depth;
    m.cancel = cc.ref;
    m.n_frames = 1;
    const bool collapse = cfg->flags & FC_FLAG_MESH_COLLAPSE;
    int32_t rc = collapse ? mesh_enqueue_collapse(c, m, 0, cc) : mesh_enqueue_uniform(c, m);
    if (rc == FC_OK) rc = mesh_finish(c, m, collapse, view.to_model ? &view.mat : nullptr, info, cc);
    guard.unlock();
    return rc == FC_ERR_CANCELLED ? no_mesh(rc) : rc;
}

int32_t fc_mesh_build_frames(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, const fc_mesh_frame* frames,
                             uint32_t n_frames, fc_mesh_info* info, fc_mesh_frame_info* per_frame) {
    if (!c || !tape || !cfg || !info) return fail(FC_ERR_INVALID, "null argument");
    return mesh_build_frames(c, tape, cfg, frames, n_frames, info, per_frame);
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
    const size_t need = 84 * size_t(c->mesh_n_frames) + size_t(c->mesh_n_tris) * 50;
    if (n_bytes) *n_bytes = need;
    if (!buf) return FC_OK;
    if (cap < need) return fail(FC_ERR_INVALID, "buffer too small");
    const bool dev = is_device_ptr(buf);
    uint8_t* d = buf;
    if (!dev) {
        CU(c->fx_out.ensure(need));
        d = c->fx_out.as<uint8_t>();
    }
    const uint32_t nf = c->mesh_n_frames;
    k_mesh_stl<<<unsigned((std::max<uint32_t>(c->mesh_n_tris, nf) + 127) / 128), 128, 0, c->stream>>>(
        c->mesh_verts.as<float3>(), c->mesh_tris.as<uint3>(), c->mesh_n_tris, nf > 1 ? c->mesh_ranges.as<uint2>() : nullptr,
        nf, d);
    CU(cudaGetLastError());
    if (!dev) CU(cudaMemcpyAsync(buf, d, need, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

}  // extern "C"
