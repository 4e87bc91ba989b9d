// Octree sampler leaves of fidget-mesh's Manifold Dual Contouring (sampling half), and the level kernel of the octree
// and quadtree samplers' trees.
#include "level_job.cuh"

// ---------------------------------------------------------------------------
// Octree sampler leaves (OctreeBuilder::leaf, fidget-mesh/src/octree.rs:590-808):
// 8 corner samples -> corner mask; for every edge whose corners differ, 4 rounds
// of 16-ary search from the inside corner to the outside one; the intersection
// is the midpoint of the final bracket.  One warp per leaf; a pass handles four
// edges (two half-warps x two points per lane), `frac` comes from a ballot.
namespace fdev {

// Edge `index` (= 4 t + 2 [start & v] + [start & u], types.rs:208-219) of a cell with corner `mask`
__device__ __forceinline__ bool edge_setup(uint32_t index, uint32_t mask, EdgeState& st) {
    const uint32_t t = index >> 2, su = index & 1u, sv = (index >> 1) & 1u;
    const uint32_t u = (t + 1u) % 3u, v = (t + 2u) % 3u;
    const uint32_t c0 = (su << u) | (sv << v), c1 = c0 | (1u << t);
    const bool in0 = (mask >> c0) & 1u, in1 = (mask >> c1) & 1u;
    if (in0 == in1) return false;
    st.s[u] = st.e[u] = su ? 65535u : 0u;
    st.s[v] = st.e[v] = sv ? 65535u : 0u;
    st.s[t] = in0 ? 0u : 65535u;   // the search runs inside -> outside
    st.e[t] = in0 ? 65535u : 0u;
    return true;
}

// STACK: a mesh frame batch's stacked octree -- the frame of the job's row supplies matrix, has_transform and vars, the
// cell's rows are the frame's, and the leaf records its frame in `pad` (0 for the one frame of a single build)
template <bool STACK>
__global__ void __launch_bounds__(128) k_octree_leaf(const __grid_constant__ OctreeLeafParams p, const MeshFrame* frames,
                                                     uint32_t rows) {
    const int lane = threadIdx.x & 31;
    float2 slots[REG_SLOTS];
    const uint32_t n_jobs = min(p.ctr->n_jobs[p.list], p.cap_jobs);
    unsigned long long n_empty = 0, n_full = 0, n_surf = 0, n_pts = 0;
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_OCTREE_LEAF, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        const TileJob* job = p.jobs + j;
        const uint32_t f = STACK ? job->y / rows : 0u;
        const uint32_t cx = job->x, cy = STACK ? job->y - f * rows : job->y, cz = job->z;
        const TapeRef tr = job->tape;
        const float h = p.cell_h;
        const float lo[3] = {float(cx) * h - 1.0f, float(cy) * h - 1.0f, float(cz) * h - 1.0f};
        const float hi[3] = {float(cx + 1u) * h - 1.0f, float(cy + 1u) * h - 1.0f, float(cz + 1u) * h - 1.0f};
        auto eval2 = [&](float x0, float y0, float z0, float x1, float y1, float z1) -> float2 {
            if (STACK ? frames[f].has_transform : p.has_transform) {
                xform_f32(STACK ? frames[f].mat : p.mat, x0, y0, z0, x0, y0, z0);
                xform_f32(STACK ? frames[f].mat : p.mat, x1, y1, z1, x1, y1, z1);
            }
            const float2 X = make_float2(x0, x1), Y = make_float2(y0, y1), Z = make_float2(z0, z1);
            return run_f32x2(tr.ptr, tr.n_ops, slots, [&](uint32_t i) {
                return pick_input(STACK ? frames[f].vb : p.vb, i, X, Y, Z, [](float v) { return make_float2(v, v); });
            });
        };
        // corners (CellBounds::corner: bit i of the corner index selects the upper bound on axis i)
        const int c = lane & 7;
        const float2 cv = eval2((c & 1) ? hi[0] : lo[0], (c & 2) ? hi[1] : lo[1], (c & 4) ? hi[2] : lo[2],
                                lo[0], lo[1], lo[2]);
        if (lane == 0) n_pts += 8;
        const uint32_t mask = __ballot_sync(FULL, cv.x < 0.0f) & 0xffu;
        if (mask == 0u) { ++n_empty; continue; }
        if (mask == 255u) { ++n_full; continue; }
        ++n_surf;
        uint32_t slot = 0;
        if (lane == 0) slot = atomicAdd(p.n_out, 1u);
        slot = __shfl_sync(FULL, slot, 0);
        if (slot >= p.cap_out) {
            if (lane == 0) atomicOr(&p.ctr->error, 2u);
            continue;
        }
        OctreeLeaf* L = p.out + slot;
        if (lane == 0) p.out_tapes[slot] = tr;
        // active edges, ascending undirected index
        uint32_t active = 0;
        for (uint32_t e = 0; e < 12u; ++e) {
            EdgeState tmp;
            if (edge_setup(e, mask, tmp)) active |= 1u << e;
        }
        const uint32_t ne = __popc(active);
        if (lane == 0) {
            n_pts += 64ull * ne;
            L->ix = uint16_t(cx); L->iy = uint16_t(cy); L->iz = uint16_t(cz);
            L->mask = uint8_t(mask); L->n_edges = uint8_t(ne);
            L->present = uint16_t(active); L->pad = uint16_t(f);
        }
        const int half = lane >> 4;
        for (uint32_t pass = 0; pass * 4u < ne; ++pass) {
            // this lane follows edges k0 (component x) and k1 (component y) of the pass
            const uint32_t k0 = pass * 4u + uint32_t(half), k1 = k0 + 2u;
            auto nth = [&](uint32_t k) {   // index of the k-th set bit of `active`
                uint32_t m = active;
                for (uint32_t q = 0; q < k; ++q) m &= m - 1u;
                return uint32_t(__ffs(m) - 1);
            };
            const bool v0 = k0 < ne, v1 = k1 < ne;
            const uint32_t e0 = v0 ? nth(k0) : nth(0), e1 = v1 ? nth(k1) : nth(0);
            EdgeState s0, s1;
            edge_setup(e0, mask, s0);
            edge_setup(e1, mask, s1);
            edge_search<3>(s0, s1, lo, hi, eval2, L->pos, v0, e0, v1, e1);
        }
    }
    if (p.stats) {
        if (lane == 0) {
            if (n_empty) atomicAdd(&p.stats[0], n_empty);
            if (n_full) atomicAdd(&p.stats[1], n_full);
            if (n_surf) atomicAdd(&p.stats[2], n_surf);
            if (n_pts) atomicAdd(&p.stats[3], n_pts);
        }
    }
}
void launch_octree_leaf(const OctreeLeafParams& p, int blocks, cudaStream_t s, const MeshFrame* frames, uint32_t rows) {
    if (frames) k_octree_leaf<true><<<blocks, 128, 0, s>>>(p, frames, rows);
    else k_octree_leaf<false><<<blocks, 128, 0, s>>>(p, nullptr, 0);
}

// Gradients at the intersections (octree.rs:780-808): one warp per surface leaf, one lane per edge,
// with the tape k_octree_leaf recorded for that leaf.
template <bool STACK>
__global__ void __launch_bounds__(128) k_octree_grads(const __grid_constant__ OctreeLeafParams p, const MeshFrame* frames) {
    grd slots[REG_SLOTS];
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t n = min(*p.n_out, p.cap_out);
    unsigned long long n_pts = 0;
    for (uint32_t i = warp; i < n; i += n_warps) {
        if (cancel_poll(p.cancel, CS_OCTREE_GRADS, i)) break;   // (uniform over the warp)
        OctreeLeaf* L = p.out + i;
        const TapeRef tr = p.out_tapes[i];
        const uint32_t active = L->present;
        const bool mine = lane < 12 && ((active >> lane) & 1u);
        const int e = mine ? lane : (__ffs(active) - 1);
        const MeshFrame* fr = STACK ? frames + L->pad : nullptr;   // (STACK: the leaf's frame)
        const grd r = grad_at(tr, slots, L->pos[e][0], L->pos[e][1], L->pos[e][2],
                              STACK ? fr->has_transform : p.has_transform, STACK ? fr->mat : p.mat, STACK ? fr->vb : p.vb);
        if (mine) {
            L->grad[e][0] = r.y; L->grad[e][1] = r.z; L->grad[e][2] = r.w; L->grad[e][3] = r.x;
            ++n_pts;
        }
    }
    if (p.stats) {
        for (int o = 16; o > 0; o >>= 1) n_pts += __shfl_xor_sync(FULL, n_pts, o);
        if (lane == 0 && n_pts) atomicAdd(&p.stats[4], n_pts);
    }
}
void launch_octree_grads(const OctreeLeafParams& p, int blocks, cudaStream_t s, const MeshFrame* frames, uint32_t) {
    if (frames) k_octree_grads<true><<<blocks, 128, 0, s>>>(p, frames);
    else k_octree_grads<false><<<blocks, 128, 0, s>>>(p, nullptr);
}

// The levels of the samplers' trees: k_interval_level's claim loop around level_job's TREE mode.  DIM 3: a mesh frame
// batch's stacked octree, one root cell per frame; DIM 2: the quadtree of a contour, one root cell, or with STACK one per
// slice of a stack.  `frames` is the frame or slice table (STACK); root cells go 32 to a warp at level 0.  MEASURE:
// fc_measure's levels of the stacked octree, proven-inside cells folded into p.measure (level_job).
template <int DIM, bool STACK, bool MEASURE = false>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) k_tree_level(const __grid_constant__ LevelParams p,
                                                                     const ContourSlice* frames) {
    __shared__ uint32_t live_s[WARPS_PER_BLOCK][8][32];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t gw = blockIdx.x * WARPS_PER_BLOCK + wib;
    uint32_t* cs = p.choice_scratch + size_t(gw) * p.choice_words * 32u + lane;
    itv slots[REG_SLOTS];
    const uint32_t n_roots = STACK ? p.roots_y : 1u;
    const uint32_t n_jobs = p.root_mode ? (n_roots + 31u) / 32u : min(p.ctr->n_jobs[p.level], p.cap_in);
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.level], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_LEVEL0 + p.level, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        level_job<DIM, false, STACK, false, true, MEASURE>(p, j, n_roots, slots, cs, live_s[wib], lane, p.epoch, frames);
    }
}
// fc_volume_build's levels: k_tree_level's loop over the stacked octree, proven cells appended to vol's tile list (a
// kernel of its own, so that the other instantiations keep their machine code)
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) k_tree_level_volume(const __grid_constant__ LevelParams p,
                                                                            const MeshFrame* frames,
                                                                            const __grid_constant__ VolumeLevel vol) {
    __shared__ uint32_t live_s[WARPS_PER_BLOCK][8][32];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t gw = blockIdx.x * WARPS_PER_BLOCK + wib;
    uint32_t* cs = p.choice_scratch + size_t(gw) * p.choice_words * 32u + lane;
    itv slots[REG_SLOTS];
    const uint32_t n_roots = p.roots_y;
    const uint32_t n_jobs = p.root_mode ? (n_roots + 31u) / 32u : min(p.ctr->n_jobs[p.level], p.cap_in);
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.level], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_LEVEL0 + p.level, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        level_job<3, false, true, false, true, false, true>(p, j, n_roots, slots, cs, live_s[wib], lane, p.epoch, frames,
                                                            &vol);
    }
}
void launch_tree_level(const LevelParams& p, int dim, const ContourSlice* frames, int blocks, cudaStream_t s) {
    if (dim == 3) k_tree_level<3, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p, frames);
    else if (frames) k_tree_level<2, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p, frames);
    else k_tree_level<2, false><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p, nullptr);
}
void launch_tree_level_measure(const LevelParams& p, const MeshFrame* frames, int blocks, cudaStream_t s) {
    k_tree_level<3, true, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p, frames);
}
void launch_tree_level_volume(const LevelParams& p, const MeshFrame* frames, const VolumeLevel& v, int blocks, cudaStream_t s) {
    k_tree_level_volume<<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p, frames, v);
}

}  // namespace fdev
