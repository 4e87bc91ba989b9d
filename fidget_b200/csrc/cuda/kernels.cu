// sm_90a kernels for the tape-evaluation hot path.
//
//  k_interval_level  -- K1: one warp per parent tile, one lane per child tile;
//                       walks the (warp-uniform) parent tape, classifies each
//                       child (fill inside / fill outside / ambiguous), then
//                       runs the reverse liveness pass that compacts a child
//                       tape into the arena (VmData::simplify semantics,
//                       fidget-core/src/vm/data.rs:123-318) and queues the
//                       ambiguous children for the next level
//                       (pixel.rs:316-398 / voxel.rs:275-357).
//  k_pixels_2d       -- K2: one warp per leaf tile, two pixels per lane
//                       (pixel.rs:400-440 + VmFloatSliceEval, vm/mod.rs:800).
//  k_fill_2d         -- paints interval-proven tiles (pixel.rs:345-369).
//  k_voxels_3d / k_zsort_* / k_normals_3d / k_merge_slabs -- the 3D leaf path
//                       (voxel.rs:359-481, 524-551).
//  k_float_slice / k_grad_slice / k_interval_batch / k_point_batch /
//  k_simplify_single -- the trait-level evaluators behind fc_*_eval.
//
// The interpreters themselves live in interp.cuh, the per-op arithmetic in dev_ops.cuh, the
// cooperative level-0 kernel in coop.cu, the octree sampler leaves in octree.cu and the
// post-processing effects in effects.cu.
#include <algorithm>
#include <cstdio>

#include "level_job.cuh"

namespace fdev {

// ---------------------------------------------------------------------------
// K1: interval level kernel.  DIM = 2: pixel::render tiles (fill records are
// painted later by k_fill_2d).  DIM = 3: voxel::render tiles; an
// interval-proven-inside tile raises the heightmap to its top + 1
// (voxel.rs:310-317), heightmap entries are (depth << 32 | leaf job id + 1).
// ONE_EACH (2D, chosen by the launcher): the list cannot be longer than the grid.  It is final when the launch starts,
// so warp w takes job w and no claim crosses the GPU (prospero 4096^2, level 1: 763 jobs, where four claims out of
// five found nothing).  Consecutive jobs go to consecutive CTAs, so that the list spreads over every SM.  Longer lists
// keep the shared cursor, which balances them: with a fixed stride the warps that draw two long jobs finish last.
template <int DIM, bool FUSED_PATH = false, bool FRAMES = false, bool SCENE = false, bool ONE_EACH = false>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
k_interval_level(const __grid_constant__ LevelParams p) {
    __shared__ uint32_t live_s[WARPS_PER_BLOCK][8][32];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t gw = blockIdx.x * WARPS_PER_BLOCK + wib;
    uint32_t* cs = p.choice_scratch + size_t(gw) * p.choice_words * 32u + lane;
    itv slots[REG_SLOTS];

    const uint32_t n_roots = SCENE ? scene_root_count(p) : root_count(p, DIM == 3);
    const uint32_t n_jobs = p.root_mode ? (n_roots + 31u) / 32u : min(p.ctr->n_jobs[p.level], p.cap_in);

    if constexpr (ONE_EACH) {
        const uint32_t j = wib * gridDim.x + blockIdx.x;
        if (j >= n_jobs || __any_sync(FULL, lane == 0 && cancel_poll(p.cancel, CS_LEVEL0 + p.level, j))) return;
        level_job<DIM, FUSED_PATH, FRAMES, SCENE>(p, j, n_roots, slots, cs, live_s[wib], lane, p.epoch);
    } else {
        for (;;) {
            uint32_t j = 0;
            if (lane == 0) {
                j = atomicAdd(&p.ctr->cursor[p.level], 1u);
                if (j < n_jobs && cancel_poll(p.cancel, CS_LEVEL0 + p.level, j)) j = ~0u;   // cancelled: claim nothing more
            }
            j = __shfl_sync(FULL, j, 0);
            if (j >= n_jobs) break;

            level_job<DIM, FUSED_PATH, FRAMES, SCENE>(p, j, n_roots, slots, cs, live_s[wib], lane, p.epoch);
        }
    }
}

void launch_interval_level_2d(const LevelParams& p, int blocks, cudaStream_t s) {
    // (diagnostic: FIDGET_B200_LEVEL_FUSED_PATH=1 runs the per-level launch with the code path of the fused tail --
    //  plain tape loads, published jobs, line-aligned arena slots -- to tell code-path cost from scheduling cost)
    static const bool fused_path = getenv("FIDGET_B200_LEVEL_FUSED_PATH") && atoi(getenv("FIDGET_B200_LEVEL_FUSED_PATH"));
    if (p.scene) k_interval_level<2, false, false, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);   // a scene
    else if (p.frames) k_interval_level<2, false, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);   // a frame batch
    else if (fused_path && !p.root_mode) k_interval_level<2, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);
    else if (!p.root_mode && p.cap_in <= uint32_t(blocks) * WARPS_PER_BLOCK)
        k_interval_level<2, false, false, false, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);
    else k_interval_level<2><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);
}
void launch_interval_level_3d(const LevelParams& p, int blocks, cudaStream_t s) {
    if (p.scene) k_interval_level<3, false, false, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);   // a scene
    else if (p.frames) k_interval_level<3, false, true><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);   // a frame batch
    else k_interval_level<3><<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p);
}

// ---------------------------------------------------------------------------
// K2 (3D): leaf voxels.  One warp per leaf tile; each lane owns two XY columns
// and walks Z front to back (k descending), two points per tape pass; the
// warp stops as soon as every column has hit the surface (voxel.rs:359-447).  FRAMES: a frame batch (the tile's
// frame supplies matrix and vars; its screen rows are relative to the frame, its heightmap rows are grid rows).
// SCENE: the tile's placement supplies them, and keys are scene ranks | id (kernels.cuh, scene_rank).
template <bool FRAMES, bool SCENE = false>
__global__ void __launch_bounds__(128) k_voxels_3d(const __grid_constant__ VoxelParams p) {
    const int lane = threadIdx.x & 31;
    float4 slots[REG_SLOTS];
    const uint32_t n_jobs = min(p.ctr->n_jobs[p.list], p.cap_jobs);
    const uint32_t T = p.tile, ncol = T * T;
    unsigned long long shaded = 0;
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_VOXELS_3D, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        if (p.order) j = p.order[j];   // front-to-back: tiles behind a finished column find it done and exit early
        const TileJob* job = p.jobs + j;
        const uint32_t cx = job->x, cy = job->y, cz = job->z;
        const TapeRef tr = job->tape;
        const uint2* tape = tr.ptr;
        const unsigned long long id = (unsigned long long)(j + 1u);
        const uint32_t pl = SCENE ? job->pad : 0u;
        const FrameView fv = view_of<FRAMES, SCENE>(p, cy, pl);   // (uniform over the warp: one tile, one frame)
        const Mat4& M = *fv.mat;
        for (uint32_t base = 0; base < ncol; base += 64u) {
            const uint32_t c0 = base + lane, c1 = c0 + 32u;
            const bool v0 = c0 < ncol, v1 = c1 < ncol;
            const uint32_t i0 = (v0 ? c0 : 0u) % T, j0 = (v0 ? c0 : 0u) / T;
            const uint32_t i1 = (v1 ? c1 : 0u) % T, j1 = (v1 ? c1 : 0u) / T;
            const uint32_t gx0 = cx + i0, gy0 = cy + j0, gx1 = cx + i1, gy1 = cy + j1;
            const uint32_t sy0 = gy0 - fv.y0, sy1 = gy1 - fv.y0;   // rows inside the frame
            const bool in0 = v0 && gx0 < p.width && sy0 < p.height, in1 = v1 && gx1 < p.width && sy1 < p.height;
            // columns already at or above this tile's top are skipped (voxel.rs:376-381); in a scene, columns whose
            // rank is at least that of this placement's top voxel (a tie with a higher placement is not a skip)
            const uint32_t zmax = cz + T;
            bool done0, done1;
            if (SCENE) {
                const unsigned long long top = scene_rank(zmax, pl, p.clamp_at, p.depth);
                done0 = !in0 || (p.heightmap[size_t(gy0) * p.width + gx0] & ~SK_ID_MASK) >= top;
                done1 = !in1 || (p.heightmap[size_t(gy1) * p.width + gx1] & ~SK_ID_MASK) >= top;
            } else {
                done0 = !in0 || uint32_t(p.heightmap[size_t(gy0) * p.width + gx0] >> 32) >= zmax;
                done1 = !in1 || uint32_t(p.heightmap[size_t(gy1) * p.width + gx1] >> 32) >= zmax;
            }
            // two Z levels per tape pass: (column 0, column 1) x (k, k - 1)
            for (int k = int(T) - 1; k >= 0; k -= 2) {
                if (__all_sync(FULL, done0 && done1)) break;
                const int k2 = k > 0 ? k - 1 : 0;
                float xa, ya, za, xb, yb, zb, xc, yc, zc, xd, yd, zd;
                xform_f32(M, float(gx0), float(sy0), float(cz + uint32_t(k)), xa, ya, za);
                xform_f32(M, float(gx1), float(sy1), float(cz + uint32_t(k)), xb, yb, zb);
                xform_f32(M, float(gx0), float(sy0), float(cz + uint32_t(k2)), xc, yc, zc);
                xform_f32(M, float(gx1), float(sy1), float(cz + uint32_t(k2)), xd, yd, zd);
                const float4 X = make_float4(xa, xb, xc, xd), Y = make_float4(ya, yb, yc, yd), Z = make_float4(za, zb, zc, zd);
                const float4 r = run_f32x4(tape, tr.n_ops, slots, [&](uint32_t i) {
                    return pick_input(*fv.vb, i, X, Y, Z, [](float f) { return make_float4(f, f, f, f); });
                });
                const unsigned long long key_hi =
                    (SCENE ? scene_rank(cz + uint32_t(k) + 1u, pl, p.clamp_at, p.depth)
                           : (unsigned long long)(cz + uint32_t(k) + 1u) << 32) | id;
                const unsigned long long key_lo =
                    (SCENE ? scene_rank(cz + uint32_t(k2) + 1u, pl, p.clamp_at, p.depth)
                           : (unsigned long long)(cz + uint32_t(k2) + 1u) << 32) | id;
                const bool two = k > 0;
                if (!done0) {
                    shaded += two ? 2 : 1;
                    if (r.x < 0.0f) { atomicMax(&p.heightmap[size_t(gy0) * p.width + gx0], key_hi); done0 = true; }
                    else if (two && r.z < 0.0f) { atomicMax(&p.heightmap[size_t(gy0) * p.width + gx0], key_lo); done0 = true; }
                }
                if (!done1) {
                    shaded += two ? 2 : 1;
                    if (r.y < 0.0f) { atomicMax(&p.heightmap[size_t(gy1) * p.width + gx1], key_hi); done1 = true; }
                    else if (two && r.w < 0.0f) { atomicMax(&p.heightmap[size_t(gy1) * p.width + gx1], key_lo); done1 = true; }
                }
            }
        }
    }
    if (p.stats) {
        for (int o = 16; o > 0; o >>= 1) shaded += __shfl_xor_sync(FULL, shaded, o);
        if (lane == 0 && shaded) atomicAdd(&p.stats->pixels, shaded);
    }
}
void launch_voxels_3d(const VoxelParams& p, int blocks, cudaStream_t s) {
    if (p.scene) k_voxels_3d<false, true><<<blocks, 128, 0, s>>>(p);
    else if (p.frames) k_voxels_3d<true><<<blocks, 128, 0, s>>>(p);
    else k_voxels_3d<false><<<blocks, 128, 0, s>>>(p);
}

// Front-to-back ordering of the leaf tiles (the reference walks Z descending, voxel.rs:244-263,
// 335-351): a counting sort by Z layer, front layer first.
__global__ void k_zsort_hist(const TileJob* jobs, const uint32_t* n_jobs, uint32_t cap, uint32_t z0, uint32_t tile,
                             uint32_t n_layers, uint32_t* hist) {
    const uint32_t n = min(*n_jobs, cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t layer = min((jobs[i].z - z0) / tile, n_layers - 1u);
        atomicAdd(&hist[n_layers - 1u - layer], 1u);
    }
}
// exclusive scan of the layer histogram: one warp, 32 layers per step (shuffle scan + running carry)
__global__ void k_zsort_scan(uint32_t n_layers, uint32_t* hist) {
    const uint32_t lane = threadIdx.x;
    uint32_t carry = 0;
    for (uint32_t base = 0; base < n_layers; base += 32u) {
        const uint32_t i = base + lane;
        const uint32_t c = i < n_layers ? hist[i] : 0u;
        uint32_t incl = c;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= uint32_t(o)) incl += v;
        }
        if (i < n_layers) hist[i] = carry + incl - c;
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
}
__global__ void k_zsort_scatter(const TileJob* jobs, const uint32_t* n_jobs, uint32_t cap, uint32_t z0, uint32_t tile,
                                uint32_t n_layers, uint32_t* hist, uint32_t* order) {
    const uint32_t n = min(*n_jobs, cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t layer = min((jobs[i].z - z0) / tile, n_layers - 1u);
        order[atomicAdd(&hist[n_layers - 1u - layer], 1u)] = i;
    }
}
void launch_leaf_zsort(const TileJob* jobs, const uint32_t* n_jobs, uint32_t cap, uint32_t z0, uint32_t tile,
                       uint32_t n_layers, uint32_t* hist, uint32_t* order, cudaStream_t s) {
    cudaMemsetAsync(hist, 0, size_t(n_layers) * 4, s);
    k_zsort_hist<<<296, 256, 0, s>>>(jobs, n_jobs, cap, z0, tile, n_layers, hist);
    k_zsort_scan<<<1, 32, 0, s>>>(n_layers, hist);
    k_zsort_scatter<<<296, 256, 0, s>>>(jobs, n_jobs, cap, z0, tile, n_layers, hist, order);
}

// Exact 3D census (FC_FLAG_EXACT_CENSUS).  The reference walks every root column front to back, depth first, and
// skips a tile when all of its pixels already hold depth >= top + 1 (voxel.rs:283-293).  Everything visited before
// a tile B that touches B's pixels lies in front of B, and from in front a pixel can only receive depth > top(B) + 1
// (a filled tile) or >= top(B) + 1 (a voxel hit at z >= top(B)); from inside B it receives at most top(B) (a voxel)
// or exactly top(B) + 1 with no leaf id (a filled descendant touching B's top).  So "finished before B was visited"
// can be read off the FINAL heightmap: depth > top + 1, or depth == top + 1 with a leaf id.  One warp per recorded
// tile applies that to the tile's footprint; tiles with an unfinished pixel are the ones the reference evaluates.
// For ambiguous tiles of the last level the unfinished columns x tile edge are the voxels it evaluates
// (voxel.rs:359-386).
__global__ void __launch_bounds__(256) k_census_3d(const __grid_constant__ CensusParams p) {
    const uint32_t n = min(*p.n_recs, p.cap);
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n; i += n_warps) {
        if (cancel_poll(p.cancel, CS_CENSUS_3D, i)) break;   // (uniform over the warp)
        const CensusRec r = p.recs[i];
        const uint32_t T = p.tile[r.level], top = uint32_t(r.z) + T;
        uint32_t open_cols = 0;
        for (uint32_t q = lane; q < T * T; q += 32u) {
            const unsigned long long key = p.heightmap[size_t(r.y + q / T) * p.width + r.x + q % T];
            const uint32_t depth = uint32_t(key >> 32), id = uint32_t(key);
            const bool done = depth > top + 1u || (depth == top + 1u && id != 0u);
            open_cols += done ? 0u : 1u;
        }
        for (int o = 16; o > 0; o >>= 1) open_cols += __shfl_xor_sync(0xffffffffu, open_cols, o);
        if (lane != 0 || open_cols == 0) continue;
        const uint32_t cls = r.flags & 3u;
        atomicAdd(&p.stats->evaluated[r.level], 1ull);
        if (cls == 1u) atomicAdd(&p.stats->filled_inside[r.level], 1ull);
        else if (cls == 0u) atomicAdd(&p.stats->filled_outside[r.level], 1ull);
        else {
            atomicAdd(&p.stats->ambiguous[r.level], 1ull);
            if (r.flags & 4u) atomicAdd(&p.stats->simplified[r.level], 1ull);
            if (int(r.level) == p.last_level) atomicAdd(&p.stats->pixels, (unsigned long long)open_cols * T);
        }
    }
}
void launch_census_3d(const CensusParams& p, int blocks, cudaStream_t s) { k_census_3d<<<blocks, 256, 0, s>>>(p); }

// K3: normals + final image.  One thread per pixel; the gradient is evaluated
// at the surface voxel (x, y, depth - 1) with the tape of the
// leaf tile that found it (voxel.rs:449-481); lanes of a warp that share a
// leaf tile run its tape together.  FRAMES: a frame batch, whose output row y is row y % height of frame
// y / height (a patch may straddle two frames: each lane takes its own frame's matrix and vars).  SCENE: the key's
// placement supplies them (kernels.cuh, scene_rank; NormalParams says which pixels a pass writes).
template <bool FRAMES, bool SCENE = false>
__global__ void __launch_bounds__(128) k_normals_3d(const __grid_constant__ NormalParams p) {
    grd slots[REG_SLOTS];
    const int lane = threadIdx.x & 31;
    // 8x4 pixel patch per warp
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (cancel_poll(p.cancel, CS_NORMALS_3D, warp)) return;   // one patch per warp: the claim is the launch itself
    if (SCENE && *p.error) return;                            // an overflowed pass is rendered again
    uint32_t x, y;
    if (p.root_list) {   // patches of the listed root tiles only
        const uint32_t ppt = (p.root_tile / 8u) * (p.root_tile / 4u), ppr = p.root_tile / 8u;
        if (warp >= p.n_root_list * ppt) return;
        const uint32_t id = __ldg(p.root_list + warp / ppt), q = warp % ppt;
        x = (id % p.roots_x) * p.root_tile + (q % ppr) * 8u + (lane & 7);
        y = p.y0 + (id / p.roots_x) * p.root_tile + (q / ppr) * 4u + (lane >> 3);
    } else {
        const uint32_t patches_x = (p.width + 7u) / 8u, patches_y = (p.y1 - p.y0 + 3u) / 4u;
        if (warp >= patches_x * patches_y) return;
        x = (warp % patches_x) * 8u + (lane & 7);
        y = p.y0 + (warp / patches_x) * 4u + (lane >> 3);
    }
    const bool inb = x < p.width && y < p.y1;
    uint32_t sy = y, hy = y;   // row inside the frame, heightmap row
    const Mat4* M = &p.mat;
    const VarBind* vb = &p.vb;
    if (FRAMES) {
        const uint32_t f = inb ? y / p.height : 0u;
        sy = y - f * p.height;
        hy = f * p.frame_rows + sy;
        M = &p.frames[f].mat;
        vb = &p.frames[f].vb;
    }
    const unsigned long long key = inb ? p.heightmap[size_t(hy) * p.width + x] : 0ull;
    uint32_t depth = uint32_t(key >> 32), id = uint32_t(key);
    bool write = inb;
    uint32_t pl = 0;
    if (SCENE) {   // decode the scene key: placement, raw depth (clamp zone: threshold + excess), leaf id
        const uint32_t sub = uint32_t(key >> SK_ID_BITS) & ((1u << SK_SUB_BITS) - 1u);
        const uint32_t prio = uint32_t(key >> (SK_ID_BITS + SK_SUB_BITS)) & (SK_MAX_SHAPES - 1u);
        const uint32_t dc = uint32_t(key >> (SK_ID_BITS + SK_SUB_BITS + SK_PRIO_BITS));
        id = uint32_t(key & SK_ID_MASK);
        pl = key ? SK_MAX_SHAPES - 1u - prio : 0u;
        depth = (p.clamp && dc == p.depth) ? p.depth - 1u + sub : dc;
        write = inb && (key == 0ull || (pl >= p.pl0 && pl < p.pl1));   // an earlier pass's winner keeps its pixel
        M = &p.frames[pl].mat;
        vb = &p.frames[pl].vb;
        if (p.clamp && p.depth <= 1u) pl = 0;   // (every image is clamped everywhere: the first one is kept)
    }
    grd g = gr(0.0f, 0.0f, 0.0f, 0.0f);
    bool pending = write && id != 0u;
    unsigned long long n = 0;
    for (;;) {
        const uint32_t m = __ballot_sync(FULL, pending);
        if (!m) break;
        const uint32_t lead_id = __shfl_sync(FULL, id, __ffs(m) - 1);
        const bool mine = pending && id == lead_id;
        const TileJob* job = p.jobs + (lead_id - 1u);
        const TapeRef tr = job->tape;
        grd gx, gy, gz;
        xform_gr(*M, gr(float(x), 1.0f, 0.0f, 0.0f), gr(float(sy), 0.0f, 1.0f, 0.0f),
                 gr(float(depth - 1u), 0.0f, 0.0f, 1.0f), gx, gy, gz);
        const grd r = run_grad(tr.ptr, tr.n_ops, slots, [&](uint32_t i) {
            return pick_input(*vb, i, gx, gy, gz, [](float f) { return gr1(f); });
        });
        if (mine) { g = r; pending = false; ++n; }
    }
    if (write) {
        float4 o;
        if (p.clamp && depth >= p.depth - 1u) {   // voxel.rs:535-546
            o = make_float4(0.0f, 0.0f, 1.0f, __uint_as_float(p.depth));
        } else {
            o = make_float4(g.y, g.z, g.w, __uint_as_float(depth));
        }
        reinterpret_cast<float4*>(p.out)[size_t(y) * p.width + x] = o;
        if (SCENE && p.index) p.index[size_t(y) * p.width + x] = uint16_t(pl);
    }
    if (p.stats) {
        for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(FULL, n, o);
        if (lane == 0 && n) atomicAdd(&p.stats->grads, n);
    }
}
void launch_normals_3d(const NormalParams& p, cudaStream_t s) {
    const uint64_t warps = p.root_list ? uint64_t(p.n_root_list) * (p.root_tile / 8u) * (p.root_tile / 4u)
                                       : uint64_t((p.width + 7u) / 8u) * ((p.y1 - p.y0 + 3u) / 4u);
    if (!warps) return;
    if (p.scene) k_normals_3d<false, true><<<unsigned((warps + 3) / 4), 128, 0, s>>>(p);
    else if (p.frames) k_normals_3d<true><<<unsigned((warps + 3) / 4), 128, 0, s>>>(p);
    else k_normals_3d<false><<<unsigned((warps + 3) / 4), 128, 0, s>>>(p);
}

// Multi-GPU: per-pixel merge of Z-ordered slab images; the highest slab with
// the greatest depth wins, then the final clamp is applied.
__global__ void k_merge_slabs(const float4* const* slabs, uint32_t n_slabs, uint32_t n_pixels, uint32_t depth,
                              float4* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pixels) return;
    float4 best = slabs[0][i];
    for (uint32_t s = 1; s < n_slabs; ++s) {
        const float4 c = slabs[s][i];
        if (__float_as_uint(c.w) >= __float_as_uint(best.w)) best = c;
    }
    if (__float_as_uint(best.w) >= depth - 1u) best = make_float4(0.0f, 0.0f, 1.0f, __uint_as_float(depth));
    out[i] = best;
}
void launch_merge_slabs(const void* const* d_slabs, uint32_t n_slabs, uint32_t n_pixels, uint32_t depth, void* out,
                        cudaStream_t s) {
    k_merge_slabs<<<(n_pixels + 255) / 256, 256, 0, s>>>(reinterpret_cast<const float4* const*>(d_slabs), n_slabs,
                                                         n_pixels, depth, reinterpret_cast<float4*>(out));
}

// Multi-GPU tile interleave: image <-> [slot][T][T] chunks.  One CTA per (tile, 8 rows); consecutive threads
// move consecutive pixels of a row, so both sides are coalesced (16-byte pixels move as one float4).
template <class PX>
__global__ void __launch_bounds__(256) k_tiles_copy(const PX* __restrict__ src, PX* __restrict__ dst, uint32_t width,
                                                    uint32_t height, uint32_t T, uint32_t roots_x, const uint32_t* __restrict__ slots,
                                                    uint32_t n_ranks, uint32_t per_rank, int rank) {
    const uint32_t tile = blockIdx.x, tx = tile % roots_x, ty = tile / roots_x;
    if (rank >= 0 && tile_owner(tx, ty, n_ranks) != uint32_t(rank)) return;
    const uint32_t slot = slots[tile];
    const size_t chunk = size_t(rank >= 0 ? slot - uint32_t(rank) * per_rank : slot) * T * T;
    for (uint32_t q = blockIdx.y * 8u * T + threadIdx.x; q < min((blockIdx.y + 1u) * 8u, T) * T; q += blockDim.x) {
        const uint32_t x = tx * T + q % T, y = ty * T + q / T;
        if (x >= width || y >= height) continue;
        const size_t img = size_t(y) * width + x;
        if (rank >= 0) dst[chunk + q] = src[img];
        else dst[img] = src[chunk + q];
    }
}
void launch_tiles_copy(const void* src, void* dst, uint32_t width, uint32_t height, uint32_t px_bytes, uint32_t T,
                       uint32_t roots_x, uint32_t roots_y, const uint32_t* slots, uint32_t n_ranks, uint32_t per_rank, int rank,
                       cudaStream_t s) {
    const dim3 grid(roots_x * roots_y, (T + 7u) / 8u);
    if (px_bytes == 16)
        k_tiles_copy<float4><<<grid, 256, 0, s>>>(static_cast<const float4*>(src), static_cast<float4*>(dst), width, height, T,
                                                  roots_x, slots, n_ranks, per_rank, rank);
    else
        k_tiles_copy<float><<<grid, 256, 0, s>>>(static_cast<const float*>(src), static_cast<float*>(dst), width, height, T,
                                                 roots_x, slots, n_ranks, per_rank, rank);
}

// ---------------------------------------------------------------------------
// K2: leaf pixels (2D); FRAMES: a frame batch (kernels.cuh, Frame2D).  SCENE: a 2D scene (kernels.cuh, Scene2D): the
// tile's placement supplies matrix, Z and vars, a tile under higher shapes' proven interiors is skipped, and a pixel
// found inside raises its key to placement + 1 instead of being written
template <bool FRAMES, bool SCENE = false, class P = PixelParams>
__global__ void __launch_bounds__(128) k_pixels_2d(const __grid_constant__ P p) {
    const int lane = threadIdx.x & 31;
    float2 slots[REG_SLOTS];
    const uint32_t n_jobs = min(p.ctr->n_jobs[p.list], 0xffffffffu);
    const uint32_t T = p.tile, npix = T * T;
    unsigned long long shaded = 0;
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_PIXELS_2D, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        const TileJob* job = p.jobs + j;
        const TapeRef tr = job->tape;
        const uint2* tape = tr.ptr;
        const uint32_t pl = SCENE ? job->pad : 0u;
        if constexpr (SCENE) {   // (the leaf tile is one block)
            if (scene2d_hidden(p.cover, p.blocks_x, p.blocks_y, T, job->x, job->y, T, pl)) continue;
        }
        const FrameView fv = view_of<FRAMES, SCENE>(p, job->y, pl);   // (uniform over the warp: one tile, one frame)
        const uint32_t cx = job->x, cy = job->y - fv.y0;
        float* const out = p.out + size_t(fv.out_row0) * p.width;
        for (uint32_t base = 0; base < npix; base += 64u) {
            uint32_t p0 = base + lane, p1 = p0 + 32u;
            bool v0 = p0 < npix, v1 = p1 < npix;
            uint32_t i0 = (v0 ? p0 : 0u) % T, j0 = (v0 ? p0 : 0u) / T;
            uint32_t i1 = (v1 ? p1 : 0u) % T, j1 = (v1 ? p1 : 0u) / T;
            float x0, y0, z0, x1, y1, z1;
            xform_f32(*fv.mat, float(cx + i0), float(cy + j0), fv.z, x0, y0, z0);
            xform_f32(*fv.mat, float(cx + i1), float(cy + j1), fv.z, x1, y1, z1);
            const float2 X = make_float2(x0, x1), Y = make_float2(y0, y1), Z = make_float2(z0, z1);
            float2 r = run_f32x2(tape, tr.n_ops, slots, [&](uint32_t i) {
                return pick_input(*fv.vb, i, X, Y, Z, [](float f) { return make_float2(f, f); });
            });
            // RawDistancePixel::from(f32): canonical NaN (pixel.rs:234-240)
            if (r.x != r.x) r.x = nanf_();
            if (r.y != r.y) r.y = nanf_();
            uint32_t gx0 = cx + i0, gy0 = cy + j0, gx1 = cx + i1, gy1 = cy + j1;
            if constexpr (SCENE) {   // RawDistancePixel::inside of a distance (a canonical NaN is outside)
                if (v0 && gx0 < p.width && gy0 < p.height && r.x < 0.0f) atomicMax(&p.key[size_t(gy0) * p.width + gx0], pl + 1u);
                if (v1 && gx1 < p.width && gy1 < p.height && r.y < 0.0f) atomicMax(&p.key[size_t(gy1) * p.width + gx1], pl + 1u);
            } else {
                if (v0 && gx0 < p.width && gy0 < p.height) out[size_t(gy0) * p.width + gx0] = r.x;
                if (v1 && gx1 < p.width && gy1 < p.height) out[size_t(gy1) * p.width + gx1] = r.y;
            }
            shaded += (v0 ? 1 : 0) + (v1 ? 1 : 0);
        }
    }
    if (p.stats) {
        for (int o = 16; o > 0; o >>= 1) shaded += __shfl_xor_sync(FULL, shaded, o);
        if (lane == 0 && shaded) atomicAdd(&p.stats->pixels, shaded);
    }
}

void launch_pixels_2d(const PixelParams& p, int blocks, cudaStream_t s) {
    if (p.frames) k_pixels_2d<true><<<blocks, 128, 0, s>>>(p);
    else k_pixels_2d<false><<<blocks, 128, 0, s>>>(p);
}
void launch_pixels_2d_scene(const ScenePixelParams& p, int blocks, cudaStream_t s) {
    k_pixels_2d<false, true, ScenePixelParams><<<blocks, 128, 0, s>>>(p);
}

// The image of a 2D scene (kernels.cuh, Scene2D): one warp per 32 consecutive pixels of a row, whose ballot is the
// 1-bit packing, as in k_to_mask
__global__ void __launch_bounds__(256) k_scene2d_resolve(const __grid_constant__ Scene2DResolveParams p) {
    const uint32_t words = (p.width + 31u) / 32u, lane = threadIdx.x & 31u;
    const uint64_t warp = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (warp >= uint64_t(words) * p.height) return;
    if (cancel_poll(p.cancel, CS_SCENE2D_RESOLVE, uint32_t(warp))) return;   // (uniform over the warp)
    const uint32_t y = uint32_t(warp / words), x = uint32_t(warp % words) * 32u + lane;
    const size_t i = size_t(y) * p.width + x;
    const uint32_t top = x < p.width ? max(p.cover[size_t(y / p.leaf) * p.blocks_x + x / p.leaf], p.key[i]) : 0u;
    if (x < p.width && p.index) p.index[i] = top ? uint16_t(top - 1u) : uint16_t(0xFFFFu);
    if (!p.out) return;
    if (p.fmt == 2u) {
        const uint32_t m = __ballot_sync(0xffffffffu, top != 0u), stride = (p.width + 7u) / 8u;
        if (lane < 4u && x - lane + lane * 8u < p.width) p.out[size_t(y) * stride + (x - lane) / 8u + lane] = uint8_t(m >> (8u * lane));
    } else if (x < p.width) {
        if (p.fmt == 1u) {
            p.out[i] = top ? 255 : 0;
        } else {
            const uint8_t* c = p.colors + 3u * (top - 1u);
            reinterpret_cast<uint32_t*>(p.out)[i] = top ? (uint32_t(c[0]) | uint32_t(c[1]) << 8 | uint32_t(c[2]) << 16 | 0xFF000000u) : 0u;
        }
    }
}
void launch_scene2d_resolve(const Scene2DResolveParams& p, cudaStream_t s) {
    const uint64_t warps = uint64_t((p.width + 31u) / 32u) * p.height;
    if (warps) k_scene2d_resolve<<<unsigned((warps * 32 + 255) / 256), 256, 0, s>>>(p);
}

// ---------------------------------------------------------------------------
// Fill painter: one warp per (record, unit of <= 1024 pixels).  Any tile edge T works: the last
// unit of a tile may be partial, and tiles whose edge is not a multiple of four (a 4-pixel group
// would straddle two rows) take the per-pixel path.
template <bool FRAMES>
__global__ void __launch_bounds__(256) k_fill_2d(const __grid_constant__ FillParams p) {
    const uint32_t n = *p.n_fills;
    const uint32_t T = p.tile;
    const uint32_t tile_px = T * T;
    const uint32_t unit_px = min(tile_px, 1024u);
    const uint32_t units = (tile_px + unit_px - 1u) / unit_px;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
    const bool vec_ok = (p.width % 4u == 0u) && ((reinterpret_cast<uintptr_t>(p.out) & 15u) == 0u) && (T % 4u == 0u);
    const unsigned long long total = (unsigned long long)n * units;
    for (unsigned long long w = warp; w < total; w += n_warps) {
        if (cancel_poll(p.cancel, CS_FILL_2D, uint32_t(w))) break;
        const uint32_t rec = uint32_t(w / units), u = uint32_t(w % units);
        const FillRec fr = p.fills[rec];
        const float v = __uint_as_float(fr.value);
        const uint32_t first = u * unit_px;
        // frame batch: the record's frame, its row inside the frame, and where that frame's rows start in `out`
        const uint32_t f = FRAMES ? fr.y / p.frame_rows : 0u, fy = fr.y - f * p.frame_rows;
        float* const out = p.out + size_t(f) * p.height * p.width;
        for (uint32_t q = lane * 4u; q < unit_px; q += 128u) {
            const uint32_t pix = first + q;
            if (pix >= tile_px) break;
            if (vec_ok) {   // T % 4 == 0: the group lies in one row, 16-byte aligned
                const uint32_t x = fr.x + pix % T, y = fy + pix / T;
                if (y >= p.height || x >= p.width) continue;
                *reinterpret_cast<float4*>(out + size_t(y) * p.width + x) = make_float4(v, v, v, v);   // width % 4 == 0
            } else {
                for (uint32_t k = 0; k < 4u && pix + k < tile_px; ++k) {
                    const uint32_t x = fr.x + (pix + k) % T, y = fy + (pix + k) / T;
                    if (x < p.width && y < p.height) out[size_t(y) * p.width + x] = v;
                }
            }
        }
    }
}

void launch_fill_2d(const FillParams& p, int blocks, cudaStream_t s) {
    if (p.frame_rows != 0xffffffffu) k_fill_2d<true><<<blocks, 256, 0, s>>>(p);
    else k_fill_2d<false><<<blocks, 256, 0, s>>>(p);
}

// ---------------------------------------------------------------------------
// Trait-level evaluators
template <int NSLOTS>
__global__ void __launch_bounds__(128) k_float_slice(const __grid_constant__ BulkParams p) {
    float slots[NSLOTS];
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    for (uint64_t idx = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < p.n; idx += stride) {
        const uint2* tape = p.tape;
        for (uint32_t i = 0; i < p.n_ops; ++i) {
            uint2 w = __ldg(tape + i);
            Dec d(w.x);
            float imm = __uint_as_float(w.y);
            float sl = slots[d.lhs], sr = slots[d.rhs];
            float a = d.form == F_IR ? imm : sl;
            float b = d.form == F_RI ? imm : sr;
            float r;
            if (d.op == OP_MEM) {
                if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                else slots[MEM_BASE + w.y] = sl;
                continue;
            } else if (d.op >= OP_ADD) r = f32_binary(d.op, a, b);
            else if (d.op >= OP_NEG) r = f32_unary(d.op, sl);
            else if (d.op == OP_COPY) r = d.form == F_RI ? imm : sl;
            else if (d.op == OP_INPUT) r = static_cast<const float*>(p.vars[w.y])[idx];
            else {
                static_cast<float*>(p.outs[w.y])[idx] = sl;
                continue;
            }
            slots[d.out] = r;
        }
    }
}

template <int NSLOTS>
__global__ void __launch_bounds__(128) k_grad_slice(const __grid_constant__ BulkParams p) {
    grd slots[NSLOTS];
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    for (uint64_t idx = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < p.n; idx += stride) {
        const uint2* tape = p.tape;
        for (uint32_t i = 0; i < p.n_ops; ++i) {
            uint2 w = __ldg(tape + i);
            Dec d(w.x);
            float imm = __uint_as_float(w.y);
            grd sl = slots[d.lhs], sr = slots[d.rhs];
            grd a = d.form == F_IR ? gr1(imm) : sl;
            grd b = d.form == F_RI ? gr1(imm) : sr;
            grd r;
            if (d.op == OP_MEM) {
                if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                else slots[MEM_BASE + w.y] = sl;
                continue;
            } else if (d.op >= OP_ADD) {
                if (d.op == OP_MUL && d.form == F_RI) r = gr_mul_f(sl, imm);
                else r = gr_binary(d.op, a, b);
            } else if (d.op >= OP_NEG) r = gr_unary(d.op, sl);
            else if (d.op == OP_COPY) r = d.form == F_RI ? gr1(imm) : sl;
            else if (d.op == OP_INPUT) r = static_cast<const grd*>(p.vars[w.y])[idx];
            else {
                static_cast<grd*>(p.outs[w.y])[idx] = sl;
                continue;
            }
            slots[d.out] = r;
        }
    }
}

static int bulk_blocks(uint64_t n) {
    uint64_t b = (n + 127) / 128;
    return int(b < 1 ? 1 : (b > 132ull * 16 ? 132ull * 16 : b));   // H100: 132 SMs x 16 blocks of 128 threads
}
void launch_float_slice(const BulkParams& p, cudaStream_t s) {
    if (p.n == 0) return;
    if (p.n_slots <= 256) k_float_slice<256><<<bulk_blocks(p.n), 128, 0, s>>>(p);
    else k_float_slice<2048><<<bulk_blocks(p.n), 128, 0, s>>>(p);
}
void launch_grad_slice(const BulkParams& p, cudaStream_t s) {
    if (p.n == 0) return;
    if (p.n_slots <= 256) k_grad_slice<256><<<bulk_blocks(p.n), 128, 0, s>>>(p);
    else k_grad_slice<2048><<<bulk_blocks(p.n), 128, 0, s>>>(p);
}

struct ByteChoiceSink {
    uint8_t* base;  // may be null
    uint32_t ci = 0;
    bool any_nonboth = false;
    __device__ __forceinline__ void push(uint32_t c) {
        if (base) base[ci] = uint8_t(c);
        ++ci;
        any_nonboth |= (c != 3u);
    }
};

template <int NSLOTS>
__global__ void __launch_bounds__(128) k_interval_batch(const __grid_constant__ TracingParams p) {
    itv slots[NSLOTS];
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    for (uint64_t idx = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < p.n; idx += stride) {
        const float* v = p.vars + idx * p.n_vars * 2;
        float* o = p.out + idx * p.n_outputs * 2;
        ByteChoiceSink sink;
        sink.base = p.choices ? p.choices + idx * p.n_choices : nullptr;
        run_interval(
            p.tape, p.n_ops, slots, [&](uint32_t i) { return iv(v[2 * i], v[2 * i + 1]); }, sink,
            [&](uint32_t oi, itv val) { o[2 * oi] = val.x; o[2 * oi + 1] = val.y; });
        if (p.simplify) p.simplify[idx] = sink.any_nonboth ? 1 : 0;
    }
}

template <int NSLOTS>
__global__ void __launch_bounds__(128) k_point_batch(const __grid_constant__ TracingParams p) {
    float slots[NSLOTS];
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    for (uint64_t idx = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < p.n; idx += stride) {
        const float* v = p.vars + idx * p.n_vars;
        float* o = p.out + idx * p.n_outputs;
        ByteChoiceSink sink;
        sink.base = p.choices ? p.choices + idx * p.n_choices : nullptr;
        for (uint32_t i = 0; i < p.n_ops; ++i) {
            uint2 w = __ldg(p.tape + i);
            Dec d(w.x);
            float imm = __uint_as_float(w.y);
            float sl = slots[d.lhs], sr = slots[d.rhs];
            float a = d.form == F_IR ? imm : sl;
            float b = d.form == F_RI ? imm : sr;
            float r;
            if (d.op == OP_MEM) {
                if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                else slots[MEM_BASE + w.y] = sl;
                continue;
            } else if (d.op >= OP_MIN) {
                r = f32_binary(d.op, a, b);
                sink.push(f32_choice(d.op, a, b));
            } else if (d.op >= OP_ADD) r = f32_binary(d.op, a, b);
            else if (d.op >= OP_NEG) r = f32_unary(d.op, sl);
            else if (d.op == OP_COPY) r = d.form == F_RI ? imm : sl;
            else if (d.op == OP_INPUT) r = v[w.y];
            else { o[w.y] = sl; continue; }
            slots[d.out] = r;
        }
        if (p.simplify) p.simplify[idx] = sink.any_nonboth ? 1 : 0;
    }
}

void launch_interval_batch(const TracingParams& p, cudaStream_t s) {
    if (p.n == 0) return;
    if (p.n_slots <= 256) k_interval_batch<256><<<bulk_blocks(p.n), 128, 0, s>>>(p);
    else k_interval_batch<2048><<<bulk_blocks(p.n), 128, 0, s>>>(p);
}
void launch_point_batch(const TracingParams& p, cudaStream_t s) {
    if (p.n == 0) return;
    if (p.n_slots <= 256) k_point_batch<256><<<bulk_blocks(p.n), 128, 0, s>>>(p);
    else k_point_batch<2048><<<bulk_blocks(p.n), 128, 0, s>>>(p);
}

__global__ void k_simplify_single(const __grid_constant__ SimplifyParams p) {
    __shared__ uint32_t live_s[8][32];
    const int lane = threadIdx.x;
    ByteChoiceSource src;
    src.base = p.choices;
    src.ci = p.n_choices;
    uint32_t n_dev = 0, ref_len = 0, nch = 0;
    simplify_lane(p.parent, p.n_ops, lane == 0, live_s, lane, src, p.out + p.n_ops, n_dev, ref_len, nch);
    if (lane == 0) {
        p.result[0] = n_dev;
        p.result[1] = ref_len;
        p.result[2] = nch;
    }
}
void launch_simplify_single(const SimplifyParams& p, cudaStream_t s) { k_simplify_single<<<1, 32, 0, s>>>(p); }

}  // namespace fdev
