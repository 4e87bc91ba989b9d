// fc_volume_build / fc_volume_read: the field of a shape on a sparse narrow-band voxel grid.  The interval levels are the
// stacked octree's (k_tree_level_volume: proven cells, tested against +-band, go to a tile list); the kernels below sort
// the bricks and tiles into their canonical order and evaluate every brick's cell centres, and its gradients with
// FC_FLAG_VOLUME_GRADS, into the volume, which stays in HBM until it is read.
#include <cub/cub.cuh>

#include <cmath>

#include "capi_internal.h"
#include "level_job.cuh"
#include "pass_plan.h"

namespace fdev {

// A pass's brick jobs as sort keys (volume_key) and their indices
__global__ void k_volume_keys(const TileJob* jobs, uint32_t n, uint32_t rows, unsigned long long* keys, uint32_t* idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t x = jobs[i].x, y = jobs[i].y, z = jobs[i].z, f = y / rows;
    keys[i] = volume_key(f, x, y - f * rows, z);
    idx[i] = i;
}

// first[f] = the index of frame f's first entry in the sorted keys (the frame is key >> shift); frames without one keep
// what first held
__global__ void k_volume_firsts(const unsigned long long* keys, uint32_t n, int shift, uint32_t* first) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t f = uint32_t(keys[i] >> shift);
    if (i == 0 || uint32_t(keys[i - 1] >> shift) != f) first[f] = i;
}

// The sorted tile keys of a pass as fc_volume_tile records (frame f of the pass is f0 + f); *n_inside counts the
// inside tiles
__global__ void k_volume_tiles(const unsigned long long* keys, uint32_t n, uint32_t f0, VolumeTile* out,
                               unsigned long long* n_inside) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < n;
    const unsigned long long k = valid ? keys[i] : 0ull, c = k >> VOLUME_TILE_LOW_BITS;
    const bool inside = valid && (k & 1ull);
    if (valid) {
        VolumeTile t;
        t.frame = f0 + uint32_t(c >> 36);
        t.ix = uint16_t(c & 0xfffu);
        t.iy = uint16_t((c >> 12) & 0xfffu);
        t.iz = uint16_t((c >> 24) & 0xfffu);
        t.log2_edge = uint8_t((k >> 1) & 0xfu);
        t.inside = inside ? 1u : 0u;
        out[i] = t;
    }
    const uint32_t m = __ballot_sync(FULL, inside);
    if ((threadIdx.x & 31u) == 0 && m) atomicAdd(n_inside, (unsigned long long)__popc(m));
}

// The world centre -1 + (2i + 1) 2^-D of cell c of the brick at (cx, cy, cz) (exact in f32), through the frame's
// world_to_model as k_measure_brick maps it
__device__ __forceinline__ void brick_centre(uint32_t cx, uint32_t cy, uint32_t cz, uint32_t c, uint32_t B, float inv,
                                             float& x, float& y, float& z) {
    x = float(2u * (cx + c % B) + 1u) * inv - 1.0f;
    y = float(2u * (cy + (c / B) % B) + 1u) * inv - 1.0f;
    z = float(2u * (cz + c / (B * B)) + 1u) * inv - 1.0f;
}

// One warp per brick, claimed in sorted order: a lane evaluates two cells at once with the brick's tape (run_f32x2), and
// the warp's stores of a step cover 64 consecutive values.  Smaller bricks (depth < 3) leave lanes idle.
__global__ void __launch_bounds__(128) k_volume_brick(const __grid_constant__ VolumeBrickParams p, const MeshFrame* frames) {
    const int lane = threadIdx.x & 31;
    float2 slots[REG_SLOTS];
    const uint32_t B = p.brick, nb = B * B * B;
    const float inv = 1.0f / float(1u << p.depth);
    for (;;) {
        uint32_t r = 0;
        if (lane == 0) {
            r = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (r < p.n && cancel_poll(p.cancel, CS_VOLUME_BRICK, r)) r = ~0u;
        }
        r = __shfl_sync(FULL, r, 0);
        if (r >= p.n) break;
        const unsigned long long key = p.keys[r];
        const uint32_t f = uint32_t(key >> 36), cx = uint32_t(key & 0xfffu), cy = uint32_t((key >> 12) & 0xfffu),
                       cz = uint32_t((key >> 24) & 0xfffu);
        const TapeRef tr = p.jobs[p.order[r]].tape;
        const MeshFrame& fr = frames[f];
        float* out = p.values + size_t(r) * nb;
        for (uint32_t q = 0; q < nb; q += 64u) {
            const uint32_t c0 = q + uint32_t(lane), c1 = c0 + 32u;
            float x0, y0, z0, x1, y1, z1;
            brick_centre(cx, cy, cz, c0 < nb ? c0 : 0u, B, inv, x0, y0, z0);
            brick_centre(cx, cy, cz, c1 < nb ? c1 : 0u, B, inv, x1, y1, z1);
            if (fr.has_transform) {
                xform_f32(fr.mat, x0, y0, z0, x0, y0, z0);
                xform_f32(fr.mat, x1, y1, z1, x1, y1, z1);
            }
            const float2 X = make_float2(x0, x1), Y = make_float2(y0, y1), Z = make_float2(z0, z1);
            const float2 v = run_f32x2(tr.ptr, tr.n_ops, slots, [&](uint32_t i) {
                return pick_input(fr.vb, i, X, Y, Z, [](float s) { return make_float2(s, s); });
            });
            if (c0 < nb) out[c0] = v.x;
            if (c1 < nb) out[c1] = v.y;
        }
        if (lane == 0) p.bricks[r] = VolumeBrick{p.f0 + f, uint16_t(cx), uint16_t(cy), uint16_t(cz), 0};
    }
}

// FC_FLAG_VOLUME_GRADS: one warp per brick, one cell per lane, grad_at with the brick's tape at the world centre
__global__ void __launch_bounds__(128) k_volume_grads(const __grid_constant__ VolumeBrickParams p, const MeshFrame* frames) {
    const int lane = threadIdx.x & 31;
    grd slots[REG_SLOTS];
    const uint32_t B = p.brick, nb = B * B * B;
    const float inv = 1.0f / float(1u << p.depth);
    for (;;) {
        uint32_t r = 0;
        if (lane == 0) {
            r = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (r < p.n && cancel_poll(p.cancel, CS_VOLUME_GRADS, r)) r = ~0u;
        }
        r = __shfl_sync(FULL, r, 0);
        if (r >= p.n) break;
        const unsigned long long key = p.keys[r];
        const uint32_t f = uint32_t(key >> 36), cx = uint32_t(key & 0xfffu), cy = uint32_t((key >> 12) & 0xfffu),
                       cz = uint32_t((key >> 24) & 0xfffu);
        const TapeRef tr = p.jobs[p.order[r]].tape;
        const MeshFrame& fr = frames[f];
        for (uint32_t q = 0; q < nb; q += 32u) {
            const uint32_t c = q + uint32_t(lane);
            float x, y, z;
            brick_centre(cx, cy, cz, c < nb ? c : 0u, B, inv, x, y, z);
            const grd g = grad_at(tr, slots, x, y, z, fr.has_transform, fr.mat, fr.vb);
            if (c < nb) {
                float* o = p.grads + (size_t(r) * nb + c) * 3u;
                o[0] = g.y; o[1] = g.z; o[2] = g.w;
            }
        }
    }
}

}  // namespace fdev

namespace {

static_assert(sizeof(fc_volume_brick) == sizeof(VolumeBrick) && sizeof(VolumeBrick) == 12, "fc_volume_brick layout");
static_assert(sizeof(fc_volume_tile) == sizeof(VolumeTile) && sizeof(VolumeTile) == 12, "fc_volume_tile layout");
static_assert(offsetof(fc_volume_tile, log2_edge) == offsetof(VolumeTile, log2_edge), "fc_volume_tile layout");
static_assert(sizeof(fc_volume_cfg) == 16 && sizeof(fc_volume_frame_info) == 32, "fc_volume layouts");
static_assert(sizeof(fc_volume_info) == 168 && offsetof(fc_volume_info, brick_edge) == 152, "fc_volume_info layout");

// Grows the volume to n_b bricks and n_t tiles, keeping its first keep_b and keep_t (the earlier passes'):
// FC_ERR_UNSUPPORTED when the buffers that must grow do not fit the device's free memory
int32_t volume_grow(fc_ctx* c, uint64_t n_b, uint64_t n_t, uint64_t keep_b, uint64_t keep_t, uint32_t cells, bool grads) {
    struct Grow { DevBuf* b; size_t need, keep; };
    const Grow g[4] = {{&c->vol_bricks, n_b * sizeof(VolumeBrick), keep_b * sizeof(VolumeBrick)},
                       {&c->vol_values, n_b * cells * 4, keep_b * cells * 4},
                       {&c->vol_grads, grads ? n_b * cells * 12 : 0, grads ? keep_b * cells * 12 : 0},
                       {&c->vol_tiles, n_t * sizeof(VolumeTile), keep_t * sizeof(VolumeTile)}};
    size_t add = 0;
    for (const Grow& x : g)
        if (x.need > x.b->cap) add += std::max(x.need, x.b->cap + x.b->cap / 2);   // (what grow_keep allocates)
    if (add) {
        size_t free_bytes = 0, total = 0;
        CU(cudaMemGetInfo(&free_bytes, &total));
        if (add > free_bytes)
            return fail(FC_ERR_UNSUPPORTED, "volume too large: " + std::to_string(n_b) + " bricks and " + std::to_string(n_t) +
                                                " tiles need " + std::to_string(add >> 20) + " MiB more device memory");
    }
    for (const Grow& x : g)
        if (int32_t rc = grow_keep(c, *x.b, x.need, x.keep)) return rc;
    return FC_OK;
}

// frame k of a pass's n starts at first[k] of its m sorted entries (0xffffffff: it has none; it starts where the next does)
void frame_ranges(uint32_t* first, uint32_t n, uint32_t m) {
    uint32_t next = m;
    for (uint32_t k = n; k-- > 0;) {
        if (first[k] == 0xffffffffu) first[k] = next;
        next = first[k];
    }
}

// The passes of a checked call, into the context's volume.  The caller holds the context's lock.
int32_t volume_passes(fc_ctx* c, const fc_tape* tape, uint32_t D, float band, bool grads, bool timing,
                      const std::vector<MeshFrame>& fr, fc_volume_info& info, std::vector<fc_volume_frame_info>& pf,
                      const CallCancel& cc) {
    const uint32_t N = uint32_t(fr.size());
    const uint32_t b = std::min<uint32_t>(D, 3), B = 1u << b, cells = B * B * B;
    const int Lb = int(D - b) + 1;   // interval levels 0 .. D - b; the bricks are list Lb
    cudaStream_t s = c->stream;
    const uint64_t cap_limit = list_cap_limit();
    // a pass's tile list: at worst every cell of every level, capped as the job lists are
    auto tile_cap = [Lb](uint64_t k, uint64_t limit) {
        uint64_t w = 0;
        for (int l = 0; l < Lb; ++l) w += k << (3 * l);
        return std::min(w, limit);
    };
    // a pass's cell rows must fit 32 bits
    PassPlan plan = tree_passes(c, N, uint32_t(std::min<uint64_t>({N, FC_MESH_MAX_PASS_FRAMES, 0xffffffffull >> D})), D, 3,
                                Lb, 0);
    const auto level_limits = plan.limits_of;
    plan.limits_of = [=](uint32_t k) {   // the tile list is the planner's measured quantity
        PassLimits lim = level_limits(k);
        lim.extra_cap = tile_cap(k, cap_limit);
        lim.extra_on = lim.extra_cap < tile_cap(k, ~0ull);
        lim.extra_scale = 1;
        return lim;
    };
    uint64_t tot_b = 0, tot_t = 0;
    std::vector<uint32_t> first;
    while (plan.more()) {
        const PassPlan::Range r = plan.take();
        MeshFrame* d_fr = nullptr;
        CU(carve(c->mesh_frames, [&](Carve& cv) { cv.take(d_fr, size_t(r.n) * sizeof(MeshFrame)); }));
        CU(cudaMemcpyAsync(d_fr, fr.data() + r.f0, size_t(r.n) * sizeof(MeshFrame), cudaMemcpyHostToDevice, s));
        TreeScratch t;
        if (int32_t trc = tree_scratch(c, tape, D, 3, r.n, 0, t)) return trc;
        uint32_t* d_n_tiles = reinterpret_cast<uint32_t*>(c->counters.as<char>() + sizeof(Counters));
        const uint64_t cap_t = tile_cap(r.n, cap_limit);
        CU(c->vol_list.ensure(cap_t * sizeof(unsigned long long)));
        CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
        const VolumeLevel v{c->vol_list.as<unsigned long long>(), d_n_tiles, uint32_t(cap_t), band};
        if (timing) CU(cudaEventRecord(get_event(c, 0), s));
        for (int l = 0; l < Lb; ++l) {
            LevelParams p = tree_level(c, tape, t, l, fr[r.f0], cc);
            p.stats = c->stats.as<Stats>();
            launch_tree_level_volume(p, d_fr, v, t.blocks(l), s);
        }
        if (timing) CU(cudaEventRecord(get_event(c, 1), s));
        CU(cudaGetLastError());
        // the pass's counters and its tile count, the word after them
        unsigned char words[sizeof(Counters) + 4];
        if (int32_t wrc = wait_read(c, s, cc, words, c->counters.p, sizeof words)) return wrc;
        Counters ctr;
        uint32_t n_t = 0;
        memcpy(&ctr, words, sizeof ctr);
        memcpy(&n_t, words + sizeof ctr, 4);
        bool split = false;
        if (!plan.observe(ctr, n_t, r, split)) return device_error(ctr.error);
        if (split) continue;
        const uint32_t n_b = ctr.n_jobs[Lb];
        if (int32_t grc = volume_grow(c, tot_b + n_b, tot_t + n_t, tot_b, tot_t, cells, grads)) return grc;
        // sort scratch: brick keys and indices in and out, tile keys out, each frame's first brick and tile
        int fbits = 0;
        for (uint32_t k = r.n - 1; k; k >>= 1) ++fbits;
        const int key_bits = 36 + fbits, tile_bits = key_bits + VOLUME_TILE_LOW_BITS;
        size_t t_b = 0, t_t = 0;
        CU(cub::DeviceRadixSort::SortPairs(nullptr, t_b, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                           (uint32_t*)nullptr, (uint32_t*)nullptr, int(n_b), 0, key_bits, s));
        CU(cub::DeviceRadixSort::SortKeys(nullptr, t_t, (unsigned long long*)nullptr, (unsigned long long*)nullptr, int(n_t),
                                          0, tile_bits, s));
        unsigned long long *bk_in, *bk, *tk, *d_inside;
        uint32_t *bi_in, *order, *d_first;
        void* cub_tmp;
        CU(carve(c->vol_scratch, [&](Carve& cv) {
            cv.take(bk_in, size_t(n_b) * 8); cv.take(bk, size_t(n_b) * 8);
            cv.take(bi_in, size_t(n_b) * 4); cv.take(order, size_t(n_b) * 4);
            cv.take(tk, size_t(n_t) * 8);
            cv.take(d_first, size_t(r.n) * 8);
            cv.take(d_inside, 8);
            cv.take(cub_tmp, std::max<size_t>(std::max(t_b, t_t), 1));
        }));
        if (timing) CU(cudaEventRecord(get_event(c, 2), s));
        CU(cudaMemsetAsync(d_first, 0xff, size_t(r.n) * 8, s));
        CU(cudaMemsetAsync(d_inside, 0, 8, s));
        const TileJob* jobs = c->jobs[Lb].as<TileJob>();
        if (n_b) {
            k_volume_keys<<<(n_b + 127) / 128, 128, 0, s>>>(jobs, n_b, 1u << D, bk_in, bi_in);
            size_t tb = t_b;
            CU(cub::DeviceRadixSort::SortPairs(cub_tmp, tb, bk_in, bk, bi_in, order, int(n_b), 0, key_bits, s));
            k_volume_firsts<<<(n_b + 127) / 128, 128, 0, s>>>(bk, n_b, 36, d_first);
        }
        if (n_t) {
            size_t tt = t_t;
            CU(cub::DeviceRadixSort::SortKeys(cub_tmp, tt, c->vol_list.as<unsigned long long>(), tk, int(n_t), 0, tile_bits, s));
            k_volume_firsts<<<(n_t + 127) / 128, 128, 0, s>>>(tk, n_t, 36 + VOLUME_TILE_LOW_BITS, d_first + r.n);
            k_volume_tiles<<<(n_t + 127) / 128, 128, 0, s>>>(tk, n_t, r.f0, c->vol_tiles.as<VolumeTile>() + tot_t, d_inside);
        }
        VolumeBrickParams q{};
        q.jobs = jobs;
        q.order = order;
        q.keys = bk;
        q.n = n_b;
        q.f0 = r.f0;
        q.depth = D;
        q.brick = B;
        q.values = c->vol_values.as<float>() + size_t(tot_b) * cells;
        q.grads = grads ? c->vol_grads.as<float>() + size_t(tot_b) * cells * 3 : nullptr;
        q.bricks = c->vol_bricks.as<VolumeBrick>() + tot_b;
        q.ctr = c->counters.as<Counters>();
        q.cursor = Lb;
        q.cancel = cc.ref;
        k_volume_brick<<<c->sm_count * 8, 128, 0, s>>>(q, d_fr);
        if (grads) {
            q.cursor = Lb + 1;
            k_volume_grads<<<c->sm_count * 8, 128, 0, s>>>(q, d_fr);
        }
        if (timing) CU(cudaEventRecord(get_event(c, 3), s));
        CU(cudaGetLastError());
        first.resize(size_t(r.n) * 2);
        if (int32_t wrc = wait_read(c, s, cc, first.data(), d_first, size_t(r.n) * 8)) return wrc;
        unsigned long long n_inside = 0;
        CU(cudaMemcpy(&n_inside, d_inside, 8, cudaMemcpyDeviceToHost));
        Stats st;
        CU(cudaMemcpy(&st, c->stats.p, sizeof st, cudaMemcpyDeviceToHost));
        frame_ranges(first.data(), r.n, n_b);
        frame_ranges(first.data() + r.n, r.n, n_t);
        for (uint32_t k = 0; k < r.n; ++k) {
            fc_volume_frame_info& o = pf[r.f0 + k];
            o.first_brick = tot_b + first[k];
            o.n_bricks = (k + 1 < r.n ? first[k + 1] : n_b) - first[k];
            o.first_tile = tot_t + first[r.n + k];
            o.n_tiles = (k + 1 < r.n ? first[r.n + k + 1] : n_t) - first[r.n + k];
        }
        for (int l = 0; l < 16 && l < MAX_LEVELS; ++l) info.evaluated[l] += st.evaluated[l];
        info.n_inside_tiles += n_inside;
        ++info.passes;
        if (timing) {
            float a = 0, z = 0;
            cudaEventElapsedTime(&a, get_event(c, 0), get_event(c, 1));
            cudaEventElapsedTime(&z, get_event(c, 2), get_event(c, 3));
            info.level_ms += a;
            info.device_ms += a + z;
        }
        tot_b += n_b;
        tot_t += n_t;
    }
    info.n_bricks = tot_b;
    info.n_tiles = tot_t;
    return FC_OK;
}

}  // namespace

extern "C" {

int32_t fc_volume_build(fc_ctx* c, const fc_tape* tape, const fc_volume_cfg* cfg, const fc_mesh_frame* frames,
                        uint32_t n_frames, fc_volume_info* info, fc_volume_frame_info* per_frame) {
    if (info) memset(info, 0, sizeof *info);
    if (per_frame && n_frames) memset(per_frame, 0, size_t(n_frames) * sizeof *per_frame);
    if (!c || !tape || !cfg) return fail(FC_ERR_INVALID, "null argument");
    {   // whatever happens below, the previous volume is gone
        std::lock_guard<std::mutex> guard(c->mu);
        c->vol_n_bricks = c->vol_n_tiles = 0;
        c->vol_grads_on = false;
    }
    if (int32_t rc = check_tree_call(tape, 3, cfg->depth, frames, n_frames, "fc_volume_build")) return rc;
    if (!(cfg->band >= 0.0f) || std::isinf(cfg->band)) return fail(FC_ERR_INVALID, "band must be finite and >= 0");
    std::vector<MeshFrame> fr(n_frames);
    for (uint32_t k = 0; k < n_frames; ++k) {
        const fc_mesh_frame& in = frames[k];
        if (int32_t vrc = bind_frame(tape, in.has_transform, in.world_to_model, 0.0f, in.var_values, in.n_var_values, fr[k]))
            return vrc;
    }
    const uint32_t D = cfg->depth, B = 1u << std::min<uint32_t>(D, 3);
    if (!n_frames) return FC_OK;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    const bool grads = (cfg->flags & FC_FLAG_VOLUME_GRADS) != 0;
    fc_volume_info in{};
    in.brick_edge = B;
    std::vector<fc_volume_frame_info> pf(n_frames);
    int32_t rc;
    {
        std::lock_guard<std::mutex> guard(c->mu);
        CU(cudaSetDevice(c->device));
        rc = volume_passes(c, tape, D, cfg->band, grads, (cfg->flags & FC_FLAG_TIMING) != 0, fr, in, pf, cc);
        if (!rc) {
            c->vol_n_bricks = in.n_bricks;
            c->vol_n_tiles = in.n_tiles;
            c->vol_cells = B * B * B;
            c->vol_grads_on = grads;
        }
    }
    if (rc) return rc;
    if (info) *info = in;
    if (per_frame) memcpy(per_frame, pf.data(), size_t(n_frames) * sizeof *per_frame);
    return FC_OK;
}

int32_t fc_volume_read(fc_ctx* c, fc_volume_brick* bricks, float* values, float* grads, fc_volume_tile* tiles) {
    if (!c) return fail(FC_ERR_INVALID, "null context");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const size_t nb = c->vol_n_bricks, nt = c->vol_n_tiles, cells = c->vol_cells;
    if (grads && nb && !c->vol_grads_on) return fail(FC_ERR_INVALID, "the volume was built without FC_FLAG_VOLUME_GRADS");
    cudaStream_t s = c->stream;
    if (bricks && nb) CU(cudaMemcpyAsync(bricks, c->vol_bricks.p, nb * sizeof(VolumeBrick), cudaMemcpyDefault, s));
    if (values && nb) CU(cudaMemcpyAsync(values, c->vol_values.p, nb * cells * 4, cudaMemcpyDefault, s));
    if (grads && nb) CU(cudaMemcpyAsync(grads, c->vol_grads.p, nb * cells * 12, cudaMemcpyDefault, s));
    if (tiles && nt) CU(cudaMemcpyAsync(tiles, c->vol_tiles.p, nt * sizeof(VolumeTile), cudaMemcpyDefault, s));
    CU(cudaStreamSynchronize(s));
    return FC_OK;
}

}  // extern "C"
