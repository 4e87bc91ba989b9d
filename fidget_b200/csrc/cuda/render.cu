// The fused tile renderers: fc_render2d (pixel::render), fc_render3d (voxel::render), their frame batches
// (fc_render2d_frames, fc_render3d_frames), scenes of several shapes (fc_render2d_scene, fc_render3d_scene),
// fc_merge_slabs.
#include <cstddef>
#include <functional>

#include "capi_internal.h"
#include "pass_plan.h"

// TileSizesRef::new (fidget-raster/src/lib.rs:59-66)
int32_t pick_tile_sizes(const uint32_t* ts_in, uint32_t n_in, const uint32_t* dflt, uint32_t n_dflt,
                               uint32_t max_size, std::vector<uint32_t>& ts) {
    std::vector<uint32_t> all(n_in ? ts_in : dflt, n_in ? ts_in + n_in : dflt + n_dflt);
    if (all.empty() || all.size() > FC_MAX_TILE_LEVELS) return fail(FC_ERR_INVALID, "bad tile size count");
    for (size_t i = 0; i < all.size(); ++i) {
        if (all[i] == 0) return fail(FC_ERR_INVALID, "tile size 0");
        if (i && (all[i - 1] <= all[i] || all[i - 1] % all[i]))
            return fail(FC_ERR_INVALID, "tile sizes must decrease and divide each other");
    }
    size_t pos = all.size();
    for (size_t i = 0; i < all.size(); ++i) if (all[i] < max_size) { pos = i; break; }
    size_t start = pos ? pos - 1 : 0;
    ts.assign(all.begin() + start, all.end());
    return FC_OK;
}

struct AxisMap { int x, y, z; };
static AxisMap axes_of(const fc_tape* t) { return AxisMap{t->ax[0], t->ax[1], t->ax[2]}; }

// ShapeVars: every non-axis input slot needs a value (MissingVar otherwise, shape/mod.rs:586-600)
int32_t bind_vars(const fc_tape* t, const float* values, uint32_t n_values, VarBind& vb) {
    AxisMap ax = axes_of(t);
    vb.x = ax.x; vb.y = ax.y; vb.z = ax.z;
    if (t->info.n_vars > uint32_t(MAX_RENDER_VARS)) return fail(FC_ERR_UNSUPPORTED, "renderers support at most 16 input variables");
    for (int i = 0; i < MAX_RENDER_VARS; ++i) vb.values[i] = 0.0f;
    for (uint32_t i = 0; i < t->info.n_vars; ++i) {
        if (int(i) == ax.x || int(i) == ax.y || int(i) == ax.z) continue;
        if (i >= n_values) return fail(FC_ERR_INVALID, "missing value for bound variable in input slot " + std::to_string(i));
        vb.values[i] = values[i];
    }
    return FC_OK;
}

cudaEvent_t get_event(fc_ctx* c, size_t i) {
    while (c->events.size() <= i) {
        cudaEvent_t ev;
        cudaEventCreate(&ev);
        c->events.push_back(ev);
    }
    return c->events[i];
}

// Tile interleave of the multi-GPU renders: the XY root tiles (tx, ty) of the band with
// tile_owner(tx, ty, stride) == offset, in row-major order, as ids (ty - row0) * roots_x + tx.
static void owned_tiles(uint32_t roots_x, uint32_t row0, uint32_t row1, uint32_t stride, uint32_t offset,
                        std::vector<uint32_t>& ids) {
    ids.clear();
    for (uint32_t ty = row0; ty < row1; ++ty)
        for (uint32_t tx = 0; tx < roots_x; ++tx)
            if (tile_owner(tx, ty, stride) == offset) ids.push_back((ty - row0) * roots_x + tx);
}
int32_t root_subset(fc_ctx* c, uint32_t roots_x, uint32_t row0, uint32_t row1, uint32_t stride, uint32_t offset,
                    cudaStream_t s, const uint32_t** d_list, uint32_t* n) {
    const uint32_t key[5] = {roots_x, row0, row1, stride, offset};
    if (memcmp(key, c->root_list_key, sizeof key) != 0 || !c->root_list.p) {
        std::vector<uint32_t> ids;
        owned_tiles(roots_x, row0, row1, stride, offset, ids);
        CU(cudaStreamSynchronize(s));   // a previous launch may still read the old list
        CU(c->root_list.ensure(std::max<size_t>(ids.size(), 1) * 4));
        if (!ids.empty()) CU(cudaMemcpy(c->root_list.p, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice));
        memcpy(c->root_list_key, key, sizeof key);
        c->root_list_n = uint32_t(ids.size());
    }
    *d_list = c->root_list.as<uint32_t>();
    *n = c->root_list_n;
    return FC_OK;
}

// Job and fill lists of a 2D render whose tile grid has n_roots root tiles: level_tiles[l] = worst-case jobs queued for
// level l (tiles of edge ts[l - 1]), which is also the worst case of the fill records level l - 1 writes
static int32_t size_lists_2d(const std::vector<uint32_t>& ts, uint64_t n_roots, std::vector<uint64_t>& level_tiles) {
    const int L = int(ts.size());
    level_tiles.assign(L + 1, 0);
    for (int l = 1; l <= L; ++l) {
        uint64_t per_root = uint64_t(ts[0] / ts[l - 1]) * (ts[0] / ts[l - 1]);
        level_tiles[l] = n_roots * per_root;
        if (level_tiles[l] > 0xfffffff0ull) return fail(FC_ERR_UNSUPPORTED, "image too large for 32-bit tile lists");
    }
    return FC_OK;
}

// The placements of a scene pass grouped by tape for level 0, which runs once per distinct tape with that tape's
// schedule: each group's placements are appended to `pl` (first: the group's offset there), groups in order of first
// appearance along `order`
struct SceneGroup { const fc_tape* tape; uint32_t first, n; };
static void group_by_tape(const fc_tape* const* tapes, const std::vector<uint32_t>& order, std::vector<uint32_t>& pl,
                          std::vector<SceneGroup>& groups) {
    for (size_t i = 0; i < order.size(); ++i) {
        const fc_tape* t = tapes[order[i]];
        bool seen = false;
        for (const SceneGroup& gr : groups) seen |= gr.tape == t;
        if (seen) continue;
        const uint32_t first = uint32_t(pl.size());
        for (size_t q = i; q < order.size(); ++q)
            if (tapes[order[q]] == t) pl.push_back(order[q]);
        groups.push_back(SceneGroup{t, first, uint32_t(pl.size()) - first});
    }
}

// The tile pipeline of fc_render2d (pixel::render), enqueued on `s`: the interval levels, the fills of every level
// (on the auxiliary stream, joined back into `s`) and the leaf pixels, into the distance image `dimg`.  The grid is
// roots_x x roots_y root tiles from root row row0 (or the listed ones, d_roots); with a frame table it stacks the
// frames of a batch (frame_rows grid rows each), else it is the one frame of vb / cfg->mat / cfg->z.  The caller has
// sized the scratch and zeroed the counters (and stats).
struct Tiles2D {
    std::vector<uint32_t> ts;
    uint32_t roots_x = 0, roots_y = 0, row0 = 0;
    const uint32_t* d_roots = nullptr;
    uint32_t n_list = 0;
    uint64_t n_roots = 0;
    std::vector<uint64_t> level_tiles;
    uint32_t choice_words = 0;
    int grid_blocks = 0;
    const Frame2D* frames = nullptr;
    uint32_t frame_rows = 0xffffffffu;
    // scene (fc_render2d_scene): `frames` is the placement table and roots_x x roots_y the grid of one placement.  Level
    // 0 runs once per group (placements listed at d_pl), every later launch is shared.  No image: inside tiles go to the
    // cover maps (read map, then write map, blocks_x x blocks_y each), inside leaf pixels to the key map (Scene2D)
    bool scene = false;
    std::vector<SceneGroup> groups;
    const uint32_t* d_pl = nullptr;
    uint32_t* cover = nullptr;
    uint32_t* key = nullptr;
    uint32_t blocks_x = 0, blocks_y = 0;
};
static int32_t enqueue_tiles_2d(fc_ctx* c, const fc_tape* tape, const fc_render2d_cfg* cfg, const Tiles2D& g,
                                const VarBind& vb, float* dimg, bool want_stats, bool timing, const CallCancel& cc,
                                cudaStream_t s, size_t& ev, uint32_t& launches, bool& fused_out) {
    const std::vector<uint32_t>& ts = g.ts;
    const int L = int(ts.size());
    const bool serial_fill = env_int("FIDGET_B200_SERIAL_FILL", 0) != 0;
    if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    if (++c->epoch == 0) c->epoch = 1;
    // experimental (FC_FLAG_FUSED_TAIL): every level after the root level, the leaf pixels and the fills as ONE
    // persistent launch draining a job queue (tail2d.cu); the default is one launch per stage
    const bool fused = !g.frames && L >= 2 && L - 1 <= TAIL_MAX_LEVELS &&
                       ((cfg->flags & FC_FLAG_FUSED_TAIL) || env_int("FIDGET_B200_FUSE", 0));
    fused_out = fused;
    Tail2DParams tail{};
    for (int l = 0; l < L; ++l) {
        LevelParams p{};
        p.level = l;
        p.epoch = c->epoch;
        p.tile = ts[l];
        p.n_axis = l ? ts[l - 1] / ts[l] : 0;
        p.is_last = (l == L - 1);
        p.pixel_perfect = cfg->pixel_perfect;
        p.root_mode = (l == 0);
        p.roots_x = g.roots_x; p.roots_y = g.roots_y; p.roots_z = 1;
        p.root_x0 = 0; p.root_y0 = g.row0 * ts[0]; p.root_z0 = 0;
        p.root_list = g.d_roots; p.n_root_list = g.n_list;
        p.root_tape = tape_ref(tape);
        p.width = cfg->width; p.height = cfg->height; p.depth = 1;
        p.z2d = cfg->z;
        memcpy(p.mat.m, cfg->mat, sizeof p.mat.m);
        p.jobs_in = l ? c->jobs[l].as<TileJob>() : nullptr;
        p.cap_in = l ? uint32_t(g.level_tiles[l]) : 0;
        p.jobs_out = c->jobs[l + 1].as<TileJob>();
        p.cap_out = uint32_t(g.level_tiles[l + 1]);
        p.fills = c->fills[l].as<FillRec>();
        p.cap_fills = uint32_t(g.level_tiles[l + 1]);
        p.arena = c->arena.as<uint2>();
        p.arena_cap = arena_clauses(c);
        p.choice_scratch = c->choice_scratch.as<uint32_t>();
        p.choice_words = g.choice_words;
        p.ctr = c->counters.as<Counters>();
        p.stats = want_stats ? c->stats.as<Stats>() : nullptr;
        p.vb = vb;
        p.cancel = cc.ref;
        p.frames = g.frames;
        p.frame_rows = g.frame_rows;
        p.fused_tail = fused;
        if (g.scene) {
            p.scene = 1;
            p.occl = g.cover;
            p.occl_w = g.blocks_x;
            p.occl_h = g.blocks_y;
            p.cull = ts[L - 1];
        }
        if (fused) {
            tail.fill_tile[l] = ts[l];
            tail.fills[l] = c->fills[l].as<FillRec>();
            tail.fill_cap[l] = uint32_t(g.level_tiles[l + 1]);
            if (l) { tail.lv[l - 1] = p; continue; }
        }
        auto launch = [&](const fc_tape* t, uint64_t n_roots) -> int32_t {
            // no more warps than the list can hold jobs (one warp per job; level 0: per 32 root tiles)
            const uint64_t warps = l ? g.level_tiles[l] : (n_roots + 31) / 32;
            const int blocks = int(std::min<uint64_t>((warps + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, uint64_t(g.grid_blocks)));
            bool coop = false;
            if (l == 0) {
                int ct = COOP_THREADS;
                int cb = coop_blocks(c, t, n_roots, p, 2, ct);
                if (cb > 0) {
                    CU(launch_interval_root_coop_2d(p, cb, ct, s));
                    coop = true;
                }
            }
            if (!coop) launch_interval_level_2d(p, std::max(blocks, 1), s);
            ++launches;
            // a scene's later launches cull against what this one proved inside: its write map becomes the read map
            if (g.scene)
                CU(cudaMemcpyAsync(g.cover, g.cover + size_t(g.blocks_x) * g.blocks_y, size_t(g.blocks_x) * g.blocks_y * 4,
                                   cudaMemcpyDeviceToDevice, s));
            return FC_OK;
        };
        if (l == 0 && g.scene) {
            // level 0 of a scene: one launch per distinct tape over the root tiles of its placements, as in a 3D scene
            for (size_t k = 0; k < g.groups.size(); ++k) {
                const SceneGroup& gr = g.groups[k];
                p.root_tape = tape_ref(gr.tape);
                p.scene_pl = g.d_pl + gr.first;
                p.n_scene_pl = gr.n;
                if (k) CU(cudaMemsetAsync(&c->counters.as<Counters>()->cursor[0], 0, sizeof(uint32_t), s));
                if (int32_t lrc = launch(gr.tape, uint64_t(g.roots_x) * g.roots_y * gr.n)) return lrc;
            }
        } else if (int32_t lrc = launch(tape, g.n_roots)) {
            return lrc;
        }
        if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
        if (!fused && !g.scene) {
            // the tiles this level proved inside/outside are painted on a second stream while the
            // next (latency-bound) levels run: fills and leaf pixels never touch the same pixel
            FillParams f{};
            f.tile = ts[l];
            f.width = cfg->width; f.height = cfg->height;
            f.fills = c->fills[l].as<FillRec>();
            f.n_fills = &c->counters.as<Counters>()->n_fills[l];
            f.out = dimg;
            f.cancel = cc.ref;
            f.frame_rows = g.frame_rows;
            cudaStream_t fs = serial_fill ? s : c->aux_stream;
            if (!serial_fill) {
                CU(cudaEventRecord(c->ev_fork[l], s));
                CU(cudaStreamWaitEvent(c->aux_stream, c->ev_fork[l], 0));
            }
            launch_fill_2d(f, c->sm_count * 2, fs);
            ++launches;
        }
    }
    if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    {
        PixelParams q{};
        q.tile = ts[L - 1];
        q.width = cfg->width; q.height = cfg->height;
        q.z2d = cfg->z;
        memcpy(q.mat.m, cfg->mat, sizeof q.mat.m);
        q.jobs = c->jobs[L].as<TileJob>();
        q.out = dimg;
        q.ctr = c->counters.as<Counters>();
        q.list = L;
        q.cursor = L;
        q.stats = want_stats ? c->stats.as<Stats>() : nullptr;
        q.vb = vb;
        q.cancel = cc.ref;
        q.frames = g.frames;
        q.frame_rows = g.frame_rows;
        if (fused) {
            tail.n_levels = L - 1;
            tail.px = q;
            tail.epoch = c->epoch;
            tail.cancel = cc.ref;
            tail.paint_fills = env_int("FIDGET_B200_TAIL_PAINTS", 0) ? 1 : 0;
            auto paint = [&](int l, cudaStream_t fs) {
                FillParams f{};
                f.tile = ts[l];
                f.width = cfg->width; f.height = cfg->height;
                f.fills = c->fills[l].as<FillRec>();
                f.n_fills = &c->counters.as<Counters>()->n_fills[l];
                f.out = dimg;
                f.cancel = cc.ref;
                f.frame_rows = g.frame_rows;
                launch_fill_2d(f, c->sm_count * 2, fs);
                ++launches;
            };
            if (!tail.paint_fills) {   // level-0 fills are final already: paint them beside the tail
                CU(cudaEventRecord(c->ev_fork[0], s));
                CU(cudaStreamWaitEvent(c->aux_stream, c->ev_fork[0], 0));
                paint(0, c->aux_stream);
            }
            CU(launch_tail_2d(tail, c->sm_count, s));
            if (!tail.paint_fills) {
                for (int l = 1; l < L; ++l) paint(l, s);
                CU(cudaEventRecord(c->ev_join, c->aux_stream));
                CU(cudaStreamWaitEvent(s, c->ev_join, 0));
            }
        } else if (g.scene) {
            ScenePixelParams sq;
            static_cast<PixelParams&>(sq) = q;
            sq.cover = g.cover;
            sq.key = g.key;
            sq.blocks_x = g.blocks_x;
            sq.blocks_y = g.blocks_y;
            launch_pixels_2d_scene(sq, c->sm_count * env_int("FIDGET_B200_PIXEL_BLOCKS_PER_SM", 8), s);
        } else {
            launch_pixels_2d(q, c->sm_count * env_int("FIDGET_B200_PIXEL_BLOCKS_PER_SM", 8), s);
        }
        ++launches;
    }
    if (!serial_fill && !fused && !g.scene) {
        CU(cudaEventRecord(c->ev_join, c->aux_stream));
        CU(cudaStreamWaitEvent(s, c->ev_join, 0));
    }
    if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    CU(cudaGetLastError());
    return FC_OK;
}

// FC_FLAG_TIMING: stage times of the passes whose events start at `first` (L + 3 events per pass), added to `stage_ms`
static void add_stage_ms_2d(fc_ctx* c, size_t first, int L, bool fused, const Stats& h, float* stage_ms) {
    float ms = 0;
    const cudaEvent_t* e = c->events.data() + first;
    if (fused) {   // [0] = root level, [12] = the fused tail (levels 1.., leaf pixels, fills)
        cudaEventElapsedTime(&ms, e[0], e[1]);
        stage_ms[0] += ms;
        cudaEventElapsedTime(&ms, e[1], e[3]);
        stage_ms[12] += ms;
        // when the last job of each list finished inside the fused launch (device clock, ms after its first warp):
        // [1 .. L-1] interval levels, [L] leaf tiles, [13] level-0 fills .. (statistics of the experiment)
        if (h.culled[0]) {
            for (int k = 1; k <= 2 * (L - 1) + 2 && k < 8; ++k)
                stage_ms[k] = h.culled[k] > h.culled[0] ? float(double(h.culled[k] - h.culled[0]) * 1e-6) : 0.0f;
            // [8], [9]: latest start of a level-1 / level-2 job; [10], [11]: the longest such job
            for (int k = 8; k <= 9; ++k)
                stage_ms[k] = h.culled[k] > h.culled[0] ? float(double(h.culled[k] - h.culled[0]) * 1e-6) : 0.0f;
            stage_ms[10] = float(double(h.culled[10]) * 1e-6);
            stage_ms[11] = float(double(h.culled[11]) * 1e-6);
        }
        cudaEventElapsedTime(&ms, e[0], e[3]);
        stage_ms[15] += ms;
    } else {
        for (int l = 0; l < L; ++l) {
            cudaEventElapsedTime(&ms, e[l], e[l + 1]);
            stage_ms[l] += ms;
        }
        cudaEventElapsedTime(&ms, e[L], e[L + 1]);
        stage_ms[8] += ms;
        cudaEventElapsedTime(&ms, e[L + 1], e[L + 2]);
        stage_ms[9] += ms;
        cudaEventElapsedTime(&ms, e[0], e[L + 2]);
        stage_ms[15] += ms;
    }
}

// A call's fc_render_stats: the census and pixels of `h`, its grads (the 3D renders only), the arena high-water mark
// in clauses and the launch count; stage_ms starts at zero for the caller to add to
static void write_stats(fc_render_stats* stats, const Stats& h, bool grads, unsigned long long arena_top, uint32_t launches) {
    memset(stats, 0, sizeof *stats);
    for (int l = 0; l < FC_MAX_TILE_LEVELS; ++l) {
        stats->evaluated[l] = h.evaluated[l];
        stats->filled_inside[l] = h.filled_inside[l];
        stats->filled_outside[l] = h.filled_outside[l];
        stats->ambiguous[l] = h.ambiguous[l];
        stats->simplified[l] = h.simplified[l];
    }
    stats->pixels = h.pixels;
    if (grads) stats->grads = h.grads;
    stats->arena_bytes_used = arena_top * sizeof(uint2);
    stats->kernel_launches = launches;
}

// Frame `f` of a batch (fc_frame2d, fc_frame3d or a scene placement) as the kernels read it: its matrix, Z and
// ShapeVars binding for `tape`
template <class F>
static int32_t bind_frame(const fc_tape* tape, const F& f, float z, Frame2D& out) {
    if (f.n_var_values > FC_MAX_VARS) return fail(FC_ERR_INVALID, "n_var_values above FC_MAX_VARS");
    memcpy(out.mat.m, f.mat, sizeof out.mat.m);
    out.z = z;
    return bind_vars(tape, f.var_values, f.n_var_values, out.vb);
}

// the tapes no renderer takes
static int32_t check_render_tape(const fc_tape* tape) {
    if (tape->info.mem_count) return fail(FC_ERR_UNSUPPORTED, "renderers need a tape without memory spills (<= 255 registers)");
    if (tape->info.n_outputs != 1) return fail(FC_ERR_INVALID, "ShapeTape has multiple outputs");
    return FC_OK;
}

// The settings of fc_render2d that the 2D batches refuse; `what` names the batch ("frame batches", "scenes")
static int32_t check_batch_2d(const fc_render2d_cfg* cfg, const std::string& what) {
    if (cfg->flags & FC_FLAG_FUSED_TAIL) return fail(FC_ERR_UNSUPPORTED, "FC_FLAG_FUSED_TAIL is not supported by " + what);
    if (cfg->root_row_begin || cfg->root_row_end) return fail(FC_ERR_UNSUPPORTED, "root row bands are not supported by " + what);
    if (cfg->root_stride > 1) return fail(FC_ERR_UNSUPPORTED, "the tile interleave is not supported by " + what);
    if (cfg->out_format > FC_OUT_RGBA8) return fail(FC_ERR_INVALID, "unknown out_format");
    return FC_OK;
}

// Validation and tile grid shared by fc_render2d and fc_render2d_frames
static int32_t check_2d(const fc_tape* tape, const fc_render2d_cfg* cfg) {
    if (cfg->width == 0 || cfg->height == 0) return fail(FC_ERR_INVALID, "empty image");
    return check_render_tape(tape);
}
static int32_t prepare_2d(fc_ctx* c, const fc_tape* tape, const fc_render2d_cfg* cfg, Tiles2D& g) {
    static const uint32_t DFLT[3] = {128, 32, 8};
    if (int32_t rc = pick_tile_sizes(cfg->tile_sizes, cfg->n_tile_sizes, DFLT, 3, std::max(cfg->width, cfg->height), g.ts))
        return rc;
    g.roots_x = (cfg->width + g.ts[0] - 1) / g.ts[0];
    // 8 CTAs per SM: a list longer than the grid (prospero 4096^2, level 2: 5520 jobs) ends sooner the more warps share
    // it (0.066 ms at 8, 0.071 at 6, 0.079 at 4 on H100), and a short list no longer pays for the grid's idle warps
    // (enqueue_tiles_2d caps a level's grid by its list's capacity)
    const int bps = env_int("FIDGET_B200_BLOCKS_PER_SM", 8);
    g.grid_blocks = c->sm_count * bps;
    g.choice_words = choice_words(tape);
    return FC_OK;
}
// scratch of a pipeline over n_roots root tiles (level_tiles sized by the caller)
static int32_t ensure_scratch_2d(fc_ctx* c, const Tiles2D& g) {
    const int L = int(g.ts.size());
    CU(c->choice_scratch.ensure(size_t(std::max(g.grid_blocks, tail_2d_blocks(c->sm_count))) * WARPS_PER_BLOCK * g.choice_words * 32 * 4));
    CU(c->arena.ensure(c->arena_bytes));
    CU(c->counters.ensure(sizeof(Counters)));
    CU(c->stats.ensure(sizeof(Stats)));
    for (int l = 1; l <= L; ++l) {
        CU(c->jobs[l].ensure(g.level_tiles[l] * sizeof(TileJob)));
        if (!g.scene) CU(c->fills[l - 1].ensure(g.level_tiles[l] * sizeof(FillRec)));   // (a scene writes no fills)
    }
    return FC_OK;
}

// bytes of one image of `fmt` (FC_OUT_*)
static size_t format_bytes(uint32_t fmt, uint32_t width, uint32_t height) {
    return fmt == FC_OUT_MASK_U8 ? size_t(width) * height
         : fmt == FC_OUT_BITMAP_1BIT ? size_t((width + 7) / 8) * height
         : size_t(width) * height * 4;
}
// ---- passes of the frame batches (fc_render2d_frames, fc_render3d_frames) ----
// The copy stream that returns a pass's images to a host `out` while the next pass runs, with two event pairs
// (ev_pass[b]: the pass in staging buffer b is complete; ev_copied[b]: its images are copied back)
static int32_t ensure_copy_stream(fc_ctx* c) {
    if (c->copy_stream) return FC_OK;
    CU(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        CU(cudaEventCreateWithFlags(&c->ev_pass[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming));
    }
    return FC_OK;
}
// Orders the copy stream after the pass in buffer b.  With a flag attached the host waits for that pass here, watching
// the flag (wait_call writes the cancel word the kernels of this pass and the next one poll): a copy into pageable
// memory blocks the host until it is done, and a blocked host could not cancel anything.  `host_wait`: the host waits
// without a flag too (it reads the pass's status next).  A cancelled pass returns FC_ERR_CANCELLED.
static int32_t wait_pass(fc_ctx* c, int b, const CallCancel& cc, bool host_wait) {
    CU(cudaStreamWaitEvent(c->copy_stream, c->ev_pass[b], 0));
    if (cc.flag) return wait_call(c, c->copy_stream, cc);
    if (host_wait) CU(cudaStreamSynchronize(c->copy_stream));
    return FC_OK;
}
// the images of the pass in staging buffer b back to the host, on the copy stream; ev_copied[b] marks b free again
static int32_t copy_pass_back(fc_ctx* c, int b, void* dst, const void* src, size_t bytes) {
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->copy_stream));
    CU(cudaEventRecord(c->ev_copied[b], c->copy_stream));
    return FC_OK;
}
// a batch that stops early (cancelled, or an error) returns once its launched work has drained, stats zeroed
static int32_t abandon_frames(fc_ctx* c, cudaStream_t s, fc_render_stats* stats, int32_t rc) {
    cudaStreamSynchronize(s);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    if (stats) memset(stats, 0, sizeof *stats);
    return rc;
}

// ---- passes of the 2D batches (fc_render2d_frames: frames; fc_render2d_scene: shapes) ----
// Items per pass: an item's worst-case lists over its n_roots root tiles, at job_bytes per job, plus its extra_bytes,
// within FC_FRAMES_PASS_BYTES (at least one item); FIDGET_B200_FRAMES_PER_PASS forces the count
static int32_t passes_2d(const std::vector<uint32_t>& ts, uint64_t n_roots, uint32_t n_items, uint64_t job_bytes,
                         uint64_t extra_bytes, uint32_t& per_pass, uint32_t& n_passes) {
    std::vector<uint64_t> item_tiles;
    if (int32_t rc = size_lists_2d(ts, n_roots, item_tiles)) return rc;
    uint64_t per_item = extra_bytes;
    for (size_t l = 1; l < item_tiles.size(); ++l) per_item += item_tiles[l] * job_bytes;
    per_pass = uint32_t(std::min<uint64_t>(n_items, std::max<uint64_t>(1, FC_FRAMES_PASS_BYTES / per_item)));
    if (const int forced = env_int("FIDGET_B200_FRAMES_PER_PASS", 0); forced > 0) per_pass = std::min<uint32_t>(n_items, forced);
    n_passes = (n_items + per_pass - 1) / per_pass;
    return FC_OK;
}
// a new pass: fresh lists, cursors and arena; error bits accumulate over the call
static int32_t reset_pass_2d(fc_ctx* c, cudaStream_t s) {
    CU(cudaMemsetAsync(c->counters.p, 0, offsetof(Counters, error), s));
    CU(cudaMemsetAsync(&c->counters.as<Counters>()->arena_top, 0, sizeof(unsigned long long), s));
    return FC_OK;
}
// pass k's arena high-water mark, into frame_tops[k] for the call's stats
static int32_t record_top_2d(fc_ctx* c, cudaStream_t s, uint32_t k) {
    CU(cudaMemcpyAsync(c->frame_tops.as<unsigned long long>() + k, &c->counters.as<Counters>()->arena_top,
                       sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s));
    return FC_OK;
}
// With a flag attached, the wait that ends a 2D batch that enqueued passes_run of its n_passes passes: FC_ERR_CANCELLED,
// stats zeroed, if the flag cancelled it
static int32_t wait_cancel_2d(fc_ctx* c, cudaStream_t s, const CallCancel& cc, uint32_t passes_run, uint32_t n_passes,
                              fc_render_stats* stats) {
    if (!cc.flag) return FC_OK;
    int32_t rc = wait_call(c, s, cc);
    // (passes_run < n_passes: the flag stopped the passes, but was cleared before the wait saw it)
    if (!rc && passes_run < n_passes) rc = fail(FC_ERR_CANCELLED, "cancelled");
    if (rc && stats) memset(stats, 0, sizeof *stats);
    return rc;
}
// The end of a 2D batch of n_passes passes (L + 3 timing events each): the device's error bits and the stats, with the
// largest arena high-water mark of frame_tops
static int32_t finish_2d(fc_ctx* c, cudaStream_t s, int L, uint32_t n_passes, bool timing, uint32_t launches,
                         fc_render_stats* stats) {
    CU(cudaStreamSynchronize(s));
    int32_t rc = check_device_errors(c);
    if (stats) {
        Stats h;
        std::vector<unsigned long long> tops(n_passes);
        CU(cudaMemcpy(&h, c->stats.p, sizeof h, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(tops.data(), c->frame_tops.p, tops.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        write_stats(stats, h, false, *std::max_element(tops.begin(), tops.end()), launches);
        if (timing)
            for (uint32_t k = 0; k < n_passes; ++k) add_stage_ms_2d(c, size_t(k) * (L + 3), L, false, h, stats->stage_ms);
    }
    return rc;
}

// the small formats, derived on the device from `rows` rows of distance image
static void derive_format(uint32_t fmt, const float* dimg, uint32_t width, uint32_t rows, uint8_t* dst, cudaStream_t s) {
    if (fmt == FC_OUT_RGBA8) launch_to_rgba(0, dimg, uint64_t(width) * rows, dst, s);
    else launch_to_mask(dimg, width, rows, dst, fmt == FC_OUT_BITMAP_1BIT, s);
}

// The tile grid of a 3D render (fc_render3d, fc_render3d_frames): the device's tile ladder, roots_x x roots_y x
// roots_z root tiles from root row row0 and Z z_begin (or the listed XY ones, d_roots), the capped work lists, the
// occlusion map and the exact census.  With a frame table the grid stacks the frames of a batch (frame_rows grid rows
// each; heightmap and occlusion map hold frame_rows rows per frame), else it is the one frame of vb / cfg->mat.
struct Tiles3D {
    std::vector<uint32_t> ts;
    uint32_t roots_x = 0, roots_y = 0, roots_z = 0, row0 = 0, z_begin = 0;
    const uint32_t* d_roots = nullptr;
    uint32_t n_list = 0;
    uint64_t n_roots = 0;
    std::vector<uint64_t> level_cap;
    uint64_t cap_census = 0;
    uint32_t choice_words = 0;
    int grid_blocks = 0, grid_blocks_last = 0;
    bool use_occl = false, exact_census = false;
    uint32_t occl_w = 0, occl_h = 0;    // occlusion blocks per row, block rows of one frame
    const Frame2D* frames = nullptr;
    uint32_t frame_rows = 0xffffffffu;
    // scene (fc_render3d_scene): `frames` is the placement table; a pass renders placements pl0 .. pl1 - 1, listed at
    // d_pl grouped by tape (level 0 runs once per group, with the group's tape); clamp_at as in scene_rank
    bool scene = false;
    std::vector<SceneGroup> groups;
    const uint32_t* d_pl = nullptr;
    uint32_t pl0 = 0, pl1 = 0, clamp_at = 0xffffffffu;
};

static int32_t check_3d(const fc_tape* tape, const fc_render3d_cfg* cfg) {
    if (cfg->width == 0 || cfg->height == 0 || cfg->depth == 0) return fail(FC_ERR_INVALID, "empty volume");
    return check_render_tape(tape);
}
// The settings of fc_render3d that the 3D batches refuse; `what` names the batch ("frame batches", "scenes")
static int32_t check_batch_3d(const fc_render3d_cfg* cfg, const std::string& what) {
    if (cfg->z_begin || cfg->z_end) return fail(FC_ERR_UNSUPPORTED, "Z slabs are not supported by " + what);
    if (cfg->root_row_begin || cfg->root_row_end) return fail(FC_ERR_UNSUPPORTED, "root row bands are not supported by " + what);
    if (cfg->root_stride > 1) return fail(FC_ERR_UNSUPPORTED, "the tile interleave is not supported by " + what);
    return FC_OK;
}
// tile ladder, launch widths, choice scratch words and the occlusion map's shape
static int32_t prepare_3d(fc_ctx* c, const fc_tape* tape, const fc_render3d_cfg* cfg, Tiles3D& g) {
    static const uint32_t DFLT[5] = {128, 64, 32, 16, 8};
    std::vector<uint32_t>& ts = g.ts;
    if (int32_t rc = pick_tile_sizes(cfg->tile_sizes, cfg->n_tile_sizes, DFLT, 5, std::max(cfg->width, cfg->height), ts))
        return rc;
    if (cfg->n_tile_sizes == 0 && !(cfg->flags & (FC_FLAG_FULL_LADDER | FC_FLAG_EXACT_CENSUS)) &&
        !env_int("FIDGET_B200_FULL_LADDER", 0)) {
        // Device ladder: every other size of the default one.  A warp then carries 32 children per pass instead of 8
        // and a whole level of launches, job records and tape writes disappears; the image cannot change, because a
        // child's interval result on its grandparent's tape equals the one on its parent's simplified tape (a choice
        // the parent's region decided is decided the same way on any sub-region, and the pruned branch never
        // contributed to the value) -- tests/test_gpu_parity.py compares the two ladders bit for bit.
        std::vector<uint32_t> fused(1, ts[0]);
        for (size_t i = 0; i + 1 < ts.size();) {
            const size_t nx = std::min(i + 2, ts.size() - 1);
            fused.push_back(ts[nx]);
            i = nx;
        }
        ts.swap(fused);
    }
    g.roots_x = (cfg->width + ts[0] - 1) / ts[0];
    // persistent CTAs per SM: 6 for the upper levels, 8 for the last one (many short jobs; measured on prospero and bear:
    // last level 1.10 -> 0.97 ms and 0.72 -> 0.61 ms, the level before it is fastest at 6)
    const int bps = env_int("FIDGET_B200_BLOCKS_PER_SM", 6);
    const int bps_last = std::max(bps, env_int("FIDGET_B200_LAST_LEVEL_BLOCKS_PER_SM", 8));
    g.grid_blocks = c->sm_count * bps;
    g.grid_blocks_last = c->sm_count * bps_last;
    g.choice_words = choice_words(tape);
    // occlusion map (16 x 16 pixel blocks); used when every tile size down to 16 is a multiple of 16
    g.occl_w = (cfg->width + 15) / 16;
    g.occl_h = (cfg->height + 15) / 16;
    g.use_occl = !env_int("FIDGET_B200_NO_CULL", 0);
    for (uint32_t t : ts) if (t >= 16 && t % 16) g.use_occl = false;
    g.exact_census = (cfg->flags & FC_FLAG_EXACT_CENSUS) != 0;
    return FC_OK;
}
// Job lists capped at list_cap_limit(); the exact census is capped at 64 Mi records
static void size_lists_3d(Tiles3D& g) {
    const std::vector<uint32_t>& ts = g.ts;
    const int L = int(ts.size());
    const uint64_t cap_limit = list_cap_limit();
    g.level_cap.assign(L + 1, 0);
    for (int l = 1; l <= L; ++l) {
        const uint64_t r = ts[0] / ts[l - 1];
        g.level_cap[l] = std::min<uint64_t>(g.n_roots * r * r * r, cap_limit);
    }
    g.cap_census = 0;
    if (g.exact_census) {
        g.cap_census = g.n_roots;
        for (int l = 1; l < L; ++l) { const uint64_t r = ts[l - 1] / ts[l]; g.cap_census += g.level_cap[l] * r * r * r; }
        g.cap_census = std::min<uint64_t>(g.cap_census, 64ull << 20);
    }
}
static uint32_t zsort_layers(const Tiles3D& g) { return (g.roots_z * g.ts[0]) / g.ts.back(); }
// scratch of a pipeline over g's lists (the z-sort's too), with heightmap pixels and occlusion blocks for hm_pixels /
// occl_blocks.  A batch sizes it for its largest pass before it enqueues any, so no pass reallocates a buffer.
static int32_t ensure_scratch_3d(fc_ctx* c, const Tiles3D& g, size_t hm_pixels, size_t occl_blocks) {
    const int L = int(g.ts.size());
    CU(c->choice_scratch.ensure(size_t(g.grid_blocks_last) * WARPS_PER_BLOCK * g.choice_words * 32 * 4));
    CU(c->arena.ensure(c->arena_bytes));
    CU(c->counters.ensure(sizeof(Counters)));
    CU(c->stats.ensure(sizeof(Stats)));
    for (int l = 1; l <= L; ++l) CU(c->jobs[l].ensure(g.level_cap[l] * sizeof(TileJob)));
    CU(c->heightmap.ensure(hm_pixels * 8));
    if (g.exact_census) CU(c->census.ensure(g.cap_census * sizeof(CensusRec)));
    if (g.use_occl) CU(c->occl.ensure(occl_blocks * 4));
    if (!env_int("FIDGET_B200_NO_ZSORT", 0)) CU(c->zsort.ensure(size_t(zsort_layers(g) + 1) * 4 + g.level_cap[L] * 4));
    return FC_OK;
}

// The tile pipeline of fc_render3d (voxel::render), enqueued on `s`: the interval levels, the front-to-back sort of
// the leaf tiles, the leaf voxels, the exact census and the normals of output rows y0 .. y1 into `dimg` (a scene pass:
// level 0 once per group of g, and the placement of every pixel it finishes into `index`, if not null).  The caller
// has sized the scratch and zeroed the counters, the heightmap rows, the occlusion map and the stats.
static int32_t enqueue_tiles_3d(fc_ctx* c, const fc_tape* tape, const fc_render3d_cfg* cfg, const Tiles3D& g,
                                const VarBind& vb, void* dimg, uint32_t y0, uint32_t y1, bool want_stats, bool timing,
                                const CallCancel& cc, cudaStream_t s, size_t& ev, uint32_t& launches,
                                uint16_t* index = nullptr) {
    const std::vector<uint32_t>& ts = g.ts;
    const int L = int(ts.size());
    const uint32_t T0 = ts[0];
    if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    for (int l = 0; l < L; ++l) {
        LevelParams p{};
        p.level = l;
        p.tile = ts[l];
        p.n_axis = l ? ts[l - 1] / ts[l] : 0;
        p.is_last = (l == L - 1);
        p.pixel_perfect = 0;
        p.root_mode = (l == 0);
        p.roots_x = g.roots_x; p.roots_y = g.roots_y; p.roots_z = g.roots_z;
        p.root_x0 = 0; p.root_y0 = g.row0 * T0; p.root_z0 = g.z_begin;
        p.root_list = g.d_roots; p.n_root_list = g.n_list;
        p.root_tape = tape_ref(tape);
        p.width = cfg->width; p.height = cfg->height; p.depth = cfg->depth;
        memcpy(p.mat.m, cfg->mat, sizeof p.mat.m);
        p.jobs_in = l ? c->jobs[l].as<TileJob>() : nullptr;
        p.cap_in = l ? uint32_t(g.level_cap[l]) : 0;
        p.jobs_out = c->jobs[l + 1].as<TileJob>();
        p.cap_out = uint32_t(g.level_cap[l + 1]);
        p.arena = c->arena.as<uint2>();
        p.arena_cap = arena_clauses(c);
        p.choice_scratch = c->choice_scratch.as<uint32_t>();
        p.choice_words = g.choice_words;
        p.ctr = c->counters.as<Counters>();
        p.stats = want_stats ? c->stats.as<Stats>() : nullptr;
        p.heightmap = c->heightmap.as<unsigned long long>();
        p.occl = g.use_occl ? c->occl.as<uint32_t>() : nullptr;
        p.occl_w = g.occl_w;
        p.occl_h = g.occl_h;
        p.cull = (g.use_occl && l >= 1 && ts[l - 1] >= 16u && ts[l - 1] <= 64u) ? 1u : 0u;   // parents made of 1, 4 or 16 blocks
        p.census = g.exact_census ? c->census.as<CensusRec>() : nullptr;
        p.cap_census = uint32_t(g.cap_census);
        p.vb = vb;
        p.cancel = cc.ref;
        p.frames = g.frames;
        p.frame_rows = g.frame_rows;
        p.scene = g.scene ? 1u : 0u;
        p.clamp_at = g.clamp_at;
        auto launch = [&](const fc_tape* t, uint64_t n_roots) -> int32_t {
            int blocks = (l == L - 1 && l > 0) ? g.grid_blocks_last : g.grid_blocks;
            if (l == 0) {
                uint64_t warps = (n_roots + 31) / 32;
                blocks = int(std::min<uint64_t>((warps + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, uint64_t(g.grid_blocks)));
            }
            bool coop = false;
            if (l == 0) {
                int ct = COOP_THREADS;
                int cb = coop_blocks(c, t, n_roots, p, 3, ct);
                if (cb > 0) {
                    CU(launch_interval_root_coop_3d(p, cb, ct, s));
                    coop = true;
                }
            }
            if (!coop) launch_interval_level_3d(p, std::max(blocks, 1), s);
            ++launches;
            return FC_OK;
        };
        if (l == 0 && g.scene) {
            // level 0 of a scene: one launch per distinct tape over the root tiles of its placements, each with that
            // tape's schedule; their children go to one shared level-1 list (the claim cursor restarts per launch)
            const uint64_t per = uint64_t(g.roots_x) * g.roots_y * g.roots_z;
            for (size_t k = 0; k < g.groups.size(); ++k) {
                const SceneGroup& gr = g.groups[k];
                p.root_tape = tape_ref(gr.tape);
                p.scene_pl = g.d_pl + gr.first;
                p.n_scene_pl = gr.n;
                if (k) CU(cudaMemsetAsync(&c->counters.as<Counters>()->cursor[0], 0, sizeof(uint32_t), s));
                if (int32_t lrc = launch(gr.tape, per * gr.n)) return lrc;
            }
        } else if (int32_t lrc = launch(tape, g.n_roots)) {
            return lrc;
        }
        if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    }
    {
        VoxelParams q{};
        q.tile = ts[L - 1];
        if (!env_int("FIDGET_B200_NO_ZSORT", 0)) {
            const uint32_t n_layers = zsort_layers(g);
            uint32_t* hist = c->zsort.as<uint32_t>();
            uint32_t* order = hist + n_layers + 1;
            launch_leaf_zsort(c->jobs[L].as<TileJob>(), &c->counters.as<Counters>()->n_jobs[L], uint32_t(g.level_cap[L]),
                              g.z_begin, ts[L - 1], n_layers, hist, order, s);
            launches += 3;
            q.order = order;
        }
        q.width = cfg->width; q.height = cfg->height;
        memcpy(q.mat.m, cfg->mat, sizeof q.mat.m);
        q.jobs = c->jobs[L].as<TileJob>();
        q.cap_jobs = uint32_t(g.level_cap[L]);
        q.heightmap = c->heightmap.as<unsigned long long>();
        q.ctr = c->counters.as<Counters>();
        q.list = L; q.cursor = L;
        q.stats = want_stats ? c->stats.as<Stats>() : nullptr;
        q.vb = vb;
        q.cancel = cc.ref;
        q.frames = g.frames;
        q.frame_rows = g.frame_rows;
        q.scene = g.scene ? 1u : 0u;
        q.depth = cfg->depth;
        q.clamp_at = g.clamp_at;
        launch_voxels_3d(q, c->sm_count * env_int("FIDGET_B200_VOXEL_BLOCKS_PER_SM", 12), s);
        ++launches;
    }
    if (g.exact_census) {
        // the counts collected so far describe what the device evaluated; replace them by the reference's census,
        // judged against the final heightmap (k_census_3d).  (A frame batch's census needs no frame: its sides are
        // multiples of the root tile, so the frames are stacked without padding rows.)
        Stats* ds = c->stats.as<Stats>();
        CU(cudaMemsetAsync(ds, 0, offsetof(Stats, grads), s));                        // evaluated .. simplified, pixels
        CensusParams cp{};
        cp.recs = c->census.as<CensusRec>();
        cp.n_recs = &c->counters.as<Counters>()->n_census;
        cp.cap = uint32_t(g.cap_census);
        for (int l = 0; l < L; ++l) cp.tile[l] = ts[l];
        cp.last_level = L - 1;
        cp.heightmap = c->heightmap.as<unsigned long long>();
        cp.width = cfg->width;
        cp.stats = ds;
        cp.cancel = cc.ref;
        launch_census_3d(cp, c->sm_count * 8, s);
        ++launches;
    }
    if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    {
        NormalParams q{};
        q.width = cfg->width; q.height = cfg->height; q.depth = cfg->depth;
        q.y0 = y0; q.y1 = y1;
        q.root_list = g.d_roots; q.n_root_list = g.n_list; q.roots_x = g.roots_x; q.root_tile = T0;
        q.clamp = (cfg->flags & FC_FLAG_NO_CLAMP) ? 0 : 1;
        memcpy(q.mat.m, cfg->mat, sizeof q.mat.m);
        q.jobs = c->jobs[L].as<TileJob>();
        q.heightmap = c->heightmap.as<unsigned long long>();
        q.out = dimg;
        q.stats = want_stats ? c->stats.as<Stats>() : nullptr;
        q.vb = vb;
        q.cancel = cc.ref;
        q.frames = g.frames;
        q.frame_rows = g.frame_rows;
        q.scene = g.scene ? 1u : 0u;
        q.pl0 = g.pl0;
        q.pl1 = g.pl1;
        q.index = index;
        q.error = &c->counters.as<Counters>()->error;
        launch_normals_3d(q, s);
        ++launches;
    }
    if (timing) CU(cudaEventRecord(get_event(c, ev++), s));
    CU(cudaGetLastError());
    return FC_OK;
}

// FC_FLAG_TIMING: stage times of the pass whose events start at `first` (L + 3 events), added to `stage_ms`
static void add_stage_ms_3d(fc_ctx* c, size_t first, int L, float* stage_ms) {
    float ms = 0;
    const cudaEvent_t* e = c->events.data() + first;
    for (int l = 0; l < L; ++l) {
        cudaEventElapsedTime(&ms, e[l], e[l + 1]);
        stage_ms[l] += ms;
    }
    cudaEventElapsedTime(&ms, e[L], e[L + 1]);
    stage_ms[9] += ms;
    cudaEventElapsedTime(&ms, e[L + 1], e[L + 2]);
    stage_ms[10] += ms;
    cudaEventElapsedTime(&ms, e[0], e[L + 2]);
    stage_ms[15] += ms;
}

// ---- passes of the 3D batches (fc_render3d_frames: frames; fc_render3d_scene: placements) ----
// The planner (pass_plan.h) of a batch of n_items whose pass of n items is the tile grid grid_of(n), lists and census
// capped.  n_max: FC_FRAMES_PASS_BYTES (at least one item) for its lists, census, z-sort order and item_bytes per item,
// 32-bit root ids and the caller's own limit n_cap.  A list's worst case is every tile of its level queued; the exact
// census counts (as the planner's measured quantity) when it is capped below every tile of every level evaluated.
static PassPlan plan_3d(const fc_ctx* c, const std::function<Tiles3D(uint32_t)>& grid_of, uint32_t n_items,
                        uint64_t item_bytes, uint32_t n_cap) {
    const int L = int(grid_of(1).ts.size());
    auto allowed = [&](uint32_t k) {
        const Tiles3D gp = grid_of(k);
        uint64_t b = uint64_t(k) * item_bytes + gp.level_cap[L] * 4 + gp.cap_census * sizeof(CensusRec);
        for (int l = 1; l <= L; ++l) b += gp.level_cap[l] * sizeof(TileJob);
        return b <= FC_FRAMES_PASS_BYTES && gp.n_roots <= 0xfffffff0ull;
    };
    uint32_t n_max = 1;
    while (n_max < std::min(n_items, n_cap) && allowed(n_max + 1)) ++n_max;
    return PassPlan(n_items, n_max, [c, grid_of, L](uint32_t n) {
        const Tiles3D gp = grid_of(n);
        PassLimits lim;
        lim.arena_cap = arena_clauses(c);
        uint64_t census_worst = gp.n_roots;
        for (int l = 1; l <= L; ++l) {
            const uint64_t r = gp.ts[0] / gp.ts[l - 1];
            lim.cap[l] = gp.level_cap[l];
            lim.worst[l] = gp.n_roots * r * r * r;
            if (l < L) { const uint64_t q = gp.ts[l - 1] / gp.ts[l]; census_worst += gp.level_cap[l] * q * q * q; }
        }
        lim.extra_on = gp.exact_census && gp.cap_census < census_worst;
        lim.extra_cap = gp.cap_census;
        return lim;
    });
}

namespace {
// The stats of a 3D batch, summed over the passes that stand: census, pixels, grads, the largest arena use and
// (FC_FLAG_TIMING) the stage times
struct PassStats {
    Stats total{};
    unsigned long long arena_top = 0;
    float stage_ms[16] = {};
    void add(fc_ctx* c, const PassStatus& ps, bool timing, size_t ev0, int L) {
        for (int l = 0; l < MAX_LEVELS; ++l) {
            total.evaluated[l] += ps.st.evaluated[l];
            total.filled_inside[l] += ps.st.filled_inside[l];
            total.filled_outside[l] += ps.st.filled_outside[l];
            total.ambiguous[l] += ps.st.ambiguous[l];
            total.simplified[l] += ps.st.simplified[l];
        }
        total.pixels += ps.st.pixels;
        total.grads += ps.st.grads;
        arena_top = std::max<unsigned long long>(arena_top, ps.ctr.arena_top);
        if (timing) add_stage_ms_3d(c, ev0, L, stage_ms);
    }
    void write(fc_render_stats* stats, uint32_t launches) const {
        write_stats(stats, total, true, arena_top, launches);
        memcpy(stats->stage_ms, stage_ms, sizeof stage_ms);
    }
};
}  // namespace
// the two pinned slots (one per staging buffer) that a 3D batch reads its passes' status from
static int32_t ensure_pass_pin(fc_ctx* c) {
    if (!c->pass_pin) CU(cudaHostAlloc(reinterpret_cast<void**>(&c->pass_pin), 2 * sizeof(PassStatus), cudaHostAllocDefault));
    return FC_OK;
}
// the finished pass's counters and (want_stats) stats, into pinned slot `slot` on s
static int32_t read_pass_status(fc_ctx* c, cudaStream_t s, int slot, bool want_stats) {
    PassStatus* hs = c->pass_pin + slot;
    CU(cudaMemcpyAsync(&hs->ctr, c->counters.p, sizeof(Counters), cudaMemcpyDeviceToHost, s));
    if (want_stats) CU(cudaMemcpyAsync(&hs->st, c->stats.p, sizeof(Stats), cudaMemcpyDeviceToHost, s));
    return FC_OK;
}

extern "C" {

int32_t fc_render2d(fc_ctx* c, const fc_tape* tape, const fc_render2d_cfg* cfg, float* out, fc_render_stats* stats) {
    if (!c || !tape || !cfg || !out) return fail(FC_ERR_INVALID, "null argument");
    if (int32_t vrc = check_2d(tape, cfg)) return vrc;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    Tiles2D g;
    int32_t rc = prepare_2d(c, tape, cfg, g);
    if (rc) return rc;
    const int L = int(g.ts.size());
    const uint32_t T0 = g.ts[0];
    const uint32_t roots_x = g.roots_x;
    uint32_t roots_y_all = (cfg->height + T0 - 1) / T0;
    uint32_t row0 = cfg->root_row_begin, row1 = cfg->root_row_end ? cfg->root_row_end : roots_y_all;
    if (row0 > row1 || row1 > roots_y_all) return fail(FC_ERR_INVALID, "bad root row band");
    const uint32_t roots_y = row1 - row0;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    const bool async = (cfg->flags & FC_FLAG_ASYNC) != 0;
    const bool want_stats = stats != nullptr;
    cudaStream_t s = c->stream;
    const uint32_t* d_roots = nullptr;
    uint32_t n_list = 0;
    if (cfg->root_stride > 1) {
        if (cfg->root_offset >= cfg->root_stride) return fail(FC_ERR_INVALID, "root_offset must be below root_stride");
        if (!is_device_ptr(out)) return fail(FC_ERR_UNSUPPORTED, "tile-interleaved renders need a device image");
        if (int32_t lrc = root_subset(c, roots_x, row0, row1, cfg->root_stride, cfg->root_offset, s, &d_roots, &n_list)) return lrc;
    }
    g.roots_y = roots_y;
    g.row0 = row0;
    g.d_roots = d_roots;
    g.n_list = n_list;
    g.n_roots = d_roots ? uint64_t(n_list) : uint64_t(roots_x) * roots_y;
    if (int32_t src = size_lists_2d(g.ts, g.n_roots, g.level_tiles)) return src;
    if (int32_t erc = ensure_scratch_2d(c, g)) return erc;
    bool out_dev = is_device_ptr(out);
    float* dimg = out;
    const size_t img_bytes = size_t(cfg->width) * cfg->height * 4;
    const uint32_t fmt = cfg->out_format;
    if (fmt > FC_OUT_RGBA8) return fail(FC_ERR_INVALID, "unknown out_format");
    if (fmt != FC_OUT_F32) {
        // the distance image lives in the context; `out` receives the derived format at the end
        if (cfg->root_stride > 1 || cfg->root_row_begin || cfg->root_row_end)
            return fail(FC_ERR_UNSUPPORTED, "out_format other than FC_OUT_F32 needs a whole-frame render");
        CU(c->image.ensure(img_bytes));
        dimg = c->image.as<float>();
    } else if (!out_dev) {
        void* alias = env_int("FIDGET_B200_ZEROCOPY", 0) ? pinned_device_alias(out) : nullptr;
        if (alias) {
            dimg = static_cast<float*>(alias);   // zero-copy: kernels store straight into the host image
            out_dev = true;
        } else {
            CU(c->image.ensure(img_bytes));
            dimg = c->image.as<float>();
        }
    }
    CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters), s));
    if (want_stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
    // (pixels outside the requested band of root rows are left untouched)

    VarBind vb;
    if (int32_t vrc = bind_vars(tape, cfg->var_values, cfg->n_var_values, vb)) return vrc;
    size_t ev = 0;
    uint32_t launches = 0;
    bool fused = false;
    if (int32_t erc = enqueue_tiles_2d(c, tape, cfg, g, vb, dimg, want_stats, timing, cc, s, ev, launches, fused)) return erc;
    CU(cudaGetLastError());
    const bool early_return = async && out_dev && !want_stats;
    if (cc.flag && !early_return) {   // a cancelled render derives no format and copies nothing to the host
        if (int32_t wrc = wait_call(c, s, cc)) {
            if (stats) memset(stats, 0, sizeof *stats);
            return wrc;
        }
    }
    if (fmt != FC_OUT_F32) {
        const size_t fb = format_bytes(fmt, cfg->width, cfg->height);
        uint8_t* dfmt = reinterpret_cast<uint8_t*>(out);
        if (!out_dev) {
            CU(c->fx_out.ensure(fb));
            dfmt = c->fx_out.as<uint8_t>();
        }
        derive_format(fmt, dimg, cfg->width, cfg->height, dfmt, s);
        ++launches;
        CU(cudaGetLastError());
        if (!out_dev) CU(cudaMemcpyAsync(out, dfmt, fb, cudaMemcpyDeviceToHost, s));
    } else if (!out_dev) {   // only the rows of the requested band are copied back
        const uint32_t by0 = std::min(row0 * T0, cfg->height), by1 = std::min(row1 * T0, cfg->height);
        if (by1 > by0)
            CU(cudaMemcpyAsync(out + size_t(by0) * cfg->width, dimg + size_t(by0) * cfg->width,
                               size_t(by1 - by0) * cfg->width * 4, cudaMemcpyDeviceToHost, s));
    }
    if (early_return) {
        c->async_call = cc;
        return FC_OK;
    }
    CU(cudaStreamSynchronize(s));
    rc = check_device_errors(c);
    if (stats) {
        memset(stats, 0, sizeof *stats);
        Stats h;
        Counters hc;
        CU(cudaMemcpy(&h, c->stats.p, sizeof h, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(&hc, c->counters.p, sizeof hc, cudaMemcpyDeviceToHost));
        write_stats(stats, h, false, hc.arena_top, launches);
        if (timing) add_stage_ms_2d(c, 0, L, fused, h, stats->stage_ms);
    }
    return rc;
}

int32_t fc_render2d_frames(fc_ctx* c, const fc_tape* tape, const fc_render2d_cfg* cfg, const fc_frame2d* frames,
                           uint32_t n_frames, void* out, fc_render_stats* stats) {
    if (!c || !tape || !cfg || !out || (n_frames && !frames)) return fail(FC_ERR_INVALID, "null argument");
    if (int32_t vrc = check_2d(tape, cfg)) return vrc;
    if (int32_t vrc = check_batch_2d(cfg, "frame batches")) return vrc;
    const uint32_t fmt = cfg->out_format;
    // every frame's ShapeVars binding, before anything is allocated or launched
    std::vector<Frame2D> table(n_frames);
    for (uint32_t k = 0; k < n_frames; ++k)
        if (int32_t brc = bind_frame(tape, frames[k], frames[k].z, table[k])) return brc;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    if (stats) memset(stats, 0, sizeof *stats);
    if (n_frames == 0) return FC_OK;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    Tiles2D g;
    if (int32_t rc = prepare_2d(c, tape, cfg, g)) return rc;
    const int L = int(g.ts.size());
    const uint32_t T0 = g.ts[0];
    const uint32_t W = cfg->width, H = cfg->height;
    const uint32_t roots_y = (H + T0 - 1) / T0;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    const bool async = (cfg->flags & FC_FLAG_ASYNC) != 0;
    const bool want_stats = stats != nullptr;
    const bool out_dev = is_device_ptr(out);
    cudaStream_t s = c->stream;

    // ---- frames per pass: the worst-case lists of a frame (jobs and fills) plus its staged images ----
    const size_t img_f32 = size_t(W) * H * 4, img_fmt = format_bytes(fmt, W, H);
    const bool stage_f32 = fmt != FC_OUT_F32 || !out_dev;             // the distance images live in the context
    const int f32_bufs = fmt == FC_OUT_F32 ? 2 : 1;                    // (a host F32 copy-back is double-buffered)
    const uint64_t staged = (stage_f32 ? uint64_t(img_f32) * f32_bufs : 0) +
                            (fmt != FC_OUT_F32 && !out_dev ? 2ull * img_fmt : 0);   // double-buffered derived images
    uint32_t per_pass, n_passes;
    if (int32_t prc = passes_2d(g.ts, uint64_t(g.roots_x) * roots_y, n_frames, sizeof(TileJob) + sizeof(FillRec), staged,
                                per_pass, n_passes))
        return prc;

    g.roots_y = roots_y * per_pass;
    g.n_roots = uint64_t(g.roots_x) * g.roots_y;
    g.frame_rows = roots_y * T0;
    if (int32_t src = size_lists_2d(g.ts, g.n_roots, g.level_tiles)) return src;
    if (int32_t erc = ensure_scratch_2d(c, g)) return erc;
    CU(c->frame_table.ensure(size_t(n_frames) * sizeof(Frame2D)));
    CU(c->frame_tops.ensure(size_t(n_passes) * sizeof(unsigned long long)));
    float* stage[2] = {nullptr, nullptr};
    uint8_t* fstage[2] = {nullptr, nullptr};
    if (stage_f32) {
        CU(c->image.ensure(img_f32 * per_pass * f32_bufs));
        stage[0] = c->image.as<float>();
        stage[1] = stage[0] + (f32_bufs == 2 ? size_t(W) * H * per_pass : 0);
    }
    if (fmt != FC_OUT_F32 && !out_dev) {
        CU(c->fx_out.ensure(img_fmt * per_pass * 2));
        fstage[0] = c->fx_out.as<uint8_t>();
        fstage[1] = fstage[0] + img_fmt * per_pass;
    }
    if (!out_dev) if (int32_t src = ensure_copy_stream(c)) return src;
    CU(cudaMemcpyAsync(c->frame_table.p, table.data(), table.size() * sizeof(Frame2D), cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters), s));
    if (want_stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));

    // host `out`: pass k's images go back on the copy stream while pass k + 1 runs (issued after pass k + 1 is
    // enqueued, so that a copy into pageable memory, which blocks the host, still overlaps the next pass).  The work
    // stream waits for the copy from then on: pass k + 2 reuses staging buffer k & 1, and the call ends with its last copy.
    auto copy_back = [&](uint32_t k) -> int32_t {
        const uint32_t f0 = k * per_pass, n = std::min(per_pass, n_frames - f0);
        const size_t fb = fmt == FC_OUT_F32 ? img_f32 : img_fmt;
        const void* src = fmt == FC_OUT_F32 ? static_cast<const void*>(stage[k & 1]) : static_cast<const void*>(fstage[k & 1]);
        if (int32_t wrc = wait_pass(c, int(k & 1), cc, false)) return wrc;   // (a cancelled pass copies nothing)
        if (int32_t crc = copy_pass_back(c, int(k & 1), static_cast<uint8_t*>(out) + size_t(f0) * fb, src, size_t(n) * fb))
            return crc;
        CU(cudaStreamWaitEvent(s, c->ev_copied[k & 1], 0));
        return FC_OK;
    };
    VarBind vb0 = table[0].vb;   // (unused by the kernels: every frame comes from the table)
    size_t ev = 0;
    uint32_t launches = 0;
    auto enqueue = [&](uint32_t k) -> int32_t {
        const uint32_t f0 = k * per_pass, n = std::min(per_pass, n_frames - f0);
        Tiles2D gp = g;
        gp.roots_y = roots_y * n;
        gp.n_roots = uint64_t(g.roots_x) * gp.roots_y;
        gp.frames = c->frame_table.as<Frame2D>() + f0;
        if (k) if (int32_t rrc = reset_pass_2d(c, s)) return rrc;
        float* dimg = stage_f32 ? stage[k & 1] : static_cast<float*>(out) + size_t(f0) * W * H;
        bool fused = false;
        if (int32_t erc = enqueue_tiles_2d(c, tape, cfg, gp, vb0, dimg, want_stats, timing, cc, s, ev, launches, fused))
            return erc;
        if (fmt != FC_OUT_F32) {
            uint8_t* dfmt = out_dev ? static_cast<uint8_t*>(out) + size_t(f0) * img_fmt : fstage[k & 1];
            derive_format(fmt, dimg, W, H * n, dfmt, s);   // the pass's frames are one image of n * H rows
            ++launches;
            CU(cudaGetLastError());
        }
        if (want_stats) if (int32_t trc = record_top_2d(c, s, k)) return trc;
        if (!out_dev) CU(cudaEventRecord(c->ev_pass[k & 1], s));
        return FC_OK;
    };
    auto abandon = [&](int32_t rc) { return abandon_frames(c, s, stats, rc); };
    uint32_t passes_run = 0;
    for (uint32_t k = 0; k < n_passes; ++k) {
        if (k && cc.flag && __atomic_load_n(cc.flag, __ATOMIC_ACQUIRE)) break;   // cancelled: enqueue no further pass
        if (int32_t erc = enqueue(k)) return abandon(erc);
        ++passes_run;
        if (!out_dev && k) if (int32_t crc = copy_back(k - 1)) return abandon(crc);
    }
    if (!out_dev) if (int32_t crc = copy_back(passes_run - 1)) return abandon(crc);
    if (async && out_dev && !want_stats) {
        c->async_call = cc;
        return FC_OK;
    }
    if (int32_t wrc = wait_cancel_2d(c, s, cc, passes_run, n_passes, stats)) return abandon(wrc);
    return finish_2d(c, s, L, n_passes, timing, launches, stats);
}

// A 2D scene (kernels.cuh, Scene2D): every placement's tiles go through the tile pipeline of fc_render2d_frames, which
// records inside tiles in the cover map and inside leaf pixels in the key map instead of painting images.  Passes run
// from the top of the draw list down, so that the shapes of a pass are culled against every shape above them; one
// resolve launch then writes the index and the image.
int32_t fc_render2d_scene(fc_ctx* c, const fc_tape* const* tapes, const fc_frame2d* placements, uint32_t n_shapes,
                          const fc_render2d_cfg* cfg, const uint8_t* colors, void* out, uint16_t* index,
                          fc_render_stats* stats) {
    static_assert(FC_OUT_MASK_U8 == 1 && FC_OUT_BITMAP_1BIT == 2 && FC_OUT_RGBA8 == 3, "Scene2DResolveParams::fmt");
    static_assert(FC_SCENE_MAX_SHAPES < FC_SCENE2D_NONE, "a shape's index is never FC_SCENE2D_NONE");
    if (!c || !cfg || (!out && !index) || (n_shapes && (!tapes || !placements))) return fail(FC_ERR_INVALID, "null argument");
    if (n_shapes > FC_SCENE_MAX_SHAPES) return fail(FC_ERR_UNSUPPORTED, "more than FC_SCENE_MAX_SHAPES shapes");
    if (int32_t vrc = check_batch_2d(cfg, "scenes")) return vrc;
    const uint32_t fmt = cfg->out_format;
    if (fmt == FC_OUT_F32) return fail(FC_ERR_UNSUPPORTED, "a 2D scene keeps no distances: FC_OUT_F32 is not supported");
    // every placement's tape and ShapeVars binding, before anything is allocated or launched
    std::vector<Frame2D> table(n_shapes);
    for (uint32_t k = 0; k < n_shapes; ++k) {
        if (!tapes[k]) return fail(FC_ERR_INVALID, "null tape in the scene");
        if (int32_t vrc = check_2d(tapes[k], cfg)) return vrc;
        if (int32_t brc = bind_frame(tapes[k], placements[k], placements[k].z, table[k])) return brc;
    }
    Tiles2D g;
    if (n_shapes)
        if (int32_t rc = prepare_2d(c, tapes[0], cfg, g)) return rc;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    if (stats) memset(stats, 0, sizeof *stats);
    if (n_shapes == 0) return FC_OK;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const int L = int(g.ts.size());
    const uint32_t T0 = g.ts[0], leaf = g.ts[L - 1];
    const uint32_t W = cfg->width, H = cfg->height;
    g.roots_y = (H + T0 - 1) / T0;
    for (uint32_t k = 0; k < n_shapes; ++k)   // choice scratch for the largest choice_count
        g.choice_words = std::max(g.choice_words, choice_words(tapes[k]));
    g.scene = true;
    g.blocks_x = (W + leaf - 1) / leaf;
    g.blocks_y = (H + leaf - 1) / leaf;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    const bool async = (cfg->flags & FC_FLAG_ASYNC) != 0;
    const bool want_stats = stats != nullptr;
    const bool host_out = out && !is_device_ptr(out), host_index = index && !is_device_ptr(index);
    const size_t npix = size_t(W) * H, n_blocks = size_t(g.blocks_x) * g.blocks_y, img_fmt = format_bytes(fmt, W, H);
    cudaStream_t s = c->stream;

    // ---- shapes per pass: their worst-case job lists (the maps are the call's) ----
    const uint64_t shape_roots = uint64_t(g.roots_x) * g.roots_y;
    uint32_t per_pass, n_passes;
    if (int32_t prc = passes_2d(g.ts, shape_roots, n_shapes, sizeof(TileJob), 0, per_pass, n_passes)) return prc;
    auto pass_range = [&](uint32_t k, uint32_t& lo, uint32_t& hi) {   // pass k: shapes [lo, hi), the top pass first
        hi = n_shapes - k * per_pass;
        lo = hi - std::min(hi, per_pass);
    };
    // each pass's level-0 groups, the top shapes' tapes first
    std::vector<uint32_t> pl_host;
    std::vector<std::vector<SceneGroup>> groups(n_passes);
    for (uint32_t k = 0; k < n_passes; ++k) {
        uint32_t lo, hi;
        pass_range(k, lo, hi);
        std::vector<uint32_t> order;
        for (uint32_t q = hi; q > lo; --q) order.push_back(q - 1);
        group_by_tape(tapes, order, pl_host, groups[k]);
    }

    g.n_roots = shape_roots * per_pass;
    if (int32_t src = size_lists_2d(g.ts, g.n_roots, g.level_tiles)) return src;
    if (int32_t erc = ensure_scratch_2d(c, g)) return erc;
    CU(c->frame_table.ensure(size_t(n_shapes) * sizeof(Frame2D)));
    CU(c->frame_tops.ensure(size_t(n_passes) * sizeof(unsigned long long)));
    CU(c->scene_pl.ensure(size_t(n_shapes) * 4));
    CU(c->scene_cover.ensure(2 * n_blocks * 4));
    CU(c->scene_key.ensure(npix * 4));
    CU(c->scene_colors.ensure(size_t(n_shapes) * 3));
    uint8_t* dout = static_cast<uint8_t*>(out);
    if (host_out) {
        CU(c->fx_out.ensure(img_fmt));
        dout = c->fx_out.as<uint8_t>();
    }
    uint16_t* dindex = index;
    if (host_index) {
        CU(c->scene_index.ensure(npix * 2));
        dindex = c->scene_index.as<uint16_t>();
    }
    const std::vector<uint8_t> white(colors ? 0 : size_t(n_shapes) * 3, 255);   // draw(): every shape white
    CU(cudaMemcpyAsync(c->frame_table.p, table.data(), table.size() * sizeof(Frame2D), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(c->scene_pl.p, pl_host.data(), pl_host.size() * 4, cudaMemcpyHostToDevice, s));
    if (out && fmt == FC_OUT_RGBA8)
        CU(cudaMemcpyAsync(c->scene_colors.p, colors ? colors : white.data(), size_t(n_shapes) * 3, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters), s));
    if (want_stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
    CU(cudaMemsetAsync(c->scene_cover.p, 0, 2 * n_blocks * 4, s));
    CU(cudaMemsetAsync(c->scene_key.p, 0, npix * 4, s));
    g.frames = c->frame_table.as<Frame2D>();
    g.d_pl = c->scene_pl.as<uint32_t>();
    g.cover = c->scene_cover.as<uint32_t>();
    g.key = c->scene_key.as<uint32_t>();

    size_t ev = 0;
    uint32_t launches = 0, passes_run = 0;
    for (uint32_t k = 0; k < n_passes; ++k) {
        if (k && cc.flag && __atomic_load_n(cc.flag, __ATOMIC_ACQUIRE)) break;   // cancelled: enqueue no further pass
        uint32_t lo, hi;
        pass_range(k, lo, hi);
        Tiles2D gp = g;
        gp.n_roots = shape_roots * (hi - lo);
        gp.groups = groups[k];
        if (k) if (int32_t rrc = reset_pass_2d(c, s)) return rrc;
        bool fused = false;
        if (int32_t erc = enqueue_tiles_2d(c, tapes[hi - 1], cfg, gp, table[hi - 1].vb, nullptr, want_stats, timing, cc, s,
                                           ev, launches, fused))
            return abandon_frames(c, s, stats, erc);
        if (want_stats) if (int32_t trc = record_top_2d(c, s, k)) return trc;
        ++passes_run;
    }
    if (passes_run == n_passes) {
        Scene2DResolveParams rp{};
        rp.cover = g.cover + n_blocks;
        rp.key = g.key;
        rp.width = W;
        rp.height = H;
        rp.leaf = leaf;
        rp.blocks_x = g.blocks_x;
        rp.fmt = fmt;
        rp.colors = c->scene_colors.as<uint8_t>();
        rp.out = out ? dout : nullptr;
        rp.index = dindex;
        rp.cancel = cc.ref;
        launch_scene2d_resolve(rp, s);
        ++launches;
        CU(cudaGetLastError());
    }
    if (async && !host_out && !host_index && !want_stats) {
        c->async_call = cc;
        return FC_OK;
    }
    // a cancelled call copies nothing to the host
    if (int32_t wrc = wait_cancel_2d(c, s, cc, passes_run, n_passes, stats)) return wrc;
    if (host_out) CU(cudaMemcpyAsync(out, dout, img_fmt, cudaMemcpyDeviceToHost, s));
    if (host_index) CU(cudaMemcpyAsync(index, dindex, npix * 2, cudaMemcpyDeviceToHost, s));
    return finish_2d(c, s, L, n_passes, timing, launches, stats);
}

int32_t fc_render3d(fc_ctx* c, const fc_tape* tape, const fc_render3d_cfg* cfg, fc_geometry_pixel* out,
                    fc_render_stats* stats) {
    if (!c || !tape || !cfg || !out) return fail(FC_ERR_INVALID, "null argument");
    if (int32_t vrc = check_3d(tape, cfg)) return vrc;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    Tiles3D g;
    int32_t rc = prepare_3d(c, tape, cfg, g);
    if (rc) return rc;
    const int L = int(g.ts.size());
    const uint32_t T0 = g.ts[0];
    const uint32_t roots_x = g.roots_x, roots_y_all = (cfg->height + T0 - 1) / T0;
    const uint32_t row0 = cfg->root_row_begin, row1 = cfg->root_row_end ? cfg->root_row_end : roots_y_all;
    if (row0 > row1 || row1 > roots_y_all) return fail(FC_ERR_INVALID, "bad root row band");
    const uint32_t roots_y = row1 - row0;
    const uint32_t band_y0 = std::min(row0 * T0, cfg->height), band_y1 = std::min(row1 * T0, cfg->height);
    const uint32_t z_begin = cfg->z_begin, z_end = cfg->z_end ? cfg->z_end : cfg->depth;
    if (z_begin % T0 || z_begin >= z_end || z_end > ((cfg->depth + T0 - 1) / T0) * T0)
        return fail(FC_ERR_INVALID, "z slab must start on a root-tile boundary inside the volume");
    const uint32_t roots_z = (std::min(z_end, ((cfg->depth + T0 - 1) / T0) * T0) - z_begin + T0 - 1) / T0;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    const bool async = (cfg->flags & FC_FLAG_ASYNC) != 0;
    const bool want_stats = stats != nullptr;
    cudaStream_t s = c->stream;
    const uint32_t* d_roots = nullptr;
    uint32_t n_list = 0;
    if (cfg->root_stride > 1) {
        if (cfg->root_offset >= cfg->root_stride) return fail(FC_ERR_INVALID, "root_offset must be below root_stride");
        if (!is_device_ptr(out)) return fail(FC_ERR_UNSUPPORTED, "tile-interleaved renders need a device image");
        if (T0 % 8) return fail(FC_ERR_UNSUPPORTED, "tile-interleaved renders need a root tile edge that is a multiple of 8");
        if (int32_t lrc = root_subset(c, roots_x, row0, row1, cfg->root_stride, cfg->root_offset, s, &d_roots, &n_list)) return lrc;
    }
    g.roots_y = roots_y; g.roots_z = roots_z; g.row0 = row0; g.z_begin = z_begin;
    g.d_roots = d_roots; g.n_list = n_list;
    g.n_roots = (d_roots ? uint64_t(n_list) : uint64_t(roots_x) * roots_y) * roots_z;
    if (g.n_roots > 0xfffffff0ull) return fail(FC_ERR_UNSUPPORTED, "volume too large");
    if (g.exact_census) {
        if (!stats) return fail(FC_ERR_INVALID, "FC_FLAG_EXACT_CENSUS needs a stats struct");
        if (cfg->width % T0 || cfg->height % T0 || d_roots || row0 || row1 != roots_y_all || z_begin || z_end < cfg->depth)
            return fail(FC_ERR_UNSUPPORTED, "the exact census needs a whole-volume render of an image whose sides are multiples of the root tile");
    }
    size_lists_3d(g);
    const size_t npix = size_t(cfg->width) * cfg->height;
    if (int32_t erc = ensure_scratch_3d(c, g, npix, size_t(g.occl_w) * g.occl_h)) return erc;
    bool out_dev = is_device_ptr(out);
    void* dimg = out;
    if (!out_dev) {
        void* alias = env_int("FIDGET_B200_ZEROCOPY", 0) ? pinned_device_alias(out) : nullptr;
        if (alias) {
            dimg = alias;
            out_dev = true;
        } else {
            CU(c->image.ensure(npix * 16));
            dimg = c->image.p;
        }
    }
    CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters), s));
    CU(cudaMemsetAsync(c->heightmap.as<char>() + size_t(band_y0) * cfg->width * 8, 0, size_t(band_y1 - band_y0) * cfg->width * 8, s));
    if (g.use_occl) CU(cudaMemsetAsync(c->occl.p, 0, size_t(g.occl_w) * g.occl_h * 4, s));
    if (want_stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));

    VarBind vb;
    if (int32_t vrc = bind_vars(tape, cfg->var_values, cfg->n_var_values, vb)) return vrc;
    size_t ev = 0;
    uint32_t launches = 0;
    if (int32_t erc = enqueue_tiles_3d(c, tape, cfg, g, vb, dimg, band_y0, band_y1, want_stats, timing, cc, s, ev, launches))
        return erc;
    const bool early_return = async && out_dev && !want_stats;
    if (cc.flag && !early_return) {   // a cancelled render copies nothing to the host
        if (int32_t wrc = wait_call(c, s, cc)) {
            if (stats) memset(stats, 0, sizeof *stats);
            return wrc;
        }
    }
    if (!out_dev && band_y1 > band_y0)
        CU(cudaMemcpyAsync(reinterpret_cast<char*>(out) + size_t(band_y0) * cfg->width * 16,
                           static_cast<char*>(dimg) + size_t(band_y0) * cfg->width * 16, size_t(band_y1 - band_y0) * cfg->width * 16,
                           cudaMemcpyDeviceToHost, s));
    if (early_return) {
        c->async_call = cc;
        return FC_OK;
    }
    CU(cudaStreamSynchronize(s));
    rc = check_device_errors(c);
    if (stats) {
        memset(stats, 0, sizeof *stats);
        Stats h;
        Counters hc;
        CU(cudaMemcpy(&h, c->stats.p, sizeof h, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(&hc, c->counters.p, sizeof hc, cudaMemcpyDeviceToHost));
        write_stats(stats, h, true, hc.arena_top, launches);
        if (timing) add_stage_ms_3d(c, 0, L, stats->stage_ms);
    }
    return rc;
}

int32_t fc_render3d_frames(fc_ctx* c, const fc_tape* tape, const fc_render3d_cfg* cfg, const fc_frame3d* frames,
                           uint32_t n_frames, fc_geometry_pixel* out, fc_render_stats* stats) {
    if (!c || !tape || !cfg || !out || (n_frames && !frames)) return fail(FC_ERR_INVALID, "null argument");
    if (int32_t vrc = check_3d(tape, cfg)) return vrc;
    if (int32_t vrc = check_batch_3d(cfg, "frame batches")) return vrc;
    // every frame's ShapeVars binding, before anything is allocated or launched (z is unused in 3D)
    std::vector<Frame2D> table(n_frames);
    for (uint32_t k = 0; k < n_frames; ++k)
        if (int32_t brc = bind_frame(tape, frames[k], 0.0f, table[k])) return brc;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    if (stats) memset(stats, 0, sizeof *stats);
    if (n_frames == 0) return FC_OK;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    Tiles3D g;
    if (int32_t rc = prepare_3d(c, tape, cfg, g)) return rc;
    const int L = int(g.ts.size());
    const uint32_t T0 = g.ts[0];
    const uint32_t W = cfg->width, H = cfg->height;
    const uint32_t roots_y = (H + T0 - 1) / T0, frame_rows = roots_y * T0;   // root rows and grid rows per frame
    g.roots_z = (cfg->depth + T0 - 1) / T0;
    const uint64_t frame_roots = uint64_t(g.roots_x) * roots_y * g.roots_z;
    if (frame_roots > 0xfffffff0ull) return fail(FC_ERR_UNSUPPORTED, "volume too large");
    if (g.exact_census) {
        if (!stats) return fail(FC_ERR_INVALID, "FC_FLAG_EXACT_CENSUS needs a stats struct");
        if (W % T0 || H % T0)
            return fail(FC_ERR_UNSUPPORTED, "the exact census needs a whole-volume render of an image whose sides are multiples of the root tile");
    }
    if (frame_rows % 16) g.use_occl = false;   // (root tiles below 16 never write the occlusion map)
    g.frame_rows = frame_rows;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    const bool async = (cfg->flags & FC_FLAG_ASYNC) != 0;
    const bool want_stats = stats != nullptr;
    const bool host_out = !is_device_ptr(out);
    const size_t img_px = size_t(W) * H;
    const size_t occl_frame = g.use_occl ? size_t(frame_rows / 16) * g.occl_w : 0;   // occlusion blocks per frame
    cudaStream_t s = c->stream;

    // ---- passes.  Lists and census of a pass of n frames are those of one grid of n stacked frames (capped as in
    // fc_render3d); its heightmap rows, occlusion blocks and (host out) two staged images per frame are its own. ----
    auto grid_of = [&](uint32_t n) {
        Tiles3D gp = g;
        gp.roots_y = roots_y * n;
        gp.n_roots = frame_roots * n;
        size_lists_3d(gp);
        return gp;
    };
    // (exact census: a pass keeps its census rows within 16 bits)
    PassPlan plan = plan_3d(c, grid_of, n_frames,
                            size_t(frame_rows) * W * 8 + occl_frame * 4 + (host_out ? 2 * img_px * 16 : 0),
                            g.exact_census ? 65536 / frame_rows : 0xffffffffu);
    const uint32_t n_max = plan.n_max;
    if (int32_t erc = ensure_scratch_3d(c, grid_of(n_max), size_t(W) * frame_rows * n_max, occl_frame * n_max)) return erc;
    CU(c->frame_table.ensure(size_t(n_frames) * sizeof(Frame2D)));
    if (int32_t prc = ensure_pass_pin(c)) return prc;
    fc_geometry_pixel* stage[2] = {nullptr, nullptr};
    if (host_out) {
        CU(c->image.ensure(2 * img_px * 16 * n_max));
        stage[0] = c->image.as<fc_geometry_pixel>();
        stage[1] = stage[0] + img_px * n_max;
    }
    if (int32_t src = ensure_copy_stream(c)) return src;
    CU(cudaMemcpyAsync(c->frame_table.p, table.data(), table.size() * sizeof(Frame2D), cudaMemcpyHostToDevice, s));

    using Range = PassPlan::Range;
    struct InFlight { Range r; int b; size_t ev0; };
    PassStats sum;
    size_t ev = 0;
    uint32_t launches = 0;
    bool copy_pending[2] = {false, false};
    const VarBind vb0 = table[0].vb;   // (unused by the kernels: every frame comes from the table)
    auto enqueue = [&](const Range& r, int b) -> int32_t {
        Tiles3D gp = grid_of(r.n);
        gp.frames = c->frame_table.as<Frame2D>() + r.f0;
        if (host_out && copy_pending[b]) CU(cudaStreamWaitEvent(s, c->ev_copied[b], 0));   // staging buffer b is free again
        CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters), s));                         // (error bits are per pass)
        CU(cudaMemsetAsync(c->heightmap.p, 0, size_t(r.n) * frame_rows * W * 8, s));
        if (g.use_occl) CU(cudaMemsetAsync(c->occl.p, 0, occl_frame * r.n * 4, s));
        if (want_stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
        void* dimg = host_out ? static_cast<void*>(stage[b]) : static_cast<void*>(out + size_t(r.f0) * img_px);
        if (int32_t erc = enqueue_tiles_3d(c, tape, cfg, gp, vb0, dimg, 0, r.n * H, want_stats, timing, cc, s, ev, launches))
            return erc;
        // the pass's status, into pinned slot b for the host to read while the next pass runs (the slot is read before
        // buffer b takes another pass)
        if (int32_t src = read_pass_status(c, s, b, want_stats)) return src;
        CU(cudaEventRecord(c->ev_pass[b], s));
        return FC_OK;
    };
    // Waits for a pass (watching the flag, as wait_call does) and reads its status.  Overflowed: its halves are queued
    // again (one frame: the error).  Else its stats are added and, with a host `out`, its images copied back on the
    // copy stream, which the host issues after the next pass is enqueued: a copy into pageable memory blocks the host.
    auto settle = [&](const InFlight& f) -> int32_t {
        if (int32_t wrc = wait_pass(c, f.b, cc, true)) return wrc;
        const PassStatus& ps = c->pass_pin[f.b];
        bool split = false;
        if (!plan.observe(ps.ctr, ps.ctr.n_census, f.r, split)) return device_error(ps.ctr.error);
        if (split) return FC_OK;
        if (want_stats) sum.add(c, ps, timing, f.ev0, L);
        if (host_out) {
            copy_pending[f.b] = true;
            return copy_pass_back(c, f.b, out + size_t(f.r.f0) * img_px, stage[f.b], size_t(f.r.n) * img_px * 16);
        }
        return FC_OK;
    };
    auto abandon = [&](int32_t rc) { return abandon_frames(c, s, stats, rc); };

    const bool early_return = async && !host_out && !want_stats;
    bool have_prev = false, stopped = false;
    InFlight prev{};
    int buf = 0;
    for (;;) {
        const bool more = plan.more();
        if (more && have_prev && cc.flag && __atomic_load_n(cc.flag, __ATOMIC_ACQUIRE)) stopped = true;   // enqueue no further pass
        if (more && !stopped) {
            if (have_prev && !plan.measured) {   // the first pass is read before the second is sized
                if (int32_t rc = settle(prev)) return abandon(rc);
                have_prev = false;
                continue;
            }
            const Range r = plan.take();
            const InFlight cur{r, buf, ev};
            if (int32_t rc = enqueue(r, buf)) return abandon(rc);
            if (have_prev)
                if (int32_t rc = settle(prev)) return abandon(rc);
            prev = cur;
            have_prev = true;
            buf ^= 1;
            continue;
        }
        if (!have_prev) break;
        if (early_return && !stopped) {   // FC_FLAG_ASYNC: the last pass is left running (its errors: fc_ctx_synchronize)
            c->async_call = cc;
            return FC_OK;
        }
        if (int32_t rc = settle(prev)) return abandon(rc);
        have_prev = false;
    }
    if (cc.flag) {
        if (int32_t wrc = wait_call(c, c->copy_stream, cc)) return abandon(wrc);
    } else {
        CU(cudaStreamSynchronize(c->copy_stream));
    }
    if (stopped) return abandon(fail(FC_ERR_CANCELLED, "cancelled"));   // the flag stopped the passes
    if (stats) sum.write(stats, launches);
    return FC_OK;
}

// A scene: every placement's tiles go through one tile pipeline over one shared heightmap and occlusion map, whose keys
// order what the fold of the per-shape images keeps (kernels.cuh, scene_rank).  Placements run in passes: a pass lists
// its placements grouped by tape for level 0, then shares every later launch; its normals finish the pixels it won.
int32_t fc_render3d_scene(fc_ctx* c, const fc_tape* const* tapes, const fc_frame3d* placements, uint32_t n_shapes,
                          const fc_render3d_cfg* cfg, fc_geometry_pixel* out, uint16_t* index, fc_render_stats* stats) {
    static_assert(FC_SCENE_MAX_SHAPES == SK_MAX_SHAPES, "FC_SCENE_MAX_SHAPES is the key's placement field");
    static_assert(FC_SCENE_MAX_DEPTH + 2 == (1u << SK_DEPTH_BITS), "FC_SCENE_MAX_DEPTH + 1 is the key's largest depth");
    static_assert(FC_SCENE_MAX_ROOT_TILE + 1 == (1u << SK_SUB_BITS) - 1, "depths reach a root tile + 1 above the clamp threshold");
    static_assert(FC_SCENE_MAX_LEAF_JOBS == SK_ID_MASK, "leaf id + 1 is the key's id field");
    if (!c || !cfg || !out || (n_shapes && (!tapes || !placements))) return fail(FC_ERR_INVALID, "null argument");
    if (n_shapes > FC_SCENE_MAX_SHAPES) return fail(FC_ERR_UNSUPPORTED, "more than FC_SCENE_MAX_SHAPES shapes");
    if (cfg->flags & FC_FLAG_EXACT_CENSUS) return fail(FC_ERR_UNSUPPORTED, "the exact census is not supported by scenes");
    if (int32_t vrc = check_batch_3d(cfg, "scenes")) return vrc;
    // every placement's tape and ShapeVars binding, and the key's limits, before anything is allocated or launched
    std::vector<Frame2D> table(n_shapes);
    for (uint32_t k = 0; k < n_shapes; ++k) {
        if (!tapes[k]) return fail(FC_ERR_INVALID, "null tape in the scene");
        if (int32_t vrc = check_3d(tapes[k], cfg)) return vrc;
        if (int32_t brc = bind_frame(tapes[k], placements[k], 0.0f, table[k])) return brc;
    }
    Tiles3D g;
    const bool clamp = !(cfg->flags & FC_FLAG_NO_CLAMP);
    if (n_shapes) {
        if (int32_t rc = prepare_3d(c, tapes[0], cfg, g)) return rc;
        const uint32_t T0 = g.ts[0];
        if (uint64_t((cfg->depth + T0 - 1) / T0) * T0 > FC_SCENE_MAX_DEPTH)
            return fail(FC_ERR_UNSUPPORTED, "scene depth (rounded up to whole root tiles) above FC_SCENE_MAX_DEPTH");
        if (clamp && T0 > FC_SCENE_MAX_ROOT_TILE)
            return fail(FC_ERR_UNSUPPORTED, "scene root tile edge above FC_SCENE_MAX_ROOT_TILE");
    }
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    if (stats) memset(stats, 0, sizeof *stats);
    if (n_shapes == 0) return FC_OK;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const int L = int(g.ts.size());
    const uint32_t T0 = g.ts[0];
    const uint32_t W = cfg->width, H = cfg->height;
    g.roots_y = (H + T0 - 1) / T0;
    g.roots_z = (cfg->depth + T0 - 1) / T0;
    const uint64_t vol_roots = uint64_t(g.roots_x) * g.roots_y * g.roots_z;
    if (vol_roots > 0xfffffff0ull) return fail(FC_ERR_UNSUPPORTED, "volume too large");
    for (uint32_t k = 0; k < n_shapes; ++k)   // choice scratch for the largest choice_count
        g.choice_words = std::max(g.choice_words, choice_words(tapes[k]));
    g.scene = true;
    g.clamp_at = clamp ? cfg->depth - 1u : 0xffffffffu;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    const bool async = (cfg->flags & FC_FLAG_ASYNC) != 0;
    const bool want_stats = stats != nullptr;
    const bool host_out = !is_device_ptr(out), host_index = index && !is_device_ptr(index);
    const size_t npix = size_t(W) * H, occl_blocks = size_t(g.occl_w) * g.occl_h;   // (scene occlusion blocks: 8 bytes)
    cudaStream_t s = c->stream;

    // Lists of a pass of n placements are those of one grid of n volumes (capped as in fc_render3d; the leaf list also
    // at FC_SCENE_MAX_LEAF_JOBS, whose ids fill the key's id field); heightmap and occlusion map are the call's.
    auto grid_of = [&](uint32_t n) {
        Tiles3D gp = g;
        gp.n_roots = vol_roots * n;
        size_lists_3d(gp);
        gp.level_cap[L] = std::min<uint64_t>(gp.level_cap[L], FC_SCENE_MAX_LEAF_JOBS);
        return gp;
    };
    PassPlan plan = plan_3d(c, grid_of, n_shapes, 0, 0xffffffffu);
    if (int32_t erc = ensure_scratch_3d(c, grid_of(plan.n_max), npix, occl_blocks * 2)) return erc;
    CU(c->frame_table.ensure(size_t(n_shapes) * sizeof(Frame2D)));
    CU(c->scene_pl.ensure(size_t(n_shapes) * 4));
    if (n_shapes > 1) CU(c->scene_backup.ensure(npix * 8 + (g.use_occl ? occl_blocks * 8 : 0)));
    if (int32_t prc = ensure_pass_pin(c)) return prc;
    void* dimg = out;
    if (host_out) {
        CU(c->image.ensure(npix * 16));
        dimg = c->image.p;
    }
    uint16_t* dindex = index;
    if (host_index) {
        CU(c->scene_index.ensure(npix * 2));
        dindex = c->scene_index.as<uint16_t>();
    }
    g.frames = c->frame_table.as<Frame2D>();
    CU(cudaMemcpyAsync(c->frame_table.p, table.data(), table.size() * sizeof(Frame2D), cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(c->heightmap.p, 0, npix * 8, s));
    if (g.use_occl) CU(cudaMemsetAsync(c->occl.p, 0, occl_blocks * 8, s));

    // Passes follow PassPlan's overflow policy per placement.  They build on each other's heightmap, so each is waited
    // for before the next; one of several placements keeps a copy of the heightmap and occlusion map from before it,
    // and if it overflows anyway (its normals write nothing) the copy is restored and its halves run instead.
    auto abandon = [&](int32_t rc) { return abandon_frames(c, s, stats, rc); };
    const size_t backup_occl = npix * 8;   // (byte offset of the occlusion map's copy)
    auto snapshot = [&](bool restore) -> int32_t {
        char* b = c->scene_backup.as<char>();
        CU(cudaMemcpyAsync(restore ? c->heightmap.p : b, restore ? b : c->heightmap.p, npix * 8, cudaMemcpyDeviceToDevice, s));
        if (g.use_occl)
            CU(cudaMemcpyAsync(restore ? c->occl.p : b + backup_occl, restore ? b + backup_occl : c->occl.p, occl_blocks * 8,
                               cudaMemcpyDeviceToDevice, s));
        return FC_OK;
    };

    PassStats sum;
    size_t ev = 0;
    uint32_t launches = 0;
    std::vector<uint32_t> pl_host;
    const bool early_return = async && !host_out && !host_index && !want_stats;
    for (bool first = true; plan.more(); first = false) {
        if (!first && cc.flag && __atomic_load_n(cc.flag, __ATOMIC_ACQUIRE))
            return abandon(fail(FC_ERR_CANCELLED, "cancelled"));   // the flag stops the passes
        const PassPlan::Range r = plan.take();
        // level-0 groups: the pass's placements by tape, in order of first appearance
        Tiles3D gp = grid_of(r.n);
        gp.pl0 = r.f0;
        gp.pl1 = r.f0 + r.n;
        pl_host.clear();
        std::vector<uint32_t> order(r.n);
        for (uint32_t k = 0; k < r.n; ++k) order[k] = r.f0 + k;
        group_by_tape(tapes, order, pl_host, gp.groups);
        gp.d_pl = c->scene_pl.as<uint32_t>();
        CU(cudaMemcpyAsync(c->scene_pl.p, pl_host.data(), pl_host.size() * 4, cudaMemcpyHostToDevice, s));
        if (r.n > 1) {
            if (int32_t brc = snapshot(false)) return abandon(brc);
        }
        CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters), s));
        if (want_stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
        const size_t ev0 = ev;
        if (int32_t erc = enqueue_tiles_3d(c, tapes[r.f0], cfg, gp, table[r.f0].vb, dimg, 0, H, want_stats, timing, cc, s, ev,
                                           launches, dindex))
            return abandon(erc);
        if (int32_t src = read_pass_status(c, s, 0, want_stats)) return src;
        const PassStatus* hs = c->pass_pin;
        if (early_return && !plan.more()) {   // FC_FLAG_ASYNC: the last pass is left running
            c->async_call = cc;
            return FC_OK;
        }
        if (cc.flag) {
            if (int32_t wrc = wait_call(c, s, cc)) return abandon(wrc);
        } else {
            CU(cudaStreamSynchronize(s));
        }
        bool split = false;
        if (!plan.observe(hs->ctr, hs->ctr.n_census, r, split)) return abandon(device_error(hs->ctr.error));
        if (split) {
            if (int32_t brc = snapshot(true)) return abandon(brc);
            continue;
        }
        if (want_stats) sum.add(c, *hs, timing, ev0, L);
    }
    if (host_out) CU(cudaMemcpyAsync(out, dimg, npix * 16, cudaMemcpyDeviceToHost, s));
    if (host_index) CU(cudaMemcpyAsync(index, dindex, npix * 2, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (stats) sum.write(stats, launches);
    return FC_OK;
}

int32_t fc_merge_slabs(fc_ctx* c, const fc_geometry_pixel* const* slabs, uint32_t n_slabs, uint32_t width,
                       uint32_t height, uint32_t depth, fc_geometry_pixel* out) {
    if (!c || !slabs || !n_slabs || !out) return fail(FC_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    for (uint32_t i = 0; i < n_slabs; ++i)
        if (!is_device_ptr(slabs[i])) return fail(FC_ERR_INVALID, "fc_merge_slabs takes device pointers");
    if (!is_device_ptr(out)) return fail(FC_ERR_INVALID, "fc_merge_slabs takes device pointers");
    CU(c->image.ensure(std::max<size_t>(n_slabs * sizeof(void*), 16)));
    CU(cudaMemcpyAsync(c->image.p, slabs, n_slabs * sizeof(void*), cudaMemcpyHostToDevice, c->stream));
    launch_merge_slabs(c->image.as<const void*>(), n_slabs, width * height, depth, out, c->stream);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

uint32_t fc_tiles_per_rank(uint32_t width, uint32_t height, uint32_t root_tile, uint32_t n_ranks) {
    if (!root_tile || !n_ranks) return 0;
    const uint32_t rx = (width + root_tile - 1) / root_tile, ry = (height + root_tile - 1) / root_tile;
    uint32_t best = 0;
    std::vector<uint32_t> ids;
    for (uint32_t r = 0; r < n_ranks; ++r) {
        owned_tiles(rx, 0, ry, n_ranks, r, ids);
        best = std::max(best, uint32_t(ids.size()));
    }
    return best;
}

static int32_t tiles_copy(fc_ctx* c, const void* src, void* dst, uint32_t width, uint32_t height, uint32_t px_bytes,
                          uint32_t T, uint32_t n_ranks, int rank /* -1: unpack all */) {
    if (!c || !src || !dst) return fail(FC_ERR_INVALID, "null argument");
    if (px_bytes != 4 && px_bytes != 16) return fail(FC_ERR_INVALID, "px_bytes must be 4 or 16");
    if (!T || !n_ranks || (rank >= 0 && uint32_t(rank) >= n_ranks)) return fail(FC_ERR_INVALID, "bad tile interleave");
    if (!is_device_ptr(src) || !is_device_ptr(dst)) return fail(FC_ERR_INVALID, "fc_tiles_pack/unpack take device pointers");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const uint32_t rx = (width + T - 1) / T, ry = (height + T - 1) / T;
    const uint32_t per = fc_tiles_per_rank(width, height, T, n_ranks);
    // slot of every image tile inside the gathered buffer: owner * per + index in the owner's list
    const uint32_t key[4] = {rx, ry, n_ranks, T};
    if (memcmp(key, c->tile_slots_key, sizeof key) != 0 || !c->tile_slots.p) {
        std::vector<uint32_t> slots(size_t(rx) * ry), ids;
        for (uint32_t r = 0; r < n_ranks; ++r) {
            owned_tiles(rx, 0, ry, n_ranks, r, ids);
            for (size_t k = 0; k < ids.size(); ++k) slots[ids[k]] = r * per + uint32_t(k);
        }
        CU(cudaStreamSynchronize(c->stream));
        CU(c->tile_slots.ensure(slots.size() * 4));
        CU(cudaMemcpy(c->tile_slots.p, slots.data(), slots.size() * 4, cudaMemcpyHostToDevice));
        memcpy(c->tile_slots_key, key, sizeof key);
    }
    launch_tiles_copy(src, dst, width, height, px_bytes, T, rx, ry, c->tile_slots.as<uint32_t>(), n_ranks, per, rank, c->stream);
    CU(cudaGetLastError());
    return FC_OK;
}
int32_t fc_tiles_pack(fc_ctx* c, const void* image, uint32_t width, uint32_t height, uint32_t px_bytes, uint32_t root_tile,
                      uint32_t n_ranks, uint32_t rank, void* packed) {
    return tiles_copy(c, image, packed, width, height, px_bytes, root_tile, n_ranks, int(rank));
}
int32_t fc_tiles_unpack(fc_ctx* c, const void* gathered, uint32_t width, uint32_t height, uint32_t px_bytes, uint32_t root_tile,
                        uint32_t n_ranks, void* image) {
    return tiles_copy(c, gathered, image, width, height, px_bytes, root_tile, n_ranks, -1);
}

}  // extern "C"
