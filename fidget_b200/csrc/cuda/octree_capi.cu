// fc_octree_sample: the sampling half of fidget-mesh's Octree::build.
#include "capi_internal.h"
#include "pass_plan.h"

template <class F>
int32_t check_tree_call(const fc_tape* tape, int dim, uint32_t depth, const F* table, uint32_t n, const char* what) {
    if (depth > uint32_t(dim == 3 ? FC_MAX_OCTREE_DEPTH : FC_MAX_QUADTREE_DEPTH))
        return fail(FC_ERR_INVALID, dim == 3 ? "octree depth too large" : "quadtree depth too large");
    if (!table && n) return fail(FC_ERR_INVALID, dim == 3 ? "null frames" : "null slices");
    for (uint32_t k = 0; k < n; ++k)
        if (table[k].n_var_values > FC_MAX_VARS) return fail(FC_ERR_INVALID, "too many variable values");
    if (tape->info.mem_count) return fail(FC_ERR_UNSUPPORTED, std::string(what) + " needs a tape without memory spills");
    if (tape->info.n_outputs != 1) return fail(FC_ERR_INVALID, "ShapeTape has multiple outputs");
    return FC_OK;
}
template int32_t check_tree_call(const fc_tape*, int, uint32_t, const fc_mesh_frame*, uint32_t, const char*);
template int32_t check_tree_call(const fc_tape*, int, uint32_t, const fc_contour_slice*, uint32_t, const char*);
template int32_t check_tree_call(const fc_tape*, int, uint32_t, const fc_raycast_cfg*, uint32_t, const char*);

int32_t bind_frame(const fc_tape* tape, uint32_t has_transform, const float* world_to_model, float z, const float* values,
                   uint32_t n_values, MeshFrame& f) {
    memcpy(f.mat.m, world_to_model, sizeof f.mat.m);
    f.z = z;
    f.has_transform = has_transform;
    bool identity = true;
    for (int i = 0; i < 16; ++i) identity &= f.mat.m[i] == (i % 5 == 0 ? 1.0f : 0.0f);
    f.to_model = has_transform && !identity;
    return bind_vars(tape, values, n_values, f.vb);
}

PassPlan tree_passes(fc_ctx* c, uint32_t n, uint32_t n_max, uint32_t D, int dim, int levels, double leaf_bytes) {
    const uint64_t cap_limit = list_cap_limit();
    return PassPlan(n, n_max, [=](uint32_t k) {
        PassLimits lim;
        lim.arena_cap = arena_clauses(c);
        for (int l = 1; l <= levels; ++l) {   // the worst case: every cell of k trees at depth min(l, D) queued
            lim.worst[l] = tree_list(k, dim, D, l, ~0ull);
            lim.cap[l] = tree_list(k, dim, D, l, cap_limit);
        }
        lim.extra_on = leaf_bytes > 0;
        lim.extra_scale = leaf_bytes;
        lim.extra_cap = FC_FRAMES_PASS_BYTES;
        return lim;
    });
}

int32_t tree_scratch(fc_ctx* c, const fc_tape* tape, uint32_t D, int dim, uint64_t n_roots, uint64_t cap, TreeScratch& t) {
    t.D = D;
    t.dim = dim;
    t.n_roots = n_roots;
    t.grid_blocks = c->sm_count * env_int("FIDGET_B200_BLOCKS_PER_SM", 6);
    t.choice_words = choice_words(tape);
    CU(c->choice_scratch.ensure(size_t(t.grid_blocks) * WARPS_PER_BLOCK * t.choice_words * 32 * 4));
    CU(c->arena.ensure(c->arena_bytes));
    CU(c->counters.ensure(sizeof(Counters) + 64));
    CU(c->stats.ensure(sizeof(Stats)));
    const uint64_t cap_limit = list_cap_limit();
    for (int l = 1; l <= int(D) + 1; ++l) {
        t.level_cap[l] = tree_list(n_roots, dim, D, l, cap_limit);
        CU(c->jobs[l].ensure(t.level_cap[l] * sizeof(TileJob)));
    }
    CU(c->leaf_tapes.ensure(std::max<uint64_t>(cap, 1) * sizeof(TapeRef)));
    CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters) + 64, c->stream));
    return FC_OK;
}

LevelParams tree_level(fc_ctx* c, const fc_tape* tape, const TreeScratch& t, int l, const ContourSlice& f0,
                       const CallCancel& cc) {
    LevelParams p{};
    p.level = l;
    p.tile = 1u << (t.D - uint32_t(l));
    p.n_axis = l ? 2 : 0;
    p.is_last = (l == int(t.D));
    p.root_mode = (l == 0);
    p.root_tape = tape_ref(tape);
    p.jobs_in = l ? c->jobs[l].as<TileJob>() : nullptr;
    p.cap_in = l ? uint32_t(t.level_cap[l]) : 0;
    p.jobs_out = c->jobs[l + 1].as<TileJob>();
    p.cap_out = uint32_t(t.level_cap[l + 1]);
    p.arena = c->arena.as<uint2>();
    p.arena_cap = arena_clauses(c);
    p.choice_scratch = c->choice_scratch.as<uint32_t>();
    p.choice_words = t.choice_words;
    p.ctr = c->counters.as<Counters>();
    p.mode = 1;
    p.has_transform = f0.has_transform;
    p.cell_h = 2.0f / float(1u << t.D);
    p.vb = f0.vb;
    p.cancel = cc.ref;
    p.roots_x = p.roots_z = 1;
    p.roots_y = uint32_t(t.n_roots);   // one root cell per frame or slice, stacked along Y
    p.frame_rows = 1u << t.D;
    p.mat = f0.mat;
    // the extents: the octree's stacked grid (2^D x n 2^D x 2^D cells), one slice of the quadtree (2^D x 2^D x 1)
    p.width = 1u << t.D;
    p.height = t.dim == 3 ? uint32_t(t.n_roots) << t.D : 1u << t.D;
    p.depth = t.dim == 3 ? 1u << t.D : 1u;
    return p;
}

// The sampler's launches over n frames (fr: host; with n > 1 also d_fr on the device): the interval levels of one root
// cell per frame, the frames stacked along Y (frame k owns the cell rows [k * 2^D, (k + 1) * 2^D)), then the leaf and
// gradient kernels into `dout` (`cap` leaves; *d_n_out counts the surface leaves, beyond cap too).  One frame takes the
// single-frame kernels with the frame in the launch parameters.  stats: the level and leaf statistics of
// fc_octree_stats (c->stats and the words after the counters).  t0 (or null) is recorded once the scratch is set up.
int32_t octree_enqueue(fc_ctx* c, const fc_tape* tape, uint32_t D, const MeshFrame* fr, uint32_t n, const MeshFrame* d_fr,
                       OctreeLeaf* dout, uint64_t cap, bool stats, cudaEvent_t t0, const CallCancel& cc, uint32_t* launches) {
    const int L = int(D) + 1;   // interval levels: depth 0 (the root cell) .. D
    cudaStream_t s = c->stream;
    const bool stack = n > 1;
    TreeScratch t;
    if (int32_t trc = tree_scratch(c, tape, D, 3, n, cap, t)) return trc;
    if (stats) CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
    // extra device words after Counters: [0] n_out, then 5 u64 leaf statistics (8-byte aligned)
    uint32_t* d_n_out = reinterpret_cast<uint32_t*>(c->counters.as<char>() + sizeof(Counters));
    unsigned long long* d_leaf_stats = reinterpret_cast<unsigned long long*>(c->counters.as<char>() + sizeof(Counters) + 8);
    if (t0) CU(cudaEventRecord(t0, s));
    for (int l = 0; l < L; ++l) {
        LevelParams p = tree_level(c, tape, t, l, fr[0], cc);
        p.stats = stats ? c->stats.as<Stats>() : nullptr;
        if (stack) launch_tree_level(p, 3, d_fr, t.blocks(l), s);
        else launch_interval_level_3d(p, t.blocks(l), s);
    }
    OctreeLeafParams q{};
    q.jobs = c->jobs[L].as<TileJob>();
    q.cap_jobs = uint32_t(t.level_cap[L]);
    q.ctr = c->counters.as<Counters>();
    q.list = L; q.cursor = L;
    q.cell_h = 2.0f / float(1u << D);
    q.has_transform = fr[0].has_transform;
    q.mat = fr[0].mat;
    q.vb = fr[0].vb;
    q.out = dout;
    q.out_tapes = c->leaf_tapes.as<TapeRef>();
    q.cap_out = uint32_t(cap);
    q.n_out = d_n_out;
    q.stats = stats ? d_leaf_stats : nullptr;
    q.cancel = cc.ref;
    launch_octree_leaf(q, c->sm_count * 8, s, stack ? d_fr : nullptr, 1u << D);
    launch_octree_grads(q, c->sm_count * 8, s, stack ? d_fr : nullptr, 1u << D);
    if (launches) *launches = uint32_t(L) + 2;
    CU(cudaGetLastError());
    return FC_OK;
}

// Device half: runs the sampler into `dout` (device memory, `cap` leaves); *n_out = surface leaves found
// (FC_ERR_INVALID when it exceeds cap).  Takes the context lock.  `cc`: the call's cancellation (begin_call).
int32_t octree_sample_device(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, OctreeLeaf* dout, uint64_t cap,
                             uint32_t* n_out_p, fc_octree_stats* stats, const CallCancel& cc) {
    static_assert(sizeof(fc_octree_leaf) == sizeof(OctreeLeaf) && sizeof(OctreeLeaf) == 348, "leaf layout");
    if (!c || !tape || !cfg || !n_out_p) return fail(FC_ERR_INVALID, "null argument");
    if (int32_t rc = check_tree_call<fc_mesh_frame>(tape, 3, cfg->depth, nullptr, 0, "the octree sampler")) return rc;
    if (cap > 0xfffffff0ull) return fail(FC_ERR_INVALID, "leaf capacity too large");
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    MeshFrame one{};
    if (int32_t vrc = bind_frame(tape, cfg->has_transform, cfg->world_to_model, 0.0f, cfg->var_values, cfg->n_var_values,
                                 one))
        return vrc;
    const uint32_t D = cfg->depth;
    cudaStream_t s = c->stream;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    uint32_t launches = 0;
    if (int32_t rc = octree_enqueue(c, tape, D, &one, 1, nullptr, dout, cap, true, timing ? get_event(c, 0) : nullptr, cc,
                                    &launches))
        return rc;
    if (timing) CU(cudaEventRecord(get_event(c, 1), s));
    uint32_t* d_n_out = reinterpret_cast<uint32_t*>(c->counters.as<char>() + sizeof(Counters));
    unsigned long long* d_leaf_stats = reinterpret_cast<unsigned long long*>(c->counters.as<char>() + sizeof(Counters) + 8);
    uint32_t n_out = 0;
    if (int32_t wrc = wait_read(c, s, cc, &n_out, d_n_out, 4)) {
        *n_out_p = 0;
        if (stats) memset(stats, 0, sizeof *stats);
        return wrc;
    }
    *n_out_p = n_out;
    int32_t rc = check_device_errors(c);
    if (n_out > cap) rc = fail(FC_ERR_INVALID, "leaf buffer too small: " + std::to_string(n_out) + " surface leaves");
    if (stats) {
        memset(stats, 0, sizeof *stats);
        Stats h;
        Counters hc;
        unsigned long long ls[5];
        CU(cudaMemcpy(&h, c->stats.p, sizeof h, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(&hc, c->counters.p, sizeof hc, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(ls, d_leaf_stats, sizeof ls, cudaMemcpyDeviceToHost));
        for (int l = 0; l < 16 && l < MAX_LEVELS; ++l) {
            stats->evaluated[l] = h.evaluated[l];
            stats->full[l] = h.filled_inside[l];
            stats->empty[l] = h.filled_outside[l];
            stats->ambiguous[l] = h.ambiguous[l];
        }
        stats->leaf_empty = ls[0]; stats->leaf_full = ls[1]; stats->leaf_surface = ls[2];
        stats->float_points = ls[3]; stats->grad_points = ls[4];
        stats->arena_bytes_used = hc.arena_top * sizeof(uint2);
        stats->kernel_launches = launches;
        if (timing) cudaEventElapsedTime(&stats->total_ms, c->events[0], c->events[1]);
    }
    return rc;
}

extern "C" {

int32_t fc_octree_sample(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, fc_octree_leaf* out, uint64_t cap,
                         uint64_t* n_leaves, fc_octree_stats* stats) {
    if (!c || !tape || !cfg || !n_leaves || (!out && cap)) return fail(FC_ERR_INVALID, "null argument");
    *n_leaves = 0;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    const bool out_dev = is_device_ptr(out);
    OctreeLeaf* dout = reinterpret_cast<OctreeLeaf*>(out);
    if (!out_dev) {
        std::lock_guard<std::mutex> guard(c->mu);
        CU(cudaSetDevice(c->device));
        CU(c->image.ensure(std::max<uint64_t>(cap, 1) * sizeof(OctreeLeaf)));
        dout = c->image.as<OctreeLeaf>();
    }
    uint32_t n_out = 0;
    int32_t rc = octree_sample_device(c, tape, cfg, dout, cap, &n_out, stats, cc);
    *n_leaves = n_out;
    if (!rc && !out_dev && n_out) CU(cudaMemcpy(out, dout, size_t(n_out) * sizeof(OctreeLeaf), cudaMemcpyDeviceToHost));
    return rc;
}

}  // extern "C"
