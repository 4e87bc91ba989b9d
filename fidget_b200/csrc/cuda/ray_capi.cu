// fc_raycast: the first inside sample along each ray (fidget_cuda.h), on ray.cu's kernels.  Rays run in passes planned
// like the tree calls' frames (pass_plan.h): each pass descends its rays' segments level by level, evaluates the leaf
// samples and finishes its hits.
#include <cmath>

#include "capi_internal.h"
#include "pass_plan.h"

namespace {

// The most rays a pass takes, and the most one pass plan covers (a call of more rays is planned in chunks)
constexpr uint32_t RAY_PASS_MAX = 1u << 16;
constexpr uint64_t RAY_PLAN_MAX = 1ull << 31;

// L of the descent: the fewest levels with 32^L >= steps, at least one
uint32_t ray_levels(uint32_t steps) {
    uint32_t L = 1;
    while ((1ull << (5 * L)) < steps) ++L;
    return L;
}
// List l (1 .. L, L being the leaf list) over n rays: at most every segment of level l - 1, which are 32^(L - l + 1)
// samples long
uint64_t ray_list(uint64_t n, uint32_t steps, uint32_t L, int l, uint64_t limit) {
    const uint64_t len = 1ull << (5 * (L - uint32_t(l) + 1));
    return std::min(n * ((steps + len - 1) / len), limit);
}

int32_t check_rays(const fc_ray* rays, uint64_t n, uint32_t steps) {
    for (uint64_t i = 0; i < n; ++i) {
        const fc_ray& r = rays[i];
        bool ok = std::isfinite(r.t0) && std::isfinite(r.dt) && r.dt > 0.0f;
        for (int a = 0; a < 3; ++a) ok = ok && std::isfinite(r.origin[a]) && std::isfinite(r.dir[a]);
        const float t_last = r.t0 + float(steps - 1u) * r.dt;
        if (!ok || !std::isfinite(t_last))
            return fail(FC_ERR_INVALID, "ray " + std::to_string(i) +
                                            ": origin, dir, t0 and dt must be finite, dt > 0, and t finite at the last sample");
    }
    return FC_OK;
}

// The passes of rays [r0, r0 + n) of a checked call into hits (offset alike).  The caller holds the context's lock.
int32_t ray_passes(fc_ctx* c, const fc_tape* tape, uint32_t steps, const VarBind& vb, bool timing, const fc_ray* rays,
                   bool rays_dev, fc_ray_hit* hits, bool hits_dev, uint64_t r0, uint32_t n, fc_raycast_info& info,
                   const CallCancel& cc) {
    const uint32_t L = ray_levels(steps);
    cudaStream_t s = c->stream;
    const uint64_t cap_limit = list_cap_limit();
    PassPlan plan(n, std::min(n, RAY_PASS_MAX), [=](uint32_t k) {
        PassLimits lim;
        lim.arena_cap = arena_clauses(c);
        for (int l = 1; l <= int(L); ++l) {
            lim.worst[l] = ray_list(k, steps, L, l, ~0ull);
            lim.cap[l] = ray_list(k, steps, L, l, cap_limit);
        }
        return lim;
    });
    const int grid = c->sm_count * env_int("FIDGET_B200_BLOCKS_PER_SM", 6);
    const uint32_t cw = choice_words(tape);
    while (plan.more()) {
        const PassPlan::Range pr = plan.take();
        const uint64_t f0 = r0 + pr.f0;
        // scratch: choice words, arena, counters and the tally after them, stats, job lists, the rays' best words and
        // staged rays and hits
        CU(c->choice_scratch.ensure(size_t(grid) * WARPS_PER_BLOCK * cw * 32 * 4));
        CU(c->arena.ensure(c->arena_bytes));
        CU(c->counters.ensure(sizeof(Counters) + 64));
        CU(c->stats.ensure(sizeof(Stats)));
        uint64_t cap[MAX_LEVELS + 1] = {};
        for (int l = 1; l <= int(L); ++l) {
            cap[l] = ray_list(pr.n, steps, L, l, cap_limit);
            CU(c->jobs[l].ensure(cap[l] * sizeof(TileJob)));
        }
        RayPass rp{};
        Ray* d_rays = nullptr;
        RayHit* d_hits = nullptr;
        CU(carve(c->image, [&](Carve& cv) {
            cv.take(rp.best, size_t(pr.n) * 4);
            if (!rays_dev) cv.take(d_rays, size_t(pr.n) * sizeof(Ray));
            if (!hits_dev) cv.take(d_hits, size_t(pr.n) * sizeof(RayHit));
        }));
        rp.rays = rays_dev ? reinterpret_cast<const Ray*>(rays + f0) : d_rays;
        rp.hits = hits_dev ? reinterpret_cast<RayHit*>(hits + f0) : d_hits;
        rp.tally = reinterpret_cast<unsigned long long*>(c->counters.as<char>() + sizeof(Counters));
        rp.n_rays = pr.n;
        rp.steps = steps;
        CU(cudaMemsetAsync(c->counters.p, 0, sizeof(Counters) + 64, s));
        CU(cudaMemsetAsync(c->stats.p, 0, sizeof(Stats), s));
        CU(cudaMemsetAsync(rp.best, 0xff, size_t(pr.n) * 4, s));
        if (!rays_dev) CU(cudaMemcpyAsync(d_rays, rays + f0, size_t(pr.n) * sizeof(Ray), cudaMemcpyHostToDevice, s));
        if (timing) CU(cudaEventRecord(get_event(c, 0), s));
        LevelParams p{};
        p.root_tape = tape_ref(tape);
        p.arena = c->arena.as<uint2>();
        p.arena_cap = arena_clauses(c);
        p.choice_scratch = c->choice_scratch.as<uint32_t>();
        p.choice_words = cw;
        p.ctr = c->counters.as<Counters>();
        p.stats = c->stats.as<Stats>();
        p.vb = vb;
        p.cancel = cc.ref;
        for (uint32_t l = 0; l <= L; ++l) {
            p.level = int(l);
            p.root_mode = l == 0;
            p.jobs_in = l ? c->jobs[l].as<TileJob>() : nullptr;
            p.cap_in = uint32_t(cap[l]);
            p.jobs_out = l < L ? c->jobs[l + 1].as<TileJob>() : nullptr;
            p.cap_out = l < L ? uint32_t(cap[l + 1]) : 0u;
            rp.seg = 1u << (5 * (L - l));
            // level 0: a warp per 32 rays; later, a warp per queued segment, at most every segment of the level above
            const uint64_t warps = l ? cap[l] : (uint64_t(pr.n) + 31) / 32;
            const int blocks = int(std::max<uint64_t>(1, std::min<uint64_t>((warps + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, grid)));
            if (l < L) launch_ray_level(p, rp, blocks, s);
            else launch_ray_leaf(p, rp, blocks, s);
        }
        launch_ray_hits(rp, tape_ref(tape), vb, cc.ref, s);
        if (timing) CU(cudaEventRecord(get_event(c, 1), s));
        CU(cudaGetLastError());
        struct { Counters ctr; unsigned long long tally[8]; } st;
        if (int32_t wrc = wait_read(c, s, cc, &st, c->counters.p, sizeof(Counters) + 64)) return wrc;
        bool split = false;
        if (!plan.observe(st.ctr, 0, pr, split)) return device_error(st.ctr.error);
        if (split) continue;
        if (!hits_dev) CU(cudaMemcpy(hits + f0, d_hits, size_t(pr.n) * sizeof(RayHit), cudaMemcpyDeviceToHost));
        Stats hs;
        CU(cudaMemcpy(&hs, c->stats.p, sizeof hs, cudaMemcpyDeviceToHost));
        for (uint32_t l = 0; l < L; ++l) info.evaluated[l] += hs.evaluated[l];
        info.n_hits += st.tally[0];
        info.n_proven += st.tally[1];
        info.leaf_samples += st.tally[2];
        ++info.passes;
        if (timing) {
            float ms = 0;
            cudaEventElapsedTime(&ms, get_event(c, 0), get_event(c, 1));
            info.device_ms += ms;
        }
    }
    return FC_OK;
}

// Every hit a miss: k = FC_RAY_MISS, the other fields 0
int32_t clear_hits(fc_ctx* c, fc_ray_hit* hits, uint64_t n) {
    if (!hits || !n) return FC_OK;
    if (!is_device_ptr(hits)) {
        memset(hits, 0, size_t(n) * sizeof *hits);
        for (uint64_t i = 0; i < n; ++i) hits[i].k = FC_RAY_MISS;
        return FC_OK;
    }
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    launch_ray_clear(reinterpret_cast<RayHit*>(hits), n, c->stream);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

int32_t raycast(fc_ctx* c, const fc_tape* tape, const fc_raycast_cfg* cfg, const fc_ray* rays, uint64_t n_rays,
                fc_ray_hit* hits, fc_raycast_info& info) {
    if (!tape || !cfg) return fail(FC_ERR_INVALID, "null argument");
    if (n_rays && (!rays || !hits)) return fail(FC_ERR_INVALID, "null rays or hits");
    if (cfg->steps == 0 || cfg->steps > FC_RAY_MAX_STEPS)
        return fail(FC_ERR_INVALID, "steps must be 1 .. FC_RAY_MAX_STEPS (2^24)");
    if (int32_t rc = check_tree_call(tape, 3, 0, cfg, 1, "fc_raycast")) return rc;
    VarBind vb;
    if (int32_t rc = bind_vars(tape, cfg->var_values, cfg->n_var_values, vb)) return rc;
    if (!n_rays) return FC_OK;
    const bool rays_dev = is_device_ptr(rays), hits_dev = is_device_ptr(hits);
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    std::vector<fc_ray> staged;
    const fc_ray* host_rays = rays;
    if (rays_dev) {   // the checks read the rays on the host: copied in the call's stream order, after the caller's work
        staged.resize(n_rays);
        CU(cudaMemcpyAsync(staged.data(), rays, size_t(n_rays) * sizeof(fc_ray), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        host_rays = staged.data();
    }
    if (int32_t rc = check_rays(host_rays, n_rays, cfg->steps)) return rc;
    const bool timing = (cfg->flags & FC_FLAG_TIMING) != 0;
    for (uint64_t r0 = 0; r0 < n_rays; r0 += RAY_PLAN_MAX)
        if (int32_t rc = ray_passes(c, tape, cfg->steps, vb, timing, rays, rays_dev, hits, hits_dev, r0,
                                    uint32_t(std::min(RAY_PLAN_MAX, n_rays - r0)), info, cc))
            return rc;
    return FC_OK;
}

}  // namespace

extern "C" {

int32_t fc_raycast(fc_ctx* c, const fc_tape* tape, const fc_raycast_cfg* cfg, const fc_ray* rays, uint64_t n_rays,
                   fc_ray_hit* hits, fc_raycast_info* info) {
    static_assert(sizeof(fc_ray) == sizeof(Ray) && sizeof(fc_ray) == 32, "fc_ray layout");
    static_assert(sizeof(fc_ray_hit) == sizeof(RayHit) && sizeof(fc_ray_hit) == 40, "fc_ray_hit layout");
    static_assert(sizeof(fc_raycast_info) == 96, "fc_raycast_info layout");
    if (info) memset(info, 0, sizeof *info);
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    fc_raycast_info acc{};
    const int32_t rc = raycast(c, tape, cfg, rays, n_rays, hits, acc);
    if (rc) {
        const std::string msg = g_err;
        clear_hits(c, hits, n_rays);
        return fail(rc, msg);
    }
    if (info) *info = acc;
    return FC_OK;
}

}  // extern "C"
