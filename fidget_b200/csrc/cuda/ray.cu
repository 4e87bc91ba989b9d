// fc_raycast's kernels: the interval levels of the descent along each ray, the leaf samples of the ambiguous 32-sample
// segments, and the value and gradient of the root tape at each hit.  The host side is ray_capi.cu; the contract is in
// fidget_cuda.h.
#include <algorithm>

#include "level_job.cuh"

namespace fdev {

// Sample k of ray r, one rounding per operation: t_k = t0 + k dt, x_k = o + t_k d
__device__ __forceinline__ float ray_t(const Ray& r, uint32_t k) { return __fadd_rn(r.t0, __fmul_rn(float(k), r.dt)); }
__device__ __forceinline__ float ray_x(const Ray& r, int a, float t) { return __fadd_rn(r.o[a], __fmul_rn(t, r.d[a])); }

// Ray i, one 4-byte load per field: a caller's device table of fc_ray is only 4-byte aligned
__device__ __forceinline__ Ray load_ray(const Ray* rays, uint32_t i) {
    const float* q = reinterpret_cast<const float*>(rays + i);
    return Ray{{q[0], q[1], q[2]}, {q[3], q[4], q[5]}, q[6], q[7]};
}

// The smallest candidate seen so far (any value that is not below the final one is good enough: a stale read only skips
// less)
__device__ __forceinline__ uint32_t best_k(const RayPass& r, uint32_t ray) { return __ldcg(r.best + ray) >> 1; }

// One interval level.  A warp evaluates 32 segments: at level 0 one whole ray per lane, later the 32 children of one
// queued segment.  A segment's box is spanned by its end samples (fidget_cuda.h: the samples are monotone in k);
// upper < 0 lowers the ray's best to the segment's first sample (proven), lower > 0 drops it, and anything else is
// queued for the next level (the leaf launch after the last), with its simplified tape when that is shorter.
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) k_ray_level(const __grid_constant__ LevelParams p,
                                                                    const __grid_constant__ RayPass rp) {
    __shared__ uint32_t live_s[WARPS_PER_BLOCK][8][32];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t gw = blockIdx.x * WARPS_PER_BLOCK + wib;
    uint32_t* cs = p.choice_scratch + size_t(gw) * p.choice_words * 32u + lane;
    itv slots[REG_SLOTS];
    const uint32_t n_jobs = p.root_mode ? (rp.n_rays + 31u) / 32u : min(p.ctr->n_jobs[p.level], p.cap_in);
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.level], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_LEVEL0 + p.level, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        uint32_t ray, a;
        bool valid;
        TapeRef tr;
        if (p.root_mode) {
            ray = j * 32u + uint32_t(lane);
            valid = ray < rp.n_rays;
            if (!valid) ray = 0;
            a = 0;
            tr = p.root_tape;
        } else {
            const TileJob jb = p.jobs_in[j];
            ray = jb.x;
            a = jb.y + uint32_t(lane) * rp.seg;
            valid = a < rp.steps && a < best_k(rp, ray);
            tr = jb.tape;
        }
        const Ray r = load_ray(rp.rays, ray);
        const uint32_t b = valid ? min(a + (rp.seg - 1u), rp.steps - 1u) : a;   // (seg - 1 first: 32^5 - 1 + a fits)
        const float ta = ray_t(r, a), tb = ray_t(r, b);
        itv box[3];
        for (int ax = 0; ax < 3; ++ax) {
            const float xa = ray_x(r, ax, ta), xb = ray_x(r, ax, tb);
            box[ax] = xb < xa ? iv(xb, xa) : iv(xa, xb);
        }
        ChoicePacker pk;
        pk.base = cs;
        itv v = iv_nan();
        run_interval(
            tr.ptr, tr.n_ops, slots,
            [&](uint32_t i) { return pick_input(p.vb, i, box[0], box[1], box[2], [](float f) { return iv1(f); }); }, pk,
            [&](uint32_t oi, itv o) { if (oi == 0) v = o; });
        pk.finish();
        const bool inside = valid && v.y < 0.0f;
        const bool outside = valid && !inside && v.x > 0.0f;
        const bool amb = valid && !inside && !outside;
        if (inside) atomicMin(rp.best + ray, a << 1 | 1u);
        if (p.stats) {
            const uint32_t mv = __ballot_sync(FULL, valid);
            if (lane == 0 && mv) atomicAdd(&p.stats->evaluated[p.level], (unsigned long long)__popc(mv));
        }
        bool kept;
        const TapeRef child = simplify_children<false>(p, tr, amb, pk, cs, live_s[wib], lane, kept);
        const uint32_t mamb = __ballot_sync(FULL, amb);
        if (mamb) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(&p.ctr->n_jobs[p.level + 1], uint32_t(__popc(mamb)));
            base = __shfl_sync(FULL, base, 0);
            if (amb) {
                const uint32_t slot = base + __popc(mamb & lanemask_lt());
                if (slot < p.cap_out) {
                    TileJob o;
                    o.x = ray;
                    o.y = a;
                    o.z = 0;
                    o.pad = 0;
                    o.tape = child;
                    p.jobs_out[slot] = o;
                } else {
                    atomicOr(&p.ctr->error, 2u);
                }
            }
        }
    }
}
void launch_ray_level(const LevelParams& p, const RayPass& r, int blocks, cudaStream_t s) {
    k_ray_level<<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(p, r);
}

// The leaf samples: one warp per ambiguous 32-sample segment, one sample per lane with the segment's tape; the first
// sample with a value < 0 lowers the ray's best.
__global__ void __launch_bounds__(128) k_ray_leaf(const __grid_constant__ LevelParams p, const __grid_constant__ RayPass rp) {
    const int lane = threadIdx.x & 31;
    float2 slots[REG_SLOTS];
    const uint32_t n_jobs = min(p.ctr->n_jobs[p.level], p.cap_in);
    unsigned long long n_samples = 0;
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.level], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_RAY_LEAF, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        const TileJob jb = p.jobs_in[j];
        const uint32_t ray = jb.x;
        uint32_t bk = lane == 0 ? best_k(rp, ray) : 0u;
        if (__shfl_sync(FULL, bk, 0) <= jb.y) continue;   // (read once: the warp must agree)
        const uint32_t k = jb.y + uint32_t(lane);
        const bool valid = k < rp.steps;
        const Ray r = load_ray(rp.rays, ray);
        const float t = ray_t(r, k);
        const float x = ray_x(r, 0, t), y = ray_x(r, 1, t), z = ray_x(r, 2, t);
        const float2 v = run_f32x2(jb.tape.ptr, jb.tape.n_ops, slots, [&](uint32_t i) {
            return pick_input(p.vb, i, make_float2(x, x), make_float2(y, y), make_float2(z, z),
                              [](float f) { return make_float2(f, f); });
        });
        const uint32_t m = __ballot_sync(FULL, valid && v.x < 0.0f);
        if (lane == 0) {
            n_samples += min(32u, rp.steps - jb.y);
            if (m) atomicMin(rp.best + ray, (jb.y + uint32_t(__ffs(m) - 1)) << 1);
        }
    }
    if (lane == 0 && n_samples) atomicAdd(rp.tally + 2, n_samples);
}
void launch_ray_leaf(const LevelParams& p, const RayPass& r, int blocks, cudaStream_t s) {
    k_ray_leaf<<<blocks, 128, 0, s>>>(p, r);
}

// The hits: one thread per ray.  A ray with a candidate gets its t, position, and the root tape's value (the f32
// interpreter, as fc_float_slice_eval) and gradient (as fc_grad_slice_eval) there; the others are misses.
__global__ void __launch_bounds__(128) k_ray_hits(const __grid_constant__ RayPass rp, const __grid_constant__ TapeRef root,
                                                  const __grid_constant__ VarBind vb, const __grid_constant__ CancelRef cancel) {
    float2 fslots[REG_SLOTS];
    grd gslots[REG_SLOTS];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (cancel_poll(cancel, CS_RAY_HITS, i >> 5)) return;   // (a cancelled call's hits are cleared by the host)
    if (i >= rp.n_rays) return;
    const uint32_t w = rp.best[i];
    RayHit h{};
    h.k = 0xFFFFFFFFu;
    if (w != 0xFFFFFFFFu) {
        const Ray r = load_ray(rp.rays, i);
        h.k = w >> 1;
        h.flags = w & 1u;
        h.t = ray_t(r, h.k);
        for (int a = 0; a < 3; ++a) h.pos[a] = ray_x(r, a, h.t);
        const float x = h.pos[0], y = h.pos[1], z = h.pos[2];
        h.value = run_f32x2(root.ptr, root.n_ops, fslots, [&](uint32_t k) {
                      return pick_input(vb, k, make_float2(x, x), make_float2(y, y), make_float2(z, z),
                                        [](float f) { return make_float2(f, f); });
                  }).x;
        const grd g = run_grad(root.ptr, root.n_ops, gslots, [&](uint32_t k) {
            return pick_input(vb, k, gr(x, 1.0f, 0.0f, 0.0f), gr(y, 0.0f, 1.0f, 0.0f), gr(z, 0.0f, 0.0f, 1.0f),
                              [](float f) { return gr1(f); });
        });
        h.grad[0] = g.y; h.grad[1] = g.z; h.grad[2] = g.w;
        atomicAdd(rp.tally + 0, 1ull);
        if (h.flags) atomicAdd(rp.tally + 1, 1ull);
    }
    rp.hits[i] = h;
}
void launch_ray_hits(const RayPass& r, const TapeRef& root, const VarBind& vb, const CancelRef& cancel, cudaStream_t s) {
    k_ray_hits<<<(r.n_rays + 127u) / 128u, 128, 0, s>>>(r, root, vb, cancel);
}

__global__ void k_ray_clear(RayHit* hits, uint64_t n) {
    for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
        RayHit h{};
        h.k = 0xFFFFFFFFu;
        hits[i] = h;
    }
}
void launch_ray_clear(RayHit* hits, uint64_t n, cudaStream_t s) {
    if (n) k_ray_clear<<<unsigned(std::min<uint64_t>((n + 255) / 256, 4096)), 256, 0, s>>>(hits, n);
}

}  // namespace fdev
