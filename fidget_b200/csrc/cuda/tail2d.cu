// Fused tail of fc_render2d: every interval level after the root level, the leaf pixels and the fill
// painting in ONE persistent launch (one CTA slot per SM x resident CTAs, each warp an independent worker).
//
// Launching one kernel per level makes the frame a chain of latency-bound stages: level 1 of prospero 4096^2
// keeps 763 warps busy for as long as its LONGEST tape takes while 92 % of the GPU idles, and level 2 cannot
// start before the last of them ends.  Here the work is a dependency-ordered queue instead: a parent tile is
// a job; finishing it publishes its ambiguous children as jobs of the next level (or as leaf-tile jobs), which
// any idle warp picks up at once; warps with nothing else to do paint the tiles the interval levels proved
// inside / outside.  The frame then lasts as long as its critical path (slowest root -> its slowest child ->
// one leaf tile), not as the sum over levels of the slowest job of each level.
//
// Queue protocol (all state in `Counters`, zeroed per render):
//   * n_jobs[l] / cursor[l]: slots reserved by producers / claimed by consumers of level l (CAS, never
//     overshooting, so a warp never holds a claim on a job that does not exist yet);
//   * a job or fill record becomes valid when its ready mark equals this render's epoch -- written after the
//     fields and a __threadfence(); consumers spin on the mark, then read the record from L2 (__ldcg);
//   * child tapes are written to whole 128-byte lines of the arena (level_job.cuh), so the cached tape loads
//     of the interpreters can never hit a line that an SM cached before another SM filled it;
//   * outstanding = jobs queued or running; a producer adds its children BEFORE retiring itself, so the count
//     reaches zero exactly when no interval / pixel work is left; fills are drained after that.
// Every spin is bounded (error bit 2) -- a logic error must not hang the device.  A cancelled call (fc_ctx_set_cancel)
// ends every spin and every warp at its next poll, without an error bit.
#include <algorithm>

#include "level_job.cuh"

namespace fdev {

// leaf tile: one warp, two pixels per lane (k_pixels_2d's body)
__device__ __forceinline__ void pixel_job(const PixelParams& p, const TileJob& job, float2* slots, int lane,
                                          unsigned long long& shaded) {
    const uint32_t T = p.tile, npix = T * T;
    const uint32_t cx = job.x, cy = job.y;
    const TapeRef tr = job.tape;
    const uint2* tape = tr.ptr;
    for (uint32_t base = 0; base < npix; base += 64u) {
        uint32_t p0 = base + lane, p1 = p0 + 32u;
        bool v0 = p0 < npix, v1 = p1 < npix;
        uint32_t i0 = (v0 ? p0 : 0u) % T, j0 = (v0 ? p0 : 0u) / T;
        uint32_t i1 = (v1 ? p1 : 0u) % T, j1 = (v1 ? p1 : 0u) / T;
        float x0, y0, z0, x1, y1, z1;
        xform_f32(p.mat, float(cx + i0), float(cy + j0), p.z2d, x0, y0, z0);
        xform_f32(p.mat, float(cx + i1), float(cy + j1), p.z2d, x1, y1, z1);
        const float2 X = make_float2(x0, x1), Y = make_float2(y0, y1), Z = make_float2(z0, z1);
        float2 r = run_f32x2<false>(tape, tr.n_ops, slots, [&](uint32_t i) {
            return pick_input(p.vb, i, X, Y, Z, [](float f) { return make_float2(f, f); });
        });
        if (r.x != r.x) r.x = nanf_();   // RawDistancePixel::from(f32): canonical NaN (pixel.rs:234-240)
        if (r.y != r.y) r.y = nanf_();
        uint32_t gx0 = cx + i0, gy0 = cy + j0, gx1 = cx + i1, gy1 = cy + j1;
        if (v0 && gx0 < p.width && gy0 < p.height) p.out[size_t(gy0) * p.width + gx0] = r.x;
        if (v1 && gx1 < p.width && gy1 < p.height) p.out[size_t(gy1) * p.width + gx1] = r.y;
        shaded += (v0 ? 1 : 0) + (v1 ? 1 : 0);
    }
}

// one interval-proven tile painted by one warp
__device__ __forceinline__ void fill_job(uint32_t T, uint32_t width, uint32_t height, float* out, uint4 rec, int lane) {
    const float v = __uint_as_float(rec.z);
    const bool vec_ok = (width % 4u == 0u) && ((reinterpret_cast<uintptr_t>(out) & 15u) == 0u) && (T % 4u == 0u);
    const uint32_t tile_px = T * T;
    for (uint32_t pix = uint32_t(lane) * 4u; pix < tile_px; pix += 128u) {
        if (vec_ok) {
            const uint32_t x = rec.x + pix % T, y = rec.y + pix / T;
            if (y >= height || x >= width) continue;
            *reinterpret_cast<float4*>(out + size_t(y) * width + x) = make_float4(v, v, v, v);
        } else {
            for (uint32_t k = 0; k < 4u && pix + k < tile_px; ++k) {
                const uint32_t x = rec.x + (pix + k) % T, y = rec.y + (pix + k) / T;
                if (x < width && y < height) out[size_t(y) * width + x] = v;
            }
        }
    }
}

// Scheduling.  Work lists are claimed with TICKETS (one atomicAdd on the list cursor hands out a range of
// indices; a compare-and-swap loop serialised thousands of idle warps on one address: 202 ms for a 0.2 ms
// frame) and the global queue is watched by ONE warp per CTA at a time (every idle warp polling the counters
// saturated the L2 slice that also serves the producers' atomics: 1.09 ms).  An idle warp first looks into its
// CTA's shared-memory ring; if that is empty and no other warp of the CTA is polling, it becomes the CTA's scout:
// one coalesced read of the reserved / claimed counters of all lists, tickets for as many entries as are
// available (at most one per warp of the CTA), valid tickets pushed into the ring.  Tickets that point past the
// reserved count (races between scouts) stay in the CTA's pending range and are honoured as soon as a producer
// reserves those indices -- a warp never blocks on them, so no cycle of waiting warps can form.
constexpr int TAIL_LISTS = 2 * TAIL_MAX_LEVELS + 2;   // interval levels, the leaf list, fill levels
constexpr uint32_t RING = 8;

struct CtaSched {
    uint32_t ring[RING];        // list << 28 | index
    uint32_t head, tail;        // consumers advance head (CAS), the scout advances tail
    uint32_t lock;              // 1 while a warp of this CTA is the scout
    uint32_t done;
    uint32_t pend_lo[TAIL_LISTS], pend_hi[TAIL_LISTS];   // tickets taken but not yet handed to a warp
};

__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) k_tail_2d(const __grid_constant__ Tail2DParams p) {
    __shared__ uint32_t live_s[WARPS_PER_BLOCK][8][32];
    __shared__ CtaSched sch;
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t gw = blockIdx.x * WARPS_PER_BLOCK + wib;
    itv slots[REG_SLOTS];   // the f32 interpreter of the leaf tiles uses the same bytes as float2[REG_SLOTS]
    Counters* ctr = p.lv[0].ctr;
    uint32_t* cs = p.lv[0].choice_scratch + size_t(gw) * p.lv[0].choice_words * 32u + lane;
    const int L = p.n_levels;   // render levels 1 .. L are interval levels here, list L + 1 holds the leaf tiles
    if (threadIdx.x == 0) { sch.head = sch.tail = 0; sch.lock = 0; sch.done = 0; }
    if (threadIdx.x < TAIL_LISTS) { sch.pend_lo[threadIdx.x] = 0; sch.pend_hi[threadIdx.x] = 0; }
    __syncthreads();
    unsigned long long shaded = 0;
    uint32_t idle = 0;
    // phase clock (statistics only): when the last job of every list finished, relative to the first warp's start
    auto now_ns = []() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; };
    Stats* st = p.px.stats;
    if (st && gw == 0 && lane == 0) st->culled[0] = now_ns();

    // list q: 0 .. L-1 interval level q + 1 (shallow first: they unlock parallelism); L: leaf tiles;
    //         L + 1 + l: fills of render level l
    auto cursor_of = [&](int q) -> uint32_t* { return q <= L ? &ctr->cursor[q + 1] : &ctr->fill_cursor[q - L - 1]; };
    auto reserved_of = [&](int q) -> uint32_t {
        if (q < L) return min(ld_volatile_u32(&ctr->n_jobs[q + 1]), p.lv[q].cap_in);
        if (q == L) return min(ld_volatile_u32(&ctr->n_jobs[L + 1]), p.lv[L - 1].cap_out);
        return min(ld_volatile_u32(&ctr->n_fills[q - L - 1]), p.fill_cap[q - L - 1]);
    };
    const int n_lists = p.paint_fills ? 2 * L + 2 : L + 1;
    volatile uint32_t* v_head = &sch.head;
    volatile uint32_t* v_tail = &sch.tail;
    volatile uint32_t* v_done = &sch.done;

    for (;;) {
        // ---- 1. the CTA's ring ----
        uint32_t entry = 0xffffffffu;
        if (lane == 0) {
            for (;;) {
                const uint32_t h = *v_head, t = *v_tail;
                if (h == t) break;
                const uint32_t e = sch.ring[h % RING];     // read before the claim: the slot may be reused right after it
                if (atomicCAS(&sch.head, h, h + 1u) == h) { entry = e; break; }
            }
            // a cancelled call claims nothing more: the warp leaves (entries still in the ring are dropped; `outstanding`
            // then never reaches zero, so no warp may wait for it)
            if (cancel_poll(p.cancel, entry == 0xffffffffu ? CS_WAIT : CS_TAIL_2D, entry & 0x0fffffffu)) entry = 0xfffffffeu;
        }
        entry = __shfl_sync(FULL, entry, 0);
        if (entry == 0xfffffffeu) break;
        if (entry == 0xffffffffu) {
            if (*v_done) break;
            // ---- 2. become the CTA's scout, or wait for the one that is ----
            uint32_t scout = 0;
            if (lane == 0) scout = atomicCAS(&sch.lock, 0u, 1u) == 0u ? 1u : 0u;
            scout = __shfl_sync(FULL, scout, 0);
            if (!scout) {
                // idle warps share their scheduler with latency-bound workers: wake rarely (measured: 200 ns naps of
                // the seven idle warps per scheduler doubled the duration of the level-1 jobs)
                __nanosleep(idle < 4u ? 250u : 1500u);
                if (++idle > (1u << 21)) { if (lane == 0) atomicOr(&ctr->error, 4u); break; }
                continue;
            }
            // one coalesced look at the queue: lane q reads what list q has reserved, lane 16 + q what is claimed
            // (`outstanding` FIRST: once it reads zero every list is final, so the counters read after it are too)
            uint32_t outst = lane == 0 ? ld_volatile_u32(&ctr->outstanding) : 0u;
            outst = __shfl_sync(FULL, outst, 0);
            __threadfence();
            const int q_l = lane & 15;
            uint32_t v = 0;
            if (q_l < n_lists) v = lane < 16 ? reserved_of(q_l) : ld_volatile_u32(cursor_of(q_l));
            bool found = false, fills_left = false;
            for (int q = 0; q < n_lists; ++q) {
                const uint32_t res = __shfl_sync(FULL, v, q), cur = __shfl_sync(FULL, v, 16 + q);
                if (lane == 0) {
                    uint32_t lo = sch.pend_lo[q], hi = sch.pend_hi[q];
                    const uint32_t space = RING - (*v_tail - *v_head);
                    if (lo == hi && cur < res && space) {
                        const uint32_t k = min(min(res - cur, uint32_t(WARPS_PER_BLOCK)), space);
                        lo = atomicAdd(cursor_of(q), k);
                        hi = lo + k;
                    }
                    uint32_t n_push = (lo < hi && lo < res) ? min(min(hi, res) - lo, space) : 0u;
                    const uint32_t t = *v_tail;
                    for (uint32_t i = 0; i < n_push; ++i) sch.ring[(t + i) % RING] = (uint32_t(q) << 28) | (lo + i);
                    if (n_push) { __threadfence_block(); *v_tail = t + n_push; found = true; }
                    lo += n_push;
                    sch.pend_lo[q] = lo;
                    sch.pend_hi[q] = hi;
                    if (q > L) fills_left |= cur < res || (lo < hi && lo < res);
                }
            }
            uint32_t flags = (found ? 1u : 0u) | (fills_left ? 2u : 0u);
            flags = __shfl_sync(FULL, flags, 0);
            if (lane == 0) {
                // nothing queued or running and no fill left to paint or to hand out: every list is final and empty
                if (!(flags & 1u) && outst == 0u && !(flags & 2u) && *v_head == *v_tail) *v_done = 1u;
                __threadfence_block();
                atomicExch(&sch.lock, 0u);
            }
            if (!(flags & 1u)) {
                __nanosleep(min(500u << min(idle, 4u), 8000u));   // back off while the queue is dry
                if (++idle > (1u << 21)) { if (lane == 0) atomicOr(&ctr->error, 4u); break; }
            }
            continue;
        }
        idle = 0;
        const int kind = int(entry >> 28);
        const uint32_t idx = entry & 0x0fffffffu;
        struct Stamp {   // statistics: finishing time of this job in its list's slot; for interval levels also the latest
            Stats* st; int slot; int lane; unsigned long long t0;      // start and the longest duration
            __device__ ~Stamp() {
                if (st && lane == 0) {
                    unsigned long long t;
                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                    atomicMax(&st->culled[slot], t);
                    if (slot <= 2) {
                        atomicMax(&st->culled[7 + slot], t0);          // [8], [9]: latest start of a level-1 / level-2 job
                        atomicMax(&st->culled[9 + slot], t - t0);      // [10], [11]: longest level-1 / level-2 job (ns)
                    }
                }
            }
        } stamp{st, 1 + min(kind, 13), lane, now_ns()};
        if (kind < L) {
            level_job<2, true>(p.lv[kind], idx, 0u, slots, cs, live_s[wib], lane, p.epoch);
            __syncwarp();
            if (lane == 0) { __threadfence(); atomicSub(&ctr->outstanding, 1u); }   // children were added before
        } else if (kind == L) {
            bool ok = true;
            const TileJob job = load_job_ready(p.px.jobs + idx, p.epoch, ctr, p.cancel, ok);
            if (!__any_sync(FULL, !ok)) pixel_job(p.px, job, reinterpret_cast<float2*>(slots), lane, shaded);
            __syncwarp();
            if (lane == 0) atomicSub(&ctr->outstanding, 1u);
        } else {
            const int l = kind - L - 1;
            const uint4* rp = reinterpret_cast<const uint4*>(p.fills[l] + idx);
            uint4 rec = __ldcg(rp);
            uint32_t spins = 0;
            while (rec.w != p.epoch) {   // reserved but not written yet
                if (cancel_poll(p.cancel, CS_WAIT, ~0u)) break;
                __nanosleep(64);
                rec = __ldcg(rp);
                if (++spins > (1u << 22)) { atomicOr(&ctr->error, 4u); break; }
            }
            if (rec.w == p.epoch) fill_job(p.fill_tile[l], p.px.width, p.px.height, p.px.out, rec, lane);
        }
    }
    if (p.px.stats) {
        for (int o = 16; o > 0; o >>= 1) shaded += __shfl_xor_sync(FULL, shaded, o);
        if (lane == 0 && shaded) atomicAdd(&p.px.stats->pixels, shaded);
    }
}

cudaError_t launch_tail_2d(const Tail2DParams& p, int sm_count, cudaStream_t s) {
    static int per_sm = 0;
    if (!per_sm) {
        // every CTA must be resident: workers wait for each other's output
        cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tail_2d, WARPS_PER_BLOCK * 32, 0);
        if (e != cudaSuccess) return e;
        per_sm = std::max(1, std::min(per_sm, 8));
    }
    k_tail_2d<<<sm_count * per_sm, WARPS_PER_BLOCK * 32, 0, s>>>(p);
    return cudaGetLastError();
}
int tail_2d_blocks(int sm_count) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tail_2d, WARPS_PER_BLOCK * 32, 0) != cudaSuccess) return 0;
    return sm_count * std::max(1, std::min(per_sm, 8));
}

}  // namespace fdev
