// The passes of the batches whose work lists are capped (fc_render3d_frames: frames; fc_render3d_scene: placements;
// fc_contour_build_slices: slices; fc_raycast: rays).  Overflow policy: a pass fails (FC_ERR_ARENA, list overflow) only where one of its
// items alone would.  The first pass holds one item; later ones are sized from the largest per-item use seen so far
// (arena clauses, jobs per level, and one more measured quantity of the caller's: census records, surface leaves) with
// headroom 1.5; a pass that still overflows is run again as two halves (the kernels report overflow, they do not
// fault), and only a one-item pass fails.  Only capped lists can overflow: a job list whose cap is the worst case of the
// pass (every tile of the level queued) never does, so the headroom applies to the arena, to the lists clamped by
// FIDGET_B200_MAX_TILES_M and to the measured quantity.  The caller runs the passes: take() the next one, observe() its
// counters once it is done, until more() is false.
#pragma once
#include <algorithm>
#include <cstdint>
#include <functional>
#include <utility>
#include <vector>

#include "env.h"
#include "kernels.cuh"

// What a pass of n items is tested against, as it stands when the pass is sized
struct PassLimits {
    uint64_t arena_cap = 0;                        // arena clauses
    uint64_t cap[fdev::MAX_LEVELS + 1] = {};       // job list of level l: its capacity ...
    uint64_t worst[fdev::MAX_LEVELS + 1] = {};     // ... and its worst case (levels left at 0 never bind)
    // the caller's measured quantity (census records, surface leaves): when on, its use times extra_scale must fit
    // extra_cap
    bool extra_on = false;
    double extra_scale = 1;
    uint64_t extra_cap = 0;
};

struct PassPlan {
    struct Range { uint32_t f0, n; };
    std::function<PassLimits(uint32_t)> limits_of;
    uint32_t n_items, n_max, next = 0;          // next: the first item no pass has taken yet
    int forced;
    double use_arena = 0, use_extra = 0, use_jobs[fdev::MAX_LEVELS + 1] = {};
    bool measured;
    std::vector<Range> redo;                    // halves of overflowed passes (a stack: the first half runs next)

    // n_max: the most items the caller allows in a pass (at least one)
    PassPlan(uint32_t n, uint32_t n_max_, std::function<PassLimits(uint32_t)> limits)
        : limits_of(std::move(limits)), n_items(n), n_max(n_max_) {
        // (diagnostic: passes of this size, at most n_max, neither measured first nor shrunk to fit)
        forced = env_int("FIDGET_B200_FRAMES_PER_PASS", 0);
        if (forced > 0) n_max = std::min<uint32_t>(n_max, uint32_t(forced));
        measured = forced > 0;
    }
    bool more() const { return next < n_items || !redo.empty(); }
    bool fits(uint32_t n) const {
        const PassLimits lim = limits_of(n);
        const double h = 1.5 * n;
        if (use_arena * h > double(lim.arena_cap)) return false;
        for (int l = 1; l <= fdev::MAX_LEVELS; ++l)
            if (lim.cap[l] < lim.worst[l] && use_jobs[l] * h > double(lim.cap[l])) return false;
        return !lim.extra_on || !(use_extra * h * lim.extra_scale > double(lim.extra_cap));
    }
    Range take() {
        if (!redo.empty()) { const Range r = redo.back(); redo.pop_back(); return r; }
        uint32_t n = std::min(n_max, n_items - next);
        if (!measured) n = 1;
        else if (forced <= 0 && !fits(n)) {
            // the largest pass that fits, by bisection: fits() holds for every size up to some bound and for none above
            // (the uses and the capped limits grow with n, and a limit at its worst case never binds); one item always
            // runs
            uint32_t lo = 1, hi = n;
            while (hi - lo > 1) {
                const uint32_t mid = lo + (hi - lo) / 2;
                (fits(mid) ? lo : hi) = mid;
            }
            n = lo;
        }
        const Range r{next, n};
        next += n;
        return r;
    }
    // Records the use of the finished pass r from its counters and its measured quantity.  False if it fails (its
    // error: device_error(ctr.error)); else `split` says that it overflowed and its halves are queued in its place.
    bool observe(const fdev::Counters& ctr, uint64_t extra, const Range& r, bool& split) {
        const double n = double(r.n);
        use_arena = std::max(use_arena, double(ctr.arena_top) / n);
        use_extra = std::max(use_extra, double(extra) / n);
        for (int l = 1; l <= fdev::MAX_LEVELS; ++l) use_jobs[l] = std::max(use_jobs[l], double(ctr.n_jobs[l]) / n);
        measured = true;
        split = false;
        if (!ctr.error) return true;
        if (r.n == 1 || (ctr.error & ~3u)) return false;
        const uint32_t h = r.n / 2;
        redo.push_back(Range{r.f0 + h, r.n - h});
        redo.push_back(Range{r.f0, h});
        split = true;
        return true;
    }
};
