// Host-side check of the pass planner of the 3D batches and contour stacks (pass_plan.h): compiled with nvcc, run on the
// CPU by tests/test_pass_plan_host.py.  Each scenario scripts what its passes report and prints one line: its name, the
// range [f0, f0 + n) of every pass taken in order, and "fail <error bits>" if the planner gives up.
#include <cstdio>
#include <cstdlib>

#include "kernels.cuh"
#include "pass_plan.h"

// Runs the passes of `plan`: report(r, ctr, extra) fills in the counters and the measured quantity of pass r
template <class F> static void run(const char* name, PassPlan plan, F report) {
    std::printf("%s", name);
    while (plan.more()) {
        const PassPlan::Range r = plan.take();
        std::printf(" [%u,%u)", r.f0, r.f0 + r.n);
        fdev::Counters ctr{};
        uint64_t extra = 0;
        report(r, ctr, extra);
        bool split = false;
        if (!plan.observe(ctr, extra, r, split)) {
            std::printf(" fail %u", ctr.error);
            break;
        }
    }
    std::printf("\n");
}

static PassLimits arena_only(uint64_t cap) {
    PassLimits lim;
    lim.arena_cap = cap;
    return lim;
}

int main() {
    setenv("FIDGET_B200_ENV_LIVE", "1", 1);   // (before the first knob is read: FRAMES_PER_PASS changes below)
    unsetenv("FIDGET_B200_FRAMES_PER_PASS");
    auto arena_1000 = [](uint32_t) { return arena_only(1000); };
    auto use_100 = [](const PassPlan::Range& r, fdev::Counters& ctr, uint64_t&) { ctr.arena_top = 100ull * r.n; };

    // (a) 100 clauses per item against 1000: one item first, then 6 (1.5 * 7 * 100 > 1000), then the rest
    run("a", PassPlan(10, 8, arena_1000), use_100);
    // (b) the pass of 6 overflows a list: its halves run next, first half first
    run("b", PassPlan(10, 8, arena_1000), [](const PassPlan::Range& r, fdev::Counters& ctr, uint64_t&) {
        ctr.arena_top = 100ull * r.n;
        if (r.f0 == 1 && r.n == 6) ctr.error = 2;
    });
    // (c) a one-item pass that exhausts the arena fails; so does a multi-item pass with an error other than overflow
    run("c1", PassPlan(10, 8, arena_1000), [](const PassPlan::Range&, fdev::Counters& ctr, uint64_t&) {
        ctr.arena_top = 1000;
        ctr.error = 1;
    });
    run("c2", PassPlan(10, 8, arena_1000), [](const PassPlan::Range& r, fdev::Counters& ctr, uint64_t&) {
        ctr.arena_top = 10ull * r.n;
        if (r.n > 1) ctr.error = 4;
    });
    // (d) a forced pass size is neither measured first nor shrunk, even where the use would not fit
    setenv("FIDGET_B200_FRAMES_PER_PASS", "3", 1);
    run("d", PassPlan(10, 8, arena_1000), [](const PassPlan::Range& r, fdev::Counters& ctr, uint64_t&) {
        ctr.arena_top = 400ull * r.n;
    });
    unsetenv("FIDGET_B200_FRAMES_PER_PASS");
    // (e) level 2's list is clamped at 300 jobs and binds at 2 items (100 per item); level 1's is the worst case of its
    // pass, so its far higher use does not count
    run("e", PassPlan(10, 8, [](uint32_t n) {
            PassLimits lim = arena_only(1ull << 30);
            lim.cap[1] = lim.worst[1] = 100ull * n;
            lim.cap[2] = 300;
            lim.worst[2] = 1000ull * n;
            return lim;
        }), [](const PassPlan::Range& r, fdev::Counters& ctr, uint64_t&) {
            ctr.n_jobs[1] = 1000 * r.n;
            ctr.n_jobs[2] = 100 * r.n;
        });
    // (f) the measured quantity: 10 per item, each costing 100 against 3000, binds at 2 items; switched off, it does not
    for (bool on : {true, false})
        run(on ? "f" : "f_off", PassPlan(10, 8, [on](uint32_t) {
                PassLimits lim = arena_only(1ull << 30);
                lim.extra_on = on;
                lim.extra_scale = 100;
                lim.extra_cap = 3000;
                return lim;
            }), [](const PassPlan::Range& r, fdev::Counters&, uint64_t& extra) { extra = 10ull * r.n; });
    // (g) the arena grows from 0 to 1000 clauses when the first pass runs: later passes are sized against 1000, as in (a)
    uint64_t arena = 0;
    run("g", PassPlan(10, 8, [&arena](uint32_t) { return arena_only(arena); }),
        [&arena](const PassPlan::Range& r, fdev::Counters& ctr, uint64_t&) {
            arena = 1000;
            ctr.arena_top = 100ull * r.n;
        });
    return 0;
}
