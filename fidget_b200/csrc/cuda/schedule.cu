// Level-0 schedule of a root tape, built on the host at fc_tape_create: SSA form, dependency waves,
// min/max chain segments, slot colouring, upload (cached per context by tape hash) and the launch
// shape of the cooperative kernel.
#include "capi_internal.h"

// Dependency-wave schedule of a register tape: value id = position of the
// defining clause; clauses are bucketed by dependency depth, sorted by opcode
// inside a bucket (keeps warps convergent); the trailing single-clause
// buckets form the serial tail.
static bool build_schedule(const std::vector<uint2>& cl, std::vector<CoopRec>& recs,
                           std::vector<uint32_t>& wave_start, uint32_t& tail_begin, std::vector<CoopSeg>& segs) {
    const size_t n = cl.size();
    if (n == 0 || n >= COOP_NONE) return false;
    std::vector<int> regdef(256, -1);
    std::vector<uint32_t> depth(n, 0);
    std::vector<CoopRec> byp(n);
    uint32_t ci = 0, max_depth = 0;
    for (size_t p = 0; p < n; ++p) {
        uint32_t x = cl[p].x, dop = x & 0xff, op = dop >> 2, form = dop & 3, out = (x >> 8) & 0xff,
                 lhs = (x >> 16) & 0xff, rhs = x >> 24;
        if (op == OP_MEM) return false;
        CoopRec r;
        r.x = x; r.y = cl[p].y; r.ia = COOP_NONE; r.ib = COOP_NONE; r.p = uint16_t(p); r.cidx = 0;
        bool use_l = false, use_r = false;
        if (op == OP_OUTPUT) use_l = true;
        else if (op == OP_INPUT) {}
        else if (op == OP_COPY) use_l = (form != F_RI);
        else if (op_is_unary(op)) use_l = true;
        else { use_l = (form != F_IR); use_r = (form != F_RI); }
        uint32_t d = 0;
        if (use_l) { if (regdef[lhs] < 0) return false; r.ia = uint16_t(regdef[lhs]); d = std::max(d, depth[r.ia] + 1); }
        if (use_r) { if (regdef[rhs] < 0) return false; r.ib = uint16_t(regdef[rhs]); d = std::max(d, depth[r.ib] + 1); }
        if (op_is_choice(op)) r.cidx = uint16_t(ci++);
        if (ci >= COOP_NONE) return false;
        depth[p] = d;
        max_depth = std::max(max_depth, d);
        if (op != OP_OUTPUT) regdef[out] = int(p);
        byp[p] = r;
    }
    std::vector<std::vector<uint32_t>> levels(max_depth + 1);
    for (size_t p = 0; p < n; ++p) levels[depth[p]].push_back(uint32_t(p));
    size_t first_tail = levels.size();
    while (first_tail > 0 && levels[first_tail - 1].size() == 1) --first_tail;
    recs.clear();
    wave_start.assign(1, 0);
    for (size_t l = 0; l < first_tail; ++l) {
        auto& v = levels[l];
        std::stable_sort(v.begin(), v.end(), [&](uint32_t a, uint32_t b) { return (cl[a].x & 0xff) < (cl[b].x & 0xff); });
        for (uint32_t p : v) recs.push_back(byp[p]);
        wave_start.push_back(uint32_t(recs.size()));
    }
    tail_begin = uint32_t(recs.size());
    for (size_t l = first_tail; l < levels.size(); ++l) recs.push_back(byp[levels[l][0]]);

    // Cut the tail into serial runs and min/max chains (see CoopSeg)
    std::vector<uint32_t> idx_of_pos(n, 0);
    for (size_t i = 0; i < recs.size(); ++i) idx_of_pos[recs[i].p] = uint32_t(i);
    segs.clear();
    const uint32_t tend = uint32_t(recs.size());
    auto chain_op = [&](uint32_t i) -> uint32_t {  // returns opcode if rec i can extend a chain, else 0
        if (i == 0 || i <= tail_begin) return 0;
        const CoopRec& r = recs[i];
        uint32_t dop = r.x & 0xff, op = dop >> 2, form = dop & 3;
        if ((op != OP_MIN && op != OP_MAX) || form != F_RR) return 0;
        uint16_t pp = recs[i - 1].p;
        if ((r.ia == pp) == (r.ib == pp)) return 0;
        return op;
    };
    uint32_t i = tail_begin, serial_start = tail_begin;
    auto flush_serial = [&](uint32_t upto) {
        if (upto > serial_start) segs.push_back(CoopSeg{serial_start, upto, 0, COOP_NONE});
        serial_start = upto;
    };
    while (i < tend) {
        uint32_t op = chain_op(i);
        if (!op) { ++i; continue; }
        uint32_t j = i;
        while (j < tend && chain_op(j) == op) {
            const CoopRec& r = recs[j];
            uint16_t pp = recs[j - 1].p;
            uint16_t side = (r.ia == pp) ? r.ib : r.ia;
            if (idx_of_pos[side] >= i) break;   // the side must be computed before the run starts
            ++j;
        }
        if (j - i >= 8 && segs.size() + 3 <= size_t(COOP_MAX_SEGS)) {
            flush_serial(i);
            segs.push_back(CoopSeg{i, j, 1, COOP_NONE});
            serial_start = j;
            i = j;
        } else {
            i = std::max(j, i + 1);
        }
    }
    flush_serial(tend);
    return segs.size() <= size_t(COOP_MAX_SEGS);
}

// Forward view of a schedule: colour the values with slots.  Execution steps are the waves,
// then every clause of a serial tail run, then each chain run as a whole; a slot is free again
// from the step after the last reader of its value.  A chain value read only by the next clause
// of the same chain needs no slot (the scan never loads it); in a chain clause the operand that
// is the previous chain value is marked COOP_NONE and the run's starting value goes to
// segs[].start_slot.  Returns the number of slots, or 0 if they do not fit 16 bits.
static uint32_t colour_slots(const std::vector<CoopRec>& recs, const std::vector<uint32_t>& wave_start,
                             std::vector<CoopSeg>& segs, std::vector<CoopFwd>& fwd) {
    const size_t m = recs.size();
    std::vector<uint32_t> step(m, 0), idx_of_pos(m, 0), chain_of(m, 0);   // chain_of: 1 + segment index for chain clauses
    uint32_t st = 0;
    for (size_t w = 0; w + 1 < wave_start.size(); ++w, ++st)
        for (uint32_t i = wave_start[w]; i < wave_start[w + 1]; ++i) step[i] = st;
    for (size_t k = 0; k < segs.size(); ++k) {
        if (segs[k].chain) {
            for (uint32_t i = segs[k].begin; i < segs[k].end; ++i) { step[i] = st; chain_of[i] = uint32_t(k) + 1; }
            ++st;
        } else {
            for (uint32_t i = segs[k].begin; i < segs[k].end; ++i) step[i] = st++;
        }
    }
    for (size_t i = 0; i < m; ++i) idx_of_pos[recs[i].p] = uint32_t(i);
    // last reading step of every value and whether anything but its chain successor reads it
    std::vector<uint32_t> last_read(m, 0), n_other(m, 0);
    std::vector<uint8_t> has_reader(m, 0);
    for (size_t i = 0; i < m; ++i) {
        for (uint16_t src : {recs[i].ia, recs[i].ib}) {
            if (src == COOP_NONE) continue;
            const uint32_t d = idx_of_pos[src];
            last_read[d] = std::max(last_read[d], step[i]);
            has_reader[d] = 1;
            const bool chain_succ = chain_of[i] && chain_of[d] == chain_of[i] && d + 1 == i;
            if (!chain_succ) ++n_other[d];
        }
    }
    std::vector<uint16_t> slot(m, uint16_t(COOP_NONE));
    std::vector<uint32_t> free_list;
    std::vector<std::vector<uint32_t>> release(st + 2);   // release[s]: record indices whose slot is free from step s on
    uint32_t n_slots = 0;
    // records sorted by step: waves and tail are already in step order
    uint32_t cur = 0;
    for (size_t i = 0; i < m; ++i) {
        while (cur <= step[i]) {
            for (uint32_t d : release[cur]) free_list.push_back(slot[d]);
            ++cur;
        }
        const bool is_output = ((recs[i].x & 0xff) >> 2) == OP_OUTPUT;
        const bool chain_internal = chain_of[i] && has_reader[i] && n_other[i] == 0 && i + 1 < m && chain_of[i + 1] == chain_of[i];
        if (is_output || chain_internal) continue;
        uint32_t sl;
        if (!free_list.empty()) { sl = free_list.back(); free_list.pop_back(); }
        else sl = n_slots++;
        if (sl >= COOP_NONE) return 0;
        slot[i] = uint16_t(sl);
        const uint32_t rel = (has_reader[i] ? last_read[i] : step[i]) + 1;
        release[std::min<uint32_t>(rel, st + 1)].push_back(uint32_t(i));
    }
    fwd.resize(m);
    for (size_t i = 0; i < m; ++i) {
        CoopFwd f;
        f.x = recs[i].x; f.y = recs[i].y; f.cidx = recs[i].cidx;
        f.sa = recs[i].ia == COOP_NONE ? uint16_t(COOP_NONE) : slot[idx_of_pos[recs[i].ia]];
        f.sb = recs[i].ib == COOP_NONE ? uint16_t(COOP_NONE) : slot[idx_of_pos[recs[i].ib]];
        f.so = slot[i];
        if (chain_of[i]) {
            // the previous chain value is the result of the record right before this one
            const uint16_t prev_pos = recs[i - 1].p;
            CoopSeg& sg = segs[chain_of[i] - 1];
            if (i == sg.begin) sg.start_slot = slot[i - 1];
            if (recs[i].ia == prev_pos) f.sa = uint16_t(COOP_NONE);
            else f.sb = uint16_t(COOP_NONE);
        }
        fwd[i] = f;
    }
    return std::max(n_slots, 1u);
}

// FNV-1a over 64-bit words (one device clause per step)
static uint64_t fnv1a(const uint2* cl, size_t n) {
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; ++i) {
        h ^= uint64_t(cl[i].x) | uint64_t(cl[i].y) << 32;
        h *= 1099511628211ull;
    }
    return h;
}

// Symbolic replay of a coloured schedule (fc_schedule_check): slots hold value ids.
static int32_t replay_schedule(const std::vector<CoopRec>& recs, const std::vector<CoopFwd>& fwd,
                               const std::vector<uint32_t>& wave_start, uint32_t tail_begin,
                               const std::vector<CoopSeg>& segs, uint32_t n_slots) {
    const uint32_t UNSET = 0xffffffffu;
    std::vector<uint32_t> holds(n_slots, UNSET);
    auto bad = [&](size_t i, const char* what) {
        return fail(FC_ERR_INVALID, std::string("schedule check: record ") + std::to_string(i) + " (clause " +
                                        std::to_string(recs[i].p) + "): " + what);
    };
    // reads of record i against the current slot contents; `skip_prev`: chain records do not load the previous chain value
    auto check_reads = [&](size_t i, bool chain) -> int32_t {
        const uint16_t def[2] = {recs[i].ia, recs[i].ib}, sl[2] = {fwd[i].sa, fwd[i].sb};
        for (int k = 0; k < 2; ++k) {
            if (def[k] == COOP_NONE) { if (sl[k] != COOP_NONE) return bad(i, "slot for an immediate operand"); continue; }
            if (chain && sl[k] == COOP_NONE) continue;                 // the previous chain value, carried by the scan
            if (sl[k] == COOP_NONE || sl[k] >= n_slots) return bad(i, "operand without a slot");
            if (holds[sl[k]] != def[k]) return bad(i, "operand slot does not hold the defining clause's value");
        }
        return FC_OK;
    };
    auto step = [&](uint32_t b, uint32_t e, bool chain) -> int32_t {   // records [b, e) run concurrently
        std::vector<uint8_t> read(n_slots, 0);
        for (uint32_t i = b; i < e; ++i) {
            if (int32_t rc = check_reads(i, chain)) return rc;
            if (fwd[i].sa != COOP_NONE) read[fwd[i].sa] = 1;
            if (fwd[i].sb != COOP_NONE) read[fwd[i].sb] = 1;
        }
        std::vector<uint8_t> written(n_slots, 0);
        for (uint32_t i = b; i < e; ++i) {
            const uint16_t so = fwd[i].so;
            if (so == COOP_NONE) continue;
            if (so >= n_slots) return bad(i, "result slot out of range");
            if (read[so] && e - b > 1) return bad(i, "writes a slot that the same step reads");
            if (written[so]) return bad(i, "two results of one step share a slot");
            written[so] = 1;
        }
        for (uint32_t i = b; i < e; ++i)
            if (fwd[i].so != COOP_NONE) holds[fwd[i].so] = recs[i].p;
        return FC_OK;
    };
    for (size_t w = 0; w + 1 < wave_start.size(); ++w)
        if (int32_t rc = step(wave_start[w], wave_start[w + 1], false)) return rc;
    if (!wave_start.empty() && wave_start.back() != tail_begin) return fail(FC_ERR_INVALID, "schedule check: waves do not end at the tail");
    uint32_t expect = tail_begin;
    for (const CoopSeg& sg : segs) {
        if (sg.begin != expect || sg.end <= sg.begin) return fail(FC_ERR_INVALID, "schedule check: tail segments are not contiguous");
        expect = sg.end;
        if (!sg.chain) {
            for (uint32_t i = sg.begin; i < sg.end; ++i)
                if (int32_t rc = step(i, i + 1, false)) return rc;
            continue;
        }
        if (sg.begin == 0 || sg.start_slot >= n_slots || holds[sg.start_slot] != recs[sg.begin - 1].p)
            return bad(sg.begin, "chain does not start from the previous record's value");
        for (uint32_t i = sg.begin; i < sg.end; ++i) {
            const uint16_t prev = recs[i - 1].p;
            const bool a_prev = recs[i].ia == prev, b_prev = recs[i].ib == prev;
            if (a_prev == b_prev) return bad(i, "chain clause does not combine the previous result with one side");
            if ((fwd[i].sa == COOP_NONE) != a_prev || (fwd[i].sb == COOP_NONE) != b_prev) return bad(i, "chain operand marking");
            const uint32_t dop = recs[i].x & 0xff, dop0 = recs[sg.begin].x & 0xff;
            if (dop != dop0) return bad(i, "mixed opcodes in a chain");
        }
        if (int32_t rc = step(sg.begin, sg.end, true)) return rc;
    }
    if (expect != recs.size()) return fail(FC_ERR_INVALID, "schedule check: tail segments do not cover the tail");
    return FC_OK;
}

extern "C" int32_t fc_schedule_check(const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count,
                                     uint32_t n_vars, uint32_t n_outputs, fc_schedule_info* info) {
    if (!info) return fail(FC_ERR_INVALID, "null argument");
    memset(info, 0, sizeof *info);
    std::vector<uint2> cl;
    uint32_t nch = 0;
    if (int32_t rc = transcode(words, n_words, reg_count, mem_count, n_vars, n_outputs, cl, nch)) return rc;
    info->n_clauses = uint32_t(cl.size());
    std::vector<CoopRec> recs;
    std::vector<uint32_t> ws;
    std::vector<CoopSeg> segs;
    uint32_t tb = 0;
    if (cl.size() < 64 || !build_schedule(cl, recs, ws, tb, segs)) return FC_OK;   // not suitable: per-lane kernel
    std::vector<CoopFwd> fwd;
    const uint32_t n_slots = colour_slots(recs, ws, segs, fwd);
    if (!n_slots) return FC_OK;
    info->suitable = 1;
    info->n_waves = uint32_t(ws.size() - 1);
    for (size_t w = 0; w + 1 < ws.size(); ++w) info->widest_wave = std::max(info->widest_wave, ws[w + 1] - ws[w]);
    info->n_tail = uint32_t(recs.size()) - tb;
    info->n_segments = uint32_t(segs.size());
    for (const CoopSeg& sg : segs) if (sg.chain) info->n_chain_clauses += sg.end - sg.begin;
    info->n_slots = n_slots;
    // every clause exactly once
    std::vector<uint8_t> seen(cl.size(), 0);
    for (const CoopRec& r : recs) {
        if (r.p >= cl.size() || seen[r.p]) return fail(FC_ERR_INVALID, "schedule check: a clause is missing or scheduled twice");
        seen[r.p] = 1;
    }
    if (recs.size() != cl.size()) return fail(FC_ERR_INVALID, "schedule check: a clause is missing or scheduled twice");
    return replay_schedule(recs, fwd, ws, tb, segs, n_slots);
}

void upload_schedule(fc_tape* t) {
    fc_ctx* c = t->ctx;
    if (t->host.size() < 64) return;   // the cooperative kernel is never used for short tapes
    const uint64_t h = fnv1a(t->host.data(), t->host.size());
    {
        std::lock_guard<std::mutex> g(c->mu);
        for (auto& sp : c->sched_cache)
            if (sp && sp->hash == h && sp->clauses.size() == t->host.size() &&
                memcmp(sp->clauses.data(), t->host.data(), t->host.size() * sizeof(uint2)) == 0) { t->sched = sp; return; }
    }
    std::vector<CoopRec> recs;
    std::vector<uint32_t> ws;
    uint32_t tb = 0;
    auto sc = std::make_shared<Sched>();
    sc->device = c->device;
    sc->hash = h;
    sc->clauses = t->host;   // a hash hit is verified against the clauses themselves
    if (!build_schedule(t->host, recs, ws, tb, sc->segs)) return;
    std::vector<CoopFwd> fwd;
    sc->n_slots = colour_slots(recs, ws, sc->segs, fwd);
    if (!sc->n_slots) return;
    if (cudaMalloc(&sc->d_fwd, fwd.size() * sizeof(CoopFwd)) != cudaSuccess) { sc->d_fwd = nullptr; cudaGetLastError(); return; }
    cudaMemcpy(sc->d_fwd, fwd.data(), fwd.size() * sizeof(CoopFwd), cudaMemcpyHostToDevice);
    if (cudaMalloc(&sc->d_recs, recs.size() * sizeof(CoopRec)) != cudaSuccess) { sc->d_recs = nullptr; cudaGetLastError(); return; }
    if (cudaMalloc(&sc->d_wave_start, ws.size() * 4) != cudaSuccess) { sc->d_wave_start = nullptr; cudaGetLastError(); return; }
    cudaMemcpy(sc->d_recs, recs.data(), recs.size() * sizeof(CoopRec), cudaMemcpyHostToDevice);
    cudaMemcpy(sc->d_wave_start, ws.data(), ws.size() * 4, cudaMemcpyHostToDevice);
    sc->n_waves = uint32_t(ws.size() - 1);
    sc->tail_begin = tb;
    sc->tail_end = uint32_t(recs.size());
    t->sched = sc;
    std::lock_guard<std::mutex> g(c->mu);
    c->sched_cache[c->sched_next++ % 4] = sc;
}

// Attach the tape's wave schedule to a level-0 launch when the cooperative kernel applies
// (long tape, few root tiles per SM); returns the grid size or 0.
int coop_blocks(fc_ctx* c, const fc_tape* tape, uint64_t n_roots, LevelParams& p, int dim, int& threads) {
    const Sched* sc = tape->sched.get();
    if (!sc || !sc->d_recs || !sc->d_fwd || !sc->d_wave_start || env_int("FIDGET_B200_NO_COOP", 0)) return 0;
    size_t smem = coop_smem_bytes(tape->info.n_ops, tape->info.choice_count, sc->n_slots);
    if (smem > 220 * 1024) return 0;
    // with one lane per tile a warp walks the tape for 32 tiles at once; that only pays when
    // there are enough root tiles to fill the machine several times over
    if (n_roots > uint64_t(c->sm_count) * 32 * 24) return 0;
    p.sched.recs = sc->d_recs;
    p.sched.fwd = sc->d_fwd;
    p.sched.n_slots = sc->n_slots;
    p.sched.wave_start = sc->d_wave_start;
    p.sched.n_waves = sc->n_waves;
    p.sched.tail_begin = sc->tail_begin;
    p.sched.tail_end = sc->tail_end;
    p.sched.n_segs = uint32_t(sc->segs.size());
    for (size_t k = 0; k < sc->segs.size(); ++k) p.sched.segs[k] = sc->segs[k];
    // Tiles are latency chains of ~55 barrier steps: what matters is how many ROUNDS of tiles the
    // launch needs.  Take the fewest CTAs per SM that reach the minimal number of rounds (wider CTAs
    // shorten a tile), within shared memory (1 KB reserved + ~1.5 KB static per CTA), 2048 threads
    // and the register file.
    const int max_by_smem = int(std::max<size_t>(1, std::min<size_t>(8, (227 * 1024) / (smem + 2560))));
    const int cap = std::min(max_by_smem, env_int("FIDGET_B200_COOP_PER_SM", 8));
    auto rounds = [&](int per_sm) { return (n_roots + uint64_t(c->sm_count) * per_sm - 1) / (uint64_t(c->sm_count) * per_sm); };
    int per_sm = 1;
    for (int k = 1; k <= cap; ++k) if (rounds(k) < rounds(per_sm)) per_sm = k;
    // widest CTA for which the runtime really keeps per_sm of them resident (register granularity
    // makes 7 x 224 threads x 40 registers NOT fit although 7 * 224 * 40 < 64 K)
    // a frame batch and a scene launch their own instantiations
    const int variant = p.scene ? 2 : p.frames != nullptr ? 1 : 0;
    auto& mm = c->coop_memo[(dim == 3 ? 3 : 0) + variant];
    if (mm.threads == 0 || mm.smem != smem || mm.per_sm != per_sm) {
        int t = COOP_THREADS;
        while (t > 64 && coop_occupancy(dim, variant, t, smem) < per_sm) t -= 32;
        mm = {smem, per_sm, t};
    }
    threads = mm.threads;
    threads = env_int("FIDGET_B200_COOP_THREADS", threads);
    if (env_int("FIDGET_B200_COOP_DEBUG", 0))
        fprintf(stderr, "coop: %u clauses, %u slots, %zu B smem, %d CTAs/SM x %d threads (%d regs), %llu roots, occupancy %d CTAs/SM, %d SMs\n",
                tape->info.n_ops, sc->n_slots, smem, per_sm, threads, coop_regs_per_thread(dim, variant), (unsigned long long)n_roots,
                coop_occupancy(dim, variant, threads, smem), c->sm_count);
    return int(std::max<uint64_t>(1, std::min<uint64_t>(n_roots, uint64_t(c->sm_count) * per_sm)));
}
