// Cooperative level-0 kernel of the tile renderers (one CTA per root tile).
#include <algorithm>
#include <cstdio>

#include "interp.cuh"

// ---------------------------------------------------------------------------
// K1-root: cooperative level-0 kernel.  The root tape is long (prospero: 6363
// clauses) and there are few root tiles (1024 at 4096^2), so one lane per
// tile is latency-bound.  Here one CTA evaluates one root tile: the tape's
// clauses run wave by wave (all clauses of a wave are independent), values
// live in shared memory indexed by the defining clause, long min/max chains
// in the tail are evaluated with a block-wide prefix scan, and the reverse
// liveness pass + compaction are parallel too.  Results are identical to
// k_interval_level_2d (same per-clause arithmetic, same simplify rules).
namespace fdev {

// shared memory of one root tile: forward values by slot, overlaid by the reverse pass's
// last_use words (one per clause; bits 16.. hold the emit code), then the 2-bit choices
size_t coop_smem_bytes(uint32_t n_ops, uint32_t n_choices, uint32_t n_slots) {
    return std::max(size_t(n_slots) * 8, size_t(n_ops) * 4) + size_t((n_choices + 15) / 16 + 1) * 4 + 16;
}

struct Fwd {
    uint32_t x, y, sa, sb, so, cidx;
    __device__ __forceinline__ explicit Fwd(const uint4 q)
        : x(q.x), y(q.y), sa(q.z & 0xffffu), sb(q.z >> 16), so(q.w & 0xffffu), cidx(q.w >> 16) {}
};
__device__ __forceinline__ Fwd load_fwd(const CoopFwd* f, uint32_t i) {
    return Fwd(__ldg(reinterpret_cast<const uint4*>(f) + i));
}
struct Rec {
    uint32_t x, y, ia, ib, p, cidx;
    __device__ __forceinline__ explicit Rec(const uint4 q)
        : x(q.x), y(q.y), ia(q.z & 0xffffu), ib(q.z >> 16), p(q.w & 0xffffu), cidx(q.w >> 16) {}
};
__device__ __forceinline__ Rec load_rec(const CoopRec* recs, uint32_t i) {
    return Rec(__ldg(reinterpret_cast<const uint4*>(recs) + i));
}

template <int DIM, bool FRAMES = false, bool SCENE = false>
__global__ void __launch_bounds__(COOP_THREADS)
k_interval_root_coop(const __grid_constant__ LevelParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t n = p.root_tape.n_ops, nch = p.root_tape.n_choices;
    const uint32_t cw = (nch + 15u) / 16u + 1u;
    itv* vals = reinterpret_cast<itv*>(smem_raw);                 // forward: values by slot
    const size_t data_bytes = max(size_t(p.sched.n_slots) * 8, size_t(n) * 4);
    uint32_t* chs = reinterpret_cast<uint32_t*>(smem_raw + data_bytes);
    // reverse: one word per clause, overlaying vals: bits 0..15 = 1 + position of the last live
    // reader (0: dead), bits 16.. = emit code
    uint32_t* last_use = reinterpret_cast<uint32_t*>(smem_raw);
    __shared__ itv s_res;
    __shared__ uint32_t s_tile, s_nonboth, s_warp_tot[COOP_THREADS / 32], s_ref, s_nch;
    __shared__ unsigned long long s_base;
    __shared__ float s_agg_lo[COOP_THREADS / 32], s_agg_hi[COOP_THREADS / 32];
    __shared__ uint8_t s_agg_f[COOP_THREADS / 32], s_agg_u[COOP_THREADS / 32];

    const uint32_t tid = threadIdx.x, T = p.tile, NT = blockDim.x;   // NT <= COOP_THREADS, a multiple of 32
    const CoopRec* __restrict__ recs = p.sched.recs;
    const CoopFwd* __restrict__ fwd = p.sched.fwd;
    const uint32_t* __restrict__ ws = p.sched.wave_start;
    const uint32_t n_roots = SCENE ? scene_root_count(p) : root_count(p, DIM == 3);
    const uint2* __restrict__ tape = p.root_tape.ptr;

    for (;;) {
        if (tid == 0) {
            s_tile = atomicAdd(&p.ctr->cursor[0], 1u);
            if (s_tile < n_roots && cancel_poll(p.cancel, CS_ROOT_COOP, s_tile)) s_tile = ~0u;   // cancelled: claim nothing more
            s_nonboth = 0;
            s_ref = 0;
            s_nch = 0;
            s_res = iv_nan();
        }
        for (uint32_t i = tid; i < cw; i += NT) chs[i] = 0;
        __syncthreads();
        const uint32_t tile = s_tile;
        if (tile >= n_roots) break;
        uint32_t cx, cy, cz, pl = 0;
        if (SCENE) pl = scene_root(p, tile, T, cx, cy, cz);
        else root_corner(p, tile, T, cx, cy, cz);
        if (DIM != 3) cz = 0u;
        if constexpr (DIM == 2 && SCENE) {   // a root tile under higher shapes' proven interiors is not evaluated
            bool open = false;
            const uint32_t nb = T / p.cull;
            for (uint32_t q = tid; q < nb * nb; q += NT) {
                const uint32_t bx = cx / p.cull + q % nb, by = cy / p.cull + q / nb;
                open |= bx >= p.occl_w || by >= p.occl_h || p.occl[size_t(by) * p.occl_w + bx] <= pl + 1u;
            }
            if (!__syncthreads_or(open)) continue;   // (every thread has read s_tile)
        }
        const FrameView fv = view_of<FRAMES, SCENE>(p, cy, pl);   // frame batch, scene
        const VarBind& vb = *fv.vb;
        itv vx, vy, vz;
        xform_iv(*fv.mat, iv(float(cx), float(cx) + float(T)),
                 iv(float(cy - fv.y0), float(cy - fv.y0) + float(T)),
                 DIM == 3 ? iv(float(cz), float(cz) + float(T)) : iv(fv.z, fv.z), vx, vy, vz);
        auto put_choice = [&](uint32_t cidx, uint32_t c) {
            atomicOr(&chs[cidx >> 4], c << ((cidx & 15u) * 2u));
            if (c != 3u) s_nonboth = 1u;
        };
        auto get_choice = [&](uint32_t cidx) { return (chs[cidx >> 4] >> ((cidx & 15u) * 2u)) & 3u; };
        auto exec = [&](const Fwd& rc, itv sl, itv sr) -> itv {
            // (records are sorted by their first byte inside a wave, so the lanes of a warp mostly share a handler)
            const float imm = __uint_as_float(rc.y);
            itv r;
            uint32_t c = 0;
            switch (c_dop.h[rc.x & 0xffu]) {
                FB_BINI(H_ADD, iv_add(a, b))
                FB_BINI(H_SUB, iv_sub(a, b))
                case H_MUL_RR: r = iv_mul(sl, sr); break;
                case H_MUL_RI: r = iv_mul_f(sl, imm); break;
                case H_MUL_IR: r = iv_mul(iv1(imm), sr); break;
                FB_BINI(H_MIN, iv_choice_op(OP_MIN, a, b, c))
                FB_BINI(H_MAX, iv_choice_op(OP_MAX, a, b, c))
                case H_NEG: r = iv_neg(sl); break;
                case H_ABS: r = iv_abs(sl); break;
                case H_SQRT: r = iv_sqrt(sl); break;
                case H_SQUARE: r = iv_square(sl); break;
                case H_COPY_REG: r = sl; break;
                case H_COPY_IMM: r = iv1(imm); break;
                default: __builtin_unreachable();
                case H_GENERIC: {
                    const Dec d(rc.x);
                    const itv a = d.form == F_IR ? iv1(imm) : sl;
                    const itv b = d.form == F_RI ? iv1(imm) : sr;
                    if (d.op >= OP_MIN) {
                        r = iv_choice_op(d.op, a, b, c);
                    } else if (d.op >= OP_ADD) {
                        r = iv_binary(d.op, a, b);
                    } else if (d.op >= OP_NEG) {
                        r = iv_unary(d.op, sl);
                    } else if (d.op == OP_COPY) {
                        r = d.form == F_RI ? iv1(imm) : sl;
                    } else if (d.op == OP_INPUT) {
                        r = pick_input(vb, rc.y, vx, vy, vz, [](float f) { return iv1(f); });
                    } else {
                        if (rc.y == 0) s_res = sl;
                        r = sl;
                    }
                }
            }
            if (c) put_choice(rc.cidx, c);
            return r;
        };
        auto ld = [&](uint32_t id) { return id != COOP_NONE ? vals[id] : iv_nan(); };

        // ---- forward: dependency waves ----
        {
            // each thread keeps the NEXT record it will execute in registers, so the
            // global (L2) latency of the schedule stream overlaps the current clause
            uint32_t w = 0, i = tid;   // recs of wave w are [ws[w], ws[w+1]); wave 0 starts at 0
            const uint32_t n_waves = p.sched.n_waves, wave_end_all = p.sched.tail_begin;
            uint32_t e = n_waves ? ws[1] : 0;
            auto advance = [&]() {     // move (w, i) to this thread's next record, crossing waves
                while (w < n_waves && i >= e) {
                    ++w;
                    if (w < n_waves) { i = e + tid; e = ws[w + 1]; }
                }
            };
            advance();
            uint4 q = (w < n_waves) ? __ldg(reinterpret_cast<const uint4*>(fwd) + i) : make_uint4(0, 0, 0, 0);
            uint32_t cur_w = 0;
            while (cur_w < n_waves) {
                // run everything this thread owns in wave cur_w
                while (w == cur_w) {
                    const Fwd rc(q);
                    i += NT;
                    advance();
                    if (w < n_waves) q = __ldg(reinterpret_cast<const uint4*>(fwd) + i);
                    const itv r = exec(rc, ld(rc.sa), ld(rc.sb));
                    if (rc.so != COOP_NONE) vals[rc.so] = r;
                }
                __syncthreads();
                ++cur_w;
            }
            (void)wave_end_all;
        }
        // ---- forward: tail segments ----
        for (uint32_t sgi = 0; sgi < p.sched.n_segs; ++sgi) {
            const uint32_t b = p.sched.segs[sgi].begin, e = p.sched.segs[sgi].end;
            if (!p.sched.segs[sgi].chain) {
                if (tid == 0) {
                    uint32_t last_s = COOP_NONE;
                    itv last_r = iv_nan();
                    for (uint32_t i = b; i < e; ++i) {
                        const Fwd rc = load_fwd(fwd, i);
                        const itv sl = (rc.sa == last_s && last_s != COOP_NONE) ? last_r : ld(rc.sa);
                        const itv sr = (rc.sb == last_s && last_s != COOP_NONE) ? last_r : ld(rc.sb);
                        const itv r = exec(rc, sl, sr);
                        if (rc.so != COOP_NONE) vals[rc.so] = r;
                        last_s = rc.so;
                        last_r = r;
                    }
                }
            } else {
                // m_i = OP(m_{i-1}, s_i): prefix scan over the sides
                const uint32_t m = e - b, ch = (m + NT - 1) / NT;
                const uint32_t c0 = min(e, b + tid * ch), c1 = min(e, c0 + ch);
                // (forward view: the operand that is the previous chain value is marked COOP_NONE,
                //  the value the chain starts from sits in segs[].start_slot)
                const Fwd first = load_fwd(fwd, b);
                const bool is_min = (Dec(first.x).op == OP_MIN);
                const uint32_t start_slot = p.sched.segs[sgi].start_slot;
                auto comb = [&](float& lo, float& hi, uint32_t& f, itv s) {
                    f |= uint32_t(iv_has_nan(s));
                    lo = is_min ? fminf(lo, s.x) : fmaxf(lo, s.x);
                    hi = is_min ? fminf(hi, s.y) : fmaxf(hi, s.y);
                };
                const float ident = is_min ? __int_as_float(0x7f800000) : __int_as_float(0xff800000);
                float alo = ident, ahi = ident;
                uint32_t af = 0;
                for (uint32_t i = c0; i < c1; ++i) {
                    const Fwd rc = load_fwd(fwd, i);
                    comb(alo, ahi, af, vals[rc.sa == COOP_NONE ? rc.sb : rc.sa]);
                }
                // exclusive block scan of the per-thread aggregates (warp shuffles + one smem hop)
                float xlo = alo, xhi = ahi;
                uint32_t xf = af;
                const uint32_t ln = tid & 31u, wp = tid >> 5;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const float vlo = __shfl_up_sync(FULL, xlo, o), vhi = __shfl_up_sync(FULL, xhi, o);
                    const uint32_t vf = __shfl_up_sync(FULL, xf, o);
                    if (ln >= uint32_t(o)) {
                        xlo = is_min ? fminf(vlo, xlo) : fmaxf(vlo, xlo);
                        xhi = is_min ? fminf(vhi, xhi) : fmaxf(vhi, xhi);
                        xf |= vf;
                    }
                }
                if (ln == 31u) { s_agg_lo[wp] = xlo; s_agg_hi[wp] = xhi; s_agg_f[wp] = uint8_t(xf); }
                // exclusive within the warp
                float elo = __shfl_up_sync(FULL, xlo, 1), ehi = __shfl_up_sync(FULL, xhi, 1);
                uint32_t ef = __shfl_up_sync(FULL, xf, 1);
                if (ln == 0u) { elo = ident; ehi = ident; ef = 0; }
                __syncthreads();
                if (c0 < c1) {
                    const itv start = vals[start_slot];
                    float lo = start.x, hi = start.y;
                    uint32_t f = uint32_t(iv_has_nan(start));
                    for (uint32_t k = 0; k < wp; ++k) {
                        f |= s_agg_f[k];
                        lo = is_min ? fminf(lo, s_agg_lo[k]) : fmaxf(lo, s_agg_lo[k]);
                        hi = is_min ? fminf(hi, s_agg_hi[k]) : fmaxf(hi, s_agg_hi[k]);
                    }
                    f |= ef;
                    lo = is_min ? fminf(lo, elo) : fmaxf(lo, elo);
                    hi = is_min ? fminf(hi, ehi) : fmaxf(hi, ehi);
                    for (uint32_t i = c0; i < c1; ++i) {
                        const Fwd rc = load_fwd(fwd, i);
                        const bool prev_is_lhs = (rc.sa == COOP_NONE);
                        const itv s = vals[prev_is_lhs ? rc.sb : rc.sa];
                        const itv mprev = f ? iv_nan() : iv(lo, hi);
                        uint32_t c;
                        const itv r = prev_is_lhs ? iv_choice_op(is_min ? OP_MIN : OP_MAX, mprev, s, c)
                                                  : iv_choice_op(is_min ? OP_MIN : OP_MAX, s, mprev, c);
                        comb(lo, hi, f, s);
                        put_choice(rc.cidx, c);
                        if (rc.so != COOP_NONE) vals[rc.so] = r;
                    }
                }
            }
            __syncthreads();
        }

        const itv r = s_res;
        const bool fill_in = !p.pixel_perfect && r.y < 0.0f;
        const bool fill_out = !p.pixel_perfect && !fill_in && r.x > 0.0f;
        const bool amb = !fill_in && !fill_out;
        if (DIM == 3 && fill_in) {   // voxel.rs:310-317 (scene: the fill's rank, kernels.cuh)
            const unsigned long long key = SCENE ? scene_rank(cz + T + 1u, pl, p.clamp_at, p.depth)
                                                 : (unsigned long long)(cz + T + 1u) << 32;
            for (uint32_t q = tid; q < T * T; q += NT) {   // (frame batch: rows below the frame are its padding)
                const uint32_t x = cx + q % T, y = cy + q / T;
                if (x < p.width && y - fv.y0 < p.height) atomicMax(&p.heightmap[size_t(y) * p.width + x], key);
            }
            if (p.occl && T % 16u == 0u)
                for (uint32_t q = tid; q < (T / 16u) * (T / 16u); q += NT) {
                    const uint32_t bx = cx / 16u + q % (T / 16u), by = cy / 16u + q / (T / 16u);
                    if (bx < p.occl_w && by - fv.y0 / 16u < p.occl_h) {
                        if (SCENE) atomicMax(reinterpret_cast<unsigned long long*>(p.occl) + size_t(by) * p.occl_w + bx, key);
                        else atomicMax(p.occl + size_t(by) * p.occl_w + bx, cz + T + 1u);
                    }
                }
        }
        if constexpr (DIM == 2 && SCENE) {   // 2D scene: the write cover map instead of a fill record
            if (fill_in)
                scene2d_cover(p.occl + size_t(p.occl_w) * p.occl_h, p.occl_w, p.occl_h, p.cull, cx, cy, T, pl, tid, NT);
        }
        if (tid == 0) {
            if (DIM == 2 && !SCENE && !amb) {
                uint32_t slot = atomicAdd(&p.ctr->n_fills[0], 1u);
                if (slot < p.cap_fills) {
                    FillRec fr;
                    fr.x = cx;
                    fr.y = cy;
                    fr.value = 0x7FC00000u | (fill_in ? 1u : 0u) | (0xF6u << 9);
                    fr.ready = p.epoch;
                    p.fills[slot] = fr;
                } else atomicOr(&p.ctr->error, 2u);
            }
            if (p.stats) {
                atomicAdd(&p.stats->evaluated[0], 1ull);
                if (fill_in) atomicAdd(&p.stats->filled_inside[0], 1ull);
                if (fill_out) atomicAdd(&p.stats->filled_outside[0], 1ull);
                if (amb) atomicAdd(&p.stats->ambiguous[0], 1ull);
            }
        }
        auto census = [&](bool kept) {   // exact 3D census record of this root tile (tid 0)
            if (DIM != 3 || !p.census) return;
            const uint32_t slot = atomicAdd(&p.ctr->n_census, 1u);
            if (slot < p.cap_census) {
                CensusRec r;
                r.x = uint16_t(cx); r.y = uint16_t(cy); r.z = uint16_t(cz);
                r.level = 0;
                r.flags = uint8_t((fill_in ? 1u : (fill_out ? 0u : 2u)) | (kept ? 4u : 0u));
                p.census[slot] = r;
            } else atomicOr(&p.ctr->error, 2u);
        };
        if (!amb) {
            if (tid == 0) census(false);
            __syncthreads();
            continue;
        }

        TapeRef child = p.root_tape;
        if (s_nonboth) {   // uniform: written before the last barrier
            // ---- R1: reverse liveness; last_use[v] = 1 + position of the last live clause reading v ----
            for (uint32_t i = tid; i < n; i += NT) last_use[i] = 0;
            __syncthreads();
            auto r1 = [&](const Rec& rc) {
                Dec d(rc.x);
                if (d.op != OP_OUTPUT && last_use[rc.p] == 0u) return;
                const uint32_t mark = rc.p + 1u;
                bool use_a = rc.ia != COOP_NONE, use_b = rc.ib != COOP_NONE;
                if (d.op >= OP_MIN) {
                    uint32_t c = get_choice(rc.cidx);
                    if (c == 1u) use_b = false;
                    else if (c == 2u) use_a = false;
                }
                if (use_a) atomicMax(&last_use[rc.ia], mark);
                if (use_b) atomicMax(&last_use[rc.ib], mark);
            };
            for (uint32_t sgi = p.sched.n_segs; sgi > 0; --sgi) {
                const uint32_t b = p.sched.segs[sgi - 1].begin, e = p.sched.segs[sgi - 1].end;
                if (!p.sched.segs[sgi - 1].chain) {
                    if (tid == 0)
                        for (uint32_t i = e; i > b; --i) r1(load_rec(recs, i - 1));
                } else {
                    // live_i = ext_i | (uses_prev_{i+1} & live_{i+1}), suffix scan over the run
                    const uint32_t m = e - b, ch = (m + NT - 1) / NT;
                    const uint32_t c0 = min(e, b + tid * ch), c1 = min(e, c0 + ch);
                    const uint32_t prev_first = load_rec(recs, b - 1).p;
                    auto uses_prev = [&](const Rec& rc, uint32_t prevp) {
                        uint32_t c = get_choice(rc.cidx);
                        return c == 3u || c == (rc.ia == prevp ? 1u : 2u);
                    };
                    // F(x) = O | (U & x), x = (uses_prev & live) of the element after the chunk
                    uint32_t O = 0, U = 1;
                    for (uint32_t i = c1; i > c0; --i) {
                        const Rec rc = load_rec(recs, i - 1);
                        const uint32_t prevp = i - 1 > b ? load_rec(recs, i - 2).p : prev_first;
                        const uint32_t ext = last_use[rc.p] != 0u, up = uses_prev(rc, prevp);
                        // y_i = up_i & live_i, live_i = ext_i | y_{i+1}
                        O = up & (ext | O);
                        U = up & U;
                    }
                    // inclusive suffix scan of F = (O, U) under composition (earlier o later)
                    uint32_t xO = O, xU = U;
                    const uint32_t ln = tid & 31u, wp = tid >> 5;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t vO = __shfl_down_sync(FULL, xO, o), vU = __shfl_down_sync(FULL, xU, o);
                        if (ln + uint32_t(o) < 32u) { xO = xO | (xU & vO); xU = xU & vU; }
                    }
                    if (ln == 0u) { s_agg_f[wp] = uint8_t(xO); s_agg_u[wp] = uint8_t(xU); }
                    // composition of the chunks AFTER this thread inside the warp
                    uint32_t eO = __shfl_down_sync(FULL, xO, 1), eU = __shfl_down_sync(FULL, xU, 1);
                    if (ln == 31u) { eO = 0; eU = 1; }
                    __syncthreads();
                    if (c0 < c1) {
                        uint32_t y = 0;   // (uses_prev & live) of the element right after this chunk
                        for (uint32_t k = (NT >> 5); k > wp + 1u; --k) y = s_agg_f[k - 1] | (s_agg_u[k - 1] & y);
                        y = eO | (eU & y);
                        for (uint32_t i = c1; i > c0; --i) {
                            const Rec rc = load_rec(recs, i - 1);
                            const uint32_t prevp = i - 1 > b ? load_rec(recs, i - 2).p : prev_first;
                            const uint32_t live = (last_use[rc.p] != 0u) | y;
                            const uint32_t c = get_choice(rc.cidx);
                            const bool prev_is_lhs = (rc.ia == prevp);
                            const bool up = c == 3u || c == (prev_is_lhs ? 1u : 2u);
                            const bool us = c == 3u || c == (prev_is_lhs ? 2u : 1u);
                            if (live) {
                                if (up) atomicMax(&last_use[prevp], rc.p + 1u);
                                if (us) atomicMax(&last_use[prev_is_lhs ? rc.ib : rc.ia], rc.p + 1u);
                            }
                            y = up & live;
                        }
                    }
                }
                __syncthreads();
            }
            for (uint32_t w = p.sched.n_waves; w > 0; --w) {
                const uint32_t e = ws[w];
                for (uint32_t i = ws[w - 1] + tid; i < e; i += NT) r1(load_rec(recs, i));
                __syncthreads();
            }
            // ---- R2a: what each clause turns into ----
            // 0 none, 1 as is, 7 as is (choice kept), 2/3 copy lhs real/alias, 4/5 copy rhs real/alias, 6 copy imm
            for (uint32_t i = tid; i < p.sched.tail_end; i += NT) {
                const Rec rc = load_rec(recs, i);
                Dec d(rc.x);
                const uint32_t pos = rc.p;
                uint32_t code;
                if (d.op != OP_OUTPUT && (last_use[pos] & 0xffffu) == 0u) code = 0;
                else if (d.op >= OP_MIN) {
                    uint32_t c = get_choice(rc.cidx);
                    if (c == 3u) code = 7;
                    else if (c == 2u && d.form == F_RI) code = 6;
                    else {
                        const bool use_rhs = (c == 2u);
                        const uint32_t src_reg = use_rhs ? d.rhs : d.lhs, src_def = use_rhs ? rc.ib : rc.ia;
                        if (src_reg == d.out) code = 0;
                        else code = (use_rhs ? 4u : 2u) + ((last_use[src_def] & 0xffffu) > pos + 1u ? 0u : 1u);
                    }
                } else if (d.op == OP_COPY && d.form != F_RI) {
                    if (d.lhs == d.out) code = 0;
                    else if (d.form == F_ALIAS) code = 3;
                    else code = (last_use[rc.ia] & 0xffffu) > pos + 1u ? 2u : 3u;
                } else code = 1;
                last_use[pos] = (last_use[pos] & 0xffffu) | (code << 16);   // only this thread writes word `pos`
            }
            __syncthreads();
            // ---- R2b: scan in tape order, then write the compacted child ----
            const uint32_t chunk = (n + NT - 1) / NT;
            const uint32_t b0 = min(n, tid * chunk), b1 = min(n, b0 + chunk);
            uint32_t my_dev = 0, my_ref = 0, my_nch = 0;
            for (uint32_t q = b0; q < b1; ++q) {
                uint32_t c = last_use[q] >> 16;
                my_dev += (c != 0u);
                my_ref += (c != 0u && c != 3u && c != 5u);
                my_nch += (c == 7u);
            }
            uint32_t incl = my_dev;
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t v = __shfl_up_sync(FULL, incl, o);
                if ((tid & 31) >= uint32_t(o)) incl += v;
            }
            if ((tid & 31) == 31) s_warp_tot[tid >> 5] = incl;
            if (my_ref) atomicAdd(&s_ref, my_ref);
            if (my_nch) atomicAdd(&s_nch, my_nch);
            __syncthreads();
            uint32_t warp_off = 0, n_dev = 0;
            for (uint32_t k = 0; k < (NT >> 5); ++k) {
                if (k < (tid >> 5)) warp_off += s_warp_tot[k];
                n_dev += s_warp_tot[k];
            }
            const uint32_t ref_len = s_ref, nch_c = s_nch;
            const bool keep = ref_len < p.root_tape.ref_len;   // render/mod.rs:125-129
            if (keep) {
                if (tid == 0) {
                    unsigned long long base = atomicAdd(&p.ctr->arena_top, (unsigned long long)n_dev);
                    if (base + n_dev > p.arena_cap) {
                        atomicOr(&p.ctr->error, 1u);
                        base = ~0ull;
                    }
                    s_base = base;
                }
                __syncthreads();
                const unsigned long long base = s_base;
                if (base != ~0ull) {
                    uint2* dst = p.arena + base + warp_off + (incl - my_dev);
                    for (uint32_t q = b0; q < b1; ++q) {
                        uint32_t c = last_use[q] >> 16;
                        if (!c) continue;
                        uint2 w = __ldg(tape + q);
                        if (c != 1u && c != 7u) {
                            Dec d(w.x);
                            if (c == 6u) w = make_uint2(enc(OP_COPY, F_RI, d.out, 0xff, 0xff), w.y);
                            else {
                                uint32_t src = (c >= 4u) ? d.rhs : d.lhs;
                                w = make_uint2(enc(OP_COPY, (c & 1u) ? F_ALIAS : F_RR, d.out, src, 0xff), 0xFF000000u);
                            }
                        }
                        *dst++ = w;
                    }
                    child.ptr = p.arena + base;
                    child.n_ops = n_dev;
                    child.ref_len = ref_len;
                    child.n_choices = nch_c;
                    if (tid == 0 && p.stats) atomicAdd(&p.stats->simplified[0], 1ull);
                }
            }
        }
        if (tid == 0) census(child.ptr != p.root_tape.ptr);
        if (tid == 0) {
            uint32_t slot = atomicAdd(&p.ctr->n_jobs[1], 1u);
            if (slot < p.cap_out) {
                TileJob o;
                o.x = cx;
                o.y = cy;
                o.z = cz;
                o.pad = SCENE ? pl : p.epoch;
                o.tape = child;
                p.jobs_out[slot] = o;
                if (p.fused_tail) atomicAdd(&p.ctr->outstanding, 1u);
            } else atomicOr(&p.ctr->error, 2u);
        }
        __syncthreads();
    }
}

template <int DIM, bool FRAMES, bool SCENE = false>
static cudaError_t launch_coop(const LevelParams& p, int blocks, int threads, cudaStream_t s) {
    size_t smem = coop_smem_bytes(p.root_tape.n_ops, p.root_tape.n_choices, p.sched.n_slots);
    static size_t configured = 0;   // (per instantiation)
    if (smem > configured) {
        cudaError_t e = cudaFuncSetAttribute(k_interval_root_coop<DIM, FRAMES, SCENE>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess) return e;
        // many small CTAs per SM: ask for the largest shared-memory carve-out
        cudaFuncSetAttribute(k_interval_root_coop<DIM, FRAMES, SCENE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        configured = smem;
    }
    k_interval_root_coop<DIM, FRAMES, SCENE><<<blocks, threads, smem, s>>>(p);
    return cudaGetLastError();
}
// the instantiation a launch takes: DIM, and whether it renders a frame batch or a 3D scene (register counts differ)
static void (*coop_kernel(int dim, int variant))(LevelParams) {
    if (dim == 3)
        return variant == 2 ? k_interval_root_coop<3, false, true>
             : variant == 1 ? k_interval_root_coop<3, true> : k_interval_root_coop<3, false>;
    return variant == 2 ? k_interval_root_coop<2, false, true>
         : variant == 1 ? k_interval_root_coop<2, true> : k_interval_root_coop<2, false>;
}
int coop_occupancy(int dim, int variant, int threads, size_t smem) {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, coop_kernel(dim, variant), threads, smem);
    return n;
}
int coop_regs_per_thread(int dim, int variant) {
    static int regs[6] = {0, 0, 0, 0, 0, 0};
    int& r = regs[(dim == 3 ? 3 : 0) + variant];
    if (!r) {
        cudaFuncAttributes a{};
        cudaError_t e = cudaFuncGetAttributes(&a, coop_kernel(dim, variant));
        r = e == cudaSuccess ? a.numRegs : 64;
    }
    return r;
}
// (a frame batch, p.frames != null, takes the instantiation that reads its frames from the table; a scene, p.scene,
// the one that reads its placements)
cudaError_t launch_interval_root_coop_2d(const LevelParams& p, int blocks, int threads, cudaStream_t s) {
    if (p.scene) return launch_coop<2, false, true>(p, blocks, threads, s);
    return p.frames ? launch_coop<2, true>(p, blocks, threads, s) : launch_coop<2, false>(p, blocks, threads, s);
}
cudaError_t launch_interval_root_coop_3d(const LevelParams& p, int blocks, int threads, cudaStream_t s) {
    if (p.scene) return launch_coop<3, false, true>(p, blocks, threads, s);
    return p.frames ? launch_coop<3, true>(p, blocks, threads, s) : launch_coop<3, false>(p, blocks, threads, s);
}

}  // namespace fdev
