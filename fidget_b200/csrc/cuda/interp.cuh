// Device-side interpreters and helpers shared by the kernels of the hot path: clause decoding,
// the interval / f32 (two and four points per lane) / gradient tape walks, choice packing and the
// reverse liveness pass that compacts a child tape (VmData::simplify semantics,
// fidget-core/src/vm/data.rs:123-318).
//
// All interpreters keep the tape's VM registers in per-thread local memory (L1-resident,
// lane-interleaved, so a warp's access to one register is one 128/256-byte line) and read tape
// clauses with warp-uniform 8-byte loads.
#pragma once
#include "kernels.cuh"

namespace fdev {

#define FULL 0xffffffffu

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// The edge searches of the octree and quadtree samplers: a point of a cell as u16 fractions of its bounds, and one
// edge's bracket (start = inside end, end = outside end), per axis
__device__ __forceinline__ float lerp_u16(float lo, float hi, uint32_t p) {
    const float frac = float(p) / 65535.0f;   // CellBounds::pos (cell.rs:183-192), Interval::lerp
    return lo * (1.0f - frac) + hi * frac;
}

struct EdgeState { uint32_t s[3], e[3]; };

// The 16-ary edge search (OctreeBuilder::leaf) on the first AXES axes of two edges per lane, in a cell with bounds lo /
// hi: each half-warp follows its own pair of edges (s0, s1), and lane jj of it probes fraction jj / 15 of both brackets
// through eval2 (x0, y0[, z0], x1, y1[, z1]) -> (v0, v1).  Each of four rounds narrows a bracket to the step that ends
// at its first probe at or outside the surface.  The half-warp's lane 0 then writes the bracket midpoint of each valid
// edge (v0, v1) to its intersection, pos[e0] / pos[e1].
template <int AXES, class Eval2>
__device__ __forceinline__ void edge_search(EdgeState& s0, EdgeState& s1, const float* lo, const float* hi,
                                            const Eval2& eval2, float (*pos)[AXES], bool v0, uint32_t e0, bool v1,
                                            uint32_t e1) {
    const int lane = threadIdx.x & 31, half = lane >> 4, jj = lane & 15;
    for (int round = 0; round < 4; ++round) {
        uint32_t q0[AXES], q1[AXES];
#pragma unroll
        for (int a = 0; a < AXES; ++a) {
            q0[a] = (s0.s[a] * uint32_t(15 - jj) + s0.e[a] * uint32_t(jj)) / 15u;
            q1[a] = (s1.s[a] * uint32_t(15 - jj) + s1.e[a] * uint32_t(jj)) / 15u;
        }
        float2 v;
        if constexpr (AXES == 3)
            v = eval2(lerp_u16(lo[0], hi[0], q0[0]), lerp_u16(lo[1], hi[1], q0[1]), lerp_u16(lo[2], hi[2], q0[2]),
                      lerp_u16(lo[0], hi[0], q1[0]), lerp_u16(lo[1], hi[1], q1[1]), lerp_u16(lo[2], hi[2], q1[2]));
        else
            v = eval2(lerp_u16(lo[0], hi[0], q0[0]), lerp_u16(lo[1], hi[1], q0[1]),
                      lerp_u16(lo[0], hi[0], q1[0]), lerp_u16(lo[1], hi[1], q1[1]));
        const uint32_t b0 = (__ballot_sync(FULL, v.x >= 0.0f) >> (16 * half)) & 0xffffu;
        const uint32_t b1 = (__ballot_sync(FULL, v.y >= 0.0f) >> (16 * half)) & 0xffffu;
        auto narrow = [&](EdgeState& st, uint32_t bits) {
            uint32_t frac = bits ? uint32_t(__ffs(bits) - 1) : 15u;
            if (frac == 0u) frac = 1u;
#pragma unroll
            for (int a = 0; a < AXES; ++a) {
                const uint32_t na = (st.s[a] * (16u - frac) + st.e[a] * (frac - 1u)) / 15u;
                const uint32_t nb = (st.s[a] * (15u - frac) + st.e[a] * frac) / 15u;
                st.s[a] = na & 0xffffu;
                st.e[a] = nb & 0xffffu;
            }
        };
        narrow(s0, b0);
        narrow(s1, b1);
    }
    if (jj == 0) {
        if (v0) for (int a = 0; a < AXES; ++a) pos[e0][a] = lerp_u16(lo[a], hi[a], ((s0.s[a] + s0.e[a]) / 2u) & 0xffffu);
        if (v1) for (int a = 0; a < AXES; ++a) pos[e1][a] = lerp_u16(lo[a], hi[a], ((s1.s[a] + s1.e[a]) / 2u) & 0xffffu);
    }
}

// INPUT clause -> value: the axes get coordinates, other slots their bound value
template <class T, class F>
__device__ __forceinline__ T pick_input(const VarBind& vb, uint32_t i, T X, T Y, T Z, F from_float) {
    const int k = int(i);
    if (k == vb.x) return X;
    if (k == vb.y) return Y;
    if (k == vb.z) return Z;
    return from_float(vb.values[k & (MAX_RENDER_VARS - 1)]);
}

// Clause loads: tapes that were complete before the launch go through the read-only path (ld.global.nc);
// in the fused 2D kernel a tape may have been written by another SM during the same launch, so it is
// read with plain loads (its 128-byte lines are exclusive to it and were never cached before).
template <bool NC>
__device__ __forceinline__ uint2 ld_clause(const uint2* p) {
    return NC ? __ldg(p) : *p;
}

struct Dec {
    uint32_t op, form, out, lhs, rhs;
    Dec() = default;
    __device__ __forceinline__ explicit Dec(uint32_t x) {
        uint32_t dop = x & 0xffu;
        op = dop >> 2;
        form = dop & 3u;
        out = (x >> 8) & 0xffu;
        lhs = (x >> 16) & 0xffu;
        rhs = x >> 24;
    }
};

// Dispatch of the f32 interpreters' hot loops: a 256-entry table (constant memory) maps the first byte of a clause
// (opcode * 4 + form) to a dense handler number, so the switch below compiles to one jump table without range
// compares, and each handler knows which operands are registers and which is the immediate (no per-component
// selects on the form; the right-hand register is only loaded by the forms that read it).  Handlers exist for the
// opcodes CSG tapes are made of; everything else is H_GENERIC.
enum : uint32_t {
    H_GENERIC = 0,
    H_ADD_RR, H_ADD_RI, H_ADD_IR, H_SUB_RR, H_SUB_RI, H_SUB_IR, H_MUL_RR, H_MUL_RI, H_MUL_IR,
    H_MIN_RR, H_MIN_RI, H_MIN_IR, H_MAX_RR, H_MAX_RI, H_MAX_IR,
    H_NEG, H_ABS, H_SQRT, H_SQUARE, H_COPY_REG, H_COPY_IMM,
    H_DIV_RR, H_DIV_RI, H_DIV_IR, H_EXP,   // c_dop_f only (bear.vm's other frequent opcodes)
    H_COUNT
};
struct DopTable {
    uint8_t h[256];
};
constexpr DopTable make_dop_table(bool f32) {
    DopTable t{};
    for (int i = 0; i < 256; ++i) t.h[i] = H_GENERIC;
    const uint32_t bin[6][2] = {{OP_ADD, H_ADD_RR}, {OP_SUB, H_SUB_RR}, {OP_MUL, H_MUL_RR}, {OP_MIN, H_MIN_RR}, {OP_MAX, H_MAX_RR},
                                {OP_DIV, H_DIV_RR}};
    for (int k = 0; k < (f32 ? 6 : 5); ++k)
        for (uint32_t f = 0; f < 3; ++f) t.h[bin[k][0] * 4u + f] = uint8_t(bin[k][1] + f);   // F_RR, F_RI, F_IR
    t.h[OP_NEG * 4u + F_RR] = H_NEG;
    t.h[OP_ABS * 4u + F_RR] = H_ABS;
    t.h[OP_SQRT * 4u + F_RR] = H_SQRT;
    t.h[OP_SQUARE * 4u + F_RR] = H_SQUARE;
    if (f32) t.h[OP_EXP * 4u + F_RR] = H_EXP;
    t.h[OP_COPY * 4u + F_RR] = H_COPY_REG;
    t.h[OP_COPY * 4u + F_ALIAS] = H_COPY_REG;
    t.h[OP_COPY * 4u + F_RI] = H_COPY_IMM;
    return t;
}
static __constant__ DopTable c_dop = make_dop_table(false);     // interval interpreters
static __constant__ DopTable c_dop_f = make_dop_table(true);    // f32 interpreters: + div, exp

// ---------------------------------------------------------------------------
// Interval interpreter.  `Input` maps a variable index to an interval,
// `Sink` receives one choice per choice clause in evaluation order, `Out`
// receives (output index, value).
// Hot loop dispatched through c_dop like the f32 interpreters; both operand registers are still loaded before the
// dispatch (a lone warp per parent tile: the loads' latency is the critical path, not their issue slots).
#define FB_BINI(H, EXPR)                                                           \
    case H##_RR: { const itv a = sl, b = sr; r = EXPR; break; }                    \
    case H##_RI: { const itv a = sl, b = iv1(imm); r = EXPR; break; }              \
    case H##_IR: { const itv a = iv1(imm), b = sr; r = EXPR; break; }
template <bool NC = true, class Input, class Sink, class Out>
__device__ __forceinline__ void run_interval(const uint2* __restrict__ tape, uint32_t n_ops, itv* slots,
                                             Input input, Sink& sink, Out out_fn) {
    if (n_ops == 0) return;
    uint2 w = ld_clause<NC>(tape);
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint2 nxt = ld_clause<NC>(tape + (i + 1 < n_ops ? i + 1 : i));
        const uint32_t x = w.x;
        const float imm = __uint_as_float(w.y);
        const itv sl = slots[(x >> 16) & 0xffu], sr = slots[x >> 24];
        itv r;
        uint32_t c = 0;   // 1 left, 2 right, 3 both for the choice opcodes
        switch (c_dop.h[x & 0xffu]) {
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
                const Dec d(x);
                const itv a = d.form == F_IR ? iv1(imm) : sl;
                const itv b = d.form == F_RI ? iv1(imm) : sr;
                if (d.op >= OP_MIN) {
                    if (d.op == OP_MEM) {
                        if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                        else slots[MEM_BASE + w.y] = sl;
                        w = nxt;
                        continue;
                    }
                    r = iv_choice_op(d.op, a, b, c);
                } else if (d.op >= OP_ADD) {
                    r = iv_binary(d.op, a, b);
                } else if (d.op >= OP_NEG) {
                    r = iv_unary(d.op, sl);
                } else if (d.op == OP_INPUT) {
                    r = input(w.y);
                } else if (d.op == OP_OUTPUT) {
                    out_fn(w.y, sl);
                    w = nxt;
                    continue;
                } else {   // a COPY form without a handler
                    r = d.form == F_RI ? iv1(imm) : sl;
                }
            }
        }
        if (c) sink.push(c);
        slots[(x >> 8) & 0xffu] = r;
        w = nxt;
    }
}

// Two-points-per-lane f32 interpreter
__device__ __forceinline__ float2 f32x2_unary(uint32_t op, float2 a) {
    switch (op) {
        case OP_NEG: return make_float2(-a.x, -a.y);
        case OP_ABS: return make_float2(fabsf(a.x), fabsf(a.y));
        case OP_SQRT: return make_float2(sqrtf(a.x), sqrtf(a.y));
        case OP_SQUARE: return make_float2(a.x * a.x, a.y * a.y);
        default: return make_float2(f32_unary(op, a.x), f32_unary(op, a.y));
    }
}
__device__ __forceinline__ float2 f32x2_binary(uint32_t op, float2 a, float2 b) {
    switch (op) {
        case OP_ADD: return make_float2(a.x + b.x, a.y + b.y);
        case OP_SUB: return make_float2(a.x - b.x, a.y - b.y);
        case OP_MUL: return make_float2(a.x * b.x, a.y * b.y);
        case OP_MIN: return make_float2(f_min(a.x, b.x), f_min(a.y, b.y));
        case OP_MAX: return make_float2(f_max(a.x, b.x), f_max(a.y, b.y));
        default: return make_float2(f32_binary(op, a.x, b.x), f32_binary(op, a.y, b.y));
    }
}

// Hot loop dispatched through c_dop (see above); H_GENERIC is the plain decode-and-select path.
#define FB_BIN2(H, EXPR)                                                                     \
    case H##_RR: { const float2 b = slots[x >> 24]; const float2 a = sl; r = EXPR; break; }  \
    case H##_RI: { const float2 b = im; const float2 a = sl; r = EXPR; break; }              \
    case H##_IR: { const float2 b = slots[x >> 24]; const float2 a = im; r = EXPR; break; }
template <bool NC = true, class Input>
__device__ __forceinline__ float2 run_f32x2(const uint2* __restrict__ tape, uint32_t n_ops, float2* slots,
                                            Input input) {
    float2 result = make_float2(nanf_(), nanf_());
    if (n_ops == 0) return result;
    uint2 w = ld_clause<NC>(tape);
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint2 nxt = ld_clause<NC>(tape + (i + 1 < n_ops ? i + 1 : i));
        const uint32_t x = w.x;
        const float imm = __uint_as_float(w.y);
        const float2 sl = slots[(x >> 16) & 0xffu];
        const float2 im = make_float2(imm, imm);
        float2 r;
        switch (c_dop_f.h[x & 0xffu]) {
            FB_BIN2(H_ADD, make_float2(a.x + b.x, a.y + b.y))
            FB_BIN2(H_SUB, make_float2(a.x - b.x, a.y - b.y))
            FB_BIN2(H_MUL, make_float2(a.x * b.x, a.y * b.y))
            FB_BIN2(H_MIN, make_float2(f_min(a.x, b.x), f_min(a.y, b.y)))
            FB_BIN2(H_MAX, make_float2(f_max(a.x, b.x), f_max(a.y, b.y)))
            case H_NEG: r = make_float2(-sl.x, -sl.y); break;
            case H_ABS: r = make_float2(fabsf(sl.x), fabsf(sl.y)); break;
            case H_SQRT: r = make_float2(sqrtf(sl.x), sqrtf(sl.y)); break;
            case H_SQUARE: r = make_float2(sl.x * sl.x, sl.y * sl.y); break;
            case H_COPY_REG: r = sl; break;
            case H_COPY_IMM: r = im; break;
            FB_BIN2(H_DIV, make_float2(a.x / b.x, a.y / b.y))
            case H_EXP: r = make_float2(expf(sl.x), expf(sl.y)); break;
            default: __builtin_unreachable();
            case H_GENERIC: {
                const Dec d(x);
                const float2 sr = slots[d.rhs];
                const float2 a = d.form == F_IR ? im : sl;
                const float2 b = d.form == F_RI ? im : sr;
                if (d.op >= OP_ADD) {
                    if (d.op == OP_MEM) {
                        if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                        else slots[MEM_BASE + w.y] = sl;
                        w = nxt;
                        continue;
                    }
                    r = f32x2_binary(d.op, a, b);
                } else if (d.op >= OP_NEG) {
                    r = f32x2_unary(d.op, sl);
                } else if (d.op == OP_COPY) {
                    r = d.form == F_RI ? im : sl;
                } else if (d.op == OP_INPUT) {
                    r = input(w.y);
                } else {
                    if (w.y == 0) result = sl;
                    w = nxt;
                    continue;
                }
            }
        }
        slots[(x >> 8) & 0xffu] = r;
        w = nxt;
    }
    return result;
}

// ---------------------------------------------------------------------------
// Choice storage for the level kernel: 2 bits per choice, 16 per word, words
// interleaved across the 32 lanes of the warp.
struct ChoicePacker {
    uint32_t* base;  // already offset by lane; stride 32
    uint32_t acc = 0, ci = 0;
    bool any_nonboth = false;
    __device__ __forceinline__ void push(uint32_t c) {
        acc |= c << ((ci & 15u) * 2u);
        any_nonboth |= (c != 3u);
        ++ci;
        if ((ci & 15u) == 0u) {
            base[((ci >> 4) - 1u) * 32u] = acc;
            acc = 0;
        }
    }
    __device__ __forceinline__ void finish() {
        if (ci & 15u) base[(ci >> 4) * 32u] = acc;
    }
};
struct ChoiceUnpacker {
    const uint32_t* base;
    uint32_t ci;       // choices remaining
    uint32_t cached_word = 0xffffffffu, cur = 0;
    __device__ __forceinline__ uint32_t pop() {
        --ci;
        uint32_t wi = ci >> 4;
        if (wi != cached_word) {
            cur = base[wi * 32u];
            cached_word = wi;
        }
        return (cur >> ((ci & 15u) * 2u)) & 3u;
    }
};
struct ByteChoiceSource {
    const uint8_t* base;
    uint32_t ci;
    __device__ __forceinline__ uint32_t pop() { return base[--ci] & 3u; }
};

// Reverse liveness pass + compaction (VmData::simplify on a register tape that
// keeps the parent's register assignment).  Writes the child tape backwards,
// ending at `wend`.  `live` is this warp's [8][32] bitset in shared memory.
template <bool NC = true, class ChoiceSrc>
__device__ __forceinline__ void simplify_lane(const uint2* __restrict__ tape, uint32_t n_ops, bool active,
                                              uint32_t (*live)[32], int lane, ChoiceSrc& cs, uint2* wend,
                                              uint32_t& n_dev, uint32_t& ref_len, uint32_t& n_choices) {
#pragma unroll
    for (int k = 0; k < 8; ++k) live[k][lane] = 0;
    auto test = [&](uint32_t r) { return (live[r >> 5][lane] >> (r & 31u)) & 1u; };
    auto set = [&](uint32_t r) { live[r >> 5][lane] |= 1u << (r & 31u); };
    auto clear = [&](uint32_t r) { live[r >> 5][lane] &= ~(1u << (r & 31u)); };
    uint2* wp = wend;
    uint32_t ref = 0, nch = 0;
    uint2 nxt = n_ops ? ld_clause<NC>(tape + (n_ops - 1)) : make_uint2(0, 0);
    for (int i = int(n_ops) - 1; i >= 0; --i) {
        const uint2 w = nxt;
        if (i > 0) nxt = ld_clause<NC>(tape + (i - 1));   // prefetch: the clause stream is the latency chain here
        Dec d(w.x);
        uint32_t c = 3u;
        bool is_choice = op_is_choice(d.op);
        if (is_choice) c = cs.pop();
        if (!active) continue;
        if (d.op == OP_OUTPUT) {
            set(d.lhs);
            *--wp = w;
            ++ref;
            continue;
        }
        if (!test(d.out)) continue;
        clear(d.out);
        if (is_choice && c != 3u) {
            if (c == 2u && d.form == F_RI) {
                *--wp = make_uint2(enc(OP_COPY, F_RI, d.out, 0xff, 0xff), w.y);
                ++ref;
            } else {
                // F_RI keeps its register in lhs; F_RR left = lhs, right = rhs
                uint32_t src = (c == 1u) ? d.lhs : d.rhs;
                if (src == d.out) {
                    set(d.out);
                } else {
                    uint32_t was = test(src);
                    set(src);
                    *--wp = make_uint2(enc(OP_COPY, was ? F_RR : F_ALIAS, d.out, src, 0xff), 0xFF000000u);
                    ref += was;
                }
            }
            continue;
        }
        if (d.op == OP_COPY && d.form != F_RI) {
            uint32_t src = d.lhs;
            if (src == d.out) { set(d.out); continue; }
            uint32_t was = test(src);
            set(src);
            uint32_t nf = (d.form == F_ALIAS || !was) ? F_ALIAS : F_RR;
            *--wp = make_uint2(enc(OP_COPY, nf, d.out, src, 0xff), w.y);
            ref += (nf == F_RR);
            continue;
        }
        *--wp = w;
        ++ref;
        if (is_choice) ++nch;
        if (d.op == OP_INPUT || d.op == OP_COPY) continue;
        if (d.op < OP_ADD) set(d.lhs);
        else {
            if (d.form != F_IR) set(d.lhs);
            if (d.form != F_RI) set(d.rhs);
        }
    }
    n_dev = uint32_t(wend - wp);
    ref_len = ref;
    n_choices = nch;
}

// Four-points-per-lane f32 interpreter (leaf voxels): decode, dispatch and register-file traffic
// are amortised over four points.
__device__ __forceinline__ float4 f32x4_unary(uint32_t op, float4 a) {
    switch (op) {
        case OP_NEG: return make_float4(-a.x, -a.y, -a.z, -a.w);
        case OP_ABS: return make_float4(fabsf(a.x), fabsf(a.y), fabsf(a.z), fabsf(a.w));
        case OP_SQRT: return make_float4(sqrtf(a.x), sqrtf(a.y), sqrtf(a.z), sqrtf(a.w));
        case OP_SQUARE: return make_float4(a.x * a.x, a.y * a.y, a.z * a.z, a.w * a.w);
        default: {
#ifndef FIDGET_UNROLLED_COLD
            // the long opcodes (libdevice transcendentals, rounding, rand ...) once in the code, not once per component:
            // the leaf kernels are instruction-cache sensitive (div and exp, frequent in bear.vm, have handlers of their own)
            float4 r = a;
#pragma unroll 1
            for (int k = 0; k < 4; ++k) {
                const float t = f32_unary(op, a.x);
                a = make_float4(a.y, a.z, a.w, a.x);
                r = make_float4(r.y, r.z, r.w, t);
            }
            return r;
#else
            return make_float4(f32_unary(op, a.x), f32_unary(op, a.y), f32_unary(op, a.z), f32_unary(op, a.w));
#endif
        }
    }
}
__device__ __forceinline__ float4 f32x4_binary(uint32_t op, float4 a, float4 b) {
    switch (op) {
        case OP_ADD: return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        case OP_SUB: return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
        case OP_MUL: return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
        case OP_MIN: return make_float4(f_min(a.x, b.x), f_min(a.y, b.y), f_min(a.z, b.z), f_min(a.w, b.w));
        case OP_MAX: return make_float4(f_max(a.x, b.x), f_max(a.y, b.y), f_max(a.z, b.z), f_max(a.w, b.w));
        default: {
#ifndef FIDGET_UNROLLED_COLD
            float4 r = a;
#pragma unroll 1
            for (int k = 0; k < 4; ++k) {
                const float t = f32_binary(op, a.x, b.x);
                a = make_float4(a.y, a.z, a.w, a.x);
                b = make_float4(b.y, b.z, b.w, b.x);
                r = make_float4(r.y, r.z, r.w, t);
            }
            return r;
#else
            return make_float4(f32_binary(op, a.x, b.x), f32_binary(op, a.y, b.y), f32_binary(op, a.z, b.z),
                               f32_binary(op, a.w, b.w));
#endif
        }
    }
}
// Hot loop dispatched through c_dop (see above); H_GENERIC is the plain decode-and-select path.
#define FB_BIN4(H, EXPR)                                                                     \
    case H##_RR: { const float4 b = slots[x >> 24]; const float4 a = sl; r = EXPR; break; }  \
    case H##_RI: { const float4 b = im; const float4 a = sl; r = EXPR; break; }              \
    case H##_IR: { const float4 b = slots[x >> 24]; const float4 a = im; r = EXPR; break; }
template <class Input>
__device__ __forceinline__ float4 run_f32x4(const uint2* __restrict__ tape, uint32_t n_ops, float4* slots, Input input) {
    float4 result = make_float4(nanf_(), nanf_(), nanf_(), nanf_());
    if (n_ops == 0) return result;
    uint2 w = __ldg(tape);
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint2 nxt = __ldg(tape + (i + 1 < n_ops ? i + 1 : i));
        const uint32_t x = w.x;
        const float imm = __uint_as_float(w.y);
        const float4 sl = slots[(x >> 16) & 0xffu];
        const float4 im = make_float4(imm, imm, imm, imm);
        float4 r;
        switch (c_dop_f.h[x & 0xffu]) {
            FB_BIN4(H_ADD, make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w))
            FB_BIN4(H_SUB, make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w))
            FB_BIN4(H_MUL, make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w))
            FB_BIN4(H_MIN, make_float4(f_min(a.x, b.x), f_min(a.y, b.y), f_min(a.z, b.z), f_min(a.w, b.w)))
            FB_BIN4(H_MAX, make_float4(f_max(a.x, b.x), f_max(a.y, b.y), f_max(a.z, b.z), f_max(a.w, b.w)))
            case H_NEG: r = make_float4(-sl.x, -sl.y, -sl.z, -sl.w); break;
            case H_ABS: r = make_float4(fabsf(sl.x), fabsf(sl.y), fabsf(sl.z), fabsf(sl.w)); break;
            case H_SQRT: r = make_float4(sqrtf(sl.x), sqrtf(sl.y), sqrtf(sl.z), sqrtf(sl.w)); break;
            case H_SQUARE: r = make_float4(sl.x * sl.x, sl.y * sl.y, sl.z * sl.z, sl.w * sl.w); break;
            case H_COPY_REG: r = sl; break;
            case H_COPY_IMM: r = im; break;
            FB_BIN4(H_DIV, make_float4(a.x / b.x, a.y / b.y, a.z / b.z, a.w / b.w))
            case H_EXP: r = make_float4(expf(sl.x), expf(sl.y), expf(sl.z), expf(sl.w)); break;
            default: __builtin_unreachable();
            case H_GENERIC: {
                const Dec d(x);
                const float4 sr = slots[d.rhs];
                const float4 a = d.form == F_IR ? im : sl;
                const float4 b = d.form == F_RI ? im : sr;
                if (d.op >= OP_ADD) {
                    if (d.op == OP_MEM) {
                        if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                        else slots[MEM_BASE + w.y] = sl;
                        w = nxt;
                        continue;
                    }
                    r = f32x4_binary(d.op, a, b);
                } else if (d.op >= OP_NEG) {
                    r = f32x4_unary(d.op, sl);
                } else if (d.op == OP_COPY) {
                    r = d.form == F_RI ? im : sl;
                } else if (d.op == OP_INPUT) {
                    r = input(w.y);
                } else {
                    if (w.y == 0) result = sl;
                    w = nxt;
                    continue;
                }
            }
        }
        slots[(x >> 8) & 0xffu] = r;
        w = nxt;
    }
    return result;
}

// Gradient interpreter (VmGradSliceEval, vm/mod.rs:1097-1396)
#define FB_BING(H, EXPR)                                                                  \
    case H##_RR: { const grd a = sl, b = slots[x >> 24]; r = EXPR; break; }               \
    case H##_RI: { const grd a = sl, b = gr1(imm); r = EXPR; break; }                     \
    case H##_IR: { const grd a = gr1(imm), b = slots[x >> 24]; r = EXPR; break; }
template <class Input>
__device__ __forceinline__ grd run_grad(const uint2* __restrict__ tape, uint32_t n_ops, grd* slots, Input input) {
    grd result = gr1(nanf_());
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint2 w = __ldg(tape + i);
        const uint32_t x = w.x;
        const float imm = __uint_as_float(w.y);
        const grd sl = slots[(x >> 16) & 0xffu];
        grd r;
        switch (c_dop_f.h[x & 0xffu]) {
            FB_BING(H_ADD, gr_add(a, b))
            FB_BING(H_SUB, gr_sub(a, b))
            case H_MUL_RR: r = gr_mul(sl, slots[x >> 24]); break;
            case H_MUL_RI: r = gr_mul_f(sl, imm); break;
            case H_MUL_IR: r = gr_mul(gr1(imm), slots[x >> 24]); break;
            FB_BING(H_MIN, gr_binary(OP_MIN, a, b))
            FB_BING(H_MAX, gr_binary(OP_MAX, a, b))
            FB_BING(H_DIV, gr_div(a, b))
            case H_NEG: r = gr_neg(sl); break;
            case H_SQUARE: r = gr_mul(sl, sl); break;
            case H_COPY_REG: r = sl; break;
            case H_COPY_IMM: r = gr1(imm); break;
            default: __builtin_unreachable();
            case H_ABS: case H_SQRT: case H_EXP:
            case H_GENERIC: {
                const Dec d(x);
                const grd sr = slots[d.rhs];
                const grd a = d.form == F_IR ? gr1(imm) : sl;
                const grd b = d.form == F_RI ? gr1(imm) : sr;
                if (d.op == OP_MEM) {
                    if (d.form == F_RI) slots[d.out] = slots[MEM_BASE + w.y];
                    else slots[MEM_BASE + w.y] = sl;
                    continue;
                } else if (d.op >= OP_ADD) {
                    r = gr_binary(d.op, a, b);
                } else if (d.op >= OP_NEG) {
                    r = gr_unary(d.op, sl);
                } else if (d.op == OP_COPY) {
                    r = d.form == F_RI ? gr1(imm) : sl;
                } else if (d.op == OP_INPUT) {
                    r = input(w.y);
                } else {
                    if (w.y == 0) result = sl;
                    continue;
                }
            }
        }
        slots[(x >> 8) & 0xffu] = r;
    }
    return result;
}

// The samplers' gradient probe (octree.rs:780-808): (v, dv/dx, dv/dy, dv/dz) of a tape at the world point (x, y, z),
// seen through `mat` when has_transform
__device__ __forceinline__ grd grad_at(const TapeRef& tr, grd* slots, float x, float y, float z, uint32_t has_transform,
                                       const Mat4& mat, const VarBind& vb) {
    grd gx = gr(x, 1.0f, 0.0f, 0.0f), gy = gr(y, 0.0f, 1.0f, 0.0f), gz = gr(z, 0.0f, 0.0f, 1.0f);
    if (has_transform) xform_gr(mat, gx, gy, gz, gx, gy, gz);
    return run_grad(tr.ptr, tr.n_ops, slots, [&](uint32_t k) {
        return pick_input(vb, k, gx, gy, gz, [](float f) { return gr1(f); });
    });
}

}  // namespace fdev
