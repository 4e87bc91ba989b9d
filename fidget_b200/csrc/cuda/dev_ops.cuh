// Device-side op semantics for the three tape interpreters (f32, interval,
// gradient) and the device tape encoding.
//
// What each function must compute is specified by the reference VM
// (fidget-core/src/vm/mod.rs:344-528 interval, 562-749 / 812-1083 f32,
// 1108-1394 grad) and its numeric types (types/interval.rs, types/grad.rs,
// types/float.rs); SURVEY.md Appendix A is the cheat-sheet.  This file is
// written for the GPU (float2 intervals, FMNMX-friendly NaN handling) and is
// NOT shared with the CPU oracle.
//
// Build flags that matter: -fmad=false (the reference never fuses a*b+c),
// -prec-div=true -prec-sqrt=true -ftz=false.
#pragma once
#ifdef __CUDACC_RTC__   // compiled tapes (compile.cu): NVRTC has no host headers
typedef unsigned char uint8_t;
typedef unsigned int uint32_t;
typedef unsigned long uint64_t;
#else
#include <cuda_runtime.h>
#include <stdint.h>
#endif

namespace fdev {

// ---- device tape encoding -------------------------------------------------
// One clause = uint2 {x: dop | out<<8 | lhs<<16 | rhs<<24, y: imm bits / index}
//   dop = opcode*4 + form; opcode numbering == fidget-bytecode's BytecodeOp.
//   form 0: reg,reg   1: reg,imm   2: imm,reg   3: device-only alias copy
//   OUTPUT: lhs = source register, y = output index
//   INPUT : out, y = variable index
//   COPY  : form 0 = CopyReg (exists in the reference tape), 1 = CopyImm,
//           3 = alias copy (the reference aliased the two SSA names, so the
//           clause does not count towards Function::size())
//   MEM   : form 1 = load out <- mem[y], form 2 = store mem[y] <- lhs
enum : uint32_t {
    OP_OUTPUT = 0, OP_INPUT, OP_COPY, OP_NEG, OP_ABS, OP_RECIP, OP_SQRT, OP_SQUARE,
    OP_FLOOR, OP_CEIL, OP_ROUND, OP_NOT, OP_RAND, OP_SIN, OP_COS, OP_TAN, OP_ASIN,
    OP_ACOS, OP_ATAN, OP_EXP, OP_LN, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_ATAN2,
    OP_COMPARE, OP_MIX, OP_MOD, OP_MIN, OP_MAX, OP_AND, OP_OR, OP_MEM, OP_COUNT
};
enum : uint32_t { F_RR = 0, F_RI = 1, F_IR = 2, F_ALIAS = 3 };
constexpr int MEM_BASE = 256;  // memory slot i lives at slot index 256 + i

__host__ __device__ inline uint32_t enc(uint32_t op, uint32_t form, uint32_t out, uint32_t lhs, uint32_t rhs) {
    return (op * 4u + form) | (out << 8) | (lhs << 16) | (rhs << 24);
}
// Multi-GPU tile interleave: which rank renders root tile (tx, ty).  A spatial hash rather than a regular
// pattern: per-tile cost is heavy-tailed and structured (text lines, silhouettes), and a pseudo-random spread keeps
// the busiest rank closer to the mean than a diagonal (tx + ty) % N, which lines such structure up on a few ranks.
__host__ __device__ inline uint32_t tile_owner(uint32_t tx, uint32_t ty, uint32_t n_ranks) {
    return ((tx * 73856093u) ^ (ty * 19349663u)) % n_ranks;
}
__host__ __device__ inline bool op_is_choice(uint32_t op) { return op >= OP_MIN && op <= OP_OR; }
__host__ __device__ inline bool op_is_binary(uint32_t op) { return op >= OP_ADD && op <= OP_OR; }
__host__ __device__ inline bool op_is_unary(uint32_t op) { return op >= OP_NEG && op <= OP_LN; }

#ifdef __CUDACC__
#define FD __device__ __forceinline__

FD float nanf_() { return __int_as_float(0x7fc00000); }

// rng/mod.rs:8-33
FD uint32_t rng_hash(uint32_t v) {
    uint32_t state = v * 747796405u + 2891336453u;
    uint32_t word = ((state >> ((state >> 28) + 4u)) ^ state) * 277803737u;
    return (word >> 22) ^ word;
}
FD float rng_rand(uint32_t seed) { return __uint_as_float((rng_hash(seed) >> 9) | 0x3f800000u) - 1.0f; }
FD uint32_t rng_mix(uint32_t a, uint32_t b) { return rng_hash(a + rng_hash(b)); }

// ---- f32 (types/float.rs:66-142) -----------------------------------------
// min_choice/max_choice values: NaN if either is NaN, ties return `b`
FD float f_min(float a, float b) { return a < b ? a : (b < a ? b : (a != a ? a : b)); }
FD float f_max(float a, float b) { return a > b ? a : (b > a ? b : (a != a ? a : b)); }
FD float f_compare(float a, float b) {
    return a < b ? -1.0f : (a > b ? 1.0f : (a == b ? 0.0f : nanf_()));
}
FD float f_rem_euclid(float a, float b) {
    float r = fmodf(a, b);
    return r < 0.0f ? r + fabsf(b) : r;
}
FD float f_div_euclid(float a, float b) {
    float q = truncf(a / b);
    if (fmodf(a, b) < 0.0f) return b > 0.0f ? q - 1.0f : q + 1.0f;
    return q;
}

FD float f32_unary(uint32_t op, float a) {
    switch (op) {
        case OP_NEG: return -a;
        case OP_ABS: return fabsf(a);
        case OP_RECIP: return 1.0f / a;
        case OP_SQRT: return sqrtf(a);
        case OP_SQUARE: return a * a;
        case OP_FLOOR: return floorf(a);
        case OP_CEIL: return ceilf(a);
        case OP_ROUND: return roundf(a);
        case OP_NOT: return a == 0.0f ? 1.0f : 0.0f;
        case OP_RAND: return rng_rand(__float_as_uint(a));
        case OP_SIN: return sinf(a);
        case OP_COS: return cosf(a);
        case OP_TAN: return tanf(a);
        case OP_ASIN: return asinf(a);
        case OP_ACOS: return acosf(a);
        case OP_ATAN: return atanf(a);
        case OP_EXP: return expf(a);
        default: return logf(a);  // OP_LN
    }
}
FD float f32_binary(uint32_t op, float a, float b) {
    switch (op) {
        case OP_ADD: return a + b;
        case OP_SUB: return a - b;
        case OP_MUL: return a * b;
        case OP_DIV: return a / b;
        case OP_ATAN2: return atan2f(a, b);
        case OP_COMPARE: return f_compare(a, b);
        case OP_MIX: return __uint_as_float(rng_mix(__float_as_uint(a), __float_as_uint(b)));
        case OP_MOD: return f_rem_euclid(a, b);
        case OP_MIN: return f_min(a, b);
        case OP_MAX: return f_max(a, b);
        case OP_AND: return a == 0.0f ? a : b;
        default: return a != 0.0f ? a : b;  // OP_OR
    }
}
// Choice of a point evaluation (1 = left, 2 = right, 3 = both)
FD uint32_t f32_choice(uint32_t op, float a, float b) {
    switch (op) {
        case OP_MIN: return a < b ? 1u : (b < a ? 2u : 3u);
        case OP_MAX: return a > b ? 1u : (b > a ? 2u : 3u);
        case OP_AND: return a == 0.0f ? 1u : 2u;
        default: return a != 0.0f ? 1u : 2u;
    }
}

// ---- intervals: float2 {x = lower, y = upper} (types/interval.rs) ----------
typedef float2 itv;
FD itv iv(float lo, float hi) { return make_float2(lo, hi); }
FD itv iv1(float f) { return make_float2(f, f); }
FD itv iv_nan() { return make_float2(nanf_(), nanf_()); }
FD bool iv_has_nan(itv a) { return a.x != a.x || a.y != a.y; }
FD bool iv_contains0(itv a) { return 0.0f >= a.x && 0.0f <= a.y; }

#define FC_PI 3.14159265358979323846f
#define FC_TAU 6.28318530717958647692f

FD itv iv_neg(itv a) { return iv(-a.y, -a.x); }
FD itv iv_abs(itv a) {
    if (a.x < 0.0f) return a.y > 0.0f ? iv(0.0f, fmaxf(a.y, -a.x)) : iv(-a.y, -a.x);
    return a;
}
FD itv iv_square(itv a) {
    if (a.y < 0.0f) return iv(a.y * a.y, a.x * a.x);
    if (a.x > 0.0f) return iv(a.x * a.x, a.y * a.y);
    if (iv_has_nan(a)) return iv_nan();
    float m = fmaxf(fabsf(a.x), fabsf(a.y));
    return iv(0.0f, m * m);
}
FD itv iv_sqrt(itv a) { return a.x < 0.0f ? iv_nan() : iv(sqrtf(a.x), sqrtf(a.y)); }
FD itv iv_recip(itv a) { return (a.x > 0.0f || a.y < 0.0f) ? iv(1.0f / a.y, 1.0f / a.x) : iv_nan(); }
FD itv iv_add(itv a, itv b) { return iv(a.x + b.x, a.y + b.y); }
FD itv iv_sub(itv a, itv b) { return iv(a.x - b.y, a.y - b.x); }
FD itv iv_mul(itv a, itv b) {
    if (iv_has_nan(a) || iv_has_nan(b)) return iv_nan();
    float o0 = a.x * b.x, o1 = a.x * b.y, o2 = a.y * b.x, o3 = a.y * b.y;
    return iv(fminf(fminf(o0, o1), fminf(o2, o3)), fmaxf(fmaxf(o0, o1), fmaxf(o2, o3)));
}
FD itv iv_mul_f(itv a, float k) {  // Mul<f32> (interval.rs:683-696)
    if (iv_has_nan(a) || k != k) return iv_nan();
    return k < 0.0f ? iv(a.y * k, a.x * k) : iv(a.x * k, a.y * k);
}
FD itv iv_div(itv a, itv b) {
    if (iv_has_nan(a)) return iv_nan();
    if (b.x > 0.0f || b.y < 0.0f) {
        float o0 = a.x / b.x, o1 = a.x / b.y, o2 = a.y / b.x, o3 = a.y / b.y;
        return iv(fminf(fminf(o0, o1), fminf(o2, o3)), fmaxf(fmaxf(o0, o1), fmaxf(o2, o3)));
    }
    return iv_nan();
}
FD int iv_quadrant(float angle) {
    float q = f_rem_euclid(floorf(angle * 2.0f / FC_PI), 4.0f);
    return (q != q) ? 0 : (int)(unsigned char)q;
}
// mode 0 = sin, 1 = cos.  cos(x) has sin's monotonicity table shifted by one
// quadrant: (ql, qu) -> (ql + 1, qu + 1) mod 4.
FD itv iv_sincos(itv a, int is_cos) {
    if (iv_has_nan(a)) return iv_nan();
    float d = a.y - a.x;
    if (d >= FC_TAU) return iv(-1.0f, 1.0f);
    float fl = is_cos ? cosf(a.x) : sinf(a.x);
    if (a.x == a.y) return iv1(fl);
    float fu = is_cos ? cosf(a.y) : sinf(a.y);
    int ql = (iv_quadrant(a.x) + is_cos) & 3, qu = (iv_quadrant(a.y) + is_cos) & 3;
    // In sin-terms: Q0,Q3 increasing; Q1,Q2 decreasing
    if (ql == qu) {
        if (d >= FC_PI) return iv(-1.0f, 1.0f);
        return (ql == 1 || ql == 2) ? iv(fu, fl) : iv(fl, fu);
    }
    if (ql == 3 && qu == 0) return d >= FC_PI ? iv(-1.0f, 1.0f) : iv(fl, fu);
    if (ql == 1 && qu == 2) return d >= FC_PI ? iv(-1.0f, 1.0f) : iv(fu, fl);
    bool l_inc = (ql == 0 || ql == 3), u_inc = (qu == 0 || qu == 3);
    if (l_inc && !u_inc) return iv(fminf(fl, fu), 1.0f);
    if (!l_inc && u_inc) return iv(-1.0f, fmaxf(fl, fu));
    return iv(-1.0f, 1.0f);  // (Q0,Q3) | (Q2,Q1)
}
FD itv iv_tan(itv a) {
    float size = a.y - a.x;
    if (size >= FC_PI) return iv_nan();
    if (a.x == a.y) return iv1(tanf(a.x));
    float l = tanf(a.x), u = tanf(a.y);
    return u >= l ? iv(l, u) : iv_nan();
}
FD itv iv_asin(itv a) {
    if (a.x < -1.0f || a.y > 1.0f) return iv_nan();
    if (a.x == a.y) return iv1(asinf(a.x));
    return iv(asinf(a.x), asinf(a.y));
}
FD itv iv_acos(itv a) {
    if (a.x < -1.0f || a.y > 1.0f) return iv_nan();
    if (a.x == a.y) return iv1(acosf(a.x));
    return iv(acosf(a.y), acosf(a.x));
}
FD itv iv_ln(itv a) { return a.x <= 0.0f ? iv_nan() : iv(logf(a.x), logf(a.y)); }
FD itv iv_not(itv a) {
    if (!iv_contains0(a) && !iv_has_nan(a)) return iv(0.0f, 0.0f);
    if (a.x == 0.0f && a.y == 0.0f) return iv(1.0f, 1.0f);
    return iv(0.0f, 1.0f);
}
FD itv iv_rand(itv a) {
    if (iv_has_nan(a) || __float_as_uint(a.x) != __float_as_uint(a.y)) return iv(0.0f, 1.0f);
    return iv1(rng_rand(__float_as_uint(a.x)));
}
FD itv iv_mix(itv a, itv b) {
    if (iv_has_nan(a) || iv_has_nan(b) || __float_as_uint(a.x) != __float_as_uint(a.y) ||
        __float_as_uint(b.x) != __float_as_uint(b.y))
        return iv_nan();
    return iv1(__uint_as_float(rng_mix(__float_as_uint(a.x), __float_as_uint(b.x))));
}
FD itv iv_compare(itv l, itv r) {
    if (iv_has_nan(l) || iv_has_nan(r)) return iv_nan();
    if (l.y < r.x) return iv1(-1.0f);
    if (l.x > r.y) return iv1(1.0f);
    if (l.x == l.y && r.x == r.y && l.x == r.x) return iv(0.0f, 0.0f);
    return iv(-1.0f, 1.0f);
}
FD itv iv_rem_euclid(itv a, itv o) {
    if (iv_has_nan(a) || iv_has_nan(o) || iv_contains0(o)) return iv_nan();
    float oabs = iv_abs(o).y;
    if (o.x == o.y && o.x > 0.0f) {
        float x = a.x / o.x, y = a.y / o.x;
        if (x != floorf(x) && floorf(x) == floorf(y))
            return iv(f_rem_euclid(a.x, o.x), f_rem_euclid(a.y, o.x));
    }
    return iv(0.0f, oabs);
}
FD itv iv_atan2(itv y, itv x) {
    if (iv_has_nan(y) || iv_has_nan(x)) return iv_nan();
    if (y.x <= 0.0f && y.y >= 0.0f && x.x < 0.0f) return iv(-FC_PI, FC_PI);
    float y0, x0, y1, x1;  // the two corner evaluations of interval.rs:560-597
    if (y.x >= 0.0f) {
        if (x.x >= 0.0f) { y0 = y.y; x0 = x.x; y1 = y.x; x1 = x.y; }
        else if (x.y <= 0.0f) { y0 = y.x; x0 = x.x; y1 = y.y; x1 = x.y; }
        else { y0 = y.x; x0 = x.x; y1 = y.x; x1 = x.y; }
    } else if (y.y <= 0.0f) {
        if (x.x >= 0.0f) { y0 = y.x; x0 = x.x; y1 = y.y; x1 = x.y; }
        else if (x.y <= 0.0f) { y0 = y.y; x0 = x.x; y1 = y.x; x1 = x.y; }
        else { y0 = y.y; x0 = x.x; y1 = y.y; x1 = x.y; }
    } else {
        y0 = y.x; x0 = x.x; y1 = y.y; x1 = x.x;
    }
    float v0 = atan2f(y0, x0), v1 = atan2f(y1, x1);
    return iv(fminf(fminf(__int_as_float(0x7f800000), v0), v1), fmaxf(fmaxf(__int_as_float(0xff800000), v0), v1));
}

FD itv iv_unary(uint32_t op, itv a) {
    switch (op) {
        case OP_NEG: return iv_neg(a);
        case OP_ABS: return iv_abs(a);
        case OP_RECIP: return iv_recip(a);
        case OP_SQRT: return iv_sqrt(a);
        case OP_SQUARE: return iv_square(a);
        case OP_FLOOR: return iv(floorf(a.x), floorf(a.y));
        case OP_CEIL: return iv(ceilf(a.x), ceilf(a.y));
        case OP_ROUND: return iv(roundf(a.x), roundf(a.y));
        case OP_NOT: return iv_not(a);
        case OP_RAND: return iv_rand(a);
        case OP_SIN: return iv_sincos(a, 0);
        case OP_COS: return iv_sincos(a, 1);
        case OP_TAN: return iv_tan(a);
        case OP_ASIN: return iv_asin(a);
        case OP_ACOS: return iv_acos(a);
        case OP_ATAN: return iv(atanf(a.x), atanf(a.y));
        case OP_EXP: return iv(expf(a.x), expf(a.y));
        default: return iv_ln(a);
    }
}
// Non-choice binary ops
FD itv iv_binary(uint32_t op, itv a, itv b) {
    switch (op) {
        case OP_ADD: return iv_add(a, b);
        case OP_SUB: return iv_sub(a, b);
        case OP_MUL: return iv_mul(a, b);
        case OP_DIV: return iv_div(a, b);
        case OP_ATAN2: return iv_atan2(a, b);
        case OP_COMPARE: return iv_compare(a, b);
        case OP_MIX: return iv_mix(a, b);
        default: return iv_rem_euclid(a, b);  // OP_MOD
    }
}
// Choice ops: returns the value, writes the choice (1 left, 2 right, 3 both)
FD itv iv_choice_op(uint32_t op, itv a, itv b, uint32_t& c) {
    if (iv_has_nan(a) || iv_has_nan(b)) { c = 3u; return iv_nan(); }
    switch (op) {
        case OP_MIN:
            c = a.y < b.x ? 1u : (b.y < a.x ? 2u : 3u);
            return iv(fminf(a.x, b.x), fminf(a.y, b.y));
        case OP_MAX:
            c = a.x > b.y ? 1u : (b.x > a.y ? 2u : 3u);
            return iv(fmaxf(a.x, b.x), fmaxf(a.y, b.y));
        case OP_AND:
            if (a.x == 0.0f && a.y == 0.0f) { c = 1u; return iv1(0.0f); }
            if (!iv_contains0(a)) { c = 2u; return b; }
            c = 3u;
            return iv(fminf(b.x, 0.0f), fmaxf(b.y, 0.0f));
        default:  // OP_OR
            if (!iv_contains0(a)) { c = 1u; return a; }
            if (a.x == 0.0f && a.y == 0.0f) { c = 2u; return b; }
            c = 3u;
            return iv(fminf(a.x, b.x), fmaxf(a.y, b.y));
    }
}

// ---- gradients: float4 {x = v, y = dx, z = dy, w = dz} (types/grad.rs) -----
typedef float4 grd;
FD grd gr(float v, float dx, float dy, float dz) { return make_float4(v, dx, dy, dz); }
FD grd gr1(float v) { return make_float4(v, 0.0f, 0.0f, 0.0f); }
FD grd gr_add(grd a, grd b) { return gr(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
FD grd gr_sub(grd a, grd b) { return gr(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
FD grd gr_neg(grd a) { return gr(-a.x, -a.y, -a.z, -a.w); }
FD grd gr_mul(grd a, grd b) {
    return gr(a.x * b.x, a.x * b.y + b.x * a.y, a.x * b.z + b.x * a.z, a.x * b.w + b.x * a.w);
}
FD grd gr_mul_f(grd a, float k) { return gr(a.x * k, a.y * k, a.z * k, a.w * k); }
FD grd gr_div(grd a, grd b) {
    float d = b.x * b.x;
    return gr(a.x / b.x, (b.x * a.y - a.x * b.y) / d, (b.x * a.z - a.x * b.z) / d, (b.x * a.w - a.x * b.w) / d);
}
FD grd gr_scale_div(grd a, float v, float r) { return gr(v, a.y / r, a.z / r, a.w / r); }
FD grd gr_unary(uint32_t op, grd a) {
    switch (op) {
        case OP_NEG: return gr_neg(a);
        case OP_ABS: return a.x < 0.0f ? gr_neg(a) : a;
        case OP_RECIP: return gr_div(gr1(1.0f), a);
        case OP_SQRT: { float v = sqrtf(a.x); return gr_scale_div(a, v, 2.0f * v); }
        case OP_SQUARE: return gr_mul(a, a);
        case OP_FLOOR: return gr1(floorf(a.x));
        case OP_CEIL: return gr1(ceilf(a.x));
        case OP_ROUND: return gr1(roundf(a.x));
        case OP_NOT: return gr1(a.x == 0.0f ? 1.0f : 0.0f);
        case OP_RAND: return gr1(rng_rand(__float_as_uint(a.x)));
        case OP_SIN: { float c = cosf(a.x); return gr(sinf(a.x), a.y * c, a.z * c, a.w * c); }
        case OP_COS: { float s = -sinf(a.x); return gr(cosf(a.x), a.y * s, a.z * s, a.w * s); }
        case OP_TAN: { float c0 = cosf(a.x); return gr_scale_div(a, tanf(a.x), c0 * c0); }
        case OP_ASIN: { float r = sqrtf(1.0f - a.x * a.x); return gr_scale_div(a, asinf(a.x), r); }
        case OP_ACOS: { float r = sqrtf(1.0f - a.x * a.x); return gr(acosf(a.x), -a.y / r, -a.z / r, -a.w / r); }
        case OP_ATAN: { float r = a.x * a.x + 1.0f; return gr_scale_div(a, atanf(a.x), r); }
        case OP_EXP: { float v = expf(a.x); return gr(v, v * a.y, v * a.z, v * a.w); }
        default: return gr_scale_div(a, logf(a.x), a.x);  // OP_LN
    }
}
FD grd gr_binary(uint32_t op, grd a, grd b) {
    switch (op) {
        case OP_ADD: return gr_add(a, b);
        case OP_SUB: return gr_sub(a, b);
        case OP_MUL: return gr_mul(a, b);
        case OP_DIV: return gr_div(a, b);
        case OP_ATAN2: {
            float d = b.x * b.x + a.x * a.x;
            return gr(atan2f(a.x, b.x), (b.x * a.y - a.x * b.y) / d, (b.x * a.z - a.x * b.z) / d,
                      (b.x * a.w - a.x * b.w) / d);
        }
        case OP_COMPARE: return gr1(f_compare(a.x, b.x));
        case OP_MIX: return gr1(__uint_as_float(rng_mix(__float_as_uint(a.x), __float_as_uint(b.x))));
        case OP_MOD: {
            float e = f_div_euclid(a.x, b.x);
            return gr(f_rem_euclid(a.x, b.x), a.y - b.y * e, a.z - b.z * e, a.w - b.w * e);
        }
        case OP_MIN: return (a.x != a.x || b.x != b.x) ? gr1(nanf_()) : (a.x < b.x ? a : b);
        case OP_MAX: return (a.x != a.x || b.x != b.x) ? gr1(nanf_()) : (a.x > b.x ? a : b);
        case OP_AND: return a.x == 0.0f ? a : b;
        default: return a.x != 0.0f ? a : b;
    }
}

// ---- transforms (shape/mod.rs:894-948) -------------------------------------
struct Mat4 { float m[16]; };  // row-major
// nalgebra transform_point: ((m0*x + m1*y) + m2*z) + m3, divided by the
// homogeneous term when that is non-zero
FD void xform_f32(const Mat4& M, float x, float y, float z, float& ox, float& oy, float& oz) {
    const float* m = M.m;
    float n = ((m[12] * x + m[13] * y) + m[14] * z) + m[15];
    float rx = ((m[0] * x + m[1] * y) + m[2] * z) + m[3];
    float ry = ((m[4] * x + m[5] * y) + m[6] * z) + m[7];
    float rz = ((m[8] * x + m[9] * y) + m[10] * z) + m[11];
    if (n != 0.0f) { rx = rx / n; ry = ry / n; rz = rz / n; }
    ox = rx; oy = ry; oz = rz;
}
FD void xform_iv(const Mat4& M, itv x, itv y, itv z, itv& ox, itv& oy, itv& oz) {
    itv o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float* r = M.m + 4 * i;
        o[i] = iv_add(iv_add(iv_add(iv_mul_f(x, r[0]), iv_mul_f(y, r[1])), iv_mul_f(z, r[2])), iv1(r[3]));
    }
    ox = iv_div(o[0], o[3]); oy = iv_div(o[1], o[3]); oz = iv_div(o[2], o[3]);
}
FD void xform_gr(const Mat4& M, grd x, grd y, grd z, grd& ox, grd& oy, grd& oz) {
    grd o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float* r = M.m + 4 * i;
        o[i] = gr_add(gr_add(gr_add(gr_mul_f(x, r[0]), gr_mul_f(y, r[1])), gr_mul_f(z, r[2])), gr1(r[3]));
    }
    ox = gr_div(o[0], o[3]); oy = gr_div(o[1], o[3]); oz = gr_div(o[2], o[3]);
}

#endif  // __CUDACC__
}  // namespace fdev
