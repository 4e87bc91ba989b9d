// ORACLE -- test infrastructure, not product code.  See vm.h for the
// reference map (file:line) of every function in this file.
#include "vm.h"

#include <algorithm>
#include <atomic>
#include <cassert>
#include <stdexcept>
#include <thread>

namespace oracle {
using namespace fhost;

Tape::Tape(TapeData t) : d(std::move(t)) {
    eval_order.assign(d.asm_.tape.rbegin(), d.asm_.tape.rend());
}

////////////////////////////////////////////////////////////////////////////
// VmIntervalEval::eval (vm/mod.rs:332-537)
bool IntervalEval::eval(const Tape& t, const Interval* vars, Interval* out) {
    slots.assign(std::max<size_t>(t.slot_count(), 1), Interval::nan());
    choices.assign(t.choice_count(), C_UNKNOWN);
    bool simplify = false;
    size_t ci = 0;
    Interval* v = slots.data();
    for (const Clause& c : t.eval_order) {
        Interval a, b;
        if (is_binary(c.op)) {
            if (c.form == F_RR) { a = v[c.a]; b = v[c.b]; }
            else if (c.form == F_RI) { a = v[c.a]; b = Interval(c.imm); }
            else { a = Interval(c.imm); b = v[c.a]; }
        } else if (is_unary(c.op)) {
            a = v[c.a];
        }
        switch (c.op) {
            case OP_OUTPUT: out[c.idx] = v[c.a]; break;
            case OP_INPUT: v[c.out] = vars[c.idx]; break;
            case OP_COPY: v[c.out] = c.form == F_RI ? Interval(c.imm) : v[c.a]; break;
            case OP_MEM:
                if (c.form == F_RI) v[c.out] = v[c.idx]; else v[c.idx] = v[c.a];
                break;
            case OP_NEG: v[c.out] = i_neg(a); break;
            case OP_ABS: v[c.out] = i_abs(a); break;
            case OP_RECIP: v[c.out] = i_recip(a); break;
            case OP_SQRT: v[c.out] = i_sqrt(a); break;
            case OP_SQUARE: v[c.out] = i_square(a); break;
            case OP_FLOOR: v[c.out] = i_floor(a); break;
            case OP_CEIL: v[c.out] = i_ceil(a); break;
            case OP_ROUND: v[c.out] = i_round(a); break;
            case OP_NOT: v[c.out] = i_not(a); break;
            case OP_RAND: v[c.out] = i_rand(a); break;
            case OP_SIN: v[c.out] = i_sin(a); break;
            case OP_COS: v[c.out] = i_cos(a); break;
            case OP_TAN: v[c.out] = i_tan(a); break;
            case OP_ASIN: v[c.out] = i_asin(a); break;
            case OP_ACOS: v[c.out] = i_acos(a); break;
            case OP_ATAN: v[c.out] = i_atan(a); break;
            case OP_EXP: v[c.out] = i_exp(a); break;
            case OP_LN: v[c.out] = i_ln(a); break;
            case OP_ADD: v[c.out] = i_add(a, b); break;
            case OP_SUB: v[c.out] = i_sub(a, b); break;
            case OP_MUL:
                // MulRegImm goes through `Mul<f32>` (vm/mod.rs:418-420)
                v[c.out] = c.form == F_RI ? i_mul_f(a, c.imm) : i_mul(a, b);
                break;
            case OP_DIV: v[c.out] = i_div(a, b); break;
            case OP_ATAN2: v[c.out] = i_atan2(a, b); break;
            case OP_COMPARE: v[c.out] = i_compare(a, b); break;
            case OP_MIX: v[c.out] = i_mix(a, b); break;
            case OP_MOD: v[c.out] = i_rem_euclid(a, b); break;
            case OP_MIN: case OP_MAX: case OP_AND: case OP_OR: {
                IC r = c.op == OP_MIN ? i_min_choice(a, b)
                     : c.op == OP_MAX ? i_max_choice(a, b)
                     : c.op == OP_AND ? i_and_choice(a, b) : i_or_choice(a, b);
                v[c.out] = r.v;
                choices[ci++] |= r.c;
                simplify |= r.c != C_BOTH;
                break;
            }
            default: throw std::runtime_error("bad opcode");
        }
    }
    return simplify;
}

////////////////////////////////////////////////////////////////////////////
// VmPointEval::eval (vm/mod.rs:551-759)
static inline float point_unary(uint8_t op, float a) {
    switch (op) {
        case OP_NEG: return -a;
        case OP_ABS: return std::fabs(a);
        case OP_RECIP: return 1.0f / a;
        case OP_SQRT: return std::sqrt(a);
        case OP_SQUARE: return a * a;
        case OP_FLOOR: return std::floor(a);
        case OP_CEIL: return std::ceil(a);
        case OP_ROUND: return std::round(a);
        case OP_NOT: return f_not(a);
        case OP_RAND: return rng_rand(f2u(a));
        case OP_SIN: return std::sin(a);
        case OP_COS: return std::cos(a);
        case OP_TAN: return std::tan(a);
        case OP_ASIN: return std::asin(a);
        case OP_ACOS: return std::acos(a);
        case OP_ATAN: return std::atan(a);
        case OP_EXP: return std::exp(a);
        default: return std::log(a);  // OP_LN
    }
}
static inline float point_binary(uint8_t op, float a, float b) {
    switch (op) {
        case OP_ADD: return a + b;
        case OP_SUB: return a - b;
        case OP_MUL: return a * b;
        case OP_DIV: return a / b;
        case OP_ATAN2: return std::atan2(a, b);
        case OP_COMPARE: return f_compare(a, b);
        case OP_MIX: return u2f(rng_mix(f2u(a), f2u(b)));
        case OP_MOD: return rem_euclid(a, b);
        case OP_MIN: return f_min_choice(a, b).v;
        case OP_MAX: return f_max_choice(a, b).v;
        case OP_AND: return f_and_choice(a, b).v;
        default: return f_or_choice(a, b).v;  // OP_OR
    }
}

bool PointEval::eval(const Tape& t, const float* vars, float* out) {
    slots.assign(std::max<size_t>(t.slot_count(), 1), NAN);
    choices.assign(t.choice_count(), C_UNKNOWN);
    bool simplify = false;
    size_t ci = 0;
    float* v = slots.data();
    for (const Clause& c : t.eval_order) {
        if (is_unary(c.op)) { v[c.out] = point_unary(c.op, v[c.a]); continue; }
        if (is_binary(c.op)) {
            float a, b;
            if (c.form == F_RR) { a = v[c.a]; b = v[c.b]; }
            else if (c.form == F_RI) { a = v[c.a]; b = c.imm; }
            else { a = c.imm; b = v[c.a]; }
            if (is_choice(c.op)) {
                FC r = c.op == OP_MIN ? f_min_choice(a, b) : c.op == OP_MAX ? f_max_choice(a, b)
                     : c.op == OP_AND ? f_and_choice(a, b) : f_or_choice(a, b);
                v[c.out] = r.v;
                choices[ci++] |= r.c;
                simplify |= r.c != C_BOTH;
            } else {
                v[c.out] = point_binary(c.op, a, b);
            }
            continue;
        }
        switch (c.op) {
            case OP_OUTPUT: out[c.idx] = v[c.a]; break;
            case OP_INPUT: v[c.out] = vars[c.idx]; break;
            case OP_COPY: v[c.out] = c.form == F_RI ? c.imm : v[c.a]; break;
            case OP_MEM:
                if (c.form == F_RI) v[c.out] = v[c.idx]; else v[c.idx] = v[c.a];
                break;
            default: throw std::runtime_error("bad opcode");
        }
    }
    return simplify;
}

////////////////////////////////////////////////////////////////////////////
// VmFloatSliceEval::eval (vm/mod.rs:800-1085): op-major over n lanes
void FloatSliceEval::eval(const Tape& t, const float* const* vars, size_t n, float* const* out) {
    size_t ns = std::max<size_t>(t.slot_count(), 1);
    if (slots.size() < ns) slots.resize(ns);
    for (size_t i = 0; i < ns; ++i)
        if (slots[i].size() < n) slots[i].resize(n, NAN);
    auto& v = slots;
    for (const Clause& c : t.eval_order) {
        if (is_unary(c.op)) {
            float* o = v[c.out].data();
            const float* a = v[c.a].data();
            switch (c.op) {
                case OP_NEG: for (size_t i = 0; i < n; ++i) o[i] = -a[i]; break;
                case OP_ABS: for (size_t i = 0; i < n; ++i) o[i] = std::fabs(a[i]); break;
                case OP_SQRT: for (size_t i = 0; i < n; ++i) o[i] = std::sqrt(a[i]); break;
                case OP_SQUARE: for (size_t i = 0; i < n; ++i) o[i] = a[i] * a[i]; break;
                default: for (size_t i = 0; i < n; ++i) o[i] = point_unary(c.op, a[i]); break;
            }
            continue;
        }
        if (is_binary(c.op)) {
            float* o = v[c.out].data();
            if (c.form == F_RR) {
                const float* a = v[c.a].data();
                const float* b = v[c.b].data();
                switch (c.op) {
                    case OP_ADD: for (size_t i = 0; i < n; ++i) o[i] = a[i] + b[i]; break;
                    case OP_SUB: for (size_t i = 0; i < n; ++i) o[i] = a[i] - b[i]; break;
                    case OP_MUL: for (size_t i = 0; i < n; ++i) o[i] = a[i] * b[i]; break;
                    case OP_MIN: for (size_t i = 0; i < n; ++i) o[i] = f_min_choice(a[i], b[i]).v; break;
                    case OP_MAX: for (size_t i = 0; i < n; ++i) o[i] = f_max_choice(a[i], b[i]).v; break;
                    default: for (size_t i = 0; i < n; ++i) o[i] = point_binary(c.op, a[i], b[i]); break;
                }
            } else if (c.form == F_RI) {
                const float* a = v[c.a].data();
                const float k = c.imm;
                switch (c.op) {
                    case OP_ADD: for (size_t i = 0; i < n; ++i) o[i] = a[i] + k; break;
                    case OP_SUB: for (size_t i = 0; i < n; ++i) o[i] = a[i] - k; break;
                    case OP_MUL: for (size_t i = 0; i < n; ++i) o[i] = a[i] * k; break;
                    default: for (size_t i = 0; i < n; ++i) o[i] = point_binary(c.op, a[i], k); break;
                }
            } else {
                const float* b = v[c.a].data();
                const float k = c.imm;
                switch (c.op) {
                    case OP_SUB: for (size_t i = 0; i < n; ++i) o[i] = k - b[i]; break;
                    default: for (size_t i = 0; i < n; ++i) o[i] = point_binary(c.op, k, b[i]); break;
                }
            }
            continue;
        }
        switch (c.op) {
            case OP_OUTPUT: std::copy(v[c.a].begin(), v[c.a].begin() + n, out[c.idx]); break;
            case OP_INPUT: std::copy(vars[c.idx], vars[c.idx] + n, v[c.out].begin()); break;
            case OP_COPY:
                if (c.form == F_RI) std::fill(v[c.out].begin(), v[c.out].begin() + n, c.imm);
                else if (c.out != c.a) std::copy(v[c.a].begin(), v[c.a].begin() + n, v[c.out].begin());
                break;
            case OP_MEM:
                if (c.form == F_RI) std::copy(v[c.idx].begin(), v[c.idx].begin() + n, v[c.out].begin());
                else std::copy(v[c.a].begin(), v[c.a].begin() + n, v[c.idx].begin());
                break;
            default: throw std::runtime_error("bad opcode");
        }
    }
}

////////////////////////////////////////////////////////////////////////////
// VmGradSliceEval::eval (vm/mod.rs:1097-1396)
static inline Grad grad_unary(uint8_t op, Grad a) {
    switch (op) {
        case OP_NEG: return g_neg(a);
        case OP_ABS: return g_abs(a);
        case OP_RECIP: return g_div(Grad(1.0f), a);
        case OP_SQRT: return g_sqrt(a);
        case OP_SQUARE: return g_mul(a, a);
        case OP_FLOOR: return Grad(std::floor(a.v));
        case OP_CEIL: return Grad(std::ceil(a.v));
        case OP_ROUND: return Grad(std::round(a.v));
        case OP_NOT: return Grad(f_not(a.v));
        case OP_RAND: return Grad(rng_rand(f2u(a.v)));
        case OP_SIN: return g_sin(a);
        case OP_COS: return g_cos(a);
        case OP_TAN: return g_tan(a);
        case OP_ASIN: return g_asin(a);
        case OP_ACOS: return g_acos(a);
        case OP_ATAN: return g_atan(a);
        case OP_EXP: return g_exp(a);
        default: return g_ln(a);
    }
}
static inline Grad grad_binary(uint8_t op, Grad a, Grad b) {
    switch (op) {
        case OP_ADD: return g_add(a, b);
        case OP_SUB: return g_sub(a, b);
        case OP_MUL: return g_mul(a, b);
        case OP_DIV: return g_div(a, b);
        case OP_ATAN2: return g_atan2(a, b);
        case OP_COMPARE: return g_compare(a, b);
        case OP_MIX: return Grad(u2f(rng_mix(f2u(a.v), f2u(b.v))));
        case OP_MOD: return g_rem_euclid(a, b);
        case OP_MIN: return g_min(a, b);
        case OP_MAX: return g_max(a, b);
        case OP_AND: return g_and(a, b);
        default: return g_or(a, b);
    }
}

void GradSliceEval::eval(const Tape& t, const Grad* const* vars, size_t n, Grad* const* out) {
    size_t ns = std::max<size_t>(t.slot_count(), 1);
    if (slots.size() < ns) slots.resize(ns);
    for (size_t i = 0; i < ns; ++i)
        if (slots[i].size() < n) slots[i].resize(n, Grad(NAN));
    auto& v = slots;
    for (const Clause& c : t.eval_order) {
        if (is_unary(c.op)) {
            for (size_t i = 0; i < n; ++i) v[c.out][i] = grad_unary(c.op, v[c.a][i]);
            continue;
        }
        if (is_binary(c.op)) {
            if (c.form == F_RR) {
                for (size_t i = 0; i < n; ++i) v[c.out][i] = grad_binary(c.op, v[c.a][i], v[c.b][i]);
            } else if (c.form == F_RI) {
                if (c.op == OP_MUL)  // `Grad * f32` (vm/mod.rs:1205-1209)
                    for (size_t i = 0; i < n; ++i) v[c.out][i] = g_mul_f(v[c.a][i], c.imm);
                else
                    for (size_t i = 0; i < n; ++i) v[c.out][i] = grad_binary(c.op, v[c.a][i], Grad(c.imm));
            } else {
                for (size_t i = 0; i < n; ++i) v[c.out][i] = grad_binary(c.op, Grad(c.imm), v[c.a][i]);
            }
            continue;
        }
        switch (c.op) {
            case OP_OUTPUT: std::copy(v[c.a].begin(), v[c.a].begin() + n, out[c.idx]); break;
            case OP_INPUT: std::copy(vars[c.idx], vars[c.idx] + n, v[c.out].begin()); break;
            case OP_COPY:
                if (c.form == F_RI) std::fill(v[c.out].begin(), v[c.out].begin() + n, Grad(c.imm));
                else if (c.out != c.a) std::copy(v[c.a].begin(), v[c.a].begin() + n, v[c.out].begin());
                break;
            case OP_MEM:
                if (c.form == F_RI) std::copy(v[c.idx].begin(), v[c.idx].begin() + n, v[c.out].begin());
                else std::copy(v[c.a].begin(), v[c.a].begin() + n, v[c.idx].begin());
                break;
            default: throw std::runtime_error("bad opcode");
        }
    }
}

////////////////////////////////////////////////////////////////////////////
// VmData::simplify (vm/data.rs:123-318)
TapeP simplify(const Tape& parent, const uint8_t* choices, size_t n_choices, uint32_t n_regs) {
    if (n_choices != parent.choice_count()) throw std::runtime_error("bad choice slice length");
    const uint32_t NONE = 0xFFFFFFFFu;
    const auto& ssa = parent.d.ssa.tape;
    std::vector<uint32_t> bind(ssa.size(), NONE);
    uint32_t count = 0;
    auto get_or_insert = [&](uint32_t i) {
        if (bind[i] == NONE) bind[i] = count++;
        return bind[i];
    };
    RegAlloc alloc(n_regs, ssa.size());
    TapeData out;
    out.n_regs = n_regs;
    out.vars = parent.d.vars;
    out.ssa.tape.reserve(ssa.size());
    size_t ci = n_choices;  // choices are consumed back to front

    for (Clause op : ssa) {
        if (op.op == OP_OUTPUT) {
            op.a = get_or_insert(op.a);
            alloc.op(op);
            out.ssa.tape.push_back(op);
            out.ssa.output_count++;
            continue;
        }
        uint32_t index = op.out;
        if (bind[index] == NONE) {
            if (is_choice(op.op)) --ci;
            continue;
        }
        uint32_t new_index = bind[index];
        if (op.op == OP_INPUT || (op.op == OP_COPY && op.form == F_RI)) {
            op.out = new_index;
        } else if (op.op == OP_COPY) {
            if (bind[op.a] != NONE) {
                op.out = new_index;
                op.a = bind[op.a];
            } else {
                bind[op.a] = new_index;
                continue;
            }
        } else if (is_choice(op.op)) {
            uint8_t choice = choices[--ci];
            if (choice == C_BOTH) {
                out.ssa.choice_count++;
                op.out = new_index;
                op.a = get_or_insert(op.a);
                if (op.form == F_RR) op.b = get_or_insert(op.b);
            } else if (choice == C_LEFT || (choice == C_RIGHT && op.form == F_RR)) {
                uint32_t arg = choice == C_LEFT ? op.a : op.b;
                if (bind[arg] != NONE) {
                    Clause cp;
                    cp.op = OP_COPY;
                    cp.form = F_RR;
                    cp.out = new_index;
                    cp.a = bind[arg];
                    op = cp;
                } else {
                    bind[arg] = new_index;
                    continue;
                }
            } else if (choice == C_RIGHT) {
                Clause cp;
                cp.op = OP_COPY;
                cp.form = F_RI;
                cp.out = new_index;
                cp.imm = op.imm;
                op = cp;
            } else {
                throw std::runtime_error("unknown choice in trace");
            }
        } else {
            op.out = new_index;
            op.a = get_or_insert(op.a);
            if (is_binary(op.op) && op.form == F_RR) op.b = get_or_insert(op.b);
        }
        alloc.op(op);
        out.ssa.tape.push_back(op);
    }
    out.asm_ = alloc.finalize();
    return std::make_shared<const Tape>(std::move(out));
}

RenderHandle* RenderHandle::simplify(const std::vector<uint8_t>& trace) {
    if (next && next_trace != trace) next.reset();
    if (!next) {
        TapeP s = oracle::simplify(*shape, trace.data(), trace.size(), shape->d.n_regs);
        if (s->size() >= shape->size()) return this;  // not shorter: keep the parent
        next_trace = trace;
        next.reset(new RenderHandle(std::move(s)));
    }
    return next.get();
}

////////////////////////////////////////////////////////////////////////////
// Matrices and transforms
Mat4 mat4_identity() {
    Mat4 m{};
    for (int i = 0; i < 4; ++i) m.m[i][i] = 1.0f;
    return m;
}
Mat4 mat4_mul(const Mat4& a, const Mat4& b) {
    Mat4 r{};
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float s = 0.0f;
            for (int k = 0; k < 4; ++k) s = s + a.m[i][k] * b.m[k][j];
            r.m[i][j] = s;
        }
    return r;
}
// region.rs:87-108: identity, append_translation(-center), then
// append_nonuniform_scaling(scale) (which scales the translation column too)
Mat4 screen_to_world_3d(uint32_t w, uint32_t h, uint32_t d) {
    float center[3] = {float(w) / 2.0f, float(h) / 2.0f - 1.0f, float(d) / 2.0f};
    float s = 2.0f / float(std::min(w, std::min(h, d)));
    float scale[3] = {s, s * -1.0f, s};
    Mat4 m = mat4_identity();
    for (int i = 0; i < 3; ++i) {
        m.m[i][i] = scale[i];
        m.m[i][3] = -center[i] * scale[i];
    }
    return m;
}
Mat4 screen_to_world_2d(uint32_t w, uint32_t h) {
    float center[2] = {float(w) / 2.0f, float(h) / 2.0f - 1.0f};
    float s = 2.0f / float(std::min(w, h));
    float scale[2] = {s, s * -1.0f};
    Mat4 m = mat4_identity();
    for (int i = 0; i < 2; ++i) {
        m.m[i][i] = scale[i];
        m.m[i][3] = -center[i] * scale[i];
    }
    return m;
}
// pixel.rs:122-124,283-287: (world_to_model * screen_to_world) as 3x3, then a
// unit Z row/column is inserted
Mat4 pixel_mat(uint32_t w, uint32_t h, const float wm[9]) {
    Mat4 s2w = screen_to_world_2d(w, h);
    float s[3][3] = {{s2w.m[0][0], s2w.m[0][1], s2w.m[0][3]},
                     {s2w.m[1][0], s2w.m[1][1], s2w.m[1][3]},
                     {0.0f, 0.0f, 1.0f}};
    float r[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            float acc = 0.0f;
            for (int k = 0; k < 3; ++k) acc = acc + wm[i * 3 + k] * s[k][j];
            r[i][j] = acc;
        }
    Mat4 m{};
    const int map[3] = {0, 1, 3};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m.m[map[i]][map[j]] = r[i][j];
    m.m[2][2] = 1.0f;
    return m;
}

// nalgebra 0.35 Matrix4::transform_point (shape/mod.rs:906-915): linear part
// accumulated left to right, plus translation, divided by the homogeneous
// term when that is non-zero.  For matrices with non-zero cross terms the
// three transforms below are pinned against float64 (tests/test_views_oracle.py);
// the summation order inside nalgebra itself stays unpinned (SURVEY.md §8c).
void transform_f32(float x, float y, float z, const Mat4& m, float out[3]) {
    float n = ((m.m[3][0] * x + m.m[3][1] * y) + m.m[3][2] * z) + m.m[3][3];
    for (int i = 0; i < 3; ++i) {
        float r = ((m.m[i][0] * x + m.m[i][1] * y) + m.m[i][2] * z) + m.m[i][3];
        out[i] = n != 0.0f ? r / n : r;
    }
}
void transform_interval(Interval x, Interval y, Interval z, const Mat4& m, Interval out[3]) {
    Interval o[4];
    for (int i = 0; i < 4; ++i)
        o[i] = i_add(i_add(i_add(i_mul_f(x, m.m[i][0]), i_mul_f(y, m.m[i][1])), i_mul_f(z, m.m[i][2])),
                     Interval(m.m[i][3]));
    for (int i = 0; i < 3; ++i) out[i] = i_div(o[i], o[3]);
}
void transform_grad(Grad x, Grad y, Grad z, const Mat4& m, Grad out[3]) {
    Grad o[4];
    for (int i = 0; i < 4; ++i)
        o[i] = g_add(g_add(g_add(g_mul_f(x, m.m[i][0]), g_mul_f(y, m.m[i][1])), g_mul_f(z, m.m[i][2])),
                     Grad(m.m[i][3]));
    for (int i = 0; i < 3; ++i) out[i] = g_div(o[i], o[3]);
}

std::vector<uint32_t> trim_tile_sizes(const std::vector<uint32_t>& ts, uint32_t max_size) {
    size_t pos = ts.size();
    for (size_t i = 0; i < ts.size(); ++i)
        if (ts[i] < max_size) { pos = i; break; }
    size_t start = pos > 0 ? pos - 1 : 0;
    return std::vector<uint32_t>(ts.begin() + start, ts.end());
}

////////////////////////////////////////////////////////////////////////////
// Shared helpers for both renderers
namespace {

struct VarSlots { int x = -1, y = -1, z = -1; size_t n = 0; };
VarSlots var_slots(const Tape& t) {
    VarSlots s;
    s.n = t.n_vars();
    for (size_t i = 0; i < t.d.vars.order.size(); ++i) {
        const auto& v = t.d.vars.order[i];
        if (v.kind == Var::X) s.x = int(i);
        else if (v.kind == Var::Y) s.y = int(i);
        else if (v.kind == Var::Z) s.z = int(i);
    }
    return s;
}

// Scratch for tracing / bulk inputs: every slot gets its bound value, then
// the axes overwrite theirs (ShapeTracingEval::eval_raw, shape/mod.rs:520-533)
template <class T>
void bind_vars(const Tape& t, const std::vector<float>& values, std::vector<T>& out) {
    out.assign(std::max<size_t>(t.n_vars(), 3), T(0.0f));
    for (size_t i = 0; i < t.n_vars(); ++i) {
        if (t.d.vars.order[i].kind != Var::V) continue;
        if (i >= values.size()) throw std::runtime_error("missing value for a bound variable");
        out[i] = T(values[i]);
    }
}

void add_stats(TileStats& a, const TileStats& b) {
    for (int i = 0; i < 8; ++i) {
        a.evaluated[i] += b.evaluated[i];
        a.filled_inside[i] += b.filled_inside[i];
        a.filled_outside[i] += b.filled_outside[i];
        a.ambiguous[i] += b.ambiguous[i];
        a.simplified[i] += b.simplified[i];
    }
    a.pixels += b.pixels;
}

template <class F>
void run_roots(uint32_t n_total, int threads, F&& f) {
    if (threads <= 1) {
        f(0, 0u, n_total, nullptr);
        return;
    }
    std::atomic<uint32_t> next{0};
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) pool.emplace_back([&, t]() { f(t, 0u, n_total, &next); });
    for (auto& th : pool) th.join();
}

}  // namespace

////////////////////////////////////////////////////////////////////////////
// pixel::render (fidget-raster/src/pixel.rs:276-492)
namespace {
struct Worker2D {
    const Render2DConfig& cfg;
    std::vector<uint32_t> ts;
    std::vector<Interval> ivars;
    std::vector<std::vector<float>> fconst;
    std::vector<const float*> bulk_vars(const Tape& t, size_t n) {
        std::vector<const float*> v(std::max<size_t>(t.n_vars(), 3), sx.data());
        fconst.resize(t.n_vars());
        for (size_t q = 0; q < t.n_vars(); ++q)
            if (t.d.vars.order[q].kind == Var::V) {
                fconst[q].assign(n, cfg.var_values.at(q));
                v[q] = fconst[q].data();
            }
        return v;
    }
    IntervalEval ieval;
    FloatSliceEval feval;
    std::vector<float> sx, sy, sz, sout;
    std::vector<float> image;  // root-tile image
    TileStats stats;

    Worker2D(const Render2DConfig& c, std::vector<uint32_t> t) : cfg(c), ts(std::move(t)) {
        size_t n = size_t(ts.back()) * ts.back();
        sx.resize(n); sy.resize(n); sz.resize(n); sout.resize(n);
    }
    size_t pixel_offset(uint32_t x, uint32_t y) const { return (x % ts[0]) + size_t(y % ts[0]) * ts[0]; }

    void recurse(RenderHandle* shape, size_t depth, uint32_t cx, uint32_t cy) {
        const Tape& tape = *shape->shape;
        uint32_t tile_size = ts[depth];
        Interval x(float(cx), float(cx) + float(tile_size));
        Interval y(float(cy), float(cy) + float(tile_size));
        Interval z(cfg.z, cfg.z);
        Interval xyz[3];
        transform_interval(x, y, z, cfg.mat, xyz);
        VarSlots vs = var_slots(tape);
        bind_vars(tape, cfg.var_values, ivars);
        Interval* vars = ivars.data();
        if (vs.x >= 0) vars[vs.x] = xyz[0];
        if (vs.y >= 0) vars[vs.y] = xyz[1];
        if (vs.z >= 0) vars[vs.z] = xyz[2];
        Interval out;
        bool has_trace = ieval.eval(tape, vars, &out);
        stats.evaluated[depth]++;
        if (!cfg.pixel_perfect) {
            int fill = out.hi < 0.0f ? 1 : (out.lo > 0.0f ? 0 : -1);
            if (fill >= 0) {
                (fill ? stats.filled_inside : stats.filled_outside)[depth]++;
                uint32_t bits = 0x7FC00000u | (uint32_t(uint8_t(depth)) << 1) | uint32_t(fill) | (0xF6u << 9);
                float f = u2f(bits);
                for (uint32_t j = 0; j < tile_size; ++j) {
                    size_t start = pixel_offset(cx, cy + j);
                    std::fill(image.begin() + start, image.begin() + start + tile_size, f);
                }
                return;
            }
        }
        stats.ambiguous[depth]++;
        RenderHandle* sub = shape;
        if (has_trace) {
            std::vector<uint8_t> trace = ieval.choices;  // the evaluator is reused by children
            sub = shape->simplify(trace);
            if (sub != shape) stats.simplified[depth]++;
        }
        if (depth + 1 < ts.size()) {
            uint32_t next = ts[depth + 1];
            uint32_t n = tile_size / next;
            for (uint32_t j = 0; j < n; ++j)
                for (uint32_t i = 0; i < n; ++i) recurse(sub, depth + 1, cx + i * next, cy + j * next);
        } else {
            pixels(sub, tile_size, cx, cy);
        }
    }

    void pixels(RenderHandle* shape, uint32_t tile_size, uint32_t cx, uint32_t cy) {
        const Tape& tape = *shape->shape;
        size_t n = size_t(tile_size) * tile_size, index = 0;
        for (uint32_t j = 0; j < tile_size; ++j)
            for (uint32_t i = 0; i < tile_size; ++i) {
                float p[3];
                transform_f32(float(cx + i), float(cy + j), cfg.z, cfg.mat, p);
                sx[index] = p[0]; sy[index] = p[1]; sz[index] = p[2];
                ++index;
            }
        VarSlots vs = var_slots(tape);
        std::vector<const float*> vars = bulk_vars(tape, n);
        if (vs.x >= 0) vars[vs.x] = sx.data();
        if (vs.y >= 0) vars[vs.y] = sy.data();
        if (vs.z >= 0) vars[vs.z] = sz.data();
        float* outs[1] = {sout.data()};
        feval.eval(tape, vars.data(), n, outs);
        stats.pixels += n;
        index = 0;
        for (uint32_t j = 0; j < tile_size; ++j) {
            size_t o = pixel_offset(cx, cy + j);
            for (uint32_t i = 0; i < tile_size; ++i) {
                float v = sout[index++];
                image[o + i] = v != v ? u2f(0x7FC00000u) : v;
            }
        }
    }
};
}  // namespace

void render2d(const TapeP& tape, const Render2DConfig& cfg, float* out, TileStats* stats_out) {
    std::vector<uint32_t> ts = trim_tile_sizes(cfg.tile_sizes, std::max(cfg.width, cfg.height));
    uint32_t t0 = ts[0];
    uint32_t nx = (cfg.width + t0 - 1) / t0, ny = (cfg.height + t0 - 1) / t0;
    uint32_t first = cfg.first_root, count = cfg.n_roots ? cfg.n_roots : nx * ny - first;
    std::fill(out, out + size_t(cfg.width) * cfg.height, 0.0f);
    std::vector<TileStats> per_thread(std::max(cfg.threads, 1));

    run_roots(count, cfg.threads, [&](int tid, uint32_t, uint32_t n_total, std::atomic<uint32_t>* next) {
        Worker2D w(cfg, ts);
        RenderHandle root(tape);
        for (uint32_t k = 0;;) {
            uint32_t r = next ? next->fetch_add(1) : k++;
            if (r >= n_total) break;
            uint32_t idx = first + r;
            uint32_t cx = (idx / ny) * t0, cy = (idx % ny) * t0;  // x-major enumeration
            w.image.assign(size_t(t0) * t0, 0.0f);
            w.recurse(&root, 0, cx, cy);
            for (uint32_t j = 0; j < t0; ++j) {
                uint32_t y = cy + j;
                if (y >= cfg.height) break;
                for (uint32_t i = 0; i < t0; ++i) {
                    uint32_t x = cx + i;
                    if (x < cfg.width) out[size_t(y) * cfg.width + x] = w.image[size_t(j) * t0 + i];
                }
            }
        }
        per_thread[tid] = w.stats;
    });
    if (stats_out) {
        *stats_out = TileStats{};
        for (auto& s : per_thread) add_stats(*stats_out, s);
    }
}

////////////////////////////////////////////////////////////////////////////
// voxel::render (fidget-raster/src/voxel.rs:216-553)
namespace {
struct Worker3D {
    const Render3DConfig& cfg;
    std::vector<uint32_t> ts;
    std::vector<Interval> ivars;
    std::vector<std::vector<float>> fconst;
    std::vector<const float*> bulk_vars(const Tape& t, size_t n) {
        std::vector<const float*> v(std::max<size_t>(t.n_vars(), 3), sx.data());
        fconst.resize(t.n_vars());
        for (size_t q = 0; q < t.n_vars(); ++q)
            if (t.d.vars.order[q].kind == Var::V) {
                fconst[q].assign(n, cfg.var_values.at(q));
                v[q] = fconst[q].data();
            }
        return v;
    }
    IntervalEval ieval;
    FloatSliceEval feval;
    GradSliceEval geval;
    std::vector<float> sx, sy, sz, sout;
    std::vector<Grad> gx, gy, gz, gout;
    std::vector<size_t> columns;
    std::vector<GeometryPixel> out;  // root-tile image
    TileStats stats;

    Worker3D(const Render3DConfig& c, std::vector<uint32_t> t) : cfg(c), ts(std::move(t)) {
        size_t b = ts.back(), n3 = b * b * b, n2 = b * b;
        sx.resize(n3); sy.resize(n3); sz.resize(n3); sout.resize(n3);
        gx.resize(n2); gy.resize(n2); gz.resize(n2); gout.resize(n2);
        columns.reserve(n2);
    }
    size_t pixel_offset(uint32_t x, uint32_t y) const { return (x % ts[0]) + size_t(y % ts[0]) * ts[0]; }

    bool recurse(RenderHandle* shape, size_t depth, uint32_t cx, uint32_t cy, uint32_t cz) {
        uint32_t tile_size = ts[depth];
        uint32_t fill_z = cz + tile_size + 1;
        bool all = true;
        for (uint32_t y = 0; y < tile_size && all; ++y) {
            size_t i = pixel_offset(cx, cy + y);
            for (uint32_t x = 0; x < tile_size; ++x)
                if (out[i + x].depth < fill_z) { all = false; break; }
        }
        if (all) return false;

        const Tape& tape = *shape->shape;
        Interval x(float(cx), float(cx) + float(tile_size));
        Interval y(float(cy), float(cy) + float(tile_size));
        Interval z(float(cz), float(cz) + float(tile_size));
        Interval xyz[3];
        transform_interval(x, y, z, cfg.mat, xyz);
        VarSlots vs = var_slots(tape);
        bind_vars(tape, cfg.var_values, ivars);
        Interval* vars = ivars.data();
        if (vs.x >= 0) vars[vs.x] = xyz[0];
        if (vs.y >= 0) vars[vs.y] = xyz[1];
        if (vs.z >= 0) vars[vs.z] = xyz[2];
        Interval r;
        bool has_trace = ieval.eval(tape, vars, &r);
        stats.evaluated[depth]++;
        if (r.hi < 0.0f) {
            stats.filled_inside[depth]++;
            for (uint32_t yy = 0; yy < tile_size; ++yy) {
                size_t i = pixel_offset(cx, cy + yy);
                for (uint32_t xx = 0; xx < tile_size; ++xx)
                    out[i + xx].depth = std::max(out[i + xx].depth, fill_z);
            }
            return false;
        } else if (r.lo > 0.0f) {
            stats.filled_outside[depth]++;
            return true;
        }
        stats.ambiguous[depth]++;
        RenderHandle* sub = shape;
        if (has_trace) {
            std::vector<uint8_t> trace = ieval.choices;
            sub = shape->simplify(trace);
            if (sub != shape) stats.simplified[depth]++;
        }
        if (depth + 1 < ts.size()) {
            uint32_t next = ts[depth + 1], n = tile_size / next;
            for (uint32_t j = 0; j < n; ++j)
                for (uint32_t i = 0; i < n; ++i)
                    for (int k = int(n) - 1; k >= 0; --k)
                        recurse(sub, depth + 1, cx + i * next, cy + j * next, cz + uint32_t(k) * next);
        } else {
            pixels(sub, tile_size, cx, cy, cz);
        }
        return true;
    }

    void pixels(RenderHandle* shape, uint32_t T, uint32_t cx, uint32_t cy, uint32_t cz) {
        const Tape& tape = *shape->shape;
        size_t index = 0;
        columns.clear();
        for (uint32_t xy = 0; xy < T * T; ++xy) {
            uint32_t i = xy % T, j = xy / T;
            size_t o = pixel_offset(cx + i, cy + j);
            uint32_t zmax = cz + T;
            if (out[o].depth >= zmax) continue;
            for (int k = int(T) - 1; k >= 0; --k) {
                float p[3];
                transform_f32(float(cx + i), float(cy + j), float(cz + uint32_t(k)), cfg.mat, p);
                sx[index] = p[0]; sy[index] = p[1]; sz[index] = p[2];
                ++index;
            }
            columns.push_back(xy);
        }
        size_t size = index;
        if (size == 0) return;  // (the reference asserts size > 0; unreachable after the early-out)
        VarSlots vs = var_slots(tape);
        std::vector<const float*> vars = bulk_vars(tape, size);
        if (vs.x >= 0) vars[vs.x] = sx.data();
        if (vs.y >= 0) vars[vs.y] = sy.data();
        if (vs.z >= 0) vars[vs.z] = sz.data();
        float* outs[1] = {sout.data()};
        feval.eval(tape, vars.data(), size, outs);
        stats.pixels += size;

        size_t grad = 0;
        for (size_t col = 0; col < columns.size(); ++col) {
            const float* d = &sout[col * T];
            int kk = -1;
            for (uint32_t q = 0; q < T; ++q)
                if (d[q] < 0.0f) { kk = int(q); break; }
            if (kk < 0) continue;
            uint32_t xy = uint32_t(columns[col]);
            uint32_t i = xy % T, j = xy / T;
            uint32_t k = T - 1 - uint32_t(kk);
            size_t o = pixel_offset(cx + i, cy + j);
            uint32_t zv = cz + k + 1;
            assert(out[o].depth < zv);
            out[o].depth = zv;
            gx[grad] = Grad(float(cx + i), 1.0f, 0.0f, 0.0f);
            gy[grad] = Grad(float(cy + j), 0.0f, 1.0f, 0.0f);
            gz[grad] = Grad(float(cz + k), 0.0f, 0.0f, 1.0f);
            columns[grad] = o;
            ++grad;
        }
        if (grad > 0) {
            for (size_t q = 0; q < grad; ++q) {
                Grad t[3];
                transform_grad(gx[q], gy[q], gz[q], cfg.mat, t);
                gx[q] = t[0]; gy[q] = t[1]; gz[q] = t[2];
            }
            std::vector<std::vector<Grad>> gconst(tape.n_vars());
            std::vector<const Grad*> gvars(std::max<size_t>(tape.n_vars(), 3), gx.data());
            for (size_t q = 0; q < tape.n_vars(); ++q)
                if (tape.d.vars.order[q].kind == Var::V) {
                    gconst[q].assign(grad, Grad(cfg.var_values.at(q)));
                    gvars[q] = gconst[q].data();
                }
            if (vs.x >= 0) gvars[vs.x] = gx.data();
            if (vs.y >= 0) gvars[vs.y] = gy.data();
            if (vs.z >= 0) gvars[vs.z] = gz.data();
            Grad* gouts[1] = {gout.data()};
            geval.eval(tape, gvars.data(), grad, gouts);
            for (size_t q = 0; q < grad; ++q) {
                GeometryPixel& p = out[columns[q]];
                p.normal[0] = gout[q].dx; p.normal[1] = gout[q].dy; p.normal[2] = gout[q].dz;
            }
        }
    }
};
}  // namespace

void render3d(const TapeP& tape, const Render3DConfig& cfg, GeometryPixel* image, TileStats* stats_out) {
    std::vector<uint32_t> ts = trim_tile_sizes(cfg.tile_sizes, std::max(cfg.width, cfg.height));
    uint32_t t0 = ts[0];
    uint32_t nx = (cfg.width + t0 - 1) / t0, ny = (cfg.height + t0 - 1) / t0;
    uint32_t first = cfg.first_root, count = cfg.n_roots ? cfg.n_roots : nx * ny - first;
    std::fill(image, image + size_t(cfg.width) * cfg.height, GeometryPixel{{0, 0, 0}, 0});
    std::vector<TileStats> per_thread(std::max(cfg.threads, 1));

    run_roots(count, cfg.threads, [&](int tid, uint32_t, uint32_t n_total, std::atomic<uint32_t>* next) {
        Worker3D w(cfg, ts);
        RenderHandle root(tape);
        for (uint32_t k = 0;;) {
            uint32_t r = next ? next->fetch_add(1) : k++;
            if (r >= n_total) break;
            uint32_t idx = first + r;
            uint32_t cx = (idx / ny) * t0, cy = (idx % ny) * t0;
            w.out.assign(size_t(t0) * t0, GeometryPixel{{0, 0, 0}, 0});
            uint32_t nk = (cfg.depth + t0 - 1) / t0;
            for (int kz = int(nk) - 1; kz >= 0; --kz)
                if (!w.recurse(&root, 0, cx, cy, uint32_t(kz) * t0)) break;
            for (uint32_t j = 0; j < t0; ++j) {
                uint32_t y = cy + j;
                if (y >= cfg.height) break;
                for (uint32_t i = 0; i < t0; ++i) {
                    uint32_t x = cx + i;
                    if (x >= cfg.width) continue;
                    const GeometryPixel& p = w.out[size_t(j) * t0 + i];
                    GeometryPixel& dst = image[size_t(y) * cfg.width + x];
                    if (p.depth >= dst.depth) {
                        uint32_t d = cfg.depth - 1;
                        if (p.depth >= d) dst = GeometryPixel{{0.0f, 0.0f, 1.0f}, d + 1};
                        else dst = p;
                    }
                }
            }
        }
        per_thread[tid] = w.stats;
    });
    if (stats_out) {
        *stats_out = TileStats{};
        for (auto& s : per_thread) add_stats(*stats_out, s);
    }
}

}  // namespace oracle
