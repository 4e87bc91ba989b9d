// TEST INFRASTRUCTURE -- the CPU mirror of fc_measure's integers (include/fidget_cuda.h), built on the oracle's public
// evaluators (oracle/vm.h) and linked against oracle/liboracle.so.  tests/measure_ref.py compiles it at test time.
//
// The descent is the octree sampler's (oracle/octree.cc, Builder::descend): interval evaluation of each cell through
// world_to_model, upper < 0 proves it inside, lower > 0 outside, and an ambiguous cell's children are evaluated with
// the tape RenderHandle::simplify gives.  It stops at cells of edge B = min(4, 2^depth): a proven-inside cell adds its
// block in closed form, an ambiguous cell of edge B (a brick) classifies its B^3 cell centres -1 + (2i + 1) 2^-depth,
// through world_to_model by transform_f32, with its simplified tape.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <exception>
#include <memory>
#include <stdexcept>
#include <vector>

#include "vm.h"

using namespace oracle;

// The handle behind oracle.Tape (oracle/capi.cc): one shared tape
struct orc_tape { TapeP t; };

namespace {

struct Sums {
    uint64_t n_inside = 0, n_proven = 0, n_undecided = 0;
    uint64_t s1[3] = {0, 0, 0}, s2[6] = {0, 0, 0, 0, 0, 0};
    uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0, 0, 0};
};

// The block of T^3 depth-D cells at x0: along one axis the odd numbers 2i + 1 sum to (x0 + T)^2 - x0^2 and their
// squares to F(x0 + T) - F(x0), F(m) = m (4 m^2 - 1) / 3
void add_block(Sums& m, const uint32_t x0[3], uint32_t T) {
    auto F = [](uint64_t v) { return v * (4 * v * v - 1) / 3; };
    const uint64_t t = T;
    uint64_t a1[3];
    for (int a = 0; a < 3; ++a) {
        const uint64_t e = x0[a] + t;
        a1[a] = e * e - uint64_t(x0[a]) * x0[a];
        m.s1[a] += t * t * a1[a];
        m.s2[a] += t * t * (F(e) - F(x0[a]));
        m.lo[a] = std::min(m.lo[a], x0[a]);
        m.hi[a] = std::max(m.hi[a], x0[a] + T - 1);
    }
    m.n_inside += t * t * t;
    m.s2[3] += t * a1[0] * a1[1];
    m.s2[4] += t * a1[0] * a1[2];
    m.s2[5] += t * a1[1] * a1[2];
}

struct Measure {
    uint32_t depth;
    bool has_transform;
    Mat4 mat;
    IntervalEval ieval;
    FloatSliceEval feval;
    std::vector<float> sx = std::vector<float>(64), sy = std::vector<float>(64), sz = std::vector<float>(64),
                       sout = std::vector<float>(64);
    Sums m;

    static void slots(const Tape& t, int s[3]) {
        s[0] = s[1] = s[2] = -1;
        for (size_t i = 0; i < t.d.vars.order.size(); ++i) {
            const auto k = t.d.vars.order[i].kind;
            if (k == fhost::Var::X) s[0] = int(i);
            else if (k == fhost::Var::Y) s[1] = int(i);
            else if (k == fhost::Var::Z) s[2] = int(i);
            else throw std::runtime_error("the measure oracle supports X/Y/Z only");
        }
    }

    void cell(RenderHandle* h, const Interval b[3], uint32_t T, uint32_t brick, const uint32_t x0[3]) {
        const Tape& tape = *h->shape;
        Interval xyz[3] = {b[0], b[1], b[2]};
        if (has_transform) transform_interval(b[0], b[1], b[2], mat, xyz);
        int s[3];
        slots(tape, s);
        Interval vars[3];
        for (int a = 0; a < 3; ++a)
            if (s[a] >= 0) vars[s[a]] = xyz[a];
        Interval r;
        const bool has_trace = ieval.eval(tape, vars, &r);
        if (r.hi < 0.0f) {
            add_block(m, x0, T);
            m.n_proven += uint64_t(T) * T * T;
            return;
        }
        if (r.lo > 0.0f) return;
        RenderHandle* sub = h;
        if (has_trace) {
            std::vector<uint8_t> trace = ieval.choices;
            sub = h->simplify(trace);
        }
        if (T == brick) {
            bricks(*sub->shape, T, x0);
            return;
        }
        for (int c = 0; c < 8; ++c) {   // CellBounds::child
            Interval cb[3];
            uint32_t x1[3];
            for (int a = 0; a < 3; ++a) {
                const float mid = (b[a].lo + b[a].hi) / 2.0f;
                const bool up = (c >> a) & 1;
                cb[a] = up ? Interval(mid, b[a].hi) : Interval(b[a].lo, mid);
                x1[a] = x0[a] + (up ? T / 2 : 0);
            }
            cell(sub, cb, T / 2, brick, x1);
        }
    }

    void bricks(const Tape& tape, uint32_t T, const uint32_t x0[3]) {
        const uint32_t n = T * T * T;
        const float inv = 1.0f / float(1u << depth);
        for (uint32_t c = 0; c < n; ++c) {
            float p[3] = {float(2u * (x0[0] + c % T) + 1u) * inv - 1.0f, float(2u * (x0[1] + (c / T) % T) + 1u) * inv - 1.0f,
                          float(2u * (x0[2] + c / (T * T)) + 1u) * inv - 1.0f};
            if (has_transform) {
                float q[3];
                transform_f32(p[0], p[1], p[2], mat, q);
                std::memcpy(p, q, sizeof p);
            }
            sx[c] = p[0]; sy[c] = p[1]; sz[c] = p[2];
        }
        int s[3];
        slots(tape, s);
        const float* vars[3] = {sx.data(), sx.data(), sx.data()};
        if (s[0] >= 0) vars[s[0]] = sx.data();
        if (s[1] >= 0) vars[s[1]] = sy.data();
        if (s[2] >= 0) vars[s[2]] = sz.data();
        float* outs[1] = {sout.data()};
        feval.eval(tape, vars, n, outs);
        for (uint32_t c = 0; c < n; ++c)
            if (sout[c] < 0.0f) {
                const uint32_t one[3] = {x0[0] + c % T, x0[1] + (c / T) % T, x0[2] + c / (T * T)};
                add_block(m, one, 1);
            }
        m.n_undecided += n;
    }
};

void store(const Sums& m, uint64_t* out, uint32_t* box) {
    out[0] = m.n_inside; out[1] = m.n_proven; out[2] = m.n_undecided;
    for (int i = 0; i < 3; ++i) { out[3 + i] = m.s1[i]; box[i] = m.lo[i]; box[3 + i] = m.hi[i]; }
    for (int i = 0; i < 6; ++i) out[6 + i] = m.s2[i];
}

}  // namespace

extern "C" {

// out = n_inside, n_proven, n_undecided, s1[3], s2[6]; box = lo[3], hi[3].  world_to_model16: row-major 4x4 or null.
// Returns 0, or -1 with nothing written when the tape has an input other than X, Y, Z.
int32_t mo_measure(const orc_tape* t, uint32_t depth, const float* world_to_model16, uint64_t* out, uint32_t* box) {
    try {
        Measure ms;
        ms.depth = depth;
        ms.has_transform = world_to_model16 != nullptr;
        if (world_to_model16) std::memcpy(ms.mat.m, world_to_model16, sizeof ms.mat.m);
        RenderHandle h(t->t);
        const Interval root[3] = {Interval(-1.0f, 1.0f), Interval(-1.0f, 1.0f), Interval(-1.0f, 1.0f)};
        const uint32_t x0[3] = {0, 0, 0};
        ms.cell(&h, root, 1u << depth, 1u << std::min<uint32_t>(depth, 2), x0);
        store(ms.m, out, box);
        return 0;
    } catch (const std::exception&) {
        return -1;
    }
}

// The closed-form sums of the block of T^3 depth-D cells at (x0, y0, z0), in mo_measure's layout
void mo_block(uint32_t x0, uint32_t y0, uint32_t z0, uint32_t T, uint64_t* out, uint32_t* box) {
    Sums m;
    const uint32_t c[3] = {x0, y0, z0};
    add_block(m, c, T);
    store(m, out, box);
}

}  // extern "C"
