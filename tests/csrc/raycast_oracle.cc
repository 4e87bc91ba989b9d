// TEST INFRASTRUCTURE -- the CPU mirror of fc_raycast's descent (include/fidget_cuda.h), built on the oracle's public
// evaluators (oracle/vm.h) and linked against oracle/liboracle.so.  tests/raycast_ref.py compiles it at test time.
//
// Ray r samples t_k = t0 + k dt, x_k = origin + t_k dir (f32, one rounding per operation: this file is compiled with
// -ffp-contract=off).  L = max(1, ceil(log2(steps) / 5)) interval levels of segments 32^(L - l) samples long, clipped to
// [0, steps); a segment's box is spanned by its end samples.  Upper < 0 makes its first sample a (proven) candidate,
// lower > 0 drops it, anything else splits it into 32 children evaluated with the tape RenderHandle::simplify gives
// (kept only when shorter); the ambiguous segments of level L - 1 evaluate their samples, and a value < 0 is a
// candidate.  The walk visits segments in sample order, so the first candidate it meets is the smallest: the hit.
// value and grad are the root tape's float and gradient evaluations at the hit.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <exception>
#include <memory>
#include <vector>

#include "vm.h"

using namespace oracle;

// The handle behind oracle.Tape (oracle/capi.cc): one shared tape
struct orc_tape { TapeP t; };

namespace {

struct Ray { float o[3], d[3], t0, dt; };

float ray_t(const Ray& r, uint32_t k) { return r.t0 + float(k) * r.dt; }
float ray_x(const Ray& r, int a, float t) { return r.o[a] + t * r.d[a]; }

struct Caster {
    uint32_t steps = 0, L = 1;
    int axis[3] = {-1, -1, -1};       // input slots of X, Y, Z
    std::vector<float> values;        // every input slot's bound value (axes ignored)
    size_t n_vars = 0;
    IntervalEval ieval;
    FloatSliceEval feval;
    GradSliceEval geval;
    uint64_t evaluated[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint64_t leaf_samples = 0;

    // The first candidate in segment [a, a + len) at level l (len = 32^(L - l)), or false
    bool segment(RenderHandle* h, const Ray& r, uint32_t a, uint64_t len, uint32_t l, uint32_t& k, bool& proven) {
        const uint32_t b = uint32_t(std::min<uint64_t>(a + len - 1, steps - 1));
        const float ta = ray_t(r, a), tb = ray_t(r, b);
        std::vector<Interval> vars(std::max<size_t>(n_vars, 1));
        for (size_t i = 0; i < n_vars; ++i) vars[i] = Interval(values[i]);
        for (int ax = 0; ax < 3; ++ax) {
            const float xa = ray_x(r, ax, ta), xb = ray_x(r, ax, tb);
            if (axis[ax] >= 0) vars[axis[ax]] = xb < xa ? Interval(xb, xa) : Interval(xa, xb);
        }
        Interval v;
        const bool has_trace = ieval.eval(*h->shape, vars.data(), &v);
        ++evaluated[l];
        if (v.hi < 0.0f) {
            k = a;
            proven = true;
            return true;
        }
        if (v.lo > 0.0f) return false;
        RenderHandle* sub = h;
        if (has_trace) {
            std::vector<uint8_t> trace = ieval.choices;
            sub = h->simplify(trace);
        }
        if (l + 1 == L) return leaf(*sub->shape, r, a, b, k, proven);
        const uint64_t child = len / 32;
        for (uint64_t c = 0; c < 32; ++c) {
            const uint64_t ca = a + c * child;
            if (ca >= steps) break;
            if (segment(sub, r, uint32_t(ca), child, l + 1, k, proven)) return true;
        }
        return false;
    }

    bool leaf(const Tape& tape, const Ray& r, uint32_t a, uint32_t b, uint32_t& k, bool& proven) {
        const uint32_t n = b - a + 1;
        std::vector<std::vector<float>> cols(std::max<size_t>(n_vars, 1));
        for (size_t i = 0; i < n_vars; ++i) cols[i].assign(n, values[i]);
        for (uint32_t s = 0; s < n; ++s) {
            const float t = ray_t(r, a + s);
            for (int ax = 0; ax < 3; ++ax)
                if (axis[ax] >= 0) cols[axis[ax]][s] = ray_x(r, ax, t);
        }
        std::vector<const float*> vp;
        for (auto& c : cols) vp.push_back(c.data());
        std::vector<float> out(n);
        float* op[1] = {out.data()};
        feval.eval(tape, vp.data(), n, op);
        leaf_samples += n;
        for (uint32_t s = 0; s < n; ++s)
            if (out[s] < 0.0f) {
                k = a + s;
                proven = false;
                return true;
            }
        return false;
    }

    // value and (d/dx, d/dy, d/dz) of the root tape at p
    void finish(const Tape& root, const float p[3], float& value, float grad[3]) {
        std::vector<float> fv(std::max<size_t>(n_vars, 1));
        std::vector<Grad> gv(std::max<size_t>(n_vars, 1));
        for (size_t i = 0; i < n_vars; ++i) { fv[i] = values[i]; gv[i] = Grad(values[i]); }
        for (int ax = 0; ax < 3; ++ax)
            if (axis[ax] >= 0) {
                fv[axis[ax]] = p[ax];
                gv[axis[ax]] = Grad(p[ax], ax == 0 ? 1.0f : 0.0f, ax == 1 ? 1.0f : 0.0f, ax == 2 ? 1.0f : 0.0f);
            }
        std::vector<const float*> fp;
        std::vector<const Grad*> gp;
        for (size_t i = 0; i < fv.size(); ++i) { fp.push_back(&fv[i]); gp.push_back(&gv[i]); }
        float out = 0.0f;
        float* fo[1] = {&out};
        feval.eval(root, fp.data(), 1, fo);
        Grad g;
        Grad* go[1] = {&g};
        geval.eval(root, gp.data(), 1, go);
        value = out;
        grad[0] = g.dx; grad[1] = g.dy; grad[2] = g.dz;
    }
};

}  // namespace

extern "C" {

// The levels of the descent for `steps` samples
uint32_t ro_levels(uint32_t steps) {
    uint32_t L = 1;
    while ((1ull << (5 * L)) < steps) ++L;
    return L;
}

// n rays (fc_ray rows of 8 floats) -> hits (fc_ray_hit rows of 10 words: k, flags, t, pos[3], value, grad[3]);
// values[i] binds input slot i (n_values of them; the axis slots are ignored).  stats: evaluated[8], leaf samples.
// Returns 0, or -1 when the tape cannot be cast (an exception in the oracle).
int32_t ro_raycast(const orc_tape* t, const float* rays, uint64_t n, uint32_t steps, const float* values,
                   uint32_t n_values, uint32_t* hits, uint64_t* stats) {
    try {
        Caster cs;
        cs.steps = steps;
        cs.L = ro_levels(steps);
        const Tape& root = *t->t;
        cs.n_vars = root.n_vars();
        cs.values.assign(std::max<size_t>(cs.n_vars, 1), 0.0f);
        for (size_t i = 0; i < cs.n_vars && i < n_values; ++i) cs.values[i] = values[i];
        for (size_t i = 0; i < root.d.vars.order.size(); ++i) {
            const auto kind = root.d.vars.order[i].kind;
            if (kind == fhost::Var::X) cs.axis[0] = int(i);
            else if (kind == fhost::Var::Y) cs.axis[1] = int(i);
            else if (kind == fhost::Var::Z) cs.axis[2] = int(i);
        }
        RenderHandle h(t->t);
        const uint64_t len0 = 1ull << (5 * cs.L);
        for (uint64_t i = 0; i < n; ++i) {
            Ray r;
            std::memcpy(&r, rays + 8 * i, sizeof r);
            uint32_t* out = hits + 10 * i;
            std::memset(out, 0, 10 * sizeof *out);
            out[0] = 0xFFFFFFFFu;
            uint32_t k = 0;
            bool proven = false;
            if (!cs.segment(&h, r, 0, len0, 0, k, proven)) continue;
            float f[8];
            f[0] = ray_t(r, k);
            for (int a = 0; a < 3; ++a) f[1 + a] = ray_x(r, a, f[0]);
            cs.finish(root, f + 1, f[4], f + 5);
            out[0] = k;
            out[1] = proven ? 1u : 0u;
            std::memcpy(out + 2, f, sizeof f);
        }
        if (stats) {
            for (int l = 0; l < 8; ++l) stats[l] = cs.evaluated[l];
            stats[8] = cs.leaf_samples;
        }
        return 0;
    } catch (const std::exception&) {
        return -1;
    }
}

}  // extern "C"
