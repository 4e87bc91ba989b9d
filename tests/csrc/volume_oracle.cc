// TEST INFRASTRUCTURE -- the CPU mirror of fc_volume_build (include/fidget_cuda.h), built on the oracle's public
// evaluators (oracle/vm.h) and linked against oracle/liboracle.so.  tests/volume_ref.py compiles it at test time.
//
// The descent is fc_measure's mirror (tests/csrc/measure_oracle.cc) with a band: interval evaluation of each cell
// through world_to_model; upper < -band makes it an inside tile, lower > band an outside tile, and an ambiguous cell's
// children are evaluated with the tape RenderHandle::simplify gives.  It stops at cells of edge B = min(8, 2^depth): an
// ambiguous cell of edge B is a brick, whose B^3 cell centres -1 + (2i + 1) 2^-depth, through world_to_model by
// transform_f32, are evaluated with its simplified tape, and with gradients by GradSliceEval on the world centre seen
// through transform_grad.  Bricks and tiles come out in the order of the descent; the caller sorts them.
#include <cstdint>
#include <cstring>
#include <exception>
#include <stdexcept>
#include <vector>

#include "vm.h"

using namespace oracle;

struct orc_tape { TapeP t; };

namespace {

struct Volume {
    uint32_t depth = 0, brick = 1;
    float band = 0.0f;
    bool has_transform = false, grads = false;
    Mat4 mat;
    IntervalEval ieval;
    FloatSliceEval feval;
    GradSliceEval geval;
    std::vector<uint32_t> bricks, tiles;   // (ix, iy, iz) / (ix, iy, iz, log2_edge, inside)
    std::vector<float> values, gvals;

    static void slots(const Tape& t, int s[3]) {
        s[0] = s[1] = s[2] = -1;
        for (size_t i = 0; i < t.d.vars.order.size(); ++i) {
            const auto k = t.d.vars.order[i].kind;
            if (k == fhost::Var::X) s[0] = int(i);
            else if (k == fhost::Var::Y) s[1] = int(i);
            else if (k == fhost::Var::Z) s[2] = int(i);
            else throw std::runtime_error("the volume oracle supports X/Y/Z only");
        }
    }

    void cell(RenderHandle* h, const Interval b[3], uint32_t T, const uint32_t x0[3]) {
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
        if (r.hi < -band || r.lo > band) {
            uint32_t lg = 0;
            while ((1u << lg) < T) ++lg;
            tiles.insert(tiles.end(), {x0[0], x0[1], x0[2], lg, r.hi < -band ? 1u : 0u});
            return;
        }
        RenderHandle* sub = h;
        if (has_trace) {
            std::vector<uint8_t> trace = ieval.choices;
            sub = h->simplify(trace);
        }
        if (T == brick) {
            evaluate(*sub->shape, x0);
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
            cell(sub, cb, T / 2, x1);
        }
    }

    void evaluate(const Tape& tape, const uint32_t x0[3]) {
        const uint32_t B = brick, n = B * B * B;
        const float inv = 1.0f / float(1u << depth);
        std::vector<float> w[3], m[3], out(n);
        for (int a = 0; a < 3; ++a) { w[a].resize(n); m[a].resize(n); }
        for (uint32_t c = 0; c < n; ++c) {
            const uint32_t ijk[3] = {x0[0] + c % B, x0[1] + (c / B) % B, x0[2] + c / (B * B)};
            float p[3];
            for (int a = 0; a < 3; ++a) p[a] = w[a][c] = float(2u * ijk[a] + 1u) * inv - 1.0f;
            if (has_transform) transform_f32(p[0], p[1], p[2], mat, p);
            for (int a = 0; a < 3; ++a) m[a][c] = p[a];
        }
        int s[3];
        slots(tape, s);
        const float* vars[3] = {m[0].data(), m[0].data(), m[0].data()};
        for (int a = 0; a < 3; ++a)
            if (s[a] >= 0) vars[s[a]] = m[a].data();
        float* outs[1] = {out.data()};
        feval.eval(tape, vars, n, outs);
        values.insert(values.end(), out.begin(), out.end());
        bricks.insert(bricks.end(), {x0[0], x0[1], x0[2]});
        if (!grads) return;
        std::vector<Grad> g[3], gout(n);
        for (int a = 0; a < 3; ++a) g[a].resize(n);
        for (uint32_t c = 0; c < n; ++c) {
            Grad gx(w[0][c], 1, 0, 0), gy(w[1][c], 0, 1, 0), gz(w[2][c], 0, 0, 1);
            if (has_transform) {
                Grad t[3];
                transform_grad(gx, gy, gz, mat, t);
                gx = t[0]; gy = t[1]; gz = t[2];
            }
            g[0][c] = gx; g[1][c] = gy; g[2][c] = gz;
        }
        const Grad* gv[3] = {g[0].data(), g[0].data(), g[0].data()};
        for (int a = 0; a < 3; ++a)
            if (s[a] >= 0) gv[s[a]] = g[a].data();
        Grad* gouts[1] = {gout.data()};
        geval.eval(tape, gv, n, gouts);
        for (uint32_t c = 0; c < n; ++c) gvals.insert(gvals.end(), {gout[c].dx, gout[c].dy, gout[c].dz});
    }
};

}  // namespace

extern "C" {

// The volume of one frame (world_to_model16: row-major 4x4 or null), or null when the tape has an input other than
// X, Y, Z.  vo_counts, vo_read, then vo_free.
void* vo_build(const orc_tape* t, uint32_t depth, float band, const float* world_to_model16, uint32_t grads) {
    try {
        Volume* v = new Volume;
        v->depth = depth;
        v->brick = 1u << (depth < 3 ? depth : 3);
        v->band = band;
        v->grads = grads != 0;
        v->has_transform = world_to_model16 != nullptr;
        if (world_to_model16) std::memcpy(v->mat.m, world_to_model16, sizeof v->mat.m);
        RenderHandle h(t->t);
        const Interval root[3] = {Interval(-1.0f, 1.0f), Interval(-1.0f, 1.0f), Interval(-1.0f, 1.0f)};
        const uint32_t x0[3] = {0, 0, 0};
        try {
            v->cell(&h, root, 1u << depth, x0);
        } catch (...) {
            delete v;
            throw;
        }
        return v;
    } catch (const std::exception&) {
        return nullptr;
    }
}

void vo_counts(const void* h, uint64_t* n_bricks, uint64_t* n_tiles) {
    const Volume* v = static_cast<const Volume*>(h);
    *n_bricks = v->bricks.size() / 3;
    *n_tiles = v->tiles.size() / 5;
}

// bricks: n_bricks * 3 words, values: n_bricks B^3, grads (with grads, or null): n_bricks B^3 3, tiles: n_tiles * 5
void vo_read(const void* h, uint32_t* bricks, float* values, float* grads, uint32_t* tiles) {
    const Volume* v = static_cast<const Volume*>(h);
    std::memcpy(bricks, v->bricks.data(), v->bricks.size() * 4);
    std::memcpy(values, v->values.data(), v->values.size() * 4);
    if (grads) std::memcpy(grads, v->gvals.data(), v->gvals.size() * 4);
    std::memcpy(tiles, v->tiles.data(), v->tiles.size() * 4);
}

void vo_free(void* h) { delete static_cast<Volume*>(h); }

}  // extern "C"
