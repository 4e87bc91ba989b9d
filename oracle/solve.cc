// ORACLE -- test infrastructure, not product code.
//
// CPU restatement of fc_solve_batch (fidget_b200/csrc/cuda/solve.cu), i.e. of fidget-solver's solve
// (fidget-solver/src/lib.rs:191-289) with the device's operation order: the same Jacobian columns, the same
// sequential sums for JtJ / Jtr / the error, and the same round-robin Jacobi eigen-solve (rotation formula, skip
// rule, sweep cap and zeroing), step for step.  The tapes run on the oracle's own point and gradient VM (vm.cc).
// Built by build.sh as oracle/libsolve_oracle.so, linked against liboracle.so (tests/solve_oracle.py is its ctypes
// face), with -ffp-contract=off, so on tapes made of IEEE operations the result equals the device's bit for bit.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "vm.h"

namespace oracle {

namespace {

constexpr int MAX_SWEEPS = 30;      // SOLVE_MAX_SWEEPS
constexpr int MAX_ATTEMPTS = 1024;  // SOLVE_MAX_ATTEMPTS
enum : uint32_t { ZERO_RESIDUAL = 0, UNCHANGED, ZERO_ERR, ZERO_DAMPING, STALLED, MAX_ITERS, NONE };

struct SolveResult { uint32_t status, iterations; float err; uint32_t pad; };

void rr_pair(uint32_t k, uint32_t r, uint32_t N, uint32_t& p, uint32_t& q) {
    const uint32_t M = N - 1;
    uint32_t a, b;
    if (k == 0) {
        a = 0;
        b = r % M + 1;
    } else {
        a = (k + r) % M + 1;
        b = (N - 1 - k + r) % M + 1;
    }
    p = a < b ? a : b;
    q = a < b ? b : a;
}

// jacobi_block (solve.cu), one thread: the phases of a round run one after the other over all pairs
void jacobi(std::vector<float>& A, std::vector<float>& V, uint32_t n) {
    const uint32_t N = n + (n & 1u), P = N / 2u;
    std::vector<float> rc(P), rs(P);
    std::vector<uint8_t> on(P);
    for (int sweep = 0; sweep < MAX_SWEEPS; ++sweep) {
        bool rotated = false;
        for (uint32_t r = 0; r + 1 < N; ++r) {
            bool any = false;
            for (uint32_t k = 0; k < P; ++k) {
                uint32_t p, q;
                rr_pair(k, r, N, p, q);
                on[k] = 0;
                if (q >= n) continue;
                const float apq = A[p * n + q], app = std::fabs(A[p * n + p]), aqq = std::fabs(A[q * n + q]);
                const float g = 100.0f * std::fabs(apq);
                if (app + g == app && aqq + g == aqq) {
                    A[p * n + q] = 0.0f;
                    A[q * n + p] = 0.0f;
                    continue;
                }
                const float h = A[q * n + q] - A[p * n + p];
                float t;
                if (std::fabs(h) + g == std::fabs(h)) {
                    t = apq / h;
                } else {
                    const float theta = 0.5f * h / apq;
                    t = 1.0f / (std::fabs(theta) + std::sqrt(1.0f + theta * theta));
                    if (theta < 0.0f) t = -t;
                }
                const float c = 1.0f / std::sqrt(1.0f + t * t);
                rc[k] = c;
                rs[k] = t * c;
                on[k] = 1;
                any = true;
            }
            if (!any) continue;
            rotated = true;
            for (int mat = 0; mat < 2; ++mat) {
                std::vector<float>& X = mat == 0 ? A : V;
                for (uint32_t i = 0; i < n; ++i)
                    for (uint32_t k = 0; k < P; ++k) {
                        if (!on[k]) continue;
                        uint32_t p, q;
                        rr_pair(k, r, N, p, q);
                        const float c = rc[k], s = rs[k], xp = X[i * n + p], xq = X[i * n + q];
                        X[i * n + p] = c * xp - s * xq;
                        X[i * n + q] = s * xp + c * xq;
                    }
            }
            for (uint32_t j = 0; j < n; ++j)
                for (uint32_t k = 0; k < P; ++k) {
                    if (!on[k]) continue;
                    uint32_t p, q;
                    rr_pair(k, r, N, p, q);
                    const float c = rc[k], s = rs[k], xp = A[p * n + j], xq = A[q * n + j];
                    A[p * n + j] = j == q ? 0.0f : c * xp - s * xq;
                    A[q * n + j] = j == p ? 0.0f : s * xp + c * xq;
                }
        }
        if (!rotated) break;
    }
}

// delta = pinv(A) b as the device forms it; A is overwritten
void pinv_apply(std::vector<float>& A, const float* b, uint32_t n, float* delta) {
    std::vector<float> V(size_t(n) * n, 0.0f), y(n);
    for (uint32_t i = 0; i < n; ++i) V[i * n + i] = 1.0f;
    jacobi(A, V, n);
    for (uint32_t i = 0; i < n; ++i) {
        float t = 0.0f;
        for (uint32_t k = 0; k < n; ++k) t = t + V[k * n + i] * b[k];
        const float w = A[i * n + i];
        y[i] = std::fabs(w) > FLT_EPSILON ? t / w : 0.0f;
    }
    for (uint32_t j = 0; j < n; ++j) {
        float d = 0.0f;
        for (uint32_t i = 0; i < n; ++i) d = d + V[j * n + i] * y[i];
        delta[j] = d;
    }
}

struct Problem {
    std::vector<TapeP> tapes;
    std::vector<std::vector<int32_t>> slots;
    uint32_t n_params, n_free, max_iters;
};

void solve_one(const Problem& pb, float* vals, SolveResult* res) {
    const uint32_t n = pb.n_free, m = uint32_t(pb.tapes.size()), G = (n + 2) / 3;
    const float* par = vals;   // fixed entries never change; free entries are read only at the start
    std::vector<float> cur(vals, vals + n), trial(n), jtr(n), r(m), e(m), J(size_t(m) * n), jtj(size_t(n) * n),
        A(size_t(n) * n), delta(n);
    std::vector<Grad> gin, gout;
    std::vector<float> fin, fout;
    GradSliceEval ge;
    PointEval pe;
    float damping = 1.0f, prev_err = INFINITY, err = 0.0f, err_buf[4] = {0, 0, 0, 0};
    uint32_t status = MAX_ITERS, iters = pb.max_iters;
    for (uint32_t it = 0; it < pb.max_iters; ++it) {
        for (uint32_t k = 0; k < m; ++k) {
            const Tape& t = *pb.tapes[k];
            gout.assign(std::max<uint32_t>(t.d.ssa.output_count, 1), Grad());
            for (uint32_t g = 0; g < G; ++g) {
                const uint32_t c0 = 3 * g;
                gin.assign(t.n_vars(), Grad());
                for (size_t s = 0; s < t.n_vars(); ++s) {
                    const uint32_t pi = uint32_t(pb.slots[k][s]);
                    gin[s] = pi < n ? Grad(cur[pi], pi == c0 ? 1.0f : 0.0f, pi == c0 + 1 ? 1.0f : 0.0f,
                                           pi == c0 + 2 ? 1.0f : 0.0f)
                                    : Grad(vals[pi]);
                }
                std::vector<const Grad*> vp(gin.size());
                for (size_t s = 0; s < gin.size(); ++s) vp[s] = &gin[s];
                std::vector<Grad*> op(gout.size());
                for (size_t o = 0; o < gout.size(); ++o) op[o] = &gout[o];
                ge.eval(t, vp.data(), 1, op.data());
                const Grad out = gout[0];
                J[k * n + c0] = out.dx;
                if (c0 + 1 < n) J[k * n + c0 + 1] = out.dy;
                if (c0 + 2 < n) J[k * n + c0 + 2] = out.dz;
                if (g == 0) r[k] = out.v;
            }
        }
        bool nonzero = false;
        for (uint32_t k = 0; k < m; ++k) nonzero |= r[k] != 0.0f;
        if (!nonzero) {
            status = ZERO_RESIDUAL;
            iters = it;
            break;
        }
        for (uint32_t a = 0; a < n; ++a)
            for (uint32_t b = 0; b < n; ++b) {
                float s = 0.0f;
                for (uint32_t k = 0; k < m; ++k) s = s + J[k * n + a] * J[k * n + b];
                jtj[a * n + b] = s;
            }
        for (uint32_t a = 0; a < n; ++a) {
            float s = 0.0f;
            for (uint32_t k = 0; k < m; ++k) s = s + J[k * n + a] * r[k];
            jtr[a] = s;
        }
        for (int attempt = 0;; ++attempt) {
            for (uint32_t a = 0; a < n; ++a)
                for (uint32_t b = 0; b < n; ++b)
                    A[a * n + b] = jtj[a * n + b] + damping * (a == b ? jtj[a * n + a] : 0.0f);
            pinv_apply(A, jtr.data(), n, delta.data());
            for (uint32_t j = 0; j < n; ++j) trial[j] = cur[j] - delta[j];
            for (uint32_t k = 0; k < m; ++k) {
                const Tape& t = *pb.tapes[k];
                fin.assign(t.n_vars(), 0.0f);
                for (size_t s = 0; s < t.n_vars(); ++s) {
                    const uint32_t pi = uint32_t(pb.slots[k][s]);
                    fin[s] = pi < n ? trial[pi] : par[pi];
                }
                fout.assign(std::max<uint32_t>(t.d.ssa.output_count, 1), 0.0f);
                pe.eval(t, fin.data(), fout.data());
                e[k] = fout[0] * fout[0];
            }
            err = 0.0f;
            for (uint32_t k = 0; k < m; ++k) err = err + e[k];
            if (err > prev_err && attempt + 1 < MAX_ATTEMPTS) {
                damping = damping * 1.5f;
            } else {
                damping = damping / 3.0f;
                break;
            }
        }
        bool changed = false;
        for (uint32_t j = 0; j < n; ++j) {
            changed |= trial[j] != cur[j];
            cur[j] = trial[j];
        }
        err_buf[it & 3u] = err;
        uint32_t st = NONE;
        if (!changed) st = UNCHANGED;
        else if (err == 0.0f) st = ZERO_ERR;
        else if (damping == 0.0f) st = ZERO_DAMPING;
        else if (err_buf[1] == err_buf[0] && err_buf[2] == err_buf[0] && err_buf[3] == err_buf[0]) st = STALLED;
        prev_err = err;
        if (st != NONE) {
            status = st;
            iters = it + 1;
            break;
        }
    }
    for (uint32_t j = 0; j < n; ++j) vals[j] = cur[j];
    if (res) *res = SolveResult{status, iters, status == ZERO_RESIDUAL ? 0.0f : err, 0};
}

}  // namespace
}  // namespace oracle

using namespace oracle;
struct orc_tape { TapeP t; };   // as in capi.cc
static thread_local std::string g_solve_err;

extern "C" {

const char* orc_solve_last_error(void) { return g_solve_err.c_str(); }

// fc_solve_batch on the CPU; values: [n_problems][n_params] (host), results: [n_problems] x 16 bytes or NULL
int32_t orc_solve_batch(const orc_tape* const* tapes, uint32_t n_constraints, const int32_t* const* slot_param,
                        uint32_t n_params, uint32_t n_free, uint32_t max_iters, float* values, uint64_t n_problems,
                        void* results) {
    try {
        if (n_free == 0 || n_free > n_params) throw std::runtime_error("bad n_free");
        Problem pb;
        pb.n_params = n_params;
        pb.n_free = n_free;
        pb.max_iters = max_iters ? max_iters : 1000u;
        for (uint32_t k = 0; k < n_constraints; ++k) {
            pb.tapes.push_back(tapes[k]->t);
            const size_t nv = tapes[k]->t->n_vars();
            std::vector<int32_t> s(slot_param[k], slot_param[k] + nv);
            for (int32_t pi : s)
                if (pi < 0 || uint32_t(pi) >= n_params) throw std::runtime_error("unbound input slot");
            pb.slots.push_back(std::move(s));
        }
        auto* res = static_cast<SolveResult*>(results);
        for (uint64_t i = 0; i < n_problems; ++i) solve_one(pb, values + i * n_params, res ? res + i : nullptr);
        return 0;
    } catch (const std::exception& e) {
        g_solve_err = e.what();
        return -1;
    }
}

// delta = pinv(A) b through the solver's Jacobi eigen-solve (A: n x n row-major, symmetric)
void orc_sym_pinv_apply(uint32_t n, const float* A, const float* b, float* out) {
    std::vector<float> a(A, A + size_t(n) * n);
    pinv_apply(a, b, n, out);
}

}  // extern "C"
