// Batched Levenberg-Marquardt solver (fc_solve_batch): fidget-solver's solve (fidget-solver/src/lib.rs:191-289) for
// many independent problems that share their constraint tapes, one thread block per problem, the whole loop in one
// launch.
//
// Per problem (the block's scratch lives in shared memory and is reused for the next problem of the batch):
//   Jacobian    one thread per (constraint k, triple g of free columns), as get_jacobian (lib.rs:107-146) groups them:
//               run_grad with the triple's unit partials seeded on the free parameters 3g, 3g+1, 3g+2 (0 past
//               n_free); J[k][3g+c] = d_c, r[k] = the value
//   JtJ, Jtr    every entry a sequential f32 sum over k = 0 .. m-1
//   step        adjusted = JtJ + damping * diag(JtJ) (element by element, as nalgebra adds the two matrices);
//               delta = pinv(adjusted) Jtr by a cyclic Jacobi eigen-solve (jacobi_block below): eigenvalues w with
//               |w| <= f32::EPSILON are dropped, t_i = sum_k V[k][i] Jtr[k], y_i = t_i / w_i, delta_j = sum_i V[j][i] y_i
//   error       one thread per constraint: point evaluation at cur - delta, squared; summed in constraint order
//               (get_err, lib.rs:148-176)
// and the damping / exit logic of solve verbatim.  Every sum has a fixed order, so the CPU oracle (oracle/solve.cc)
// reproduces the result bit for bit on tapes made of IEEE operations.
//
// The reference's outer loop has no cap; here it stops after max_iters steps (FC_SOLVE_MAX_ITERS).  Its inner loop
// needs none: damping grows by 1.5 per rejected attempt, reaches inf after at most ~480 attempts (from the smallest
// denormal), and then adjusted is NaN (inf * 0 off the diagonal) or, for one column, inf; the step is NaN or 0 and
// is accepted.  SOLVE_MAX_ATTEMPTS only guards the device against a hang should that argument ever fail.
#include <cfloat>

#include "interp.cuh"
#include "solve.cuh"

namespace fdev {

enum : uint32_t { ST_ZERO_RESIDUAL = 0, ST_UNCHANGED, ST_ZERO_ERR, ST_ZERO_DAMPING, ST_STALLED, ST_MAX_ITERS, ST_NONE };

// Round-robin ("circle") pairing of N (even) indices: in each of the N - 1 rounds the N / 2 pairs are disjoint, and
// every pair meets once per sweep.  Pair k of round r is (p, q), p < q; q >= n marks the dummy index of odd n.
__host__ __device__ inline void rr_pair(uint32_t k, uint32_t r, uint32_t N, uint32_t& p, uint32_t& q) {
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

// Symmetric n x n eigen-decomposition A = V diag(w) V^T (w = the diagonal left in A), by cyclic Jacobi rotations
// with the round-robin ordering: per round, the rotation angles of the n/2 disjoint pairs are computed from A, then
// A <- A J and V <- V J (column updates), then A <- J^T A (row updates), and the rotated pairs' off-diagonal entries
// are set to 0.  A pair is skipped (and its entries zeroed) when 100 |a_pq| is negligible against both |a_pp| and
// |a_qq| in f32.  Stops after a sweep without a rotation, or after SOLVE_MAX_SWEEPS sweeps (NaN / inf input).
// V must hold the identity on entry.  The caller synchronised A and V; returns synchronised.
__device__ void jacobi_block(float* A, float* V, uint32_t n, float* rc, float* rs, uint32_t* on) {
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    const uint32_t N = n + (n & 1u), P = N / 2u;
    for (int sweep = 0; sweep < SOLVE_MAX_SWEEPS; ++sweep) {
        int rotated = 0;
        for (uint32_t r = 0; r + 1 < N; ++r) {
            int mine = 0;
            for (uint32_t k = tid; k < P; k += nt) {
                uint32_t p, q, o = 0;
                rr_pair(k, r, N, p, q);
                if (q < n) {
                    const float apq = A[p * n + q], app = fabsf(A[p * n + p]), aqq = fabsf(A[q * n + q]);
                    const float g = 100.0f * fabsf(apq);
                    if (app + g == app && aqq + g == aqq) {
                        A[p * n + q] = 0.0f;
                        A[q * n + p] = 0.0f;
                    } else {
                        const float h = A[q * n + q] - A[p * n + p];
                        float t;
                        if (fabsf(h) + g == fabsf(h)) {
                            t = apq / h;
                        } else {
                            const float theta = 0.5f * h / apq;
                            t = 1.0f / (fabsf(theta) + sqrtf(1.0f + theta * theta));
                            if (theta < 0.0f) t = -t;
                        }
                        const float c = 1.0f / sqrtf(1.0f + t * t);
                        rc[k] = c;
                        rs[k] = t * c;
                        o = 1;
                    }
                }
                on[k] = o;
                mine |= int(o);
            }
            if (!__syncthreads_or(mine)) continue;   // uniform
            rotated = 1;
            for (uint32_t task = tid; task < 2u * n * P; task += nt) {   // columns p, q of A (first half) and of V
                const uint32_t k = task % P, i = (task / P) % n;
                if (!on[k]) continue;
                float* X = task < n * P ? A : V;
                uint32_t p, q;
                rr_pair(k, r, N, p, q);
                const float c = rc[k], s = rs[k], xp = X[i * n + p], xq = X[i * n + q];
                X[i * n + p] = c * xp - s * xq;
                X[i * n + q] = s * xp + c * xq;
            }
            __syncthreads();
            for (uint32_t task = tid; task < n * P; task += nt) {   // rows p, q of A
                const uint32_t k = task % P, j = task / P;
                if (!on[k]) continue;
                uint32_t p, q;
                rr_pair(k, r, N, p, q);
                const float c = rc[k], s = rs[k], xp = A[p * n + j], xq = A[q * n + j];
                A[p * n + j] = j == q ? 0.0f : c * xp - s * xq;
                A[q * n + j] = j == p ? 0.0f : s * xp + c * xq;
            }
            __syncthreads();
        }
        if (!rotated) break;
    }
}

size_t solve_smem_bytes(uint32_t m, uint32_t n_params, uint32_t n_free) {
    const size_t n = n_free, P = (n + 1) / 2;
    return 4 * (size_t(n_params) + 5 * n + 2 * size_t(m) + size_t(m) * n + 3 * n * n + 3 * P);
}
uint32_t solve_threads(uint32_t n_free) { return n_free > 16 ? 256u : 128u; }

__global__ void __launch_bounds__(256) k_solve(const __grid_constant__ SolveParams p) {
    extern __shared__ float sm[];
    __shared__ float s_damping, s_prev, s_err, s_errbuf[4];
    __shared__ uint32_t s_again, s_status;
    union {
        grd g[REG_SLOTS];
        float2 f[REG_SLOTS];
    } slots;
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    const uint32_t n = p.n_free, m = p.m, np_ = p.n_params;
    const uint32_t G = (n + 2u) / 3u, P = (n + 1u) / 2u;
    float* par = sm;
    float* cur = par + np_;
    float* trial = cur + n;
    float* delta = trial + n;
    float* jtr = delta + n;
    float* ybuf = jtr + n;
    float* r = ybuf + n;
    float* e = r + m;
    float* J = e + m;
    float* jtj = J + size_t(m) * n;
    float* A = jtj + n * n;
    float* V = A + n * n;
    float* rc = V + n * n;
    float* rs = rc + P;
    uint32_t* on = reinterpret_cast<uint32_t*>(rs + P);

    for (uint64_t prob = blockIdx.x; prob < p.n_problems; prob += gridDim.x) {
        float* vrow = p.values + prob * np_;
        for (uint32_t i = tid; i < np_; i += nt) par[i] = vrow[i];
        for (uint32_t i = tid; i < n; i += nt) cur[i] = vrow[i];
        if (tid == 0) {
            s_damping = 1.0f;
            s_prev = __int_as_float(0x7f800000);
            for (int k = 0; k < 4; ++k) s_errbuf[k] = 0.0f;
        }
        __syncthreads();
        uint32_t status = ST_MAX_ITERS, iters = p.max_iters;
        for (uint32_t it = 0; it < p.max_iters; ++it) {
            // Jacobian and residuals
            for (uint32_t t = tid; t < m * G; t += nt) {
                const uint32_t k = t / G, g = t % G, c0 = 3u * g;
                const TapeRef tr = p.tapes[k];
                const int32_t* sp = p.slot_param + p.slot_off[k];
                const grd res = run_grad(tr.ptr, tr.n_ops, slots.g, [&](uint32_t s) {
                    const uint32_t pi = uint32_t(sp[s]);
                    if (pi < n) return gr(cur[pi], pi == c0 ? 1.0f : 0.0f, pi == c0 + 1u ? 1.0f : 0.0f,
                                          pi == c0 + 2u ? 1.0f : 0.0f);
                    return gr1(par[pi]);
                });
                J[k * n + c0] = res.y;
                if (c0 + 1u < n) J[k * n + c0 + 1u] = res.z;
                if (c0 + 2u < n) J[k * n + c0 + 2u] = res.w;
                if (g == 0) r[k] = res.x;
            }
            __syncthreads();
            int nonzero = 0;
            for (uint32_t k = tid; k < m; k += nt) nonzero |= r[k] != 0.0f;
            if (!__syncthreads_or(nonzero)) {
                status = ST_ZERO_RESIDUAL;
                iters = it;
                break;
            }
            for (uint32_t x = tid; x < n * n; x += nt) {
                const uint32_t a = x / n, b = x % n;
                float s = 0.0f;
                for (uint32_t k = 0; k < m; ++k) s = s + J[k * n + a] * J[k * n + b];
                jtj[x] = s;
            }
            for (uint32_t a = tid; a < n; a += nt) {
                float s = 0.0f;
                for (uint32_t k = 0; k < m; ++k) s = s + J[k * n + a] * r[k];
                jtr[a] = s;
            }
            __syncthreads();
            // step search
            for (int attempt = 0;; ++attempt) {
                const float damping = s_damping;
                for (uint32_t x = tid; x < n * n; x += nt) {
                    const uint32_t a = x / n, b = x % n;
                    A[x] = jtj[x] + damping * (a == b ? jtj[a * n + a] : 0.0f);
                    V[x] = a == b ? 1.0f : 0.0f;
                }
                __syncthreads();
                jacobi_block(A, V, n, rc, rs, on);
                for (uint32_t i = tid; i < n; i += nt) {
                    float t = 0.0f;
                    for (uint32_t k = 0; k < n; ++k) t = t + V[k * n + i] * jtr[k];
                    const float w = A[i * n + i];
                    ybuf[i] = fabsf(w) > FLT_EPSILON ? t / w : 0.0f;
                }
                __syncthreads();
                for (uint32_t j = tid; j < n; j += nt) {
                    float d = 0.0f;
                    for (uint32_t i = 0; i < n; ++i) d = d + V[j * n + i] * ybuf[i];
                    delta[j] = d;
                    trial[j] = cur[j] - d;
                }
                __syncthreads();
                for (uint32_t k = tid; k < m; k += nt) {
                    const TapeRef tr = p.tapes[k];
                    const int32_t* sp = p.slot_param + p.slot_off[k];
                    const float2 v = run_f32x2(tr.ptr, tr.n_ops, slots.f, [&](uint32_t s) {
                        const uint32_t pi = uint32_t(sp[s]);
                        const float x = pi < n ? trial[pi] : par[pi];
                        return make_float2(x, x);
                    });
                    e[k] = v.x * v.x;
                }
                __syncthreads();
                if (tid == 0) {
                    float err = 0.0f;
                    for (uint32_t k = 0; k < m; ++k) err = err + e[k];
                    s_err = err;
                    if (err > s_prev && attempt + 1 < SOLVE_MAX_ATTEMPTS) {
                        s_damping = s_damping * 1.5f;
                        s_again = 1;
                    } else {
                        s_damping = s_damping / 3.0f;
                        s_again = 0;
                    }
                }
                __syncthreads();
                if (!s_again) break;
            }
            // take the step
            int changed = 0;
            for (uint32_t j = tid; j < n; j += nt) {
                changed |= trial[j] != cur[j];
                cur[j] = trial[j];
            }
            changed = __syncthreads_or(changed);
            if (tid == 0) {
                const float err = s_err;
                s_errbuf[it & 3u] = err;
                uint32_t st = ST_NONE;
                if (!changed) st = ST_UNCHANGED;
                else if (err == 0.0f) st = ST_ZERO_ERR;
                else if (s_damping == 0.0f) st = ST_ZERO_DAMPING;
                else if (s_errbuf[1] == s_errbuf[0] && s_errbuf[2] == s_errbuf[0] && s_errbuf[3] == s_errbuf[0])
                    st = ST_STALLED;
                s_status = st;
                s_prev = err;
            }
            __syncthreads();
            if (s_status != ST_NONE) {
                status = s_status;
                iters = it + 1u;
                break;
            }
        }
        for (uint32_t i = tid; i < n; i += nt) vrow[i] = cur[i];
        if (tid == 0 && p.results) {
            SolveResultDev res;
            res.status = status;
            res.iterations = iters;
            res.err = status == ST_ZERO_RESIDUAL ? 0.0f : s_err;
            res.pad = 0;
            p.results[prob] = res;
        }
        __syncthreads();   // the next problem reuses the scratch
    }
}

int solve_blocks_per_sm(uint32_t m, uint32_t n_params, uint32_t n_free) {
    const size_t smem = solve_smem_bytes(m, n_params, n_free);
    if (cudaFuncSetAttribute(k_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int blocks = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, k_solve, int(solve_threads(n_free)), smem) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return blocks;
}

void launch_solve(const SolveParams& p, int blocks, cudaStream_t s) {
    k_solve<<<blocks, solve_threads(p.n_free), solve_smem_bytes(p.m, p.n_params, p.n_free), s>>>(p);
}

}  // namespace fdev
