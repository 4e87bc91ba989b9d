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

#include <cooperative_groups.h>

#include "interp.cuh"
#include "solve.cuh"

namespace fdev {

namespace cg = cooperative_groups;

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
    __shared__ uint32_t s_again, s_status, s_cancel;
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
            s_cancel = cancel_poll(p.cancel, CS_SOLVE, uint32_t(prob));
        }
        __syncthreads();
        if (s_cancel) break;   // (uniform) claim nothing more
        uint32_t status = ST_MAX_ITERS, iters = p.max_iters;
        bool cancelled = false;
        for (uint32_t it = 0; it < p.max_iters; ++it) {
            if (tid == 0) s_cancel = cancel_poll(p.cancel, CS_SOLVE, uint32_t(prob));   // read after the Jacobian
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
            if (s_cancel) {   // (uniform) the problem stops unsolved and its row is not written
                cancelled = true;
                break;
            }
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
        if (cancelled) break;
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

// ---------------------------------------------------------------------------------------------------------------
// fc_solve_large_batch: one problem per cluster of C CTAs (solve_plan.h), k_solve's phases with the work of each spread
// over the whole cluster and separated by cluster barriers.  The matrices live in the cluster's slice of a global
// workspace (L2-resident at moderate n); each CTA keeps the round tables and its copy of the scalar state in shared
// memory.  Every element keeps k_solve's operation sequence (each sum in the same order), so the bits are k_solve's;
// only the assignment of elements to threads differs.  Control flow is uniform over the cluster: every decision is
// recomputed identically in every CTA from the same global data read after a barrier (residual test, attempt loop,
// Jacobi round / sweep exits, exit status), except cancellation, which rank 0 polls and publishes in its shared memory
// (a sticky flag: cancellation ends the launch, so it is never reset).  Details and the hazard list: DESIGN.md.
constexpr uint32_t SOLVE_LARGE_THREADS = 256;
constexpr uint32_t JT_TILE = 64, JT_K = 32;   // JtJ: 64 x 64 entries per tile, J staged 32 rows at a time
static_assert(2 * JT_TILE * JT_K >= SOLVE_LARGE_MAX_CONSTRAINTS, "s_buf also stages e[]");
static_assert(JT_TILE * JT_TILE == 16 * SOLVE_LARGE_THREADS, "4 x 4 JtJ entries per thread");

// jacobi_block over a cluster.  Per round: every CTA computes every pair's angle (identical inputs, identical results,
// so "no rotation this round / sweep" is the same decision everywhere); barrier (all reads of A done); each skipped
// pair's zeros are written by one owner thread (the one that computed its angle, in one CTA), and the column updates
// of A and V run; barrier; row updates; barrier.  A round without a rotation takes only the first barrier.  The zeros
// may land in any order against the column and row updates: those touch the columns and rows of rotated pairs only,
// which are disjoint from the skipped ones.
__device__ void jacobi_cluster(float* A, float* V, uint32_t n, float* rc, float* rs, uint32_t* on, uint32_t gt,
                               uint32_t GT) {
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t tid = threadIdx.x, nt = blockDim.x, C = cluster.num_blocks(), rank = cluster.block_rank();
    const uint32_t N = n + (n & 1u), P = N / 2u;
    for (int sweep = 0; sweep < SOLVE_MAX_SWEEPS; ++sweep) {
        int rotated = 0;
        for (uint32_t r = 0; r + 1 < N; ++r) {
            int mine = 0;
            for (uint32_t k = tid; k < P; k += nt) {
                uint32_t p, q, o = 0;   // 0: dummy pair, 1: rotate, 2: skip (zero a_pq, a_qp)
                rr_pair(k, r, N, p, q);
                if (q < n) {
                    const float apq = A[p * n + q], app = fabsf(A[p * n + p]), aqq = fabsf(A[q * n + q]);
                    const float g = 100.0f * fabsf(apq);
                    if (app + g == app && aqq + g == aqq) {
                        o = 2;
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
                mine |= int(o == 1);
            }
            const int any = __syncthreads_or(mine);   // the same in every CTA
            cluster.sync();
            // the zeros: pair k by CTA (k / nt) mod C, thread k mod nt -- the thread that wrote on[k] above and writes
            // it next round, so a round without a rotation needs no barrier between this read and that write
            for (uint32_t k = tid; k < P; k += nt) {
                if (on[k] != 2 || (k / nt) % C != rank) continue;
                uint32_t p, q;
                rr_pair(k, r, N, p, q);
                A[p * n + q] = 0.0f;
                A[q * n + p] = 0.0f;
            }
            if (!any) continue;
            rotated = 1;
            for (uint32_t task = gt; task < 2u * n * P; task += GT) {   // columns p, q of A (first half) and of V
                const uint32_t k = task % P, i = (task / P) % n;
                if (on[k] != 1) continue;
                float* X = task < n * P ? A : V;
                uint32_t p, q;
                rr_pair(k, r, N, p, q);
                const float c = rc[k], s = rs[k], xp = X[i * n + p], xq = X[i * n + q];
                X[i * n + p] = c * xp - s * xq;
                X[i * n + q] = s * xp + c * xq;
            }
            cluster.sync();
            for (uint32_t task = gt; task < n * P; task += GT) {   // rows p, q of A (consecutive threads: consecutive j)
                const uint32_t j = task % n, k = task / n;
                if (on[k] != 1) continue;
                uint32_t p, q;
                rr_pair(k, r, N, p, q);
                const float c = rc[k], s = rs[k], xp = A[p * n + j], xq = A[q * n + j];
                A[p * n + j] = j == q ? 0.0f : c * xp - s * xq;
                A[q * n + j] = j == p ? 0.0f : s * xp + c * xq;
            }
            cluster.sync();
        }
        if (!rotated) break;
    }
}

// JtJ entries [a0, a0 + 64) x [b0, b0 + 64) by one CTA, each a sequential sum over k = 0 .. m-1 as in k_solve; J
// goes through shared memory 32 rows at a time.  With a0 != b0 the mirrored entries get the same values (x * y ==
// y * x bit for bit; the device's NaNs are canonical).
__device__ void jtj_tile(const float* J, uint32_t m, uint32_t n, uint32_t a0, uint32_t b0, float* jtj, float* s_buf) {
    const uint32_t tid = threadIdx.x, nt = blockDim.x, tx = tid % 16u, ty = tid / 16u;
    float* Ja = s_buf;
    float* Jb = s_buf + JT_K * JT_TILE;
    float acc[4][4];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    for (uint32_t k0 = 0; k0 < m; k0 += JT_K) {
        const uint32_t kn = min(JT_K, m - k0);
        __syncthreads();   // the previous rows are consumed
        for (uint32_t x = tid; x < JT_K * JT_TILE; x += nt) {
            const uint32_t kk = x / JT_TILE, c = x % JT_TILE;
            float va = 0.0f, vb = 0.0f;
            if (kk < kn) {
                if (a0 + c < n) va = J[size_t(k0 + kk) * n + a0 + c];
                if (b0 + c < n) vb = J[size_t(k0 + kk) * n + b0 + c];
            }
            Ja[x] = va;
            Jb[x] = vb;
        }
        __syncthreads();
        for (uint32_t kk = 0; kk < kn; ++kk) {
            float a[4], b[4];
            for (int i = 0; i < 4; ++i) a[i] = Ja[kk * JT_TILE + ty + 16u * i];
            for (int j = 0; j < 4; ++j) b[j] = Jb[kk * JT_TILE + tx + 16u * j];
            for (int i = 0; i < 4; ++i)
                for (int j = 0; j < 4; ++j) acc[i][j] = acc[i][j] + a[i] * b[j];
        }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const uint32_t a = a0 + ty + 16u * i, b = b0 + tx + 16u * j;
            if (a >= n || b >= n) continue;
            jtj[a * n + b] = acc[i][j];
            if (a0 != b0) jtj[b * n + a] = acc[i][j];
        }
    __syncthreads();   // s_buf is free again
}

__global__ void __launch_bounds__(SOLVE_LARGE_THREADS) k_solve_large(const __grid_constant__ SolveParams p) {
    __shared__ float s_rc[SOLVE_LARGE_MAX_FREE / 2], s_rs[SOLVE_LARGE_MAX_FREE / 2];
    __shared__ uint32_t s_on[SOLVE_LARGE_MAX_FREE / 2];
    __shared__ float s_buf[2 * JT_TILE * JT_K];   // JtJ: two staged J tiles; error: e[] staged for the sum
    __shared__ float s_damping, s_prev, s_err, s_errbuf[4];
    __shared__ uint32_t s_again, s_status, s_cancel;
    union {
        grd g[REG_SLOTS];
        float2 f[REG_SLOTS];
    } slots;
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t C = cluster.num_blocks(), rank = cluster.block_rank();
    const uint32_t tid = threadIdx.x, nt = blockDim.x, gt = rank * nt + tid, GT = C * nt;
    const uint32_t n = p.n_free, m = p.m, np_ = p.n_params;
    const uint32_t G = (n + 2u) / 3u, T = (n + JT_TILE - 1u) / JT_TILE;
    const uint64_t cid = blockIdx.x / C, n_clusters = gridDim.x / C;
    float* par = p.work + cid * p.slice_floats;
    float* cur = par + np_;
    float* trial = cur + n;
    float* jtr = trial + n;
    float* ybuf = jtr + n;
    float* r = ybuf + n;
    float* e = r + m;
    float* J = e + m;
    float* jtj = J + size_t(m) * n;
    float* A = jtj + size_t(n) * n;
    float* V = A + size_t(n) * n;
    // The cluster's cancel decision: rank 0's flag, set only by rank 0's thread 0 at a poll and read by every thread right
    // after the next cluster barrier.  Every write is separated from every read of the previous value by a cluster
    // barrier (the read after the Jacobian is followed by the JtJ barrier or, on the zero-residual exit, by the
    // end-of-problem barrier), so all threads of the cluster read the same value between two barriers.
    const volatile uint32_t* cancelled_flag = cluster.map_shared_rank(&s_cancel, 0);
    const bool poller = rank == 0 && tid == 0;
    if (poller) s_cancel = 0;

    for (uint64_t prob = cid; prob < p.n_problems; prob += n_clusters) {
        if (poller && cancel_poll(p.cancel, CS_SOLVE_LARGE, uint32_t(prob))) s_cancel = 1;
        cluster.sync();
        if (*cancelled_flag) break;
        float* vrow = p.values + prob * np_;
        for (uint32_t i = gt; i < np_; i += GT) par[i] = vrow[i];
        for (uint32_t i = gt; i < n; i += GT) cur[i] = vrow[i];
        if (tid == 0) {
            s_damping = 1.0f;
            s_prev = __int_as_float(0x7f800000);
            for (int k = 0; k < 4; ++k) s_errbuf[k] = 0.0f;
        }
        cluster.sync();
        uint32_t status = ST_MAX_ITERS, iters = p.max_iters;
        bool cancelled = false;
        for (uint32_t it = 0; it < p.max_iters; ++it) {
            if (poller && cancel_poll(p.cancel, CS_SOLVE_LARGE, uint32_t(prob))) s_cancel = 1;
            // Jacobian and residuals
            for (uint32_t t = gt; t < m * G; t += GT) {
                const uint32_t k = t / G, g = t % G, c0 = 3u * g;
                const TapeRef tr = p.tapes[k];
                const int32_t* sp = p.slot_param + p.slot_off[k];
                const grd res = run_grad(tr.ptr, tr.n_ops, slots.g, [&](uint32_t s) {
                    const uint32_t pi = uint32_t(sp[s]);
                    if (pi < n) return gr(cur[pi], pi == c0 ? 1.0f : 0.0f, pi == c0 + 1u ? 1.0f : 0.0f,
                                          pi == c0 + 2u ? 1.0f : 0.0f);
                    return gr1(par[pi]);
                });
                J[size_t(k) * n + c0] = res.y;
                if (c0 + 1u < n) J[size_t(k) * n + c0 + 1u] = res.z;
                if (c0 + 2u < n) J[size_t(k) * n + c0 + 2u] = res.w;
                if (g == 0) r[k] = res.x;
            }
            cluster.sync();
            if (*cancelled_flag) {   // the problem stops unsolved and its row is not written
                cancelled = true;
                break;
            }
            int nonzero = 0;   // every CTA tests every residual: the same answer everywhere
            for (uint32_t k = tid; k < m; k += nt) nonzero |= r[k] != 0.0f;
            if (!__syncthreads_or(nonzero)) {
                status = ST_ZERO_RESIDUAL;
                iters = it;
                break;
            }
            for (uint32_t tile = rank; tile < T * (T + 1u) / 2u; tile += C) {   // upper-triangle tiles of JtJ
                uint32_t ta = 0, rem = tile;
                while (rem >= T - ta) rem -= T - ta++;
                jtj_tile(J, m, n, ta * JT_TILE, (ta + rem) * JT_TILE, jtj, s_buf);
            }
            for (uint32_t a = gt; a < n; a += GT) {
                float s = 0.0f;
                for (uint32_t k = 0; k < m; ++k) s = s + J[size_t(k) * n + a] * r[k];
                jtr[a] = s;
            }
            cluster.sync();
            // step search
            for (int attempt = 0;; ++attempt) {
                const float damping = s_damping;
                for (uint32_t x = gt; x < n * n; x += GT) {
                    const uint32_t a = x / n, b = x % n;
                    A[x] = jtj[x] + damping * (a == b ? jtj[a * n + a] : 0.0f);
                    V[x] = a == b ? 1.0f : 0.0f;
                }
                cluster.sync();
                jacobi_cluster(A, V, n, s_rc, s_rs, s_on, gt, GT);
                for (uint32_t i = gt; i < n; i += GT) {
                    float t = 0.0f;
                    for (uint32_t k = 0; k < n; ++k) t = t + V[k * n + i] * jtr[k];
                    const float w = A[i * n + i];
                    ybuf[i] = fabsf(w) > FLT_EPSILON ? t / w : 0.0f;
                }
                cluster.sync();
                for (uint32_t j = gt; j < n; j += GT) {
                    float d = 0.0f;
                    for (uint32_t i = 0; i < n; ++i) d = d + V[j * n + i] * ybuf[i];
                    trial[j] = cur[j] - d;
                }
                cluster.sync();
                for (uint32_t k = gt; k < m; k += GT) {
                    const TapeRef tr = p.tapes[k];
                    const int32_t* sp = p.slot_param + p.slot_off[k];
                    const float2 v = run_f32x2(tr.ptr, tr.n_ops, slots.f, [&](uint32_t s) {
                        const uint32_t pi = uint32_t(sp[s]);
                        const float x = pi < n ? trial[pi] : par[pi];
                        return make_float2(x, x);
                    });
                    e[k] = v.x * v.x;
                }
                cluster.sync();
                for (uint32_t k = tid; k < m; k += nt) s_buf[k] = e[k];   // every CTA sums e[] in constraint order
                __syncthreads();
                if (tid == 0) {
                    float err = 0.0f;
                    for (uint32_t k = 0; k < m; ++k) err = err + s_buf[k];
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
            // take the step: every CTA compares every entry, then cur and trial swap roles (k_solve copies trial
            // into cur; the next trial overwrites the other buffer before reading it)
            int changed = 0;
            for (uint32_t j = tid; j < n; j += nt) changed |= trial[j] != cur[j];
            changed = __syncthreads_or(changed);
            float* const was = cur;
            cur = trial;
            trial = was;
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
        if (cancelled) break;
        for (uint32_t i = gt; i < n; i += GT) vrow[i] = cur[i];
        if (poller && p.results) {
            SolveResultDev res;
            res.status = status;
            res.iterations = iters;
            res.err = status == ST_ZERO_RESIDUAL ? 0.0f : s_err;
            res.pad = 0;
            p.results[prob] = res;
        }
        // every read of the flag in this problem precedes the next claim's poll, and the row is written out before the
        // workspace is reused
        cluster.sync();
    }
    cluster.sync();   // rank 0's shared memory (the cancel flag) outlives every reader
}

static cudaLaunchConfig_t large_config(uint32_t cluster, uint64_t clusters, cudaStream_t s, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(uint32_t(uint64_t(cluster) * clusters), 1, 1);
    cfg.blockDim = dim3(SOLVE_LARGE_THREADS, 1, 1);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = cluster;
    attr->val.clusterDim.y = 1;
    attr->val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

int solve_large_max_clusters(uint32_t cluster) {
    if (cluster > 8) {
        const cudaError_t e = cudaFuncSetAttribute(k_solve_large, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        if (e != cudaSuccess) return -int(e);
    }
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = large_config(cluster, 1, nullptr, &attr);
    int clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&clusters, k_solve_large, &cfg) != cudaSuccess) {
        cudaGetLastError();   // (a cluster size the device cannot place)
        return 0;
    }
    return clusters;
}

cudaError_t launch_solve_large(const SolveParams& p, uint32_t cluster, uint64_t clusters, cudaStream_t s) {
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = large_config(cluster, clusters, s, &attr);
    return cudaLaunchKernelEx(&cfg, k_solve_large, p);
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
