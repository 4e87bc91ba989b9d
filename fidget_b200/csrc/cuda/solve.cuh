// Batched Levenberg-Marquardt solvers (fc_solve_batch, fc_solve_large_batch): launch parameters shared by solve.cu and
// solve_capi.cu.
#pragma once
#include "kernels.cuh"
#include "solve_plan.h"

namespace fdev {

constexpr uint32_t SOLVE_MAX_FREE = 64;           // free parameters (Jacobian columns)
constexpr uint32_t SOLVE_MAX_CONSTRAINTS = 256;   // constraint tapes (Jacobian rows)
constexpr uint32_t SOLVE_MAX_PARAMS = 1024;       // free + fixed parameters of one problem
constexpr int SOLVE_MAX_SWEEPS = 30;              // Jacobi sweep cap (reached only by NaN / inf matrices)
constexpr int SOLVE_MAX_ATTEMPTS = 1024;          // step-size attempts per iteration (unreachable, see solve.cu)

struct SolveResultDev { uint32_t status, iterations; float err; uint32_t pad; };   // == fc_solve_result

struct SolveParams {
    const TapeRef* tapes;          // [m] constraint tapes (only ptr / n_ops are read)
    const uint32_t* slot_off;      // [m + 1]: slot map of constraint k is slot_param[slot_off[k] .. slot_off[k + 1])
    const int32_t* slot_param;     // tape input slot -> parameter index
    uint32_t m, n_params, n_free, max_iters;
    float* values;                 // [n_problems][n_params], free entries overwritten with the solution
    SolveResultDev* results;       // [n_problems] or null
    uint64_t n_problems;
    CancelRef cancel;              // polled before a problem is claimed and at the top of every iteration
    float* work;                   // k_solve_large: [clusters][slice_floats] workspace (solve_plan.h)
    size_t slice_floats;
};

// Dynamic shared memory of one block (bytes)
size_t solve_smem_bytes(uint32_t m, uint32_t n_params, uint32_t n_free);
uint32_t solve_threads(uint32_t n_free);
// Sets the kernel's shared-memory limit and returns its resident blocks per SM for this shape (0: does not fit)
int solve_blocks_per_sm(uint32_t m, uint32_t n_params, uint32_t n_free);
void launch_solve(const SolveParams& p, int blocks, cudaStream_t s);

// k_solve_large: one problem per cluster of `cluster` CTAs.  Sets the kernel's attributes and returns the device's
// resident clusters of that size (cudaOccupancyMaxActiveClusters; 0: none fits), or a negative CUDA error
int solve_large_max_clusters(uint32_t cluster);
cudaError_t launch_solve_large(const SolveParams& p, uint32_t cluster, uint64_t clusters, cudaStream_t s);

}  // namespace fdev
