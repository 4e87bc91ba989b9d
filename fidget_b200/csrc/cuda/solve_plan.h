// Launch planning of fc_solve_large_batch (solve.cu, k_solve_large): the cluster size, the workspace of one cluster and
// the clusters in flight.  Plain host arithmetic with no CUDA runtime call, so tests/csrc/solve_plan_check.cu can check it
// on the CPU; solve_capi.cu feeds it the occupancy query.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>

namespace fdev {

constexpr uint32_t SOLVE_LARGE_MAX_FREE = 1024;          // free parameters (Jacobian columns)
constexpr uint32_t SOLVE_LARGE_MAX_CONSTRAINTS = 4096;   // constraint tapes (Jacobian rows)
constexpr uint32_t SOLVE_LARGE_MAX_PARAMS = 16384;       // free + fixed parameters of one problem
constexpr uint32_t SOLVE_LARGE_MAX_CLUSTER = 16;         // CTAs per cluster (above 8: a non-portable cluster size)
constexpr uint32_t SOLVE_LARGE_COLS_PER_CTA = 64;        // free columns per CTA of the cluster-size rule

// CTAs per problem: one per 64 free columns, rounded up to a power of two, 1 .. 16 (n <= 64: 1, <= 128: 2, <= 256: 4,
// <= 512: 8, else 16).  `forced` > 0 (FIDGET_B200_SOLVE_CLUSTER) fixes it instead, clamped to 1 .. 16.
inline uint32_t solve_cluster_size(uint32_t n_free, int forced) {
    if (forced > 0) return std::min<uint32_t>(uint32_t(forced), SOLVE_LARGE_MAX_CLUSTER);
    uint32_t c = 1;
    while (c < SOLVE_LARGE_MAX_CLUSTER && uint64_t(c) * SOLVE_LARGE_COLS_PER_CTA < n_free) c *= 2;
    return c;
}

// The workspace of one cluster in floats: the parameter row [n_params], cur / trial / Jtr / y [n_free each], r / e [m],
// J [m][n_free], JtJ / A / V [n_free][n_free]
inline size_t solve_large_slice_floats(uint32_t m, uint32_t n_params, uint32_t n_free) {
    const size_t n = n_free;
    return size_t(n_params) + 4 * n + 2 * size_t(m) + size_t(m) * n + 3 * n * n;
}
// ... in bytes, rounded up to 256 so that every cluster's slice starts aligned
inline size_t solve_large_slice_bytes(uint32_t m, uint32_t n_params, uint32_t n_free) {
    return (4 * solve_large_slice_floats(m, n_params, n_free) + 255) & ~size_t(255);
}

// Clusters in flight: min(n_problems, the device's resident clusters scaled to `sm_count` of its `device_sms` SMs
// (FIDGET_B200_SM_COUNT), the slices that fit `budget` bytes), and never fewer than one: a lone problem always gets its
// workspace.  `max_active`: cudaOccupancyMaxActiveClusters for the whole device.
inline uint64_t solve_large_clusters(uint64_t n_problems, int max_active, int sm_count, int device_sms,
                                     size_t slice_bytes, size_t budget) {
    uint64_t resident = uint64_t(std::max(max_active, 1));
    if (device_sms > 0 && sm_count < device_sms) resident = resident * uint64_t(std::max(sm_count, 1)) / uint64_t(device_sms);
    const uint64_t by_budget = slice_bytes ? budget / slice_bytes : resident;
    return std::max<uint64_t>(1, std::min({n_problems, resident, by_budget}));
}

}  // namespace fdev
