// Host-side check of fc_solve_large_batch's launch planning (solve_plan.h): compiled with nvcc, run on the CPU by
// tests/test_solve_large_api.py.  Each line is a name and the values the planner gives.
#include <cstdio>

#include "solve_plan.h"

using namespace fdev;

int main() {
    // cluster size from n_free, unforced
    std::printf("cluster");
    for (uint32_t n : {1u, 64u, 65u, 128u, 129u, 256u, 257u, 512u, 513u, 1024u}) std::printf(" %u", solve_cluster_size(n, 0));
    std::printf("\n");
    // forced sizes (FIDGET_B200_SOLVE_CLUSTER), clamped to 1 .. 16
    std::printf("forced");
    for (int f : {1, 3, 8, 16, 17, 64}) std::printf(" %u", solve_cluster_size(1024, f));
    std::printf("\n");
    // workspace of one cluster: floats and bytes (the limits, a tiny problem, a 100-free sketch-sized one)
    std::printf("slice_floats %zu %zu %zu\n", solve_large_slice_floats(4096, 16384, 1024), solve_large_slice_floats(1, 1, 1),
                solve_large_slice_floats(149, 120, 100));
    std::printf("slice_bytes %zu %zu %zu\n", solve_large_slice_bytes(4096, 16384, 1024), solve_large_slice_bytes(1, 1, 1),
                solve_large_slice_bytes(149, 120, 100));
    const size_t big = solve_large_slice_bytes(4096, 16384, 1024), budget = size_t(512) << 20;
    // clusters in flight: problems, resident clusters, SM scaling, budget, and the lone problem
    std::printf("clusters %llu %llu %llu %llu %llu %llu %llu\n",
                (unsigned long long)solve_large_clusters(1, 8, 132, 132, big, budget),        // one problem
                (unsigned long long)solve_large_clusters(1000, 8, 132, 132, 4096, budget),    // resident clusters
                (unsigned long long)solve_large_clusters(1000, 60, 132, 132, big, budget),    // the budget
                (unsigned long long)solve_large_clusters(1000, 66, 3, 132, 4096, budget),     // 3 of 132 SMs
                (unsigned long long)solve_large_clusters(1000, 8, 1, 132, 4096, budget),      // never fewer than one
                (unsigned long long)solve_large_clusters(5, 66, 132, 132, 4096, budget),      // fewer problems
                (unsigned long long)solve_large_clusters(1, 8, 132, 132, budget * 2, budget)); // a lone problem over budget
    return 0;
}
