// fc_solve_batch and fc_solve_large_batch (include/fidget_cuda.h, "constraint solver"): argument checks, the tape table
// and slot maps, staging of host values / results, cancellation, and the launch of k_solve or k_solve_large (solve.cu).
#include "capi_internal.h"
#include "solve.cuh"

static_assert(sizeof(fc_solve_result) == sizeof(SolveResultDev), "fc_solve_result layout");
static_assert(FC_SOLVE_LARGE_MAX_FREE == SOLVE_LARGE_MAX_FREE &&
                  FC_SOLVE_LARGE_MAX_CONSTRAINTS == SOLVE_LARGE_MAX_CONSTRAINTS &&
                  FC_SOLVE_LARGE_MAX_PARAMS == SOLVE_LARGE_MAX_PARAMS, "fc_solve_large_batch limits");

static int32_t solve_call(fc_ctx* c, const fc_tape* const* constraints, uint32_t n_constraints,
                          const int32_t* const* slot_param, const fc_solve_cfg* cfg, float* values, uint64_t n_problems,
                          fc_solve_result* results, bool large) {
    const std::string fn = large ? "fc_solve_large_batch" : "fc_solve_batch";
    if (!c || !cfg || (n_constraints && (!constraints || !slot_param)) || (n_problems && !values))
        return fail(FC_ERR_INVALID, "null argument");
    const uint32_t n_params = cfg->n_params, n_free = cfg->n_free;
    const uint32_t max_free = large ? SOLVE_LARGE_MAX_FREE : SOLVE_MAX_FREE;
    const uint32_t max_constraints = large ? SOLVE_LARGE_MAX_CONSTRAINTS : SOLVE_MAX_CONSTRAINTS;
    const uint32_t max_params = large ? SOLVE_LARGE_MAX_PARAMS : SOLVE_MAX_PARAMS;
    if (n_free == 0) return fail(FC_ERR_INVALID, fn + ": no free parameter");
    if (n_free > n_params) return fail(FC_ERR_INVALID, fn + ": n_free > n_params");
    if (n_free > max_free)
        return fail(FC_ERR_UNSUPPORTED, fn + ": more than " + std::to_string(max_free) + " free parameters");
    if (n_constraints > max_constraints)
        return fail(FC_ERR_UNSUPPORTED, fn + ": more than " + std::to_string(max_constraints) + " constraints");
    if (n_params > max_params)
        return fail(FC_ERR_UNSUPPORTED, fn + ": more than " + std::to_string(max_params) + " parameters");

    // tape table [m] | slot offsets [m + 1] | slot -> parameter
    std::vector<TapeRef> refs(n_constraints);
    std::vector<uint32_t> offs(n_constraints + 1, 0);
    std::vector<int32_t> slots;
    for (uint32_t k = 0; k < n_constraints; ++k) {
        const fc_tape* t = constraints[k];
        const std::string who = fn + ": constraint " + std::to_string(k);
        if (!t) return fail(FC_ERR_INVALID, who + " is null");
        if (t->ctx != c) return fail(FC_ERR_INVALID, who + " belongs to another context");
        if (t->info.mem_count) return fail(FC_ERR_UNSUPPORTED, who + " uses memory slots");
        if (t->info.n_outputs == 0) return fail(FC_ERR_INVALID, who + " has no output");
        if (t->info.n_vars && !slot_param[k]) return fail(FC_ERR_INVALID, who + ": null slot map");
        for (uint32_t s = 0; s < t->info.n_vars; ++s) {
            const int32_t pi = slot_param[k][s];
            if (pi < 0 || uint32_t(pi) >= n_params)
                return fail(FC_ERR_INVALID, who + ": input slot " + std::to_string(s) + " is not bound to a parameter");
            slots.push_back(pi);
        }
        offs[k + 1] = uint32_t(slots.size());
        refs[k] = TapeRef{t->dev, t->info.n_ops, t->info.ref_len, t->info.choice_count, 0};
    }
    if (n_problems == 0) return FC_OK;

    CallCancel cc;
    if (int32_t rc = begin_call(c, cc)) return rc;
    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    // launch shape: k_solve's blocks per SM, or k_solve_large's cluster size and clusters in flight (solve_plan.h)
    int per_sm = 0;
    uint32_t cluster = 1;
    uint64_t clusters = 0;
    size_t slice = 0;
    if (!large) {
        per_sm = solve_blocks_per_sm(n_constraints, n_params, n_free);
        if (per_sm <= 0) return fail(FC_ERR_UNSUPPORTED, fn + ": problem too large for one thread block's shared memory");
    } else {
        const int forced = env_int("FIDGET_B200_SOLVE_CLUSTER", 0);
        cluster = solve_cluster_size(n_free, forced);
        int resident = solve_large_max_clusters(cluster);
        // without a forced size, a cluster the device cannot place is halved: every size gives the same bits
        while (resident == 0 && forced <= 0 && cluster > 1) resident = solve_large_max_clusters(cluster /= 2);
        if (resident < 0) CU(cudaError_t(-resident));
        if (resident == 0)
            return fail(FC_ERR_UNSUPPORTED, fn + ": the device cannot place a cluster of " + std::to_string(cluster) + " CTAs");
        int device_sms = 0;
        CU(cudaDeviceGetAttribute(&device_sms, cudaDevAttrMultiProcessorCount, c->device));
        slice = solve_large_slice_bytes(n_constraints, n_params, n_free);
        clusters = solve_large_clusters(n_problems, resident, c->sm_count, device_sms, slice, FC_FRAMES_PASS_BYTES);
        if (cudaError_t e = c->solve_work.ensure(slice * clusters))
            return fail(FC_ERR_CUDA, fn + ": cannot allocate the " + std::to_string(slice * clusters >> 20) +
                                         " MiB solver workspace: " + cudaGetErrorString(e));
    }

    const size_t b_refs = refs.size() * sizeof(TapeRef), b_offs = offs.size() * 4, b_slots = slots.size() * 4;
    const size_t o_offs = (b_refs + 15) & ~size_t(15), o_slots = (o_offs + b_offs + 15) & ~size_t(15);
    std::vector<uint8_t> meta(o_slots + b_slots + 16, 0);
    if (b_refs) memcpy(meta.data(), refs.data(), b_refs);
    memcpy(meta.data() + o_offs, offs.data(), b_offs);
    if (b_slots) memcpy(meta.data() + o_slots, slots.data(), b_slots);
    CU(c->solve_meta.ensure(meta.size()));
    CU(cudaMemcpyAsync(c->solve_meta.p, meta.data(), meta.size(), cudaMemcpyHostToDevice, c->stream));

    SolveParams p{};
    p.tapes = c->solve_meta.as<TapeRef>();
    p.slot_off = reinterpret_cast<const uint32_t*>(c->solve_meta.as<uint8_t>() + o_offs);
    p.slot_param = reinterpret_cast<const int32_t*>(c->solve_meta.as<uint8_t>() + o_slots);
    p.m = n_constraints;
    p.n_params = n_params;
    p.n_free = n_free;
    p.max_iters = cfg->max_iters ? cfg->max_iters : 1000u;
    p.n_problems = n_problems;
    p.cancel = cc.ref;
    p.work = large ? c->solve_work.as<float>() : nullptr;
    p.slice_floats = slice / 4;

    const size_t b_vals = size_t(n_problems) * n_params * 4, b_res = size_t(n_problems) * sizeof(fc_solve_result);
    const bool dvals = is_device_ptr(values), dres = is_device_ptr(results);
    if (dvals) {
        p.values = values;
    } else {
        CU(c->solve_vals.ensure(b_vals));
        CU(cudaMemcpyAsync(c->solve_vals.p, values, b_vals, cudaMemcpyHostToDevice, c->stream));
        p.values = c->solve_vals.as<float>();
    }
    if (results) {
        if (dres) p.results = reinterpret_cast<SolveResultDev*>(results);
        else {
            CU(c->solve_res.ensure(b_res));
            p.results = c->solve_res.as<SolveResultDev>();
        }
    }
    if (large) {
        CU(launch_solve_large(p, cluster, clusters, c->stream));
    } else {
        const uint64_t cap = uint64_t(per_sm) * uint64_t(c->sm_count);
        launch_solve(p, int(n_problems < cap ? n_problems : cap), c->stream);
    }
    CU(cudaGetLastError());
    // with a cancel flag attached the (cancellable) wait comes first, and a cancelled call copies nothing back
    if (cc.flag)
        if (int32_t rc = wait_call(c, c->stream, cc)) return rc;
    if (!dvals) CU(cudaMemcpyAsync(values, p.values, b_vals, cudaMemcpyDeviceToHost, c->stream));
    if (results && !dres) CU(cudaMemcpyAsync(results, p.results, b_res, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

extern "C" int32_t fc_solve_batch(fc_ctx* c, const fc_tape* const* constraints, uint32_t n_constraints,
                                  const int32_t* const* slot_param, const fc_solve_cfg* cfg, float* values,
                                  uint64_t n_problems, fc_solve_result* results) {
    return solve_call(c, constraints, n_constraints, slot_param, cfg, values, n_problems, results, false);
}

extern "C" int32_t fc_solve_large_batch(fc_ctx* c, const fc_tape* const* constraints, uint32_t n_constraints,
                                        const int32_t* const* slot_param, const fc_solve_cfg* cfg, float* values,
                                        uint64_t n_problems, fc_solve_result* results) {
    return solve_call(c, constraints, n_constraints, slot_param, cfg, values, n_problems, results, true);
}
