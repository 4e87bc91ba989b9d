// fc_solve_batch (include/fidget_cuda.h, "constraint solver"): argument checks, the tape table and slot maps, staging
// of host values / results, and the launch of k_solve (solve.cu).
#include "capi_internal.h"
#include "solve.cuh"

static_assert(sizeof(fc_solve_result) == sizeof(SolveResultDev), "fc_solve_result layout");

extern "C" int32_t fc_solve_batch(fc_ctx* c, const fc_tape* const* constraints, uint32_t n_constraints,
                                  const int32_t* const* slot_param, const fc_solve_cfg* cfg, float* values,
                                  uint64_t n_problems, fc_solve_result* results) {
    if (!c || !cfg || (n_constraints && (!constraints || !slot_param)) || (n_problems && !values))
        return fail(FC_ERR_INVALID, "null argument");
    const uint32_t n_params = cfg->n_params, n_free = cfg->n_free;
    if (n_free == 0) return fail(FC_ERR_INVALID, "fc_solve_batch: no free parameter");
    if (n_free > n_params) return fail(FC_ERR_INVALID, "fc_solve_batch: n_free > n_params");
    if (n_free > SOLVE_MAX_FREE)
        return fail(FC_ERR_UNSUPPORTED, "fc_solve_batch: more than " + std::to_string(SOLVE_MAX_FREE) + " free parameters");
    if (n_constraints > SOLVE_MAX_CONSTRAINTS)
        return fail(FC_ERR_UNSUPPORTED, "fc_solve_batch: more than " + std::to_string(SOLVE_MAX_CONSTRAINTS) + " constraints");
    if (n_params > SOLVE_MAX_PARAMS)
        return fail(FC_ERR_UNSUPPORTED, "fc_solve_batch: more than " + std::to_string(SOLVE_MAX_PARAMS) + " parameters");

    // tape table [m] | slot offsets [m + 1] | slot -> parameter
    std::vector<TapeRef> refs(n_constraints);
    std::vector<uint32_t> offs(n_constraints + 1, 0);
    std::vector<int32_t> slots;
    for (uint32_t k = 0; k < n_constraints; ++k) {
        const fc_tape* t = constraints[k];
        const std::string who = "fc_solve_batch: constraint " + std::to_string(k);
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

    std::lock_guard<std::mutex> guard(c->mu);
    CU(cudaSetDevice(c->device));
    const int per_sm = solve_blocks_per_sm(n_constraints, n_params, n_free);
    if (per_sm <= 0) return fail(FC_ERR_UNSUPPORTED, "fc_solve_batch: problem too large for one thread block's shared memory");

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
    const uint64_t cap = uint64_t(per_sm) * uint64_t(c->sm_count);
    launch_solve(p, int(n_problems < cap ? n_problems : cap), c->stream);
    CU(cudaGetLastError());
    if (!dvals) CU(cudaMemcpyAsync(values, p.values, b_vals, cudaMemcpyDeviceToHost, c->stream));
    if (results && !dres) CU(cudaMemcpyAsync(results, p.results, b_res, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}
