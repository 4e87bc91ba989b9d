// C ABI of libfidget_cuda (include/fidget_cuda.h): contexts, tapes, the trait-level evaluators and
// fc_simplify.  The renderers live in render.cu, the octree sampler in octree_capi.cu, the effects in
// effects_capi.cu, the level-0 schedule in schedule.cu.
#include <functional>
#include <thread>

#include "capi_internal.h"

thread_local std::string g_err;

////////////////////////////////////////////////////////////////////////////
// bytecode <-> device clauses
int32_t transcode(const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count,
                         uint32_t n_vars, uint32_t n_outputs, std::vector<uint2>& out, uint32_t& n_choices) {
    if (!words || n_words < 4 || (n_words & 1)) return fail(FC_ERR_INVALID, "bytecode: bad length");
    if (words[0] != 0xFFFFFFFFu || words[1] != 0u) return fail(FC_ERR_INVALID, "bytecode: missing start marker");
    if (words[n_words - 2] != 0xFFFFFFFFu || words[n_words - 1] != 0xFFFFFFFFu)
        return fail(FC_ERR_INVALID, "bytecode: missing end marker");
    out.clear();
    n_choices = 0;
    auto reg_ok = [&](uint32_t r) { return r < reg_count; };
    for (size_t i = 2; i + 2 < n_words; i += 2) {
        uint32_t w = words[i], imm = words[i + 1];
        uint32_t op = w & 0xff, b1 = (w >> 8) & 0xff, b2 = (w >> 16) & 0xff, b3 = w >> 24;
        if (op >= OP_COUNT) return fail(FC_ERR_INVALID, "bytecode: unknown opcode " + std::to_string(op));
        uint32_t x;
        bool ok = true;
        if (op == OP_OUTPUT) {
            ok = reg_ok(b1) && imm < n_outputs;
            x = enc(op, F_RR, 0xff, b1, 0xff);
        } else if (op == OP_INPUT) {
            ok = reg_ok(b1) && imm < n_vars;
            x = enc(op, F_RR, b1, 0xff, 0xff);
        } else if (op == OP_COPY) {
            if (b2 == 0xff) { ok = reg_ok(b1); x = enc(op, F_RI, b1, 0xff, 0xff); }
            else { ok = reg_ok(b1) && reg_ok(b2); x = enc(op, F_RR, b1, b2, 0xff); }
        } else if (op_is_unary(op)) {
            ok = reg_ok(b1) && reg_ok(b2);
            x = enc(op, F_RR, b1, b2, 0xff);
        } else if (op_is_binary(op)) {
            if (b2 == 0xff && b3 == 0xff) ok = false;
            else if (b2 == 0xff) { ok = reg_ok(b1) && reg_ok(b3); x = enc(op, F_IR, b1, 0xff, b3); }
            else if (b3 == 0xff) { ok = reg_ok(b1) && reg_ok(b2); x = enc(op, F_RI, b1, b2, 0xff); }
            else { ok = reg_ok(b1) && reg_ok(b2) && reg_ok(b3); x = enc(op, F_RR, b1, b2, b3); }
            if (op_is_choice(op)) {
                if (b2 == 0xff) ok = false;  // choice ops never have an immediate lhs (ssa_tape.rs:151-176)
                ++n_choices;
            }
        } else {  // OP_MEM
            if (imm >= mem_count) ok = false;
            else if (b2 == 0xff && b1 != 0xff) { ok = reg_ok(b1); x = enc(op, F_RI, b1, 0xff, 0xff); }
            else if (b1 == 0xff && b2 != 0xff) { ok = reg_ok(b2); x = enc(op, F_IR, 0xff, b2, 0xff); }
            else ok = false;
        }
        if (!ok) return fail(FC_ERR_INVALID, "bytecode: malformed clause at word " + std::to_string(i));
        out.push_back(make_uint2(x, imm));
    }
    return FC_OK;
}

static void to_bytecode(const std::vector<uint2>& cl, std::vector<uint32_t>& words) {
    words.assign({0xFFFFFFFFu, 0u});
    for (const uint2& c : cl) {
        uint32_t dop = c.x & 0xff, op = dop >> 2, form = dop & 3, out = (c.x >> 8) & 0xff, lhs = (c.x >> 16) & 0xff,
                 rhs = c.x >> 24;
        uint32_t b1 = 0xff, b2 = 0xff, b3 = 0xff;
        if (op == OP_OUTPUT) b1 = lhs;
        else if (op == OP_INPUT) b1 = out;
        else if (op == OP_COPY) { b1 = out; if (form != F_RI) b2 = lhs; }
        else if (op_is_unary(op)) { b1 = out; b2 = lhs; }
        else if (op_is_binary(op)) { b1 = out; if (form != F_IR) b2 = lhs; if (form != F_RI) b3 = rhs; }
        else { if (form == F_RI) b1 = out; else b2 = lhs; }
        words.push_back(op | b1 << 8 | b2 << 16 | b3 << 24);
        words.push_back(c.y);
    }
    words.push_back(0xFFFFFFFFu);
    words.push_back(0xFFFFFFFFu);
}

extern "C" {

const char* fc_last_error(void) { return g_err.c_str(); }
uint32_t fc_abi_version(void) { return 2; }

int32_t fc_ctx_create(int32_t device, fc_ctx** out) {
    if (!out) return fail(FC_ERR_INVALID, "null out");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(FC_ERR_NO_DEVICE, std::string("no CUDA device available (") + cudaGetErrorString(e) +
                                          "); libfidget_cuda has no CPU fallback");
    }
    if (device < 0 || device >= n) return fail(FC_ERR_INVALID, "bad device index");
    CU(cudaSetDevice(device));
    fc_ctx* c = new fc_ctx();
    c->device = device;
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    // FIDGET_B200_SM_COUNT=<n> sizes every SM-scaled grid of this context as if the device had n SMs (clamped to
    // 1 .. the real count): the launch shapes of a MIG slice or a smaller part, on the whole device.  Never more than
    // the real count, because the fused 2D tail needs all of its CTAs resident.
    c->sm_count = std::max(1, std::min(env_int("FIDGET_B200_SM_COUNT", prop.multiProcessorCount), prop.multiProcessorCount));
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code loads on compute capability 9.0 and nothing else
        delete c;
        return fail(FC_ERR_NO_DEVICE, "libfidget_cuda is built for sm_90a (H100) only; found sm_" +
                                          std::to_string(prop.major) + std::to_string(prop.minor));
    }
    CU(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&c->aux_stream, cudaStreamNonBlocking));
    for (auto& e : c->ev_fork) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    c->stream = c->own_stream;
    *out = c;
    return FC_OK;
}

void fc_ctx_destroy(fc_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->arena.release();
    for (auto& b : c->jobs) b.release();
    for (auto& b : c->fills) b.release();
    c->choice_scratch.release();
    c->counters.release();
    c->stats.release();
    c->image.release();
    c->heightmap.release();
    c->leaf_tapes.release();
    c->zsort.release();
    c->census.release();
    c->occl.release();
    c->root_list.release();
    c->mesh_leaves.release();
    c->mesh_scratch.release();
    c->mesh_verts.release();
    c->mesh_tris.release();
    c->mesh_tree.release();
    c->mesh_herm.release();
    c->mesh_cells.release();
    c->contour_leaves.release();
    c->contour_scratch.release();
    c->contour_out.release();
    c->contour_offs.release();
    c->contour_flags.release();
    c->contour_slices.release();
    c->vol_bricks.release();
    c->vol_values.release();
    c->vol_grads.release();
    c->vol_tiles.release();
    c->vol_list.release();
    c->vol_scratch.release();
    c->tile_slots.release();
    c->fx_in.release();
    c->fx_out.release();
    c->fx_tmp.release();
    c->fx_tables.release();
    c->solve_meta.release();
    c->solve_vals.release();
    c->solve_res.release();
    c->solve_work.release();
    c->frame_table.release();
    c->frame_tops.release();
    c->scene_pl.release();
    c->scene_backup.release();
    c->scene_index.release();
    c->scene_cover.release();
    c->scene_key.release();
    c->scene_colors.release();
    if (c->pass_pin) cudaFreeHost(c->pass_pin);
    if (c->copy_stream) {
        cudaStreamSynchronize(c->copy_stream);
        cudaStreamDestroy(c->copy_stream);
    }
    for (int i = 0; i < 2; ++i) {
        if (c->ev_pass[i]) cudaEventDestroy(c->ev_pass[i]);
        if (c->ev_copied[i]) cudaEventDestroy(c->ev_copied[i]);
    }
    for (auto& pb : c->tape_pool) cudaFree(pb.second);
    if (c->stage) cudaFreeHost(c->stage);
    if (c->stage_ev) cudaEventDestroy(c->stage_ev);
    for (auto ev : c->events) cudaEventDestroy(ev);
    for (auto e : c->ev_fork) if (e) cudaEventDestroy(e);
    if (c->ev_join) cudaEventDestroy(c->ev_join);
    if (c->cancel_word) cudaFree(c->cancel_word);
    if (c->cancel_pin) cudaFreeHost(c->cancel_pin);
    if (c->cancel_ev) cudaEventDestroy(c->cancel_ev);
    if (c->cancel_stream) cudaStreamDestroy(c->cancel_stream);
    cudaStreamDestroy(c->aux_stream);
    cudaStreamDestroy(c->own_stream);
    delete c;
}

int32_t fc_ctx_set_stream(fc_ctx* c, void* s, int32_t use_own) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    cudaStream_t ns = use_own ? c->own_stream : static_cast<cudaStream_t>(s);
    if (ns != c->stream) {
        cudaSetDevice(c->device);
        cudaStreamSynchronize(c->stream);   // tape uploads and scratch reuse are ordered on the context's stream
    }
    c->stream = ns;
    return FC_OK;
}

int32_t fc_ctx_set_cancel(fc_ctx* c, const uint8_t* flag) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    if (flag && !c->cancel_word) {
        std::lock_guard<std::mutex> guard(c->mu);
        CU(cudaSetDevice(c->device));
        CU(cudaStreamCreateWithFlags(&c->cancel_stream, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&c->cancel_ev, cudaEventDisableTiming));
        CU(cudaHostAlloc(reinterpret_cast<void**>(&c->cancel_pin), 4, cudaHostAllocDefault));
        uint32_t* w = nullptr;
        CU(cudaMalloc(&w, 4));
        CU(cudaMemsetAsync(w, 0, 4, c->cancel_stream));   // 0 is no call's id
        CU(cudaStreamSynchronize(c->cancel_stream));
        c->cancel_word = w;
    }
    c->cancel_flag.store(flag);
    return FC_OK;
}

}  // extern "C"

// FIDGET_B200_CANCEL_AT=<site>:<n> names the poll sites of kernels.cuh (CancelSite)
static int32_t cancel_site_of(const std::string& name) {
    static const char* const names[] = {
        "k_interval_root_coop", "k_fill_2d", "k_pixels_2d", "k_tail_2d", "k_voxels_3d", "k_normals_3d", "k_census_3d",
        "k_octree_leaf", "k_octree_grads", "k_mesh_hash", "k_mesh_vertices", "k_mesh_faces0", "k_mesh_faces1",
        "k_mesh_assign", "k_tree_parents", "k_tree_collapse", "k_tree_final", "k_tree_faces0", "k_tree_faces1"};
    static_assert(sizeof(names) / sizeof(names[0]) == CS_WAIT - CS_ROOT_COOP, "one name per poll site");
    for (int i = 0; i < MAX_LEVELS; ++i)
        if (name == "k_interval_level" + std::to_string(i)) return CS_LEVEL0 + i;
    for (int i = 0; i < CS_WAIT - CS_ROOT_COOP; ++i)
        if (name == names[i]) return CS_ROOT_COOP + i;
    static_assert(CS_SCENE2D_RESOLVE + 1 == CS_CONTOUR_LEAF, "one name per poll site");
    if (name == "k_scene2d_resolve") return CS_SCENE2D_RESOLVE;
    static const char* const contour[] = {"k_contour_leaf", "k_contour_grads", "k_contour_vertices", "k_contour_segments",
                                          "k_contour_link", "k_contour_emit"};
    static_assert(sizeof(contour) / sizeof(contour[0]) == CS_SOLVE - CS_CONTOUR_LEAF, "one name per poll site");
    for (int i = 0; i < CS_SOLVE - CS_CONTOUR_LEAF; ++i)
        if (name == contour[i]) return CS_CONTOUR_LEAF + i;
    static const char* const solve[] = {"k_solve", "k_solve_large"};
    static_assert(sizeof(solve) / sizeof(solve[0]) == CS_MEASURE_BRICK - CS_SOLVE, "one name per poll site");
    for (int i = 0; i < CS_MEASURE_BRICK - CS_SOLVE; ++i)
        if (name == solve[i]) return CS_SOLVE + i;
    static_assert(CS_VOLUME_GRADS + 1 == CS_COUNT, "one name per poll site");
    if (name == "k_measure_brick") return CS_MEASURE_BRICK;
    if (name == "k_ray_leaf") return CS_RAY_LEAF;
    if (name == "k_ray_hits") return CS_RAY_HITS;
    if (name == "k_volume_brick") return CS_VOLUME_BRICK;
    if (name == "k_volume_grads") return CS_VOLUME_GRADS;
    return -1;
}

int32_t begin_call(fc_ctx* c, CallCancel& cc) {
    cc = CallCancel{};
    const uint8_t* flag = c->cancel_flag.load();
    if (!flag) return FC_OK;
    if (__atomic_load_n(flag, __ATOMIC_ACQUIRE)) return fail(FC_ERR_CANCELLED, "cancelled before the call started");
    cc.flag = flag;
    cc.ref.word = c->cancel_word;
    {
        std::lock_guard<std::mutex> guard(c->mu);
        if (++c->call_id == 0) c->call_id = 1;
        cc.ref.id = c->call_id;
    }
    // diagnostic: the poll at <site> that claims item <n> cancels this call, as the host would
    const std::string at = env_str("FIDGET_B200_CANCEL_AT");
    if (!at.empty()) {
        const size_t colon = at.rfind(':');
        const int32_t site = colon == std::string::npos ? -1 : cancel_site_of(at.substr(0, colon));
        if (site < 0) return fail(FC_ERR_INVALID, "FIDGET_B200_CANCEL_AT: expected <kernel site>:<item>, got " + at);
        cc.ref.site = site;
        cc.ref.item = uint32_t(strtoul(at.c_str() + colon + 1, nullptr, 10));
    }
    return FC_OK;
}

int32_t wait_call(fc_ctx* c, cudaStream_t s, const CallCancel& cc) {
    if (!cc.flag) {
        CU(cudaStreamSynchronize(s));
        return FC_OK;
    }
    CU(cudaEventRecord(c->cancel_ev, s));
    bool written = false;
    for (;;) {
        const cudaError_t q = cudaEventQuery(c->cancel_ev);
        if (q == cudaSuccess) break;
        if (q != cudaErrorNotReady) return fail(FC_ERR_CUDA, std::string("cudaEventQuery: ") + cudaGetErrorString(q));
        if (!written && __atomic_load_n(cc.flag, __ATOMIC_ACQUIRE)) {
            // the kernels of this call read the word from L2 at their next claim; the copy engine runs beside them
            *c->cancel_pin = cc.ref.id;
            CU(cudaMemcpyAsync(c->cancel_word, c->cancel_pin, 4, cudaMemcpyHostToDevice, c->cancel_stream));
            written = true;
        }
        std::this_thread::yield();
    }
    CU(cudaStreamSynchronize(s));
    bool cancelled = written;
    if (written) CU(cudaStreamSynchronize(c->cancel_stream));   // (the pinned word is reused by the next call)
    else if (cc.ref.site >= 0) {                                 // FIDGET_B200_CANCEL_AT: did a poll cancel the call?
        CU(cudaMemcpyAsync(c->cancel_pin, c->cancel_word, 4, cudaMemcpyDeviceToHost, c->cancel_stream));
        CU(cudaStreamSynchronize(c->cancel_stream));
        cancelled = *c->cancel_pin == cc.ref.id;
    }
    return cancelled ? fail(FC_ERR_CANCELLED, "cancelled") : FC_OK;
}

int32_t wait_read(fc_ctx* c, cudaStream_t s, const CallCancel& cc, void* dst, const void* src, size_t bytes) {
    if (cc.flag)
        if (int32_t rc = wait_call(c, s, cc)) return rc;
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return FC_OK;
}

int32_t check_device_errors(fc_ctx* c) {
    if (!c->counters.p) return FC_OK;
    Counters h;
    CU(cudaMemcpy(&h, c->counters.p, sizeof h, cudaMemcpyDeviceToHost));
    return device_error(h.error);
}
int32_t device_error(uint32_t bits) {
    if (bits & 1u) return fail(FC_ERR_ARENA, "tape arena exhausted during on-device simplification; raise it with fc_ctx_set_arena_bytes");
    if (bits & 2u) return fail(FC_ERR_CUDA, "internal work list overflow");
    if (bits & 4u) return fail(FC_ERR_CUDA, "fused 2D kernel: a queued job never became ready (watchdog)");
    return FC_OK;
}
extern "C" {

int32_t fc_ctx_synchronize(fc_ctx* c) {
    if (!c) return fail(FC_ERR_INVALID, "null ctx");
    CU(cudaSetDevice(c->device));
    // a flag attached now applies to the last FC_FLAG_ASYNC render / sampler / mesh call still in flight
    CallCancel cc = c->async_call;
    c->async_call = CallCancel{};
    cc.flag = cc.ref.word ? c->cancel_flag.load() : nullptr;
    if (!cc.flag) cc = CallCancel{};
    if (int32_t rc = wait_call(c, c->stream, cc)) return rc;
    return check_device_errors(c);
}

int32_t fc_ctx_set_arena_bytes(fc_ctx* c, uint64_t bytes) {
    if (!c || bytes < (1u << 20)) return fail(FC_ERR_INVALID, "arena must be at least 1 MiB");
    c->arena_bytes = bytes;
    return FC_OK;
}

////////////////////////////////////////////////////////////////////////////
int32_t fc_tape_create(fc_ctx* c, const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count,
                       uint32_t n_vars, uint32_t n_outputs, uint32_t choice_count, fc_tape** out) {
    if (!c || !out) return fail(FC_ERR_INVALID, "null argument");
    if (mem_count > 2048 - MEM_BASE) return fail(FC_ERR_UNSUPPORTED, "too many memory slots (max 1792)");
    std::vector<uint2> cl;
    uint32_t nch = 0;
    int32_t rc = transcode(words, n_words, reg_count, mem_count, n_vars, n_outputs, cl, nch);
    if (rc) return rc;
    if (nch != choice_count)
        return fail(FC_ERR_INVALID, "choice_count mismatch: bytecode has " + std::to_string(nch));
    CU(cudaSetDevice(c->device));
    fc_tape* t = new fc_tape();
    t->ctx = c;
    t->host = std::move(cl);
    t->info.n_ops = uint32_t(t->host.size());
    t->info.ref_len = uint32_t(t->host.size());
    t->info.choice_count = nch;
    t->info.reg_count = reg_count;
    t->info.mem_count = mem_count;
    t->info.n_vars = n_vars;
    t->info.n_outputs = n_outputs;
    for (int k = 0; k < 3; ++k) t->ax[k] = uint32_t(k) < n_vars ? k : -1;
    const size_t need = std::max<size_t>(t->host.size(), 1) * sizeof(uint2);
    cudaError_t e = cudaSuccess;
    {
        std::lock_guard<std::mutex> g(c->mu);
        for (size_t k = 0; k < c->tape_pool.size(); ++k)
            if (c->tape_pool[k].first >= need && c->tape_pool[k].first <= 2 * need + 4096) {
                t->dev = c->tape_pool[k].second;
                t->dev_cap = c->tape_pool[k].first;
                c->tape_pool.erase(c->tape_pool.begin() + k);
                break;
            }
        if (!t->dev) {
            e = cudaMalloc(&t->dev, need);
            t->dev_cap = need;
        }
        if (e == cudaSuccess && !t->host.empty()) {
            if (!c->stage_ev) e = cudaEventCreateWithFlags(&c->stage_ev, cudaEventDisableTiming);
            else e = cudaEventSynchronize(c->stage_ev);          // the previous upload has left the staging buffer
            if (e == cudaSuccess && c->stage_cap < need) {
                if (c->stage) cudaFreeHost(c->stage);
                c->stage = nullptr;
                c->stage_cap = 0;
                e = cudaHostAlloc(&c->stage, need * 2, cudaHostAllocDefault);
                if (e == cudaSuccess) c->stage_cap = need * 2;
            }
            if (e == cudaSuccess) {
                memcpy(c->stage, t->host.data(), t->host.size() * sizeof(uint2));
                e = cudaMemcpyAsync(t->dev, c->stage, t->host.size() * sizeof(uint2), cudaMemcpyHostToDevice, c->stream);
            }
            if (e == cudaSuccess) e = cudaEventRecord(c->stage_ev, c->stream);
        }
    }
    if (e != cudaSuccess) {
        if (t->dev) cudaFree(t->dev);
        delete t;
        return fail(FC_ERR_CUDA, cudaGetErrorString(e));
    }
    upload_schedule(t);
    *out = t;
    return FC_OK;
}

int32_t fc_tape_retain(fc_tape* t) {
    if (!t) return fail(FC_ERR_INVALID, "null tape");
    t->refs.fetch_add(1);
    return FC_OK;
}
int32_t fc_tape_release(fc_tape* t) {
    if (!t) return fail(FC_ERR_INVALID, "null tape");
    if (t->refs.fetch_sub(1) == 1) {
        fc_ctx* c = t->ctx;
        cudaSetDevice(c->device);
        bool pooled = false;
        if (t->pooled_ok) {
            // reuse is ordered on the context's stream, behind whatever still reads this tape
            std::lock_guard<std::mutex> g(c->mu);
            if (c->tape_pool.size() < 8) { c->tape_pool.push_back({t->dev_cap, t->dev}); pooled = true; }
        }
        if (!pooled) cudaFree(t->dev);
        delete t;
    }
    return FC_OK;
}
int32_t fc_tape_get_info(const fc_tape* t, fc_tape_info* info) {
    if (!t || !info) return fail(FC_ERR_INVALID, "null argument");
    *info = t->info;
    return FC_OK;
}
int32_t fc_tape_read(const fc_tape* t, uint32_t* words, size_t cap, size_t* n_words) {
    if (!t) return fail(FC_ERR_INVALID, "null tape");
    std::vector<uint32_t> w;
    to_bytecode(t->host, w);
    if (n_words) *n_words = w.size();
    if (words) {
        if (cap < w.size()) return fail(FC_ERR_INVALID, "buffer too small");
        memcpy(words, w.data(), w.size() * 4);
    }
    return FC_OK;
}

int32_t fc_tape_serialize(const fc_tape* t, uint8_t* buf, size_t cap, size_t* n_bytes) {
    if (!t) return fail(FC_ERR_INVALID, "null tape");
    std::vector<uint32_t> w;
    to_bytecode(t->host, w);
    const size_t need = 4 + 6 * 4 + 3 * 4 + 8 + w.size() * 4;
    if (n_bytes) *n_bytes = need;
    if (!buf) return FC_OK;
    if (cap < need) return fail(FC_ERR_INVALID, "buffer too small");
    uint8_t* q = buf;
    auto put32 = [&](uint32_t v) { memcpy(q, &v, 4); q += 4; };
    memcpy(q, "FTAP", 4); q += 4;
    put32(1); put32(t->info.reg_count); put32(t->info.mem_count); put32(t->info.n_vars); put32(t->info.n_outputs);
    put32(t->info.choice_count);
    for (int k = 0; k < 3; ++k) put32(uint32_t(t->ax[k]));
    const uint64_t nw = w.size();
    memcpy(q, &nw, 8); q += 8;
    memcpy(q, w.data(), nw * 4);
    return FC_OK;
}
int32_t fc_tape_deserialize(fc_ctx* c, const uint8_t* buf, size_t n_bytes, fc_tape** out) {
    if (!c || !buf || !out) return fail(FC_ERR_INVALID, "null argument");
    const size_t hdr = 4 + 6 * 4 + 3 * 4 + 8;
    if (n_bytes < hdr || memcmp(buf, "FTAP", 4) != 0) return fail(FC_ERR_INVALID, "not a tape blob (bad magic)");
    uint32_t f[9];
    memcpy(f, buf + 4, sizeof f);
    if (f[0] != 1) return fail(FC_ERR_INVALID, "unsupported tape blob version " + std::to_string(f[0]));
    uint64_t nw;
    memcpy(&nw, buf + 4 + 9 * 4, 8);
    if (nw > (n_bytes - hdr) / 4) return fail(FC_ERR_INVALID, "truncated tape blob");
    if (f[1] > 255) return fail(FC_ERR_INVALID, "bad register count");
    std::vector<uint32_t> words(nw);
    memcpy(words.data(), buf + hdr, nw * 4);
    fc_tape* t = nullptr;
    int32_t rc = fc_tape_create(c, words.data(), words.size(), uint8_t(f[1]), f[2], f[3], f[4], f[5], &t);
    if (rc) return rc;
    rc = fc_tape_set_axes(t, int32_t(f[6]), int32_t(f[7]), int32_t(f[8]));
    if (rc) { fc_tape_release(t); return rc; }
    *out = t;
    return FC_OK;
}

////////////////////////////////////////////////////////////////////////////
int32_t fc_eval_create(fc_ctx* c, fc_eval** out) {
    if (!c || !out) return fail(FC_ERR_INVALID, "null argument");
    fc_eval* e = new fc_eval();
    e->ctx = c;
    *out = e;
    return FC_OK;
}
void fc_eval_destroy(fc_eval* e) {
    if (!e) return;
    cudaSetDevice(e->ctx->device);
    cudaStreamSynchronize(e->ctx->stream);
    e->in.release(); e->out.release(); e->choices.release(); e->simplify.release(); e->ptrs.release(); e->tmp.release();
    delete e;
}

}  // extern "C"

// Staging shared by the tracing batch calls (interpreted and compiled): host buffers go through the evaluator's
// device buffers, results come back, and the call ends with a synchronise; `launch` enqueues the kernel
int32_t tracing_eval(fc_eval* e, const fc_tape* t, const float* vars, uint64_t n, float* out, uint8_t* choices,
                     uint8_t* simplify, bool interval, const std::function<int32_t(TracingParams&)>& launch) {
    if (!e || !t || (!vars && t->info.n_vars) || !out) return fail(FC_ERR_INVALID, "null argument");
    fc_ctx* c = e->ctx;
    CU(cudaSetDevice(c->device));
    const size_t w = interval ? 2 : 1;
    const size_t in_bytes = n * t->info.n_vars * w * 4, out_bytes = n * t->info.n_outputs * w * 4;
    const size_t ch_bytes = n * t->info.choice_count;
    TracingParams p{};
    p.tape = t->dev;
    p.n_ops = t->info.n_ops;
    p.n_vars = t->info.n_vars;
    p.n_outputs = t->info.n_outputs;
    p.n_choices = t->info.choice_count;
    p.n_slots = MEM_BASE + t->info.mem_count;
    p.n = n;
    const bool dv = is_device_ptr(vars), dout = is_device_ptr(out), dch = is_device_ptr(choices),
               dsi = is_device_ptr(simplify);
    if (dv || !in_bytes) p.vars = vars;
    else {
        CU(e->in.ensure(in_bytes));
        CU(cudaMemcpyAsync(e->in.p, vars, in_bytes, cudaMemcpyHostToDevice, c->stream));
        p.vars = e->in.as<float>();
    }
    if (dout) p.out = out; else { CU(e->out.ensure(std::max<size_t>(out_bytes, 4))); p.out = e->out.as<float>(); }
    if (choices && ch_bytes) {
        if (dch) p.choices = choices; else { CU(e->choices.ensure(ch_bytes)); p.choices = e->choices.as<uint8_t>(); }
    }
    if (simplify) {
        if (dsi) p.simplify = simplify; else { CU(e->simplify.ensure(n)); p.simplify = e->simplify.as<uint8_t>(); }
    }
    if (int32_t rc = launch(p)) return rc;
    CU(cudaGetLastError());
    if (!dout && out_bytes) CU(cudaMemcpyAsync(out, p.out, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    if (choices && ch_bytes && !dch) CU(cudaMemcpyAsync(choices, p.choices, ch_bytes, cudaMemcpyDeviceToHost, c->stream));
    if (simplify && !dsi) CU(cudaMemcpyAsync(simplify, p.simplify, n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

static int32_t interpret_interval(fc_eval* e, TracingParams& p) {
    launch_interval_batch(p, e->ctx->stream);
    return FC_OK;
}

extern "C" {

int32_t fc_interval_eval(fc_eval* e, const fc_tape* t, const float* vars, float* out, uint8_t* choices, uint8_t* simplify) {
    return tracing_eval(e, t, vars, 1, out, choices, simplify, true, [&](TracingParams& p) { return interpret_interval(e, p); });
}
int32_t fc_point_eval(fc_eval* e, const fc_tape* t, const float* vars, float* out, uint8_t* choices, uint8_t* simplify) {
    return tracing_eval(e, t, vars, 1, out, choices, simplify, false, [&](TracingParams& p) {
        launch_point_batch(p, e->ctx->stream);
        return FC_OK;
    });
}
int32_t fc_interval_eval_batch(fc_eval* e, const fc_tape* t, const float* vars, uint64_t n, float* out, uint8_t* choices,
                               uint8_t* simplify) {
    return tracing_eval(e, t, vars, n, out, choices, simplify, true, [&](TracingParams& p) { return interpret_interval(e, p); });
}

}  // extern "C"

// The interpreters' launch: the TMA-fed kernel when the tape and the buffers fit it, else the per-thread kernel
static int32_t interpret_slice(fc_eval* e, const fc_tape* t, BulkParams& p, const std::vector<const void*>& dptr, bool grad) {
    fc_ctx* c = e->ctx;
    const uint32_t nv = p.n_vars, no = p.n_outputs;
    const uint64_t n = p.n;
    unsigned tma_ctas = 0;
    if (!t->info.mem_count && n >= 4096 && nv <= 4 && no <= 2 && !env_int("FIDGET_B200_NO_TMA", 0)) {
        SliceTmaParams q{};
        q.tape = t->dev;
        q.n_ops = t->info.n_ops;
        q.n_vars = nv;
        q.n_outputs = no;
        q.n_regs = t->info.reg_count;
        q.n = n;
        for (uint32_t i = 0; i < nv; ++i) q.vars[i] = static_cast<const float4*>(dptr[i]);
        for (uint32_t o = 0; o < no; ++o) q.outs[o] = static_cast<float4*>(const_cast<void*>(dptr[nv + o]));
        tma_ctas = launch_slice_tma(q, grad, c->sm_count, c->stream);
    }
    if (!tma_ctas) { if (grad) launch_grad_slice(p, c->stream); else launch_float_slice(p, c->stream); }
    if (env_int("FIDGET_B200_SLICE_DEBUG", 0)) {   // which kernel ran, and how many tiles each TMA CTA had to cycle
        const uint64_t tile = uint64_t(SLICE_TMA_TILE) * (grad ? 1 : 4);
        if (tma_ctas)
            fprintf(stderr, "slice: TMA kernel, %llu points, %llu full tiles, %u CTAs, %d SMs\n", (unsigned long long)n,
                    (unsigned long long)(n / tile), tma_ctas, c->sm_count);
        else
            fprintf(stderr, "slice: per-thread kernel, %llu points\n", (unsigned long long)n);
    }
    return FC_OK;
}

// Staging shared by the slice calls (interpreted and compiled), as tracing_eval's
int32_t bulk_eval(fc_eval* e, const fc_tape* t, const void* const* vars, void* const* outs, uint64_t n, size_t elem,
                  const std::function<int32_t(BulkParams&, const std::vector<const void*>&)>& launch) {
    if (!e || !t || (!vars && t->info.n_vars) || !outs) return fail(FC_ERR_INVALID, "null argument");
    fc_ctx* c = e->ctx;
    CU(cudaSetDevice(c->device));
    const uint32_t nv = t->info.n_vars, no = t->info.n_outputs;
    std::vector<const void*> dptr(nv + no);
    // stage host inputs / outputs in the evaluator's buffers
    size_t in_need = 0, out_need = 0;
    for (uint32_t i = 0; i < nv; ++i) if (!is_device_ptr(vars[i])) in_need += n * elem;
    for (uint32_t o = 0; o < no; ++o) if (!is_device_ptr(outs[o])) out_need += n * elem;
    CU(e->in.ensure(std::max<size_t>(in_need, 16)));
    CU(e->out.ensure(std::max<size_t>(out_need, 16)));
    size_t io = 0, oo = 0;
    std::vector<std::pair<void*, void*>> copy_back;
    for (uint32_t i = 0; i < nv; ++i) {
        if (is_device_ptr(vars[i])) dptr[i] = vars[i];
        else {
            char* d = e->in.as<char>() + io;
            if (n) CU(cudaMemcpyAsync(d, vars[i], n * elem, cudaMemcpyHostToDevice, c->stream));
            dptr[i] = d;
            io += n * elem;
        }
    }
    for (uint32_t o = 0; o < no; ++o) {
        if (is_device_ptr(outs[o])) dptr[nv + o] = outs[o];
        else {
            char* d = e->out.as<char>() + oo;
            dptr[nv + o] = d;
            copy_back.push_back({outs[o], d});
            oo += n * elem;
        }
    }
    CU(e->ptrs.ensure(std::max<size_t>(dptr.size(), 1) * sizeof(void*)));
    if (!dptr.empty())
        CU(cudaMemcpyAsync(e->ptrs.p, dptr.data(), dptr.size() * sizeof(void*), cudaMemcpyHostToDevice, c->stream));
    BulkParams p{};
    p.tape = t->dev;
    p.n_ops = t->info.n_ops;
    p.n_vars = nv;
    p.n_outputs = no;
    p.n_slots = MEM_BASE + t->info.mem_count;
    p.n = n;
    p.vars = e->ptrs.as<const void*>();
    p.outs = reinterpret_cast<void* const*>(e->ptrs.as<void*>() + nv);
    if (int32_t rc = launch(p, dptr)) return rc;
    CU(cudaGetLastError());
    for (auto& cb : copy_back)
        if (n) CU(cudaMemcpyAsync(cb.first, cb.second, n * elem, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FC_OK;
}

extern "C" {

int32_t fc_float_slice_eval(fc_eval* e, const fc_tape* t, const float* const* vars, float* const* out, uint64_t n) {
    return bulk_eval(e, t, reinterpret_cast<const void* const*>(vars), reinterpret_cast<void* const*>(out), n, 4,
                     [&](BulkParams& p, const std::vector<const void*>& dptr) { return interpret_slice(e, t, p, dptr, false); });
}
int32_t fc_grad_slice_eval(fc_eval* e, const fc_tape* t, const fc_grad* const* vars, fc_grad* const* out, uint64_t n) {
    return bulk_eval(e, t, reinterpret_cast<const void* const*>(vars), reinterpret_cast<void* const*>(out), n, 16,
                     [&](BulkParams& p, const std::vector<const void*>& dptr) { return interpret_slice(e, t, p, dptr, true); });
}

int32_t fc_simplify(fc_eval* e, const fc_tape* parent, const uint8_t* choices, size_t n_choices, fc_tape** child) {
    if (!e || !parent || !child || (!choices && n_choices)) return fail(FC_ERR_INVALID, "null argument");
    if (n_choices != parent->info.choice_count)
        return fail(FC_ERR_INVALID, "choice slice length (" + std::to_string(n_choices) + ") does not match choice count (" +
                                        std::to_string(parent->info.choice_count) + ")");
    if (parent->info.mem_count) return fail(FC_ERR_UNSUPPORTED, "fc_simplify: parent tape uses memory slots");
    for (size_t i = 0; i < n_choices; ++i)
        if (choices[i] < 1 || choices[i] > 3) return fail(FC_ERR_INVALID, "trace contains Choice::Unknown");
    fc_ctx* c = e->ctx;
    CU(cudaSetDevice(c->device));
    const uint32_t n = parent->info.n_ops;
    CU(e->tmp.ensure(std::max<size_t>(n, 1) * sizeof(uint2) + 16));
    CU(e->choices.ensure(std::max<size_t>(n_choices, 1)));
    if (n_choices) CU(cudaMemcpyAsync(e->choices.p, choices, n_choices, cudaMemcpyHostToDevice, c->stream));
    SimplifyParams p{};
    p.parent = parent->dev;
    p.n_ops = n;
    p.parent_ref_len = parent->info.ref_len;
    p.choices = e->choices.as<uint8_t>();
    p.n_choices = uint32_t(n_choices);
    p.out = e->tmp.as<uint2>();
    p.result = reinterpret_cast<uint32_t*>(e->tmp.as<char>() + size_t(n) * sizeof(uint2));
    launch_simplify_single(p, c->stream);
    CU(cudaGetLastError());
    uint32_t res[3];
    CU(cudaMemcpyAsync(res, p.result, sizeof res, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    fc_tape* t = new fc_tape();
    t->ctx = c;
    t->info = parent->info;
    memcpy(t->ax, parent->ax, sizeof t->ax);
    t->info.n_ops = res[0];
    t->info.ref_len = res[1];
    t->info.choice_count = res[2];
    t->host.resize(res[0]);
    t->dev_cap = std::max<size_t>(res[0], 1) * sizeof(uint2);
    cudaError_t err = cudaMalloc(&t->dev, t->dev_cap);
    if (err == cudaSuccess && res[0]) {
        err = cudaMemcpy(t->dev, p.out + (n - res[0]), res[0] * sizeof(uint2), cudaMemcpyDeviceToDevice);
        if (err == cudaSuccess) err = cudaMemcpy(t->host.data(), t->dev, res[0] * sizeof(uint2), cudaMemcpyDeviceToHost);
    }
    if (err != cudaSuccess) {
        if (t->dev) cudaFree(t->dev);
        delete t;
        return fail(FC_ERR_CUDA, cudaGetErrorString(err));
    }
    *child = t;
    return FC_OK;
}

// Binds tape input slots to the X, Y, Z axes (ShapeTape::vars(),
// shape/mod.rs:355-376); -1 = axis unused.
int32_t fc_tape_set_axes(fc_tape* t, int32_t x, int32_t y, int32_t z) {
    if (!t) return fail(FC_ERR_INVALID, "null tape");
    int nv = int(t->info.n_vars);
    if (x >= nv || y >= nv || z >= nv) return fail(FC_ERR_INVALID, "axis slot out of range");
    t->ax[0] = x; t->ax[1] = y; t->ax[2] = z;
    return FC_OK;
}

}  // extern "C"
