// Internal declarations shared by the host-side sources of libfidget_cuda (include/fidget_cuda.h):
// error reporting, device buffers, the context / tape / evaluator objects and the helpers that more
// than one translation unit uses.
#pragma once
#include <algorithm>
#include <atomic>
#include <memory>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "../../../include/fidget_cuda.h"
#include "env.h"
#include "kernels.cuh"
#include "effects.cuh"

using namespace fdev;

extern thread_local std::string g_err;   // defined in capi.cu
inline int32_t fail(int32_t code, const std::string& msg) {
    g_err = msg;
    return code;
}
#define CU(call)                                                                          \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess)                                                            \
            return fail(FC_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T> T* as() { return static_cast<T*>(p); }
};

// Consecutive 256-byte-aligned arrays of one device buffer: take() points each at its place
struct Carve {
    char* base;
    size_t used = 0;
    template <class T> void take(T*& p, size_t bytes) {
        p = base ? reinterpret_cast<T*>(base + used) : nullptr;
        used += (bytes + 255) & ~size_t(255);
    }
};
// Grows `buf` to the arrays lay_out(Carve&) takes, then points them into it
template <class F> cudaError_t carve(DevBuf& buf, F lay_out) {
    Carve size{nullptr};
    lay_out(size);
    if (cudaError_t e = buf.ensure(size.used)) return e;
    Carve at{buf.as<char>()};
    lay_out(at);
    return cudaSuccess;
}

inline bool is_device_ptr(const void* p) {
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Pinned (page-locked, mapped) host memory can be written by kernels directly over PCIe.
// Scattered SM stores over PCIe move an image more slowly than one DMA copy of it, so this is opt-in
// (FIDGET_B200_ZEROCOPY=1); the default stages the image in HBM and copies it with the DMA engine.
// Returns the device alias of `p` or null.
inline void* pinned_device_alias(const void* p) {
    if (!p) return nullptr;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return a.type == cudaMemoryTypeHost ? a.devicePointer : nullptr;
}

// Cancellation of one call (fc_ctx_set_cancel): the flag attached when the call began and the device side's view
// (ref.word == null when no flag is attached)
struct CallCancel {
    const uint8_t* flag = nullptr;
    CancelRef ref{nullptr, 0, -1, 0};
};

struct fc_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t aux_stream = nullptr;        // fills are painted here, concurrently with the next levels
    cudaEvent_t ev_fork[MAX_LEVELS] = {}, ev_join = nullptr;
    uint64_t arena_bytes = 1ull << 30;
    uint32_t epoch = 0;                       // ready mark of the current render's job / fill records
    // render scratch
    DevBuf arena, jobs[MAX_LEVELS + 1], fills[MAX_LEVELS], choice_scratch, counters, stats, image, heightmap, leaf_tapes, zsort, census, occl;
    DevBuf mesh_leaves, mesh_scratch, mesh_verts, mesh_tris;   // fc_mesh_build: sampler output and the mesh, resident in HBM
    uint32_t mesh_n_verts = 0, mesh_n_tris = 0;
    DevBuf mesh_tree, mesh_herm, mesh_cells;                    // FC_FLAG_MESH_COLLAPSE: cell tree, Hermite records, final leaves
    uint32_t mesh_n_cells = 0;
    // fc_mesh_build_frames: a pass's frame table, and each frame's first vertex and triangle in the mesh (uint2 per frame,
    // for fc_mesh_write_stl; unused with one frame).  No mesh is one frame of nothing.
    DevBuf mesh_frames, mesh_ranges;
    uint32_t mesh_n_frames = 1;
    DevBuf contour_leaves, contour_scratch, contour_out;        // fc_contour_build: sampler output, link scratch, vertices
    DevBuf contour_offs, contour_flags, contour_slices;         // offsets, closed flags, a stack pass's slice table
    uint32_t contour_n_verts = 0, contour_n_polys = 0;
    uint32_t* contour_offsets = nullptr;                        // in contour_offs
    uint8_t* contour_closed = nullptr;                          // in contour_flags
    // fc_volume_build: the volume, resident in HBM until read (brick records, values, gradients, tile records), a pass's
    // tile list and sort scratch; the counts of the volume (0: none) and its values per brick
    DevBuf vol_bricks, vol_values, vol_grads, vol_tiles, vol_list, vol_scratch;
    uint64_t vol_n_bricks = 0, vol_n_tiles = 0;
    uint32_t vol_cells = 0;
    bool vol_grads_on = false;
    DevBuf fx_in, fx_out, fx_tmp, fx_tables;  // effects: staged host images, intermediate maps, SSAO tables
    DevBuf solve_meta, solve_vals, solve_res; // the solvers: tape table + slot maps, staged host values / results
    DevBuf solve_work;                        // fc_solve_large_batch: one workspace slice per cluster in flight
    // the batches (fc_render2d_frames, fc_render3d_frames, fc_render3d_scene): the frame or placement table, and the copy
    // stream that returns a frame batch's pass to a host `out` while the next pass runs (ev_pass: the pass in staging
    // buffer b is complete; ev_copied: copied back).  fc_render2d_frames: each pass's arena high-water mark.
    DevBuf frame_table, frame_tops;
    // the 3D batches: each in-flight pass's counters and stats (two pinned host slots, one per staging buffer; a scene
    // waits for every pass and uses the first)
    struct PassStatus* pass_pin = nullptr;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_pass[2] = {}, ev_copied[2] = {};
    // fc_render3d_scene: each pass's placements grouped by tape, the heightmap and occlusion map as they were before a
    // pass of several placements (restored when it overflows), and the staged index image of a host `index`
    DevBuf scene_pl, scene_backup, scene_index;
    // fc_render2d_scene: the cover maps (read, write), the pixel key map and the colour table (kernels.cuh, Scene2D)
    DevBuf scene_cover, scene_key, scene_colors;
    // tile interleave: device list of this rank's XY root tiles (cached on its key), and the
    // tile -> gathered-slot table of fc_tiles_unpack
    DevBuf root_list, tile_slots;
    uint32_t root_list_key[5] = {0, 0, 0, 0, 0}, root_list_n = 0;
    uint32_t tile_slots_key[4] = {0, 0, 0, 0};
    std::vector<cudaEvent_t> events;
    std::mutex mu;
    // tape uploads: released device buffers are reused (no cudaMalloc / cudaFree per tape) and the
    // clauses go through a pinned staging buffer with a stream-ordered copy (no host synchronisation)
    std::vector<std::pair<size_t, uint2*>> tape_pool;
    void* stage = nullptr;
    size_t stage_cap = 0;
    cudaEvent_t stage_ev = nullptr;
    // level-0 launch shape (occupancy query cached) per instantiation: 2D, 2D frame batch, 2D scene, 3D, 3D frame batch,
    // 3D scene
    struct { size_t smem; int per_sm, threads; } coop_memo[6] = {};
    std::shared_ptr<struct Sched> sched_cache[4];
    unsigned sched_next = 0;
    // cancellation (fc_ctx_set_cancel): the caller's flag; the device word kernels poll, written from pinned memory on
    // a non-blocking side stream while the work stream runs; ids of the calls, so that a late write cancels nothing newer
    std::atomic<const uint8_t*> cancel_flag{nullptr};
    uint32_t* cancel_word = nullptr;
    uint32_t* cancel_pin = nullptr;
    cudaStream_t cancel_stream = nullptr;
    cudaEvent_t cancel_ev = nullptr;
    uint32_t call_id = 0;
    CallCancel async_call;                    // the last FC_FLAG_ASYNC call that returned before its work was done
};

// What the host reads of a finished pass of fc_render3d_frames or fc_render3d_scene: its counters (error bits, list and
// arena use) and stats
struct PassStatus {
    Counters ctr;
    Stats st;
};

struct fc_tape {
    fc_ctx* ctx = nullptr;
    std::atomic<int> refs{1};
    uint2* dev = nullptr;
    size_t dev_cap = 0;       // bytes behind `dev` (a pooled buffer may be larger than the tape)
    bool pooled_ok = true;    // false for tapes whose buffer is not a plain cudaMalloc of their own
    std::vector<uint2> host;  // copy of the device clauses
    fc_tape_info info{};
    int ax[3] = {-1, -1, -1};  // input slots of X, Y, Z
    // cooperative level-0 schedule (null when the tape is unsuitable); shared between tapes
    // created from identical bytecode (re-uploading an unchanged shape every frame is the
    // common interactive pattern)
    std::shared_ptr<struct Sched> sched;
};

// A tape as the kernels take it, its choice scratch words per lane (LevelParams::choice_words) and the arena a launch
// may fill, in clauses
inline TapeRef tape_ref(const fc_tape* t) { return TapeRef{t->dev, t->info.n_ops, t->info.ref_len, t->info.choice_count}; }
inline uint32_t choice_words(const fc_tape* t) { return (t->info.choice_count + 15) / 16 + 1; }
inline uint64_t arena_clauses(const fc_ctx* c) { return std::min<uint64_t>(c->arena.cap, c->arena_bytes) / sizeof(uint2); }
// Work lists hold only ambiguous tiles (a surface-like set), so they are capped well below the N^3 tile count
// (FIDGET_B200_MAX_TILES_M, 16 Mi jobs); overflow is reported, not ignored
inline uint64_t list_cap_limit() { return uint64_t(env_int("FIDGET_B200_MAX_TILES_M", 16)) << 20; }

struct Sched {
    int device = 0;
    uint64_t hash = 0;
    std::vector<uint2> clauses;
    CoopRec* d_recs = nullptr;
    CoopFwd* d_fwd = nullptr;
    uint32_t* d_wave_start = nullptr;
    uint32_t n_waves = 0, tail_begin = 0, tail_end = 0, n_slots = 0;
    std::vector<CoopSeg> segs;
    ~Sched() {
        cudaSetDevice(device);
        if (d_recs) cudaFree(d_recs);
        if (d_fwd) cudaFree(d_fwd);
        if (d_wave_start) cudaFree(d_wave_start);
    }
};
struct fc_eval {
    fc_ctx* ctx = nullptr;
    DevBuf in, out, choices, simplify, ptrs, tmp;
};

// schedule.cu
void upload_schedule(fc_tape* t);
int coop_blocks(fc_ctx* c, const fc_tape* tape, uint64_t n_roots, LevelParams& p, int dim, int& threads);
// capi.cu
int32_t check_device_errors(fc_ctx* c);
// the error of a render's Counters::error bits (FC_OK for none)
int32_t device_error(uint32_t bits);
// Start of a cancellable call: FC_ERR_CANCELLED if the attached flag is already set, else `cc` for its kernels
int32_t begin_call(fc_ctx* c, CallCancel& cc);
// cudaStreamSynchronize(s) of a cancellable call.  With a flag attached it polls the work and the flag, writes the
// cancel word once it sees the flag, drains the stream and returns FC_ERR_CANCELLED if the call was cancelled.
int32_t wait_call(fc_ctx* c, cudaStream_t s, const CallCancel& cc);
// The readback of device counters that ends a wait: a copy to pageable memory would block the host until the stream
// drains, so with a flag attached the (cancellable) wait comes first
int32_t wait_read(fc_ctx* c, cudaStream_t s, const CallCancel& cc, void* dst, const void* src, size_t bytes);
// The batch evaluators' staging of host / device inputs and outputs around one kernel launch (`launch`), shared by the
// interpreted calls and the compiled ones (compile.cu); both end with a synchronise of the context's stream
int32_t tracing_eval(fc_eval* e, const fc_tape* t, const float* vars, uint64_t n, float* out, uint8_t* choices,
                     uint8_t* simplify, bool interval, const std::function<int32_t(TracingParams&)>& launch);
int32_t bulk_eval(fc_eval* e, const fc_tape* t, const void* const* vars, void* const* outs, uint64_t n, size_t elem,
                  const std::function<int32_t(BulkParams&, const std::vector<const void*>&)>& launch);
int32_t transcode(const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count, uint32_t n_vars,
                  uint32_t n_outputs, std::vector<uint2>& out, uint32_t& n_choices);
// octree_capi.cu
// The refusals every uniform-tree call (octree sample, mesh frames, contours, fc_measure) makes before it begins, locks
// or allocates: a depth above the tree's limit (FC_MAX_OCTREE_DEPTH for dim 3, FC_MAX_QUADTREE_DEPTH for 2), a null
// `table` of n > 0 frames or slices, more than FC_MAX_VARS values in one, a tape with memory slots (`what` names the
// caller), a multi-output tape.  F: fc_mesh_frame or fc_contour_slice (fc_raycast: its cfg, depth 0).
template <class F>
int32_t check_tree_call(const fc_tape* tape, int dim, uint32_t depth, const F* table, uint32_t n, const char* what);
// A frame or slice as the tree kernels take it, its vars bound (bind_vars' refusals).  to_model: map the vertices back
// through world_to_model (row-major 4x4) unless it is the identity, as Octree::build does (octree.rs:58-65).  The
// kernels read the matrix only with has_transform.
int32_t bind_frame(const fc_tape* tape, uint32_t has_transform, const float* world_to_model, float z, const float* values,
                   uint32_t n_values, MeshFrame& f);
// Level l's job list over n root cells of 2^dim children per level: every cell at depth min(l, D), at most `limit`
inline uint64_t tree_list(uint64_t n, int dim, uint32_t D, int l, uint64_t limit) {
    return std::min(n << (dim * std::min(l, int(D))), limit);
}
// The passes of a batch of n frames or slices (pass_plan.h), at most n_max each: the job lists of levels 1 .. `levels`
// as tree_scratch sizes them, and with leaf_bytes > 0 the surface leaves within FC_FRAMES_PASS_BYTES
struct PassPlan;
PassPlan tree_passes(fc_ctx* c, uint32_t n, uint32_t n_max, uint32_t D, int dim, int levels, double leaf_bytes);
// The uniform-tree samplers (octree_enqueue, contour_sample) over n_roots root cells stacked along Y (one per frame or
// slice), each with 2^dim children per level down to depth D: their scratch (choice scratch, arena, counters with 64
// zeroed bytes after them, stats, the job lists, `cap` leaf tapes), the LevelParams every level of both shares, and the
// size of each level's launch
struct TreeScratch {
    uint32_t D = 0;
    int dim = 0;
    uint64_t n_roots = 0;
    int grid_blocks = 0;
    uint32_t choice_words = 0;
    uint64_t level_cap[MAX_LEVELS + 1] = {};   // level l's job list: the cells at depth min(l, D), capped
    // blocks of level l's launch, within the grid: a warp per parent cell, or per 32 root cells at level 0
    int blocks(int l) const {
        const uint64_t warps = l ? std::max<uint64_t>(1, (n_roots << (dim * l)) >> dim) : (n_roots + 31) / 32;
        return std::max(int(std::min<uint64_t>((warps + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, uint64_t(grid_blocks))), 1);
    }
};
int32_t tree_scratch(fc_ctx* c, const fc_tape* tape, uint32_t D, int dim, uint64_t n_roots, uint64_t cap, TreeScratch& t);
// level l's launch parameters, with the matrix, transform flag and vars of the first frame or slice, f0
LevelParams tree_level(fc_ctx* c, const fc_tape* tape, const TreeScratch& t, int l, const ContourSlice& f0,
                       const CallCancel& cc);
int32_t octree_enqueue(fc_ctx* c, const fc_tape* tape, uint32_t D, const MeshFrame* fr, uint32_t n, const MeshFrame* d_fr,
                       OctreeLeaf* dout, uint64_t cap, bool stats, cudaEvent_t t0, const CallCancel& cc, uint32_t* launches);
// contour.cu
// Grows `b` to at least `need` bytes, keeping its first `keep` bytes (the output of a batch's earlier passes)
int32_t grow_keep(fc_ctx* c, DevBuf& b, size_t need, size_t keep);
// render.cu
int32_t pick_tile_sizes(const uint32_t* ts_in, uint32_t n_in, const uint32_t* dflt, uint32_t n_dflt, uint32_t max_size,
                        std::vector<uint32_t>& ts);
int32_t bind_vars(const fc_tape* t, const float* values, uint32_t n_values, VarBind& vb);
cudaEvent_t get_event(fc_ctx* c, size_t i);
int32_t root_subset(fc_ctx* c, uint32_t roots_x, uint32_t row0, uint32_t row1, uint32_t stride, uint32_t offset,
                    cudaStream_t s, const uint32_t** d_list, uint32_t* n);
