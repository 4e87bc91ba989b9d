// Kernel-side data structures shared between kernels.cu and capi.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dev_ops.cuh"

namespace fdev {

constexpr int MAX_LEVELS = 16;             // 3D renders use <= 8; the octree sampler uses depth + 1
constexpr int WARPS_PER_BLOCK = 4;          // interval kernels
constexpr int REG_SLOTS = 256;              // register slots of the fast interpreters

// Cancellation (fc_ctx_set_cancel).  The context owns one device word; the host writes the id of a cancelled call into
// it from a side stream while the call's kernels run.  Kernels poll it where a warp or CTA is about to claim new work
// (cancel_poll) and stop claiming once it equals their own call's id; a claimed job always runs to its end, so every
// record a producer has reserved is written.  word == null: no flag attached, the poll is one uniform predicate.
// Poll sites, for the FIDGET_B200_CANCEL_AT diagnostic (the poll at `site` that claims item `item` cancels the call
// itself, as the host would); the host maps their names (cancel_site_of, capi.cu) to these ids.
enum CancelSite : int32_t {
    CS_LEVEL0 = 0,                                        // k_interval_level, level l = CS_LEVEL0 + l (< MAX_LEVELS)
    CS_ROOT_COOP = 16, CS_FILL_2D, CS_PIXELS_2D, CS_TAIL_2D, CS_VOXELS_3D, CS_NORMALS_3D, CS_CENSUS_3D,
    CS_OCTREE_LEAF, CS_OCTREE_GRADS,
    CS_MESH_HASH, CS_MESH_VERTICES, CS_MESH_FACES0, CS_MESH_FACES1, CS_MESH_ASSIGN,
    CS_TREE_PARENTS, CS_TREE_COLLAPSE, CS_TREE_FINAL, CS_TREE_FACES0, CS_TREE_FACES1,
    CS_WAIT,                                              // polls inside spin waits: not a claim, never a trigger site
    CS_SCENE2D_RESOLVE,                                   // (after CS_WAIT: the ids the kernels above compare stay put)
    CS_CONTOUR_LEAF, CS_CONTOUR_GRADS, CS_CONTOUR_VERTICES, CS_CONTOUR_SEGMENTS, CS_CONTOUR_LINK, CS_CONTOUR_EMIT,
    CS_SOLVE, CS_SOLVE_LARGE,                             // the solvers: item = problem index (claim and every iteration)
    CS_MEASURE_BRICK,                                     // fc_measure's brick kernel: item = brick
    CS_RAY_LEAF, CS_RAY_HITS,                             // fc_raycast's leaf (item = segment) and hit (item = warp) kernels
    CS_VOLUME_BRICK, CS_VOLUME_GRADS,                     // fc_volume_build's brick and gradient kernels: item = brick
    CS_COUNT
};
struct CancelRef {
    uint32_t* word;       // the context's cancel word, or null
    uint32_t id;          // this call's id (never 0)
    int32_t site;         // FIDGET_B200_CANCEL_AT: poll site that cancels (-1: none) ...
    uint32_t item;        // ... when it claims this item
};
#ifdef __CUDACC__
// true when the call is cancelled; `item` is the job / record / block being claimed (0xffffffff: not a claim)
__device__ __forceinline__ bool cancel_poll(const CancelRef& c, int32_t site, uint32_t item) {
    if (!c.word) return false;
    if (site == c.site && item == c.item) { atomicExch(c.word, c.id); return true; }
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(c.word) : "memory");
    return v == c.id;
}
#endif

// A tape living in the device arena (units of uint2 clauses)
struct TapeRef {
    const uint2* ptr;     // first clause (device memory: a root tape buffer or the arena)
    uint32_t n_ops;       // device clauses
    uint32_t ref_len;     // RegTape::len() of the reference's equivalent tape
    uint32_t n_choices;   // choice clauses (== reference choice_count)
    uint32_t pad;
};

// One tile that survived the previous level ("ambiguous"), plus the tape its
// children are evaluated with.
struct TileJob {
    uint32_t x, y, z;     // corner in pixels/voxels
    uint32_t pad;
    TapeRef tape;
};  // 40 bytes

struct FillRec { uint32_t x, y, value, ready; };  // 2D fill: corner + RawDistancePixel bits + this render's ready mark

// One interval-evaluated 3D tile, recorded for the exact census (FC_FLAG_EXACT_CENSUS): the reference visits
// tiles front to back and skips those whose pixels are all finished (voxel.rs:283-293); which tiles that
// are is decided afterwards from the final heightmap (k_census_3d)
struct CensusRec { uint16_t x, y, z; uint8_t level, flags; };   // flags: 0 outside, 1 inside, 2 ambiguous; | 4 simplified tape kept

struct Stats {
    unsigned long long evaluated[MAX_LEVELS];
    unsigned long long filled_inside[MAX_LEVELS];
    unsigned long long filled_outside[MAX_LEVELS];
    unsigned long long ambiguous[MAX_LEVELS];
    unsigned long long simplified[MAX_LEVELS];
    unsigned long long pixels;
    unsigned long long grads;
    unsigned long long culled[MAX_LEVELS];
};

// Device-side counters of one render call.  The words that every warp of a launch bumps (the next level's list
// length, the fill count, the arena top, a shared cursor) sit in different 128-byte lines, so that their atomics queue
// at different L2 slices instead of one; the host resets and reads the struct as a whole.
struct Counters {
    alignas(128) uint32_t n_jobs[MAX_LEVELS + 1];   // n_jobs[l] = tiles queued FOR level l (parents whose children are evaluated at l)
    alignas(128) uint32_t n_fills[MAX_LEVELS];      // 2D fill records produced by level l
    alignas(128) uint32_t cursor[MAX_LEVELS + 2];   // dynamic work cursors (one per kernel)
    alignas(128) uint32_t error;       // bit 0: arena exhausted, bit 1: list overflow, bit 2: fused kernel watchdog
    uint32_t outstanding;              // fused 2D kernel: interval / pixel jobs queued or running
    uint32_t fill_cursor[MAX_LEVELS];  // fused 2D kernel: fill records painted so far, per level
    uint32_t n_census;                 // exact 3D census: records appended
    uint32_t pad;
    alignas(128) unsigned long long arena_top;      // bump pointer (clauses)
};

// Cooperative level-0 schedule (built on the host at fc_tape_create): the root
// tape in SSA form (value id = position of the defining clause), clauses
// grouped into dependency waves; a trailing run of single-clause waves is the
// serial tail.
constexpr int COOP_THREADS = 256;
constexpr uint32_t COOP_NONE = 0xFFFFu;
struct CoopRec {
    uint32_t x, y;        // the device clause
    uint16_t ia, ib;      // defining positions of the lhs / rhs register operands (COOP_NONE: immediate/unused)
    uint16_t p;           // position of this clause in the tape (== id of the value it defines)
    uint16_t cidx;        // choice index (choice clauses only)
};
// The tail is cut into segments: SERIAL runs are executed by one thread,
// CHAIN runs (>= 8 consecutive min- or max-clauses, each combining the
// previous clause's result with a value computed before the run) are
// evaluated with a block-wide prefix scan: min/max of intervals is exactly
// associative, and the choices follow from the prefix values.
struct CoopSeg { uint32_t begin, end, chain, start_slot; };   // start_slot: slot of the value a chain starts from
// The forward pass addresses values by SLOT, not by defining clause: the host colours the
// values of the schedule so that a slot is reused once every reader of its value has run
// (prospero: 6363 values -> ~2700 slots), which is what lets seven root tiles share an SM.
// A chain value whose only reader is the next clause of the same chain gets no slot at all.
struct CoopFwd {
    uint32_t x, y;        // the device clause
    uint16_t sa, sb;      // slots of the lhs / rhs register operands (COOP_NONE: immediate/unused)
    uint16_t so;          // slot of the result (COOP_NONE: not stored)
    uint16_t cidx;        // choice index (choice clauses only)
};
constexpr int COOP_MAX_SEGS = 16;
struct CoopSched {
    const CoopFwd* fwd;           // forward view of the same records (slots instead of positions)
    uint32_t n_slots;
    const CoopRec* recs;
    const uint32_t* wave_start;   // [n_waves + 1] offsets into recs
    uint32_t n_waves;
    uint32_t tail_begin, tail_end;
    uint32_t n_segs;
    CoopSeg segs[COOP_MAX_SEGS];
};

// Where the renderers feed coordinates: input slots of X, Y, Z (-1 = unused) and the
// values bound to every other input slot (ShapeVars, shape/mod.rs:548-640).
constexpr int MAX_RENDER_VARS = 16;
struct VarBind {
    int x, y, z;
    float values[MAX_RENDER_VARS];
};

// One frame of a 2D frame batch (fc_render2d_frames): what fc_render2d takes from its cfg per call.  The batch's
// tile grid stacks its frames vertically: frame k owns the grid rows [k * frame_rows, (k + 1) * frame_rows), where
// frame_rows is the frame's height rounded up to whole root tiles, so no tile straddles two frames.  A tile's screen
// coordinates are taken relative to its frame, and its frame's pixel rows land at k * height in the output.  A
// single render is the batch of one frame with frame_rows = 0xffffffff and the frame in the launch parameters.
// A 3D frame batch (fc_render3d_frames) uses the same table with z unused: its frames stack their XY root rows the
// same way (the Z layers are shared), and its heightmap and occlusion map hold frame_rows rows per frame.
struct Frame2D {
    Mat4 mat;
    float z;
    VarBind vb;
};

// One slice of a contour stack (fc_contour_build_slices): what fc_contour_build takes from its cfg per call.  The
// stacked quadtree gives slice k the cell rows [k * 2^depth, (k + 1) * 2^depth), and a cell's rows are taken relative
// to its slice.  has_transform stays a flag of its own: skipping the transform is not applying the identity (0 * z is
// NaN for a non-finite z, and a sum can flip a signed zero).  to_model: vertices go back through `mat` (has_transform
// and a matrix other than the identity).
struct ContourSlice {
    Mat4 mat;
    float z;
    uint32_t has_transform, to_model;
    VarBind vb;
};
// One frame of a mesh frame batch (fc_mesh_build_frames) is the same record with z unused: the stacked octree gives frame
// k the cell rows [k * 2^depth, (k + 1) * 2^depth), a cell's rows are taken relative to its frame, and to_model sends the
// frame's vertices back through `mat`.
using MeshFrame = ContourSlice;

// Scene renders (fc_render3d_scene): K placements (a tape and its Frame2D) share one heightmap and one occlusion map.
// Placement k's jobs carry k in TileJob::pad.  A heightmap key orders what the merged image keeps: the greater clamped
// depth, then the lower placement, then, inside one placement, what fc_render3d orders by (raw depth, then a leaf id
// over a fill).  Packed high to low: clamped depth (SK_DEPTH_BITS), priority 1023 - k (SK_PRIO_BITS), raw depth above
// the clamp threshold D - 1 (SK_SUB_BITS: 0 outside the clamp zone), leaf job id + 1 (SK_ID_BITS, 0 for a fill).  The
// key without its id is the placement's rank of a depth: what a skipped tile is compared against.  The occlusion map of
// a scene holds 64-bit ranks.  The host checks the limits the field widths imply (FC_SCENE_* in fidget_cuda.h).
constexpr uint32_t SK_ID_BITS = 26, SK_SUB_BITS = 10, SK_PRIO_BITS = 10, SK_DEPTH_BITS = 18;
constexpr uint32_t SK_MAX_SHAPES = 1u << SK_PRIO_BITS;
constexpr unsigned long long SK_ID_MASK = (1ull << SK_ID_BITS) - 1ull;
#ifdef __CUDACC__
// rank of raw depth `raw` for placement `pl`; clamp_at = D - 1 when the final clamp applies (depths >= D - 1 compare
// as D), 0xffffffff without it
__device__ __forceinline__ unsigned long long scene_rank(uint32_t raw, uint32_t pl, uint32_t clamp_at, uint32_t depth) {
    const bool zone = raw >= clamp_at;
    const unsigned long long dc = zone ? depth : raw, sub = zone ? raw - clamp_at : 0u;
    return ((((dc << SK_PRIO_BITS) | (SK_MAX_SHAPES - 1u - pl)) << SK_SUB_BITS) | sub) << SK_ID_BITS;
}
#endif

struct LevelParams {
    CoopSched sched;
    int level;                 // index into tile sizes
    uint32_t tile;             // edge of the tiles evaluated by this launch
    uint32_t n_axis;           // children per axis of each parent job (level > 0)
    uint32_t is_last;          // children are leaf tiles
    uint32_t pixel_perfect;
    // level 0 enumerates root tiles itself
    uint32_t root_mode;
    uint32_t roots_x, roots_y, roots_z;     // root grid
    uint32_t root_x0, root_y0, root_z0;     // origin of the root grid (pixels)
    // multi-GPU tile interleave: when non-null only the XY root tiles listed here (ty * roots_x + tx inside
    // the band) are evaluated, at every Z layer
    const uint32_t* root_list;
    uint32_t n_root_list;
    TapeRef root_tape;
    uint32_t epoch;                // ready mark of this render's job and fill records (never 0)
    // image
    uint32_t width, height, depth;
    float z2d;
    Mat4 mat;
    // lists
    const TileJob* jobs_in;
    uint32_t cap_in;
    TileJob* jobs_out;
    uint32_t cap_out;
    FillRec* fills;
    uint32_t cap_fills;
    // arena
    uint2* arena;
    unsigned long long arena_cap;   // clauses
    // scratch: per-warp choice words [choice_words][32]
    uint32_t* choice_scratch;
    uint32_t choice_words;          // words per lane
    Counters* ctr;
    Stats* stats;
    // octree sampler (mode 1): coordinates are cells at the finest depth; bounds = coord * cell_h - 1
    uint32_t mode;
    uint32_t has_transform;
    float cell_h;
    // 3D
    unsigned long long* heightmap;  // 3D: width*height keys (depth << 32 | leaf job id + 1), atomicMax
    // 3D occlusion map: per 16 x 16 block of pixels, a lower bound of the depth EVERY pixel of the block already has
    // (raised by interval-proven-inside tiles that cover whole blocks).  A parent whose blocks all reach its top + 1
    // cannot show anything: its children are skipped (cull != 0: this level's parents are made of whole blocks).
    // 2D scene (fc_render2d_scene): occl holds the two cover maps of kernels.cuh (Scene2D), the read map then the write
    // map, occl_w x occl_h leaf blocks each, and cull is the leaf tile edge (the block edge)
    uint32_t* occl;
    uint32_t occl_w, occl_h;        // blocks per row, block rows (tiles may overhang a ragged image: blocks outside are skipped)
    uint32_t cull;
    CensusRec* census;              // exact 3D census records (or null)
    uint32_t cap_census;
    VarBind vb;
    CancelRef cancel;
    // frame batch (2D or 3D): the frame table (null: the one frame is mat / z2d / vb above) and the grid rows per
    // frame; 3D: occl_h counts the block rows of one frame, and frame k's blocks start at row k * frame_rows / 16
    const Frame2D* frames;
    uint32_t frame_rows;
    // scene (fc_render3d_scene): `frames` is the placement table; level 0 evaluates the root tiles of the n_scene_pl
    // placements listed in scene_pl (those of root_tape), roots_x * roots_y * roots_z per placement; the heightmap
    // keys and the occlusion map hold scene ranks (clamp_at: see scene_rank)
    uint32_t scene;
    const uint32_t* scene_pl;
    uint32_t n_scene_pl;
    uint32_t clamp_at;
    uint32_t fused_tail;           // the fused 2D tail consumes this level's jobs: count them in Counters::outstanding
    // fc_measure (k_tree_level with MEASURE): one accumulator per frame of the pass, which the frame's proven-inside
    // cells are folded into
    struct MeasureAcc* measure;
};

// fc_measure's exact per-frame sums (fc_measure_result's integer fields, in its order).  Over the inside cells (i, j, k)
// at depth D, with u = 2i + 1, v = 2j + 1, w = 2k + 1: the counts, s1 = (Σu, Σv, Σw), s2 = (Σuu, Σvv, Σww, Σuv, Σuw,
// Σvw) and the inclusive cell-index box (lo starts at 0xffffffff, hi at 0).  Every word only ever grows by atomic adds,
// minima and maxima of integers, so the result does not depend on the order of the work.
struct MeasureAcc {
    unsigned long long n_inside, n_proven, n_undecided;
    unsigned long long s1[3], s2[6];
    uint32_t lo[3], hi[3];
};
// The brick kernel (measure.cu): every ambiguous cell of edge `brick` in list `list`, its brick^3 cell centres evaluated
// with the cell's simplified tape; frame f owns the cell rows [f * rows, (f + 1) * rows) and accumulator acc[f]
struct MeasureBrickParams {
    const TileJob* jobs;
    uint32_t cap_jobs;
    Counters* ctr;
    int list, cursor;
    uint32_t depth, brick, rows;
    MeasureAcc* acc;
    CancelRef cancel;
};

// fc_volume_build (volume.cu).  Its interval levels (k_tree_level_volume) take the band and the tile list in a kernel
// argument of their own, so that LevelParams keeps the layout the other level kernels are built with: a cell whose
// interval lies below -band or above band is proven, appended to `tiles` as its volume_tile_key and not split;
// *n_tiles counts the proven cells, beyond cap_tiles too (an overflow also sets error bit 1).
struct VolumeLevel {
    unsigned long long* tiles;
    uint32_t* n_tiles;
    uint32_t cap_tiles;
    float band;
};
// Sort keys of a pass's bricks and tiles: (frame of the pass, iz, iy, ix) of the first cell, 12 bits per coordinate
// (FC_MAX_OCTREE_DEPTH), so that sorting them gives the canonical order; a tile's key also carries its log2 edge and
// whether it is inside in its 5 low bits (below the cell, which alone orders the unique tiles of a frame)
constexpr int VOLUME_TILE_LOW_BITS = 5;
__host__ __device__ __forceinline__ unsigned long long volume_key(uint32_t f, uint32_t x, uint32_t y, uint32_t z) {
    return (((((unsigned long long)f << 12) | z) << 12 | y) << 12) | x;
}
__host__ __device__ __forceinline__ unsigned long long volume_tile_key(uint32_t f, uint32_t x, uint32_t y, uint32_t z,
                                                                       uint32_t log2_edge, bool inside) {
    return (volume_key(f, x, y, z) << VOLUME_TILE_LOW_BITS) | (log2_edge << 1) | (inside ? 1u : 0u);
}
// fc_volume_brick and fc_volume_tile
struct VolumeBrick { uint32_t frame; uint16_t ix, iy, iz, pad; };
struct VolumeTile { uint32_t frame; uint16_t ix, iy, iz; uint8_t log2_edge, inside; };
// The brick and gradient kernels: brick r of the pass (r < n) is job order[r] of `jobs` (list `list` of the levels),
// with sort key keys[r]; its brick^3 values go to values[r], its gradients to grads[r], its record to bricks[r].  frame
// f of the pass is fc_volume_build's frame f0 + f, and frames[f] its record.
struct VolumeBrickParams {
    const TileJob* jobs;
    const uint32_t* order;
    const unsigned long long* keys;
    uint32_t n, f0;
    uint32_t depth, brick;
    float* values;
    float* grads;
    VolumeBrick* bricks;
    Counters* ctr;
    int cursor;
    CancelRef cancel;
};
void launch_tree_level_volume(const LevelParams& p, const MeshFrame* frames, const VolumeLevel& v, int blocks, cudaStream_t s);

// fc_raycast (ray.cu).  A ray and a hit as fc_ray and fc_ray_hit lay them out.  The interval levels take their lists,
// arena, tape and vars from LevelParams and the pass from RayPass: a job is a segment of ray x starting at sample y,
// whose 32 children (seg samples each) are the lanes of one warp; level 0 takes 32 rays per warp, whole.  best[r] is ray
// r's smallest candidate so far, (k << 1) | proven (0xffffffff: none), lowered with atomicMin.
struct Ray { float o[3], d[3], t0, dt; };
struct RayHit { uint32_t k, flags; float t, pos[3], value, grad[3]; };
struct RayPass {
    const Ray* rays;
    RayHit* hits;
    uint32_t* best;
    unsigned long long* tally;   // [0] hits, [1] proven hits, [2] samples evaluated by the leaf launch
    uint32_t n_rays, steps;
    uint32_t seg;                // samples per segment this launch evaluates (level 0: 32^L, the whole ray)
};
void launch_ray_level(const LevelParams& p, const RayPass& r, int blocks, cudaStream_t s);
// the ambiguous 32-sample segments of list p.level, one warp each (p.jobs_in, p.cap_in, cursor p.level)
void launch_ray_leaf(const LevelParams& p, const RayPass& r, int blocks, cudaStream_t s);
void launch_ray_hits(const RayPass& r, const TapeRef& root, const VarBind& vb, const CancelRef& cancel, cudaStream_t s);
void launch_ray_clear(RayHit* hits, uint64_t n, cudaStream_t s);

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t root_count(const LevelParams& p, bool with_z) {
    return (p.root_list ? p.n_root_list : p.roots_x * p.roots_y) * (with_z ? p.roots_z : 1u);
}
// corner of root tile `idx` (XY-major, then Z layers)
__device__ __forceinline__ void root_corner(const LevelParams& p, uint32_t idx, uint32_t T, uint32_t& cx, uint32_t& cy,
                                            uint32_t& cz) {
    const uint32_t n_xy = p.root_list ? p.n_root_list : p.roots_x * p.roots_y;
    uint32_t xy = idx % n_xy;
    const uint32_t zl = idx / n_xy;
    if (p.root_list) xy = __ldg(p.root_list + xy);
    cx = p.root_x0 + (xy % p.roots_x) * T;
    cy = p.root_y0 + (xy / p.roots_x) * T;
    cz = p.root_z0 + zl * T;
}
// scene: the root tiles of every listed placement, placement-major; corner and placement of root `idx`
__device__ __forceinline__ uint32_t scene_root_count(const LevelParams& p) {
    return p.n_scene_pl * p.roots_x * p.roots_y * p.roots_z;
}
__device__ __forceinline__ uint32_t scene_root(const LevelParams& p, uint32_t idx, uint32_t T, uint32_t& cx, uint32_t& cy,
                                               uint32_t& cz) {
    const uint32_t per = p.roots_x * p.roots_y * p.roots_z;
    root_corner(p, idx % per, T, cx, cy, cz);
    return __ldg(p.scene_pl + idx / per);
}
#endif

struct PixelParams {
    uint32_t tile;             // leaf tile edge
    uint32_t width, height;
    float z2d;
    Mat4 mat;
    const TileJob* jobs;
    float* out;
    Counters* ctr;
    int list;                  // which n_jobs entry holds the leaf count
    int cursor;
    Stats* stats;
    VarBind vb;
    CancelRef cancel;
    const Frame2D* frames;     // 2D frame batch, as in LevelParams
    uint32_t frame_rows;
};

// The frame a 2D tile at grid row `y` belongs to: its parameters (in the launch parameters or the frame table),
// the first grid row of its frame and the first output row of its frame
struct FrameView {
    const Mat4* mat;
    float z;
    const VarBind* vb;
    uint32_t y0, out_row0;
};
#ifdef __CUDACC__
// FRAMES is a compile-time switch: the kernels of a single fc_render2d / fc_render3d (FRAMES = false) read their one
// frame from the launch parameters exactly as before the frame dimension existed (a runtime choice cost 2.7 % on
// prospero 4096^2).  (3D launch parameters have no z2d: their FrameView.z is 0 and unused.)
template <class P> __device__ __forceinline__ float single_z(const P&) { return 0.0f; }
__device__ __forceinline__ float single_z(const LevelParams& p) { return p.z2d; }
__device__ __forceinline__ float single_z(const PixelParams& p) { return p.z2d; }
template <bool FRAMES, class P>
__device__ __forceinline__ FrameView frame_of(const P& p, uint32_t y) {
    if (!FRAMES) return FrameView{&p.mat, single_z(p), &p.vb, 0u, 0u};
    const uint32_t f = y / p.frame_rows;
    const Frame2D* fr = p.frames + f;
    return FrameView{&fr->mat, fr->z, &fr->vb, f * p.frame_rows, f * p.height};
}
// SCENE (another compile-time switch): the placement `pl` of the tile supplies matrix and vars; all placements share
// the screen grid, so coordinates are not offset
template <bool FRAMES, bool SCENE, class P>
__device__ __forceinline__ FrameView view_of(const P& p, uint32_t y, uint32_t pl) {
    if (SCENE) return FrameView{&p.frames[pl].mat, p.frames[pl].z, &p.frames[pl].vb, 0u, 0u};
    return frame_of<FRAMES>(p, y);
}
// TREE (contours): the one slice of fc_contour_build in the launch parameters, or with STACK the slice of cell row y in
// the table `slices` (a kernel argument of its own: LevelParams keeps the layout the other level kernels are built with),
// frame_rows rows each
template <bool STACK>
__device__ __forceinline__ FrameView quad_view(const LevelParams& p, const ContourSlice* slices, uint32_t y) {
    if (!STACK) return FrameView{&p.mat, p.z2d, &p.vb, 0u, 0u};
    const uint32_t s = y / p.frame_rows;
    const ContourSlice* sl = slices + s;
    return FrameView{&sl->mat, sl->z, &sl->vb, s * p.frame_rows, 0u};
}
template <bool STACK>
__device__ __forceinline__ uint32_t quad_has_transform(const LevelParams& p, const ContourSlice* slices, uint32_t y) {
    return STACK ? slices[y / p.frame_rows].has_transform : p.has_transform;
}
#endif

// 2D scenes (fc_render2d_scene).  Placement k's jobs carry k in TileJob::pad, as a 3D scene's do.  Two maps replace the
// per-shape images:
//  - the cover map, one word per leaf block (leaf tile edge, aligned to the grid): max(k + 1) over the tiles of shape k
//    proven inside by interval arithmetic that cover the block.  Every tile is a union of whole blocks (each tile size
//    divides the one before it), so an inside fill is recorded exactly; outside fills record nothing.
//  - the key map, one word per pixel: max(k + 1) over the shapes whose leaf pixel evaluation found the pixel inside.
// The topmost shape inside pixel p is max(cover[block(p)], key[p]) - 1.  Both maps only take maxima of proven facts, so
// the result does not depend on the order of the work.  A tile of shape j whose every block already holds cover > j + 1
// cannot change that maximum and is not evaluated (culled).  Cull decisions read a copy of the cover map that only
// changes between launches (the read map; launches write the write map, which is copied over the read map after each
// launch), so which tiles are evaluated, and the census, do not depend on the launch grid or the timing of the work.
struct ScenePixelParams : PixelParams {
    const uint32_t* cover;     // the read cover map
    uint32_t* key;             // width * height words
    uint32_t blocks_x, blocks_y;
};
#ifdef __CUDACC__
// true when every leaf block of the T x T tile at (x, y) holds cover > pl + 1 (blocks outside the map count as open)
__device__ __forceinline__ bool scene2d_hidden(const uint32_t* cover, uint32_t blocks_x, uint32_t blocks_y, uint32_t leaf,
                                               uint32_t x, uint32_t y, uint32_t T, uint32_t pl) {
    const uint32_t nb = T / leaf, bx0 = x / leaf, by0 = y / leaf;
    for (uint32_t q = 0; q < nb * nb; ++q) {
        const uint32_t bx = bx0 + q % nb, by = by0 + q / nb;
        if (bx >= blocks_x || by >= blocks_y || cover[size_t(by) * blocks_x + bx] <= pl + 1u) return false;
    }
    return true;
}
// an interval-proven-inside T x T tile of placement pl at (x, y): its blocks of the write cover map, lanes lane0,
// lane0 + stride, ...
__device__ __forceinline__ void scene2d_cover(uint32_t* cover_out, uint32_t blocks_x, uint32_t blocks_y, uint32_t leaf,
                                              uint32_t x, uint32_t y, uint32_t T, uint32_t pl, uint32_t lane0,
                                              uint32_t stride) {
    const uint32_t nb = T / leaf;
    for (uint32_t q = lane0; q < nb * nb; q += stride) {
        const uint32_t bx = x / leaf + q % nb, by = y / leaf + q / nb;
        if (bx < blocks_x && by < blocks_y) atomicMax(cover_out + size_t(by) * blocks_x + bx, pl + 1u);
    }
}
#endif
// The image of a 2D scene from its maps: index (or null) and `out` (or null) in `fmt` (FC_OUT_MASK_U8 = 1,
// FC_OUT_BITMAP_1BIT = 2, FC_OUT_RGBA8 = 3 with colors[3 * k .. 3 * k + 2] the RGB of shape k)
struct Scene2DResolveParams {
    const uint32_t* cover;     // the final cover map
    const uint32_t* key;
    uint32_t width, height, leaf, blocks_x;
    uint32_t fmt;
    const uint8_t* colors;
    uint8_t* out;
    uint16_t* index;
    CancelRef cancel;
};

struct FillParams {
    uint32_t tile, width, height;
    const FillRec* fills;
    const uint32_t* n_fills;
    float* out;
    CancelRef cancel;
    uint32_t frame_rows;       // 2D frame batch: grid rows per frame (0xffffffff: one frame)
};

struct VoxelParams {
    uint32_t tile, width, height;
    const uint32_t* order;      // leaf jobs sorted front to back (descending z), or null
    Mat4 mat;
    const TileJob* jobs;
    uint32_t cap_jobs;
    unsigned long long* heightmap;
    Counters* ctr;
    int list, cursor;
    Stats* stats;
    VarBind vb;
    CancelRef cancel;
    const Frame2D* frames;      // 3D frame batch, as in LevelParams (job y is a grid row; the heightmap has its rows)
    uint32_t frame_rows;
    uint32_t scene, depth, clamp_at;   // scene: `frames` is the placement table, keys are scene ranks | id
};
struct NormalParams {
    uint32_t width, height, depth;
    uint32_t y0, y1;            // rows to finish (a Y band of a sharded render, else 0..height)
    // tile interleave: only these root tiles (ty * roots_x + tx inside the band, edge `root_tile`) are finished
    const uint32_t* root_list;
    uint32_t n_root_list, roots_x, root_tile;
    uint32_t clamp;             // apply the final `depth >= D-1` clamp (voxel.rs:535-546)
    Mat4 mat;
    const TileJob* jobs;        // leaf jobs
    const unsigned long long* heightmap;
    void* out;                  // GeometryPixel[width*height]
    Stats* stats;
    VarBind vb;
    CancelRef cancel;
    // 3D frame batch: rows y0 .. y1 are output rows of the stacked frames (frame k's row y is k * height + y, its
    // heightmap row k * frame_rows + y), each frame with its matrix and vars from the table
    const Frame2D* frames;
    uint32_t frame_rows;
    // scene: `frames` is the placement table.  Only pixels whose key belongs to placements pl0 .. pl1 - 1 (this pass's:
    // their leaf ids index this pass's leaf list) or is empty are written, with the placement into `index` (or null),
    // and nothing at all when the pass overflowed (`error` != 0: it is rendered again)
    uint32_t scene, pl0, pl1;
    uint16_t* index;
    const uint32_t* error;
};

// One leaf of the Manifold-Dual-Contouring octree (LeafHermiteData, fidget-mesh/src/octree.rs:864-900)
struct OctreeLeaf {
    uint16_t ix, iy, iz;
    uint8_t mask, n_edges;
    uint16_t present, pad;
    float pos[12][3];
    float grad[12][4];   // dx, dy, dz, v
};
struct OctreeLeafParams {
    const TileJob* jobs;
    uint32_t cap_jobs;
    Counters* ctr;
    int list, cursor;
    float cell_h;
    uint32_t has_transform;
    Mat4 mat;
    VarBind vb;
    OctreeLeaf* out;
    TapeRef* out_tapes;         // tape of each emitted leaf (consumed by the gradient pass)
    uint32_t cap_out;
    uint32_t* n_out;            // device counter
    unsigned long long* stats;  // [0] leaf_empty [1] leaf_full [2] leaf_surface [3] float points [4] grad points
    CancelRef cancel;
};

// launchers (kernels.cu)
// frames == null: the one frame in the launch parameters (fc_octree_sample, fc_mesh_build); else a mesh frame batch's
// table, `rows` cell rows per frame (the leaves record their frame in OctreeLeaf::pad)
void launch_octree_leaf(const OctreeLeafParams& p, int blocks, cudaStream_t s, const MeshFrame* frames = nullptr,
                        uint32_t rows = 0);
void launch_octree_grads(const OctreeLeafParams& p, int blocks, cudaStream_t s, const MeshFrame* frames = nullptr,
                         uint32_t rows = 0);
// the interval levels of the samplers' trees (octree.cu, k_tree_level): dim 3, a mesh frame batch's stacked octree (one
// root cell per frame, p.roots_y frames); dim 2, a contour's quadtree (frames == null: one root cell, the slice in the
// launch parameters; else a slice stack's table, one root cell per slice)
void launch_tree_level(const LevelParams& p, int dim, const ContourSlice* frames, int blocks, cudaStream_t s);
// fc_measure's levels: the stacked octree of dim 3 with its proven-inside cells folded into p.measure
void launch_tree_level_measure(const LevelParams& p, const MeshFrame* frames, int blocks, cudaStream_t s);
void launch_measure_bricks(const MeasureBrickParams& p, const MeshFrame* frames, int blocks, cudaStream_t s);
void launch_interval_level_3d(const LevelParams& p, int blocks, cudaStream_t s);
void launch_voxels_3d(const VoxelParams& p, int blocks, cudaStream_t s);
// Counting sort of the leaf jobs by descending Z layer: hist/offsets are device scratch of n_layers+1 words
void launch_leaf_zsort(const TileJob* jobs, const uint32_t* n_jobs, uint32_t cap, uint32_t z0, uint32_t tile,
                       uint32_t n_layers, uint32_t* hist, uint32_t* order, cudaStream_t s);
void launch_normals_3d(const NormalParams& p, cudaStream_t s);
struct CensusParams {
    const CensusRec* recs;
    const uint32_t* n_recs;
    uint32_t cap;
    uint32_t tile[MAX_LEVELS];
    int last_level;
    const unsigned long long* heightmap;
    uint32_t width;
    Stats* stats;
    CancelRef cancel;
};
void launch_census_3d(const CensusParams& p, int blocks, cudaStream_t s);
void launch_merge_slabs(const void* const* d_slabs, uint32_t n_slabs, uint32_t n_pixels, uint32_t depth, void* out,
                        cudaStream_t s);
// tile interleave: rank >= 0 packs that rank's tiles of `src` (an image) into `dst` (its chunk);
// rank < 0 unpacks every tile of the gathered chunks in `src` into the image `dst`
void launch_tiles_copy(const void* src, void* dst, uint32_t width, uint32_t height, uint32_t px_bytes, uint32_t T,
                       uint32_t roots_x, uint32_t roots_y, const uint32_t* slots, uint32_t n_ranks, uint32_t per_rank, int rank,
                       cudaStream_t s);
void launch_interval_level_2d(const LevelParams& p, int blocks, cudaStream_t s);
// occupancy of the level-0 kernel instantiation a launch takes (variant 0: one frame, 1: a frame batch, 2: a scene)
int coop_regs_per_thread(int dim, int variant);
int coop_occupancy(int dim, int variant, int threads, size_t smem);
size_t coop_smem_bytes(uint32_t n_ops, uint32_t n_choices, uint32_t n_slots);
cudaError_t launch_interval_root_coop_2d(const LevelParams& p, int blocks, int threads, cudaStream_t s);
cudaError_t launch_interval_root_coop_3d(const LevelParams& p, int blocks, int threads, cudaStream_t s);
void launch_pixels_2d(const PixelParams& p, int blocks, cudaStream_t s);
void launch_pixels_2d_scene(const ScenePixelParams& p, int blocks, cudaStream_t s);
void launch_scene2d_resolve(const Scene2DResolveParams& p, cudaStream_t s);
// Fused 2D tail (tail2d.cu): every level after the root level, the leaf pixels and the fills in ONE
// persistent launch that drains a dependency-ordered queue
constexpr int TAIL_MAX_LEVELS = 4;
struct Tail2DParams {
    int n_levels;                      // interval levels handled here (levels 1 .. n_levels of the render)
    LevelParams lv[TAIL_MAX_LEVELS];   // lv[k] = parameters of render level k + 1
    PixelParams px;
    uint32_t fill_tile[TAIL_MAX_LEVELS + 1];        // tile edge of the fill records of render level l
    const FillRec* fills[TAIL_MAX_LEVELS + 1];
    uint32_t fill_cap[TAIL_MAX_LEVELS + 1];
    uint32_t epoch;
    uint32_t paint_fills;              // 1: idle warps paint the fill records; 0: k_fill_2d launches do (after / beside this kernel)
    CancelRef cancel;
};
cudaError_t launch_tail_2d(const Tail2DParams& p, int sm_count, cudaStream_t s);
int tail_2d_blocks(int sm_count);
void launch_fill_2d(const FillParams& p, int blocks, cudaStream_t s);

// trait-level evaluators
struct BulkParams {
    const uint2* tape;
    uint32_t n_ops;
    uint32_t n_vars, n_outputs;
    uint32_t n_slots;           // 256 + mem_count
    uint64_t n;
    const void* const* vars;    // device array of device pointers (n_vars)
    void* const* outs;          // device array of device pointers (n_outputs)
};
void launch_float_slice(const BulkParams& p, cudaStream_t s);
// TMA-fed persistent bulk evaluators (bulk.cu): float4 columns, i.e. four consecutive f32 points or one
// gradient per thread
struct SliceTmaParams {
    const uint2* tape;
    uint32_t n_ops, n_vars, n_outputs, n_regs;
    uint64_t n;                 // points
    const float4* vars[4];
    float4* outs[2];
};
constexpr uint32_t SLICE_TMA_TILE = 256;   // float4 per variable in a tile of k_slice_tma: 1024 points f32, 256 gradients
unsigned launch_slice_tma(const SliceTmaParams& p, bool grad, int sm_count, cudaStream_t s);
void launch_grad_slice(const BulkParams& p, cudaStream_t s);

struct TracingParams {
    const uint2* tape;
    uint32_t n_ops, n_vars, n_outputs, n_choices, n_slots;
    uint64_t n;
    const float* vars;   // interval: [n][n_vars][2]; point: [n][n_vars]
    float* out;          // interval: [n][n_outputs][2]; point: [n][n_outputs]
    uint8_t* choices;    // [n][n_choices] or null
    uint8_t* simplify;   // [n] or null
};
void launch_interval_batch(const TracingParams& p, cudaStream_t s);
void launch_point_batch(const TracingParams& p, cudaStream_t s);

struct SimplifyParams {
    const uint2* parent;
    uint32_t n_ops, parent_ref_len;
    const uint8_t* choices;   // [n_choices] bytes
    uint32_t n_choices;
    uint2* out;               // capacity n_ops; child occupies the TAIL
    uint32_t* result;         // {n_dev, ref_len, n_choices_child}
};
void launch_simplify_single(const SimplifyParams& p, cudaStream_t s);

}  // namespace fdev
