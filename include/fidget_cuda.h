/* libfidget_cuda -- H100 (sm_90a) backend for Fidget's tape-evaluation hot path.
 *
 * C ABI, plain pointers and sizes only.  Every entry point cites the reference
 * interface it replaces (paths relative to the mkeeter/fidget checkout);
 * INTEGRATION.md shows the Rust `extern "C"` block and the `CudaFunction`
 * shim a maintainer would add on the reference side.
 *
 * Conventions
 *  - every function returns FC_OK (0) or a negative fc_status; nothing throws
 *    or aborts across the boundary.  fc_last_error() returns a message for the
 *    most recent failure on the calling thread.
 *  - handles are opaque.  fc_tape is reference counted (Arc semantics, like
 *    `GenericVmTape(Arc<VmData>)`, fidget-core/src/vm/mod.rs:47-48).
 *  - an fc_eval owns its scratch + output buffers and one CUDA stream; use one
 *    per thread, like the reference's evaluators (eval/bulk.rs:23-58).
 *  - pointers marked "host or device" are classified with
 *    cudaPointerGetAttributes; device (or managed) memory is used in place.
 *  - numerics: IEEE f32, round-to-nearest, no FMA contraction, denormals kept
 *    (the library is built with -fmad=false -prec-div=true -prec-sqrt=true
 *    -ftz=false).  add/sub/mul/div/sqrt/neg/abs/min/max/square/floor/ceil/
 *    round/mod and all comparisons are bit-identical to the reference VM;
 *    sin/cos/tan/asin/acos/atan/atan2/exp/ln use CUDA libdevice (<= 2 ulp).
 */
#ifndef FIDGET_CUDA_H
#define FIDGET_CUDA_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum fc_status {
    FC_OK = 0,
    FC_ERR_INVALID = -1,      /* bad argument / malformed bytecode */
    FC_ERR_CUDA = -2,         /* CUDA runtime error (message has the detail) */
    FC_ERR_UNSUPPORTED = -3,  /* valid input the device path cannot take (e.g. spilled tape in a renderer) */
    FC_ERR_ARENA = -4,        /* tape arena exhausted during on-device simplification */
    FC_ERR_NO_DEVICE = -5,    /* no usable CUDA device; there is NO CPU fallback */
    FC_ERR_CANCELLED = -6     /* the cancel flag attached with fc_ctx_set_cancel was set (never returned without one) */
} fc_status;

typedef struct fc_ctx fc_ctx;    /* one GPU + stream + scratch arenas */
typedef struct fc_tape fc_tape;  /* device-resident tape */
typedef struct fc_eval fc_eval;  /* per-thread evaluator scratch */

const char* fc_last_error(void);
/* Library/ABI version; bumped on any signature change */
uint32_t fc_abi_version(void);   /* 2: root_stride/root_offset, fc_tiles_* */

/* ---- lifecycle ---------------------------------------------------------- */
int32_t fc_ctx_create(int32_t device, fc_ctx** out);
void fc_ctx_destroy(fc_ctx* ctx);
/* Enqueue all subsequent work of this context on `cuda_stream` (a
 * cudaStream_t, e.g. torch.cuda.current_stream().cuda_stream; NULL is the
 * CUDA default stream).  use_own != 0 restores the context's own stream. */
int32_t fc_ctx_set_stream(fc_ctx* ctx, void* cuda_stream, int32_t use_own);
/* Wait for enqueued work and report deferred device-side errors
 * (FC_ERR_ARENA, ...). */
int32_t fc_ctx_synchronize(fc_ctx* ctx);
/* Size of the tape arena used by on-device simplification (bytes; default
 * 1 GiB).  Takes effect at the next render call. */
int32_t fc_ctx_set_arena_bytes(fc_ctx* ctx, uint64_t bytes);
/* Cancellation (CancelToken, fidget-core/src/render/config.rs:59-80).  `flag` points to a caller-owned byte with the
 * layout of Rust's AtomicBool (CancelToken::into_raw() as *const u8): nonzero = cancelled.  The library reads it with
 * an acquire load, from any thread; NULL detaches it.  Context-wide, like fc_ctx_set_stream, and consulted only by
 * fc_render2d, fc_render2d_frames, fc_render3d, fc_render3d_frames, fc_render3d_scene, fc_octree_sample, fc_mesh_build, and
 * fc_ctx_synchronize after the most recent FC_FLAG_ASYNC call of those.  With a flag attached:
 *  - set on entry: the call returns FC_ERR_CANCELLED before it allocates or launches anything;
 *  - set while the call runs: the kernels stop claiming work and the call returns FC_ERR_CANCELLED ("cancelled" in
 *    fc_last_error); `out` is unspecified (a host `out` receives no copy), stats / info are zeroed, and the context
 *    stays usable.  A cancelled fc_mesh_build leaves no mesh (fc_mesh_read copies nothing, fc_mesh_read_cells
 *    reports 0, fc_mesh_write_stl 84 bytes);
 *  - FC_OK: the result, stats included, is exactly that of the same call without a flag. */
int32_t fc_ctx_set_cancel(fc_ctx* ctx, const uint8_t* flag);

/* ---- tapes -------------------------------------------------------------- */
/* `words` is exactly what fidget_bytecode::Bytecode::new emits
 * (fidget-bytecode/src/lib.rs:203-332): [0xFFFFFFFF,0] op pairs ...
 * [0xFFFFFFFF,0xFFFFFFFF]; reg_count / mem_count from Bytecode::{reg_count,
 * mem_count}; n_vars = VarMap::len, n_outputs = VmData::output_count,
 * choice_count = VmData::choice_count (checked against the words). */
int32_t fc_tape_create(fc_ctx* ctx, const uint32_t* words, size_t n_words, uint8_t reg_count,
                       uint32_t mem_count, uint32_t n_vars, uint32_t n_outputs, uint32_t choice_count,
                       fc_tape** out);
int32_t fc_tape_retain(fc_tape* tape);
int32_t fc_tape_release(fc_tape* tape);

typedef struct fc_tape_info {
    uint32_t n_ops;         /* clauses in the device tape */
    uint32_t ref_len;       /* RegTape::len() of the equivalent reference tape (Function::size) */
    uint32_t choice_count;
    uint32_t reg_count;
    uint32_t mem_count;
    uint32_t n_vars;
    uint32_t n_outputs;
} fc_tape_info;
int32_t fc_tape_get_info(const fc_tape* tape, fc_tape_info* info);
/* Which input slots carry X, Y, Z (VarMap lookup of Var::X/Y/Z, shape/mod.rs:355-376;
 * -1 = the shape does not use that axis).  Default: x=0,y=1,z=2 clipped to n_vars.
 * The renderers feed transformed coordinates into these slots. */
int32_t fc_tape_set_axes(fc_tape* tape, int32_t x, int32_t y, int32_t z);
/* Copies the device tape back as bytecode words (same framing as the input;
 * device-only alias copies appear as plain Copy clauses).  words==NULL
 * queries the count. */
int32_t fc_tape_read(const fc_tape* tape, uint32_t* words, size_t cap, size_t* n_words);

/* Wire / on-disk form (the counterpart of serde on VmData, fidget-core/src/vm/data.rs:64):
 *   "FTAP" | version u32 = 1 | reg_count | mem_count | n_vars | n_outputs | choice_count (u32 each)
 *   | axis slots i32[3] | n_words u64 | bytecode words u32[n_words]          (little endian)
 * fc_tape_serialize writes the tape's blob (buf == NULL queries the size); fc_tape_deserialize is
 * fc_tape_create + fc_tape_set_axes from a blob (as written by fc_tape_serialize or by the host front end). */
int32_t fc_tape_serialize(const fc_tape* tape, uint8_t* buf, size_t cap, size_t* n_bytes);
int32_t fc_tape_deserialize(fc_ctx* ctx, const uint8_t* buf, size_t n_bytes, fc_tape** out);

/* ---- trait-level evaluators -------------------------------------------- */
/* These mirror TracingEvaluator / BulkEvaluator (eval/tracing.rs:26-61,
 * eval/bulk.rs:23-58) the way fidget-jit's raw function pointers do
 * (fidget-jit/src/lib.rs:1058-1065,1172-1178). */
int32_t fc_eval_create(fc_ctx* ctx, fc_eval** out);
void fc_eval_destroy(fc_eval* e);

/* VmIntervalEval::eval (vm/mod.rs:332-537).  vars: [n_vars][2] = lower,upper.
 * out: [n_outputs][2].  choices: [choice_count] bytes (Choice as u8:
 * 0 unknown, 1 left, 2 right, 3 both), may be NULL.  *simplify = 1 iff a
 * trace is available (some choice != Both).  Host pointers. */
int32_t fc_interval_eval(fc_eval* e, const fc_tape* tape, const float* vars_lo_hi, float* out_lo_hi,
                         uint8_t* choices, uint8_t* simplify);
/* VmPointEval::eval (vm/mod.rs:551-759) */
int32_t fc_point_eval(fc_eval* e, const fc_tape* tape, const float* vars, float* out, uint8_t* choices,
                      uint8_t* simplify);
/* n independent boxes in one launch (one lane per box; what the octree
 * sampler and the conformance tests use).  vars: [n][n_vars][2];
 * out: [n][n_outputs][2]; choices: [n][choice_count] or NULL;
 * simplify: [n] or NULL.  Host or device pointers. */
int32_t fc_interval_eval_batch(fc_eval* e, const fc_tape* tape, const float* vars, uint64_t n, float* out,
                               uint8_t* choices, uint8_t* simplify);
/* VmFloatSliceEval::eval (vm/mod.rs:800-1085): vars[i] -> n floats (SoA),
 * out[o] -> n floats.  The arrays of pointers are host arrays; the pointed-to
 * buffers may be host or device. */
int32_t fc_float_slice_eval(fc_eval* e, const fc_tape* tape, const float* const* vars, float* const* out,
                            uint64_t n);
typedef struct fc_grad { float v, dx, dy, dz; } fc_grad; /* types/grad.rs:2-13, #[repr(C)] */
/* VmGradSliceEval::eval (vm/mod.rs:1097-1396) */
int32_t fc_grad_slice_eval(fc_eval* e, const fc_tape* tape, const fc_grad* const* vars,
                           fc_grad* const* out, uint64_t n);
/* VmData::simplify (vm/data.rs:123-318) run on the device for one trace.
 * The child keeps the parent's register assignment (no re-allocation), is
 * value-identical to the reference's child, and reports the reference's
 * child length in fc_tape_info.ref_len.  Parent must not use memory slots. */
int32_t fc_simplify(fc_eval* e, const fc_tape* parent, const uint8_t* choices, size_t n_choices,
                    fc_tape** child);

/* ---- fused renderers (the measured path) -------------------------------- */
#define FC_MAX_TILE_LEVELS 8
#define FC_MAX_VARS 16
#define FC_FLAG_ASYNC 1u        /* enqueue only; errors surface in fc_ctx_synchronize */
#define FC_FLAG_TIMING 2u       /* record per-stage CUDA events (fc_render_stats.stage_ms) */
#define FC_FLAG_FUSED_TAIL 8u   /* fc_render2d, EXPERIMENTAL: the levels after the root level, the leaf pixels and the fills as one
                                   persistent launch draining a job queue (tail2d.cu) instead of one launch per stage.
                                   Same image and census; measured SLOWER on H100 (0.32 vs 0.25 ms for prospero 4096², profiles/), so off
                                   by default */
#define FC_FLAG_EXACT_CENSUS 16u /* fc_render3d with stats: report the tile census and voxel count of the reference's front-to-back
                                   walk (voxel.rs:244-357), computed from the final heightmap; without it the census counts what
                                   the device evaluated (a superset: it only culls whole parents behind interval-proven tiles).  Whole-volume renders of
                                   images whose sides are multiples of the root tile */
#define FC_FLAG_FULL_LADDER 32u /* fc_render3d with the default tile sizes: evaluate every size of the reference's ladder
                                   {128,64,32,16,8}.  Without it the device skips every other size ({128,32,8}: a 4x4x4 split
                                   evaluated with the parent's tape, as fidget-wgpu's interval_tiles.wgsl does) -- the image is
                                   the same bit for bit (interval results of a sub-region never contradict its parent's
                                   choices), 7-10 % faster, and fc_render_stats then describes those three levels.
                                   FC_FLAG_EXACT_CENSUS implies the full ladder; explicit tile_sizes are always used as given */
#define FC_FLAG_NO_CLAMP 4u     /* fc_render3d: skip the final depth clamp (slab renders; fc_merge_slabs applies it) */

#define FC_OUT_F32 0u          /* width*height RawDistancePixel bits as f32 (pixel::render's own output) */
#define FC_OUT_MASK_U8 1u      /* width*height bytes: 255 inside, 0 outside */
#define FC_OUT_BITMAP_1BIT 2u  /* height rows of (width+7)/8 bytes; bit x%8 (LSB first) of byte x/8 set = inside */
#define FC_OUT_RGBA8 3u        /* width*height*4 bytes: effects::to_rgba_bitmap(image, false) */
typedef struct fc_render2d_cfg {
    uint32_t width, height;
    float mat[16];              /* row-major 4x4, screen -> model: RenderConfig::mat() embedded as in
                                   fidget-raster/src/pixel.rs:283-287 */
    float z;                    /* pixel::RenderConfig::z */
    uint32_t pixel_perfect;     /* pixel::RenderConfig::pixel_perfect */
    uint32_t n_tile_sizes;      /* 0 => the VM default {128,32,8} (vm/mod.rs:254-256) */
    uint32_t tile_sizes[FC_MAX_TILE_LEVELS];
    uint32_t flags;
    /* Y band [row_begin,row_end) of root-tile rows to render (multi-GPU
     * sharding); row_end = 0 means all rows. */
    uint32_t root_row_begin, root_row_end;
    /* ShapeVars (shape/mod.rs:548-640): value for each tape input slot that is not an axis
     * (entries at axis slots are ignored); n_var_values may be 0 for plain X/Y/Z shapes. */
    uint32_t n_var_values;
    float var_values[FC_MAX_VARS];
    /* Multi-GPU tile interleave: with root_stride = N > 1 only the root tiles (tx, ty) with
     * ((tx * 73856093) ^ (ty * 19349663)) % N == root_offset (32-bit arithmetic: a spatial hash that spreads
     * heavy-tailed per-tile cost evenly) are rendered (the analogue of rayon handing root tiles to worker
     * threads, fidget-raster/src/lib.rs:152-165); other pixels are left untouched, and `out` must be a
     * device image.  0 or 1 = every root tile. */
    uint32_t root_stride, root_offset;
    /* What `out` receives (FC_OUT_*).  The distance image is always produced in HBM; the smaller formats
     * are derived from it on the device (RawDistancePixel::inside, pixel.rs:177-183 / effects::to_rgba_bitmap,
     * effects.rs:446-466), so a host caller pays the PCIe copy of the small image only. */
    uint32_t out_format;
} fc_render2d_cfg;

typedef struct fc_geometry_pixel { float normal[3]; uint32_t depth; } fc_geometry_pixel; /* voxel.rs:126-134 */

typedef struct fc_render3d_cfg {
    uint32_t width, height, depth;
    float mat[16];              /* row-major 4x4: voxel::RenderConfig::mat() (voxel.rs:107-109) */
    uint32_t n_tile_sizes;      /* 0 => {128,64,32,16,8} (vm/mod.rs:250-252) */
    uint32_t tile_sizes[FC_MAX_TILE_LEVELS];
    uint32_t flags;
    /* Z slab [z_begin,z_end) in voxels (multiples of tile_sizes[0]);
     * z_end = 0 means the whole depth. */
    uint32_t z_begin, z_end;
    uint32_t n_var_values;      /* as in fc_render2d_cfg */
    float var_values[FC_MAX_VARS];
    /* Y band [row_begin,row_end) of root-tile rows to render, full depth (multi-GPU sharding that
     * balances surface-like work better than Z slabs); row_end = 0 means all rows.  Only the rows
     * of the band are written. */
    uint32_t root_row_begin, root_row_end;
    uint32_t root_stride, root_offset;   /* tile interleave, as in fc_render2d_cfg (full depth per tile column) */
} fc_render3d_cfg;

typedef struct fc_render_stats {
    uint64_t evaluated[FC_MAX_TILE_LEVELS];      /* interval evaluations per level */
    uint64_t filled_inside[FC_MAX_TILE_LEVELS];
    uint64_t filled_outside[FC_MAX_TILE_LEVELS];
    uint64_t ambiguous[FC_MAX_TILE_LEVELS];
    uint64_t simplified[FC_MAX_TILE_LEVELS];     /* simplifications kept (shorter than parent) */
    uint64_t pixels;                             /* points shaded by the bulk kernel */
    uint64_t grads;                              /* points shaded by the gradient kernel */
    uint64_t arena_bytes_used;
    uint32_t kernel_launches;
    float stage_ms[16];                          /* FC_FLAG_TIMING: interval levels 0..7, then [8]=fill,
                                                    [9]=bulk f32, [10]=grad, [11]=merge, [12]=fused 2D tail (levels 1.., leaf pixels, fills), [15]=total */
} fc_render_stats;

/* pixel::render (fidget-raster/src/pixel.rs:452-492).  out: width*height
 * RawDistancePixel bit patterns as f32, row-major; host or device. */
int32_t fc_render2d(fc_ctx* ctx, const fc_tape* tape, const fc_render2d_cfg* cfg, float* out,
                    fc_render_stats* stats /* may be NULL */);

/* Many 2D frames of one tape in one call: Z-slice stacks, ShapeVars sweeps, view sequences.  The reference has no
 * batched call: frame k is pixel::render of its own RenderConfig, and here it is bit-identical to fc_render2d called
 * with `cfg` plus frame k's mat, z and var_values (same device arithmetic, libm operations included), for every
 * out_format and for pixel_perfect.  The frames of a pass share each launch of the tile pipeline, so every level
 * launch holds the ambiguous tiles of all of them.
 *  - cfg supplies what the frames share: width, height, pixel_perfect, tile_sizes, flags, out_format; its mat, z and
 *    var_values are ignored.
 *  - out (host or device) receives n_frames images back to back in fc_render2d's layout for out_format: frame k
 *    starts at k * (one image's bytes).  A host out gets each pass's images while the next pass runs.
 *  - stats: the per-level census and pixels summed over all frames (the sum of the per-frame fc_render2d stats),
 *    arena_bytes_used the largest of any pass, stage_ms summed over passes.
 *  - frames run in passes of as many as fit FC_FRAMES_PASS_BYTES of device memory: the worst-case job and fill lists
 *    of a frame (4096^2 with {128,32,8}: 15.7 MB), plus its distance image (two with a host F32 out) when out_format
 *    is not FC_OUT_F32 or out is on the host, plus two images of out_format with a host out.  The tape arena is
 *    reset per pass; FC_ERR_ARENA if a pass exhausts it.
 *  - n_frames == 0 launches nothing and returns FC_OK.  Errors follow fc_render2d (a spilled tape or more than 16
 *    inputs: FC_ERR_UNSUPPORTED; a frame without a value for a bound variable: FC_ERR_INVALID).  FC_ERR_UNSUPPORTED
 *    also for FC_FLAG_FUSED_TAIL, root row bands (root_row_begin / root_row_end) and the tile interleave
 *    (root_stride > 1).
 *  - FC_FLAG_ASYNC and the cancel flag (fc_ctx_set_cancel) behave as in fc_render2d; a cancelled call leaves `out`
 *    unspecified.  With a flag attached and a host `out`, the host waits for each pass while watching the flag before
 *    it copies that pass back (a copy into pageable memory would block it), so a flag set mid-call always stops the
 *    work in flight. */
#define FC_FRAMES_PASS_BYTES 536870912u   /* 512 MiB */
typedef struct fc_frame2d {
    float mat[16];                  /* row-major 4x4 screen -> model, as fc_render2d_cfg.mat */
    float z;                        /* pixel::RenderConfig::z */
    uint32_t n_var_values;          /* ShapeVars of this frame, as in fc_render2d_cfg */
    float var_values[FC_MAX_VARS];
} fc_frame2d;
int32_t fc_render2d_frames(fc_ctx* ctx, const fc_tape* tape, const fc_render2d_cfg* cfg,
                           const fc_frame2d* frames /* host */, uint32_t n_frames, void* out,
                           fc_render_stats* stats /* may be NULL */);
/* voxel::render (fidget-raster/src/voxel.rs:500-553).  out: width*height
 * GeometryPixel; host or device. */
int32_t fc_render3d(fc_ctx* ctx, const fc_tape* tape, const fc_render3d_cfg* cfg, fc_geometry_pixel* out,
                    fc_render_stats* stats /* may be NULL */);

/* Many 3D frames of one tape in one call: turntables, thumbnail views, camera paths, ShapeVars animations.  Frame k is
 * bit-identical to fc_render3d called with `cfg` plus frame k's mat and var_values (depth and all three normal floats;
 * same device arithmetic, libm operations included).  The frames of a pass share each launch of the tile pipeline.
 *  - cfg supplies what the frames share: width, height, depth, tile_sizes, flags (FC_FLAG_FULL_LADDER,
 *    FC_FLAG_NO_CLAMP, FC_FLAG_EXACT_CENSUS, FC_FLAG_TIMING, FC_FLAG_ASYNC); its mat and var_values are ignored.
 *  - out (host or device) receives n_frames images of width*height fc_geometry_pixel back to back.
 *  - stats: the per-level census, pixels and grads summed over all frames (the sum of the per-frame fc_render3d
 *    stats, FC_FLAG_EXACT_CENSUS included), arena_bytes_used the largest of any pass, stage_ms summed over passes,
 *    kernel_launches counting every pass run.
 *  - passes: at most as many frames as fit FC_FRAMES_PASS_BYTES of device memory (heightmaps, occlusion maps, job
 *    lists, and two staged images per frame with a host out).  FC_ERR_ARENA or a work-list overflow comes back only
 *    where one frame alone overflows: the first pass renders one frame, later passes are sized from the largest
 *    per-frame arena and list use seen so far, and a pass that still overflows is rendered again in halves.
 *  - n_frames == 0 launches nothing and returns FC_OK.  FC_ERR_UNSUPPORTED for a spilled tape (as fc_render3d), Z slabs
 *    (z_begin / z_end), root row bands and the tile interleave (root_stride > 1); FC_ERR_INVALID for a frame without a
 *    value for a bound variable, a multi-output tape, and frames == NULL with n_frames > 0.
 *  - The cancel flag behaves as in fc_render3d.  FC_FLAG_ASYNC (device out, no stats) returns once the last pass is
 *    enqueued; every earlier pass has been waited on, because its overflow status decides whether it runs again.  An
 *    overflow of the last pass is then reported by fc_ctx_synchronize, as fc_render3d's is. */
typedef struct fc_frame3d {
    float mat[16];                  /* row-major 4x4, as fc_render3d_cfg.mat (voxel::RenderConfig::mat) */
    uint32_t n_var_values;          /* ShapeVars of this frame, as in fc_render3d_cfg */
    float var_values[FC_MAX_VARS];
} fc_frame3d;
int32_t fc_render3d_frames(fc_ctx* ctx, const fc_tape* tape, const fc_render3d_cfg* cfg,
                           const fc_frame3d* frames /* host */, uint32_t n_frames, fc_geometry_pixel* out,
                           fc_render_stats* stats /* may be NULL */);
/* Several shapes rendered into one image: a viewer's draw list (every draw(shape) of a script rendered and composited),
 * or the merge of several voxel images that fidget-wgpu's effects pipeline starts with (merge.wgsl).  Shape k is
 * tapes[k] placed by placements[k] (its mat and var_values, as in fc_render3d_frames; the same tape may appear any number
 * of times).  Let img_k be fc_render3d(tapes[k], cfg with placements[k]'s mat and var_values), final clamp included
 * unless FC_FLAG_NO_CLAMP.  Then, bit for bit (depth and all three normal floats):
 *    out = img_0, then for k = 1 .. n_shapes - 1: out = (out.depth >= img_k.depth) ? out : img_k
 * per pixel -- the greatest (clamped) depth wins, and on equal depth the lowest k; index (may be NULL) receives the k
 * kept, 0 where every image is empty (depth 0).  All shapes share one heightmap and one occlusion map, so a tile proven
 * full for a front shape culls the tiles of the shapes behind it.
 *  - cfg supplies width, height, depth, tile_sizes and the flags FC_FLAG_NO_CLAMP, FC_FLAG_FULL_LADDER, FC_FLAG_TIMING
 *    and FC_FLAG_ASYNC; its mat and var_values are ignored.  out and index are host or device memory.
 *  - stats: the per-level census of the tiles evaluated across the scene (tiles culled behind other shapes are not
 *    counted), pixels, grads (normals evaluated), arena_bytes_used the largest of any pass, kernel_launches and stage_ms
 *    over all passes.  Every field but pixels is the same for two identical calls.
 *  - passes: placements go in passes that share the heightmap; FC_ERR_ARENA or a work-list overflow comes back only
 *    where one placement alone overflows (the first pass renders one placement, later ones are sized from the largest
 *    per-placement use so far, and a pass that overflows anyway is restored and rendered again in halves).
 *  - n_shapes == 0 launches nothing and returns FC_OK.  FC_ERR_UNSUPPORTED for a spilled tape, FC_FLAG_EXACT_CENSUS,
 *    Z slabs, root row bands, the tile interleave, n_shapes > FC_SCENE_MAX_SHAPES, a volume depth rounded up to whole
 *    root tiles above FC_SCENE_MAX_DEPTH, and (with the clamp) a root tile edge above FC_SCENE_MAX_ROOT_TILE.
 *    FC_ERR_INVALID for a multi-output tape, a placement without a value for a bound variable, a NULL entry of tapes,
 *    and tapes or placements NULL with n_shapes > 0.  All of these before anything is allocated or launched.
 *  - The cancel flag and FC_FLAG_ASYNC (device out and index, no stats) behave as in fc_render3d_frames.
 * Limits of the heightmap key (clamped depth, shape, depth above the clamp threshold, leaf tile): the shapes, the depth
 * and the root tile edge below; a pass holds at most FC_SCENE_MAX_LEAF_JOBS leaf tiles (more is a list overflow). */
#define FC_SCENE_MAX_SHAPES 1024
#define FC_SCENE_MAX_DEPTH 262142        /* depth rounded up to whole root tiles */
#define FC_SCENE_MAX_ROOT_TILE 1022      /* with the clamp: the root tile edge */
#define FC_SCENE_MAX_LEAF_JOBS 67108863  /* leaf tiles of one pass */
int32_t fc_render3d_scene(fc_ctx* ctx, const fc_tape* const* tapes /* host, n_shapes */,
                          const fc_frame3d* placements /* host, n_shapes */, uint32_t n_shapes,
                          const fc_render3d_cfg* cfg, fc_geometry_pixel* out, uint16_t* index /* may be NULL */,
                          fc_render_stats* stats /* may be NULL */);
/* Per-pixel merge of `n_slabs` slab images (each width*height, device
 * pointers, Z-ordered) into `out`, applying the final depth clamp of
 * voxel.rs:535-546.  Used after the all-gather in multi-GPU renders. */
int32_t fc_merge_slabs(fc_ctx* ctx, const fc_geometry_pixel* const* slabs, uint32_t n_slabs,
                       uint32_t width, uint32_t height, uint32_t depth, fc_geometry_pixel* out);

/* Tile-interleaved sharding (root_stride / root_offset above): the root tiles of rank r, in row-major
 * order, packed as [tile][root_tile rows][root_tile pixels] -- the contiguous chunk an all-gather needs.
 * Every rank's chunk holds fc_tiles_per_rank() tiles (ranks owning fewer leave the tail unused).
 * px_bytes is 4 (fc_render2d images) or 16 (fc_render3d images).  Device pointers; the calls only
 * ENQUEUE on the context's stream. */
uint32_t fc_tiles_per_rank(uint32_t width, uint32_t height, uint32_t root_tile, uint32_t n_ranks);
int32_t fc_tiles_pack(fc_ctx* ctx, const void* image, uint32_t width, uint32_t height, uint32_t px_bytes,
                      uint32_t root_tile, uint32_t n_ranks, uint32_t rank, void* packed);
/* gathered: n_ranks chunks in rank order (the output of the all-gather); writes every pixel of `image`. */
int32_t fc_tiles_unpack(fc_ctx* ctx, const void* gathered, uint32_t width, uint32_t height, uint32_t px_bytes,
                        uint32_t root_tile, uint32_t n_ranks, void* image);

/* ---- octree sampler (fidget-mesh) ----------------------------------------- */
/* The sampling half of Octree::build (fidget-mesh/src/octree.rs:521-808): interval
 * descent of the [-1,1]^3 octree with tape simplification at every cell, then for
 * each surface leaf the corner mask, the 16-ary edge searches and the gradient at
 * every intersection -- i.e. LeafHermiteData.intersections.  QEF solve, cell
 * collapse and walk_dual stay on the host (SURVEY.md section 8f). */
#define FC_MAX_OCTREE_DEPTH 12
typedef struct fc_octree_cfg {
    uint32_t depth;             /* mesh::Settings::depth */
    uint32_t has_transform;     /* 0 when Settings::world_to_model is the identity (octree.rs:493-498) */
    float world_to_model[16];   /* row-major 4x4 */
    uint32_t flags;
    uint32_t n_var_values;
    float var_values[FC_MAX_VARS];
} fc_octree_cfg;
typedef struct fc_octree_leaf {
    uint16_t ix, iy, iz;        /* cell coordinates at `depth` */
    uint8_t mask;               /* CellMask: bit c = corner c inside (bit 0 of c = +X, 1 = +Y, 2 = +Z) */
    uint8_t n_edges;
    uint16_t present, pad;      /* bit e = undirected edge e (types.rs:208-219) carries an intersection */
    float pos[12][3];           /* LeafIntersection::pos.xyz */
    float grad[12][4];          /* LeafIntersection::grad = (dx, dy, dz, v) */
} fc_octree_leaf;
typedef struct fc_octree_stats {
    uint64_t evaluated[16], full[16], empty[16], ambiguous[16];   /* interval census per depth */
    uint64_t leaf_empty, leaf_full, leaf_surface, float_points, grad_points;
    uint64_t arena_bytes_used;
    uint32_t kernel_launches;
    float total_ms;             /* FC_FLAG_TIMING */
} fc_octree_stats;
/* out: `cap` leaves, host or device; leaves arrive in no particular order.  *n_leaves receives
 * the number of surface leaves (if it exceeds cap the call fails with FC_ERR_INVALID). */
int32_t fc_octree_sample(fc_ctx* ctx, const fc_tape* tape, const fc_octree_cfg* cfg, fc_octree_leaf* out,
                         uint64_t cap, uint64_t* n_leaves, fc_octree_stats* stats /* may be NULL */);

/* ---- meshing back half (fidget-mesh: QEF vertices, dual walk, STL) ---------------------------------------- */
/* fc_mesh_build = fc_octree_sample + the rest of the Manifold Dual Contouring pipeline on the device, the mesh
 * staying in HBM until it is read: one vertex per connected group of inside corners of every surface leaf,
 * positioned by QuadraticErrorSolver::solve (fidget-mesh/src/qef.rs:67-168); four triangles around every
 * sign-changing cell edge as in dc_edge (fidget-mesh/src/dc.rs:104-213).  By default there is no cell collapse:
 * the result is the uniform-depth mesh.  With FC_FLAG_MESH_COLLAPSE in fc_octree_cfg.flags the eight children of a
 * cell are merged into one leaf as Octree::check_done / try_collapse do (octree.rs:252-440: manifold topology and a
 * merged QEF error below twice the children's), and the dual is walked over leaves of different depths, as
 * Octree::build(..).walk_dual() does: fewer triangles in flat regions.  Edges on the boundary of the [-1,1]^3 domain
 * get no triangles (open_edges).
 * With fc_octree_cfg.has_transform the octree is built over the [-1,1]^3 world cube in the field seen through
 * world_to_model, and, as the last step of Octree::build (octree.rs:58-65), every vertex is mapped back to model space
 * through Matrix4::transform_point (f32, divided by the homogeneous term where that is not zero) unless the matrix is
 * the identity: fc_mesh_read, fc_mesh_write_stl and fc_mesh_cell.vertex are in model space, the cell coordinates of
 * fc_mesh_read_cells stay those of the world cube. */
#define FC_FLAG_MESH_COLLAPSE 64u /* fc_mesh_build: cell collapse and the adaptive dual walk */
typedef struct fc_mesh_info {
    uint64_t n_leaves, n_vertices, n_triangles, open_edges;
    float sampler_ms, mesh_ms;   /* device time of the sampler / of QEF + dual walk */
} fc_mesh_info;
int32_t fc_mesh_build(fc_ctx* ctx, const fc_tape* tape, const fc_octree_cfg* cfg, fc_mesh_info* info);
/* vertices: n_vertices * 3 floats, triangles: n_triangles * 3 vertex indices; host or device; either may be NULL */
int32_t fc_mesh_read(fc_ctx* ctx, float* vertices, uint32_t* triangles);
/* One final leaf of the octree of the last fc_mesh_build, when it ran with FC_FLAG_MESH_COLLAPSE */
typedef struct fc_mesh_cell {
    uint16_t ix, iy, iz;        /* cell coordinates at `depth` */
    uint8_t depth;
    uint8_t mask;               /* CellMask of the leaf */
    float vertex[3];            /* the leaf's first cell vertex */
} fc_mesh_cell;
/* out: `cap` cells, host or device, in no particular order; *n receives the number of final leaves (0 after a build
 * without FC_FLAG_MESH_COLLAPSE).  out == NULL queries the count. */
int32_t fc_mesh_read_cells(fc_ctx* ctx, fc_mesh_cell* out, uint64_t cap, uint64_t* n);
/* Mesh::write_stl (fidget-mesh/src/output.rs:7-38): binary STL of the last mesh, assembled on the device.
 * buf == NULL queries the size (84 + 50 * n_triangles). */
int32_t fc_mesh_write_stl(fc_ctx* ctx, uint8_t* buf, size_t cap, size_t* n_bytes);

/* ---- constraint solver (fidget-solver) ----------------------------------------------------------------------- */
/* fidget_solver::solve (fidget-solver/src/lib.rs:191-289) for a batch of independent problems that share their
 * constraint tapes (multi-start solves, parameter sweeps, one sketch re-solved for many drag positions), the whole
 * Levenberg-Marquardt loop of every problem in one launch.  Per problem exactly the reference's loop: the Jacobian
 * from the gradient of output 0 of each constraint, damping 1.0 (x1.5 per rejected step, /3 per accepted one),
 * delta = pinv(JtJ + damping diag(JtJ)) Jtr with eigenvalues |w| <= f32::EPSILON dropped, err = the sum of the
 * squared constraint values in constraint order, and the reference's exits (FC_SOLVE_*).  Differences:
 *  - the loop stops after max_iters steps (FC_SOLVE_MAX_ITERS); the reference's has no cap;
 *  - every tape input slot must be bound to a parameter (FC_ERR_INVALID otherwise): the reference shares one input
 *    buffer across its tapes, so an unbound slot would read whatever another tape last wrote there;
 *  - Jacobian columns follow the caller's parameter order (the reference's come from HashMap iteration order);
 *  - the pseudo-inverse is a cyclic Jacobi eigen-solve in f32 with a fixed operation order (the reference calls
 *    nalgebra's SVD): results agree with the reference to rounding, and bit for bit with the project's CPU oracle.
 * Limits (FC_ERR_UNSUPPORTED beyond them): n_free <= 64, n_constraints <= 256, n_params <= 1024, constraint tapes
 * without memory slots.  n_free == 0 is FC_ERR_INVALID (the reference indexes an empty Jacobian).  Not cancellable. */
#define FC_SOLVE_MAX_FREE 64
#define FC_SOLVE_MAX_CONSTRAINTS 256
#define FC_SOLVE_MAX_PARAMS 1024
/* problem parameters: indices [0, n_free) are free (Parameter::Free), [n_free, n_params) fixed (Parameter::Fixed) */
typedef struct fc_solve_cfg {
    uint32_t n_params, n_free;
    uint32_t max_iters;          /* 0 => 1000 */
} fc_solve_cfg;
#define FC_SOLVE_ZERO_RESIDUAL 0u /* every residual == 0 before a step */
#define FC_SOLVE_UNCHANGED 1u     /* the step changed no free value */
#define FC_SOLVE_ZERO_ERR 2u      /* the accepted step's error is 0 */
#define FC_SOLVE_ZERO_DAMPING 3u  /* damping underflowed to 0 */
#define FC_SOLVE_STALLED 4u       /* four equal errors in a row */
#define FC_SOLVE_MAX_ITERS 5u     /* max_iters steps taken without another exit */
/* iterations: steps applied to the free values; err: the last accepted step's error (0 for FC_SOLVE_ZERO_RESIDUAL) */
typedef struct fc_solve_result { uint32_t status, iterations; float err; uint32_t pad; } fc_solve_result;
/* slot_param[k]: n_vars(constraints[k]) entries, tape input slot -> parameter index (host arrays).
 * values: [n_problems][n_params], host or device; free entries are overwritten with the solution.
 * results: [n_problems], host or device, or NULL.  n_problems == 0 launches nothing. */
int32_t fc_solve_batch(fc_ctx* ctx, const fc_tape* const* constraints, uint32_t n_constraints,
                       const int32_t* const* slot_param, const fc_solve_cfg* cfg, float* values, uint64_t n_problems,
                       fc_solve_result* results);

/* ---- diagnostics ---------------------------------------------------------- */
/* Host-only (no device needed): builds the level-0 schedule fc_tape_create would build for this
 * bytecode -- dependency waves, serial / chain tail segments, slot colouring -- and replays it
 * symbolically: every operand slot must hold the value of the clause that defines the operand at the
 * moment it is read, and no clause of a wave (or chain run) may overwrite a slot another clause of
 * the same step reads.  FC_ERR_INVALID with a message if the check fails; suitable == 0 when the
 * tape takes the per-lane kernel instead (too short, uses memory slots, ...). */
typedef struct fc_schedule_info {
    uint32_t suitable, n_clauses, n_waves, widest_wave, n_tail, n_segments, n_chain_clauses, n_slots;
} fc_schedule_info;
int32_t fc_schedule_check(const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count,
                          uint32_t n_vars, uint32_t n_outputs, fc_schedule_info* info);

/* ---- post-processing effects (fidget-raster/src/effects.rs) ---------------- */
/* Every image pointer may be a host or a device pointer (host images are staged
 * through HBM); images are row-major width*height.  All results are bit-identical
 * to the reference's arithmetic except fc_to_rgba_distance (exp/cos: within one
 * 8-bit step). */

/* effects::denoise_normals (effects.rs:17-36): back-facing normals are replaced by
 * the best-scoring mean of four 3x3 neighbourhoods.  Not in place. */
int32_t fc_denoise_normals(fc_ctx* ctx, const fc_geometry_pixel* image, uint32_t width, uint32_t height,
                           fc_geometry_pixel* out);
/* effects::compute_ssao (effects.rs:72-95).  `kernel`: n_kernel hemisphere samples
 * (x,y,z each), `noise`: n_noise unit XY rotations (x,y each) -- the reference draws
 * them from rand::rng() on every call (ssao_kernel(64) / ssao_noise(256),
 * effects.rs:385-440), so they are inputs here.  out: width*height f32, NaN where
 * the pixel is empty. */
int32_t fc_compute_ssao(fc_ctx* ctx, const fc_geometry_pixel* image, uint32_t width, uint32_t height,
                        uint32_t depth, const float* kernel, uint32_t n_kernel, const float* noise,
                        uint32_t n_noise, float* out);
/* effects::blur_ssao (effects.rs:98-115).  Not in place. */
int32_t fc_blur_ssao(fc_ctx* ctx, const float* ssao, uint32_t width, uint32_t height, float* out);
/* effects::apply_shading (effects.rs:42-66): three-light diffuse shading, optionally
 * modulated by compute_ssao + blur_ssao (ssao != 0; then the tables are required).
 * out_rgb: width*height*3 bytes (ColorImage). */
int32_t fc_apply_shading(fc_ctx* ctx, const fc_geometry_pixel* image, uint32_t width, uint32_t height,
                         uint32_t depth, int32_t ssao, const float* kernel, uint32_t n_kernel,
                         const float* noise, uint32_t n_noise, uint8_t* out_rgb);
/* The last stage of apply_shading alone (shade_pixel, effects.rs:118-154) with an
 * already blurred occlusion map (or NULL). */
int32_t fc_shade_with_occlusion(fc_ctx* ctx, const fc_geometry_pixel* image, uint32_t width, uint32_t height,
                                uint32_t depth, const float* blurred_ssao, uint8_t* out_rgb);
/* GeometryPixel::to_color per pixel (voxel.rs:136-153). out_rgb: width*height*3 bytes. */
int32_t fc_normals_to_color(fc_ctx* ctx, const fc_geometry_pixel* image, uint32_t width, uint32_t height,
                            uint8_t* out_rgb);
/* effects::to_rgba_bitmap / to_debug_bitmap / to_rgba_distance (effects.rs:446-547) on a
 * RawDistancePixel image (fc_render2d's output).  out_rgba: width*height*4 bytes. */
int32_t fc_to_rgba_bitmap(fc_ctx* ctx, const float* image, uint32_t width, uint32_t height, int32_t transparent,
                          uint8_t* out_rgba);
int32_t fc_to_debug_bitmap(fc_ctx* ctx, const float* image, uint32_t width, uint32_t height, uint8_t* out_rgba);
int32_t fc_to_rgba_distance(fc_ctx* ctx, const float* image, uint32_t width, uint32_t height, uint8_t* out_rgba);

#ifdef __cplusplus
}
#endif
#endif /* FIDGET_CUDA_H */
