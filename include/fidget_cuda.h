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
 * fc_render2d, fc_render2d_frames, fc_render2d_scene, fc_render3d, fc_render3d_frames, fc_render3d_scene, fc_octree_sample,
 * fc_mesh_build, fc_mesh_build_frames, fc_contour_build, fc_raycast, fc_volume_build, fc_solve_batch, fc_solve_large_batch, and
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
/* ---- compiled tapes (JitFunction / JitShape, fidget-jit) ----------------------------------------------------
 * fc_tape_compile turns one tape into straight-line sm_90a kernels for the bulk evaluators, compiled at run time
 * with NVRTC: every VM register and memory slot is a local variable, so values stay in registers instead of the
 * interpreters' per-thread register file.  Compiling takes host time (seconds for a tape of thousands of clauses), so
 * it is explicit and per kind; the compiled calls pay off over many points.
 *  - Results: for every tape fc_tape_create accepts (multi-output tapes and tapes with memory slots included), each
 *    compiled call writes exactly the bits its interpreter counterpart (fc_float_slice_eval, fc_grad_slice_eval,
 *    fc_interval_eval_batch) writes on the same inputs -- for intervals the values, the choice bytes and the simplify
 *    flags -- for every opcode and form, NaN payloads of rand / mix included.  NVRTC compiles the library's own device
 *    arithmetic with the numeric flags the library is built with.
 *  - Errors: kinds == 0, a kind that was not compiled, or an NVRTC compile error (log in fc_last_error):
 *    FC_ERR_INVALID.  NVRTC that cannot be loaded: FC_ERR_UNSUPPORTED, and the message says where it looked.
 *  - NVRTC is opened with dlopen at the first compile, never linked: the path in FIDGET_B200_NVRTC (a file, or the
 *    directory holding libnvrtc.so.12) and nothing else if it is set; else libnvrtc.so.12 by soname; else
 *    $CUDA_HOME/lib64 (default /usr/local/cuda).
 *  - Lifetime: a compiled tape belongs to the context and must be released before fc_ctx_destroy, like a tape; it
 *    retains its fc_tape.  Work goes on the context's stream (fc_ctx_set_stream).  Not cancellable (nor are the
 *    calls it shadows). */
typedef struct fc_compiled fc_compiled;     /* a tape compiled for some evaluator kinds; retains its fc_tape */
#define FC_COMPILE_FLOAT 1u                 /* fc_compiled_float_slice_eval */
#define FC_COMPILE_GRAD 2u                  /* fc_compiled_grad_slice_eval */
#define FC_COMPILE_INTERVAL 4u              /* fc_compiled_interval_eval_batch */
typedef struct fc_compiled_info {
    uint32_t kinds;                 /* kinds compiled */
    uint32_t nvrtc_version;         /* major * 1000 + minor * 10 of the NVRTC that compiled it */
    uint32_t regs[3];               /* per kind (float, grad, interval): registers per thread, 0 if not compiled */
    uint32_t local_bytes[3];        /* per kind: local memory (stack frame, spills included) per thread */
    float compile_ms[3];            /* per kind: host wall time of source generation + NVRTC */
    uint64_t cubin_bytes;
} fc_compiled_info;
int32_t fc_tape_compile(fc_ctx* ctx, const fc_tape* tape, uint32_t kinds, fc_compiled** out);
int32_t fc_compiled_get_info(const fc_compiled* c, fc_compiled_info* info);
int32_t fc_compiled_release(fc_compiled* c);
/* Same arguments, layouts, host / device pointer rules and results as the interpreter calls they shadow */
int32_t fc_compiled_float_slice_eval(fc_eval* e, const fc_compiled* c, const float* const* vars, float* const* out,
                                     uint64_t n);
int32_t fc_compiled_grad_slice_eval(fc_eval* e, const fc_compiled* c, const fc_grad* const* vars, fc_grad* const* out,
                                    uint64_t n);
int32_t fc_compiled_interval_eval_batch(fc_eval* e, const fc_compiled* c, const float* vars, uint64_t n, float* out,
                                        uint8_t* choices, uint8_t* simplify);
/* Host-only, no device needed (like fc_schedule_check): generate and compile the given bytecode for `kinds`, fill
 * *info (regs / local_bytes read from the cubin), and optionally copy the generated source, NUL-terminated and cut
 * to cap - 1 characters (source == NULL or cap == 0: only *n_source, the full length, is set). */
int32_t fc_compile_check(const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count, uint32_t n_vars,
                         uint32_t n_outputs, uint32_t kinds, char* source, size_t cap, size_t* n_source,
                         fc_compiled_info* info);

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
/* A 2D draw list in one call: the reference viewer's 2D mode, where each draw(shape) / draw_rgb(shape, r, g, b) of a
 * script is rendered and painted over the layers before it, opaque (BlendComponent::OVER).  Shape k is tapes[k] placed
 * by placements[k] (its mat, z and var_values, as fc_render2d_frames reads a frame; the same tape may appear any number
 * of times).  Let in_k(p) be RawDistancePixel::inside of pixel p in fc_render2d(tapes[k], cfg with placements[k]'s mat,
 * z and var_values).  Then, bit for bit:
 *  - index (may be NULL) receives the largest k with in_k(p), or FC_SCENE2D_NONE where no shape is inside: later shapes
 *    are on top, as the viewer paints them.
 *  - out (may be NULL) receives the image in cfg->out_format: FC_OUT_RGBA8 [r_k, g_k, b_k, 255] for k = index[p] and
 *    [0, 0, 0, 0] where no shape is inside, with colors[3k .. 3k + 2] (host, n_shapes * 3 bytes; NULL: white for every
 *    shape, the colour of draw()); FC_OUT_MASK_U8 and FC_OUT_BITMAP_1BIT: the union of the shapes' inside sets, in
 *    fc_render2d's layouts.  FC_OUT_F32 is FC_ERR_UNSUPPORTED: no per-shape distance is kept.
 *  - cfg supplies what the shapes share: width, height, pixel_perfect, tile_sizes, out_format and the flags
 *    FC_FLAG_TIMING and FC_FLAG_ASYNC; its mat, z and var_values are ignored.  out and index are host or device memory.
 *  - The shapes share one cover map (per leaf tile block: the topmost shape with an interval-proven-inside tile over
 *    it) and one key map (per pixel: the topmost shape whose leaf evaluation found it inside).  A tile whose every block
 *    is covered by a higher shape is not evaluated.  With pixel_perfect no tile is proven inside, so nothing is culled.
 *  - stats: the per-level census of the tiles evaluated (culled tiles are not counted) and the leaf pixels evaluated,
 *    arena_bytes_used the largest of any pass, stage_ms and kernel_launches summed over passes.  Every field is the same
 *    for two identical calls and at any launch grid: a cull decision only reads what earlier launches proved.
 *  - passes: as many shapes as their worst-case job lists fit FC_FRAMES_PASS_BYTES, from the top of the draw list down,
 *    so that lower shapes are culled against everything above them.  The tape arena is reset per pass; FC_ERR_ARENA if
 *    a pass exhausts it.
 *  - n_shapes == 0 launches nothing and returns FC_OK.  Refused before anything is allocated or launched, with out and
 *    index untouched: every tape fc_render2d refuses (with its code); FC_ERR_INVALID for a placement without a value
 *    for a bound variable, a NULL entry of tapes, tapes or placements NULL with n_shapes > 0, and out and index both
 *    NULL; FC_ERR_UNSUPPORTED for n_shapes > FC_SCENE_MAX_SHAPES, FC_FLAG_FUSED_TAIL, root row bands, the tile
 *    interleave and FC_OUT_F32.
 *  - The cancel flag and FC_FLAG_ASYNC (device out and index, no stats) behave as in fc_render2d_frames. */
#define FC_SCENE2D_NONE 0xFFFFu
int32_t fc_render2d_scene(fc_ctx* ctx, const fc_tape* const* tapes /* host, n_shapes */,
                          const fc_frame2d* placements /* host, n_shapes */, uint32_t n_shapes,
                          const fc_render2d_cfg* cfg, const uint8_t* colors /* host, n_shapes * 3 RGB, or NULL */,
                          void* out /* may be NULL */, uint16_t* index /* may be NULL */,
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
 * buf == NULL queries the size (84 + 50 * n_triangles; after fc_mesh_build_frames one file per frame, back to back). */
int32_t fc_mesh_write_stl(fc_ctx* ctx, uint8_t* buf, size_t cap, size_t* n_bytes);
/* Many meshes of one tape in one call: an animation through a ShapeVars parameter, a design sweep, one part under several
 * placements or views.  Frame k's mesh is what fc_mesh_build gives for cfg's depth and flags (FC_FLAG_MESH_COLLAPSE,
 * FC_FLAG_TIMING) plus frame k's has_transform, world_to_model and var_values: the same vertices bit for bit and the same
 * triangles as triples of vertex positions with their winding (both compared as multisets, since fc_mesh_build writes
 * in atomic order), the same n_leaves, n_vertices, n_triangles and open_edges, and with collapse the same final leaves
 * and cell vertices.  The frames of a pass share each launch: one tall octree grid holds them (frame k owns the cell
 * rows [k * 2^depth, (k + 1) * 2^depth)), and the mesher keys every cell by its frame, so nothing crosses frames.
 *  - cfg supplies depth and flags; its has_transform, world_to_model and var_values are ignored.
 *  - fc_mesh_read returns the whole batch: vertices and triangles frame-contiguous in frame order, each frame's
 *    triangle indices relative to its first vertex, so frame k's rows of the two arrays are a complete mesh on their own
 *    (per_frame gives the row counts).  fc_mesh_read_cells lists the final leaves frame by frame (n_cells each), and
 *    fc_mesh_write_stl writes one complete binary STL per frame, back to back: frame k's file takes
 *    84 + 50 * n_triangles_k bytes.  After a single fc_mesh_build the reads give what a batch of its one frame would;
 *    whichever of the two ran last is what they return.
 *  - per_frame (may be NULL, n_frames entries): frame k's counts.  info: their sums (n_cells has no field there), and
 *    sampler_ms (with FC_FLAG_TIMING) and mesh_ms summed over passes.
 *  - passes: the first pass holds one frame, later ones are sized from the largest per-frame arena, job-list and
 *    surface-leaf use seen so far (leaves and mesh scratch within FC_FRAMES_PASS_BYTES, at most
 *    FC_MESH_MAX_PASS_FRAMES frames), and a pass that overflows anyway is run again in halves: FC_ERR_ARENA, a work-list
 *    overflow or "mesh too large for cell collapse" comes back only where one frame alone would give it.
 *  - Errors are fc_mesh_build's, checked for every frame before anything is allocated or launched (depth above
 *    FC_MAX_OCTREE_DEPTH, a multi-output tape, more than FC_MAX_VARS values or a frame without a value for a bound
 *    variable: FC_ERR_INVALID; a tape with memory slots: FC_ERR_UNSUPPORTED), and FC_ERR_INVALID for frames == NULL
 *    with n_frames > 0.  A failed or cancelled call (the cancel flag behaves as in fc_mesh_build) leaves no mesh, as
 *    does n_frames == 0, which launches nothing. */
#define FC_MESH_MAX_PASS_FRAMES 4096u

typedef struct fc_mesh_frame {
    uint32_t has_transform;         /* as fc_octree_cfg.has_transform */
    float world_to_model[16];       /* as fc_octree_cfg.world_to_model (row-major 4x4) */
    uint32_t n_var_values;          /* ShapeVars of this frame, as fc_octree_cfg */
    float var_values[FC_MAX_VARS];
} fc_mesh_frame;
typedef struct fc_mesh_frame_info {
    uint64_t n_leaves, n_vertices, n_triangles, open_edges, n_cells;
} fc_mesh_frame_info;
int32_t fc_mesh_build_frames(fc_ctx* ctx, const fc_tape* tape, const fc_octree_cfg* cfg /* depth, flags */,
                             const fc_mesh_frame* frames /* host */, uint32_t n_frames,
                             fc_mesh_info* info /* totals */, fc_mesh_frame_info* per_frame /* may be NULL */);

/* ---- Measurement: volume, centre of mass, inertia and bounding box ------------------------------------------------
 * fc_measure measures the voxel solid of a shape at depth D (0 <= D <= FC_MAX_OCTREE_DEPTH): the world cube [-1,1]^3 is
 * split into 2^D cells per axis, cell (i, j, k) spanning [-1 + i h, -1 + (i + 1) h] on X (likewise Y, Z), h = 2 / 2^D,
 * and the solid is the union of the cells that count as inside, as solid cubes of unit density.  With has_transform the
 * field is seen through world_to_model, as fc_mesh_build sees it.  Which cells count as inside is fixed by the descent:
 *  - with B = min(4, 2^D) the brick edge, interval levels run from the root cell down to cells of edge B, one octree
 *    depth per level, with fc_octree_sample's bounds, transform, tape simplification and classification: upper < 0
 *    proves the cell inside (all its depth-D cells count), lower > 0 proves it outside (dropped), anything else is
 *    split further;
 *  - every ambiguous cell of edge B is a brick: each of its B^3 depth-D cells counts as inside iff the f32 value at its
 *    centre (-1 + (2i + 1) 2^-D, ...; exact in f32), through world_to_model as the octree leaf's corners are, with the
 *    brick's own simplified tape, is < 0.
 * For tapes of IEEE operations an interval never contradicts a point value in its box, so the result should equal a
 * classification of every cell centre.
 * Exact results (integers, independent of the launch grid, the order of the work and the passes), with u = 2i + 1,
 * v = 2j + 1, w = 2k + 1 over the inside cells: n_inside; n_proven, those in interval-proven-inside cells; n_undecided,
 * B^3 times the number of bricks; s1 = (Σu, Σv, Σw); s2 = (Σuu, Σvv, Σww, Σuv, Σuw, Σvw); lo / hi, the inclusive
 * cell-index box (0xFFFFFFFF and 0 when n_inside is 0).  Every sum fits u64 up to depth 12 (Σuv <= 2^62).
 * Derived results, float64, computed from the integers on the host.  In world space the volume is N h^3, the centroid
 * -1 + s1 / (N 2^D), the covariance (N s2 - s1 s1^T) / (N^2 4^D) plus h^2 / 12 on the diagonal (the numerators formed
 * exactly), and [volume_lo, volume_hi] = [n_proven, n_proven + n_undecided] h^3 encloses the shape's true volume inside
 * the cube, up to rounding (the intervals are not outward-rounded).  The fields below are in model space: with
 * has_transform and a matrix other than the identity, world_to_model = [A t; 0 1] scales the volumes by |det A|, maps
 * the centroid, and turns the covariance C into A C A^T; inertia = volume (tr(C) I - C) about the centroid (Ixx, Iyy,
 * Izz, Ixy, Ixz, Iyz; the products of inertia are -∫xy dV); bbox is the box of the 8 mapped corners of the world box
 * [lo h - 1, (hi + 1) h - 1].  An empty frame has volume 0 and NaN centroid, inertia and box.
 *  - frames (host, n_frames entries): each frame's has_transform, world_to_model and var_values; cfg supplies depth and
 *    flags (FC_FLAG_TIMING: *device_ms, when not NULL, receives the device time summed over passes).
 *  - passes: the frames of a pass share each launch in one stacked octree (frame k owns the cell rows
 *    [k 2^D, (k + 1) 2^D)); the first pass holds one frame, later ones are sized from the largest per-frame arena and
 *    job-list use seen so far, and a pass that overflows anyway is run again in halves: FC_ERR_ARENA or a work-list
 *    overflow comes back only where one frame alone gives it.
 *  - Checked for every frame before anything is allocated or launched: depth above FC_MAX_OCTREE_DEPTH, a multi-output
 *    tape, more than FC_MAX_VARS values, a frame without a value for a bound variable, and NULL frames or out with
 *    n_frames > 0 give FC_ERR_INVALID; a tape with memory slots or a projective world_to_model (last row other than
 *    0 0 0 1, with has_transform) gives FC_ERR_UNSUPPORTED.  n_frames == 0 launches nothing and returns FC_OK.
 *  - The cancel flag behaves as in fc_mesh_build: a cancelled call returns FC_ERR_CANCELLED with out zeroed, and the
 *    context stays usable.  A failed call zeroes out too. */
typedef struct fc_measure_result {
    uint64_t n_inside, n_proven, n_undecided;
    uint64_t s1[3];                 /* Σu, Σv, Σw */
    uint64_t s2[6];                 /* Σuu, Σvv, Σww, Σuv, Σuw, Σvw */
    uint32_t lo[3], hi[3];          /* inclusive cell-index box of the inside cells */
    double volume, volume_lo, volume_hi;
    double centroid[3];
    double inertia[6];              /* Ixx, Iyy, Izz, Ixy, Ixz, Iyz about the centroid */
    double bbox_min[3], bbox_max[3];
} fc_measure_result;
int32_t fc_measure(fc_ctx* ctx, const fc_tape* tape, const fc_octree_cfg* cfg /* depth, flags */,
                   const fc_mesh_frame* frames /* host */, uint32_t n_frames, fc_measure_result* out /* host */,
                   float* device_ms /* FC_FLAG_TIMING, may be NULL */);

/* ---- Sparse narrow-band volumes: the field on a voxel grid ---------------------------------------------------------
 * fc_volume_build samples the field of a shape at the cell centres of the depth-D grid of the world cube [-1,1]^3
 * (0 <= D <= FC_MAX_OCTREE_DEPTH), densely near the surface and as proven tiles everywhere else, the result staying in
 * HBM until fc_volume_read copies it out (VDB-style exports, SDF textures, collision lookups, training data):
 *  - Grid.  Cell (i, j, k) is centred at -1 + (2i + 1) 2^-D on X, likewise on Y and Z (exact in f32).  With
 *    has_transform the centre is mapped through world_to_model in f32 (Matrix4::transform_point, divided by the
 *    homogeneous term where that is not zero), as fc_measure maps it; projective matrices are allowed.
 *  - Band.  cfg->band, 0 <= band < inf.  With B = min(8, 2^D) the brick edge, interval levels run from the root cell
 *    down to cells of edge B, one octree depth per level, with fc_octree_sample's bounds, transform and tape
 *    simplification.  A cell whose interval [lo, hi] has hi < -band is an inside tile, lo > band an outside tile; a tile
 *    is recorded and not split.  Anything else, NaN included, is split; an unsplit cell of edge B is a brick.  With
 *    band == 0 this is exactly the classification of fc_measure and the octree sampler.
 *  - Brick values.  Every brick stores its B^3 values, values[brick][(k B + j) B + i] (x fastest): the f32 result of
 *    the brick's simplified tape at the mapped centre, the evaluation fc_measure makes.
 *  - Gradients.  With FC_FLAG_VOLUME_GRADS each brick also stores grads[brick][cell][3], the world-space partials
 *    (d/dx, d/dy, d/dz) of the brick's tape at the cell centre, as fc_octree_leaf.grad gives them.
 *  - Partition.  The tiles and bricks of a frame partition its cube exactly; every tile has edge 2^log2_edge >= B.
 *  - Order.  Bricks and tiles are each sorted by (frame, iz, iy, ix) of their first cell: the output is byte for byte
 *    independent of the launch grid, the order of the work and the passes.
 *  - Which values are exact.  For tapes of IEEE operations an interval never contradicts a point value in its box, so:
 *    every centre whose root-tape value v has |v| <= band lies in a brick; every centre in an inside tile has
 *    v < -band and every centre in an outside tile has v > band; brick values equal fc_float_slice_eval of the root
 *    tape at the mapped centre, bit for bit.
 *  - frames (host, n_frames entries): each frame's has_transform, world_to_model and var_values.  Passes: the frames of
 *    a pass share each launch in one stacked octree; the first pass holds one frame, later ones are sized from the
 *    largest per-frame arena, job-list and tile-list use seen so far, and a pass that overflows anyway is run again in
 *    halves: FC_ERR_ARENA or a work-list overflow (the tile list included) comes back only where one frame alone gives
 *    it.  Once a pass's levels are done its brick and tile counts are known, and the volume grows to hold them before
 *    its bricks are evaluated: n_bricks B^3 4 (1 + 3 grads) bytes of values and gradients, 12 bytes per brick and per
 *    tile.  When that would exceed the device's free memory the call returns FC_ERR_UNSUPPORTED ("volume too large")
 *    and the context stays usable.
 *  - info (may be NULL): the counts of the whole volume, the cells evaluated per interval level, B, the passes run, and
 *    with FC_FLAG_TIMING the device time (level_ms: of the interval levels alone) summed over passes.  per_frame (may be
 *    NULL, n_frames entries): frame k's counts and its first brick and tile in the volume.
 *  - Checked before anything is allocated or launched: fc_measure's refusals but the projective matrix (depth above
 *    FC_MAX_OCTREE_DEPTH, a multi-output tape, more than FC_MAX_VARS values, a frame without a value for a bound
 *    variable, NULL frames with n_frames > 0: FC_ERR_INVALID; a tape with memory slots: FC_ERR_UNSUPPORTED), and a NaN,
 *    negative or infinite band: FC_ERR_INVALID.  n_frames == 0 launches nothing and leaves an empty volume.
 *  - The cancel flag behaves as in fc_mesh_build.  A cancelled or failed call leaves no volume: fc_volume_read copies
 *    nothing and info and per_frame are zeroed.
 * fc_volume_read copies the volume of the last fc_volume_build into host or device memory; any pointer may be NULL:
 * bricks (n_bricks), values (n_bricks B^3 floats), grads (n_bricks B^3 3 floats; FC_ERR_INVALID unless the volume was
 * built with FC_FLAG_VOLUME_GRADS), tiles (n_tiles). */
#define FC_FLAG_VOLUME_GRADS 128u
typedef struct fc_volume_cfg {
    uint32_t depth;
    uint32_t flags;                 /* FC_FLAG_VOLUME_GRADS, FC_FLAG_TIMING */
    float band;
    uint32_t pad;
} fc_volume_cfg;
typedef struct fc_volume_brick {
    uint32_t frame;
    uint16_t ix, iy, iz, pad;       /* first cell */
} fc_volume_brick;
typedef struct fc_volume_tile {
    uint32_t frame;
    uint16_t ix, iy, iz;            /* first cell */
    uint8_t log2_edge;              /* edge 2^log2_edge cells */
    uint8_t inside;                 /* 1: hi < -band, 0: lo > band */
} fc_volume_tile;
typedef struct fc_volume_info {
    uint64_t n_bricks, n_tiles, n_inside_tiles;
    uint64_t evaluated[16];         /* cells evaluated per interval level */
    uint32_t brick_edge, passes;
    float device_ms, level_ms;      /* FC_FLAG_TIMING */
} fc_volume_info;
typedef struct fc_volume_frame_info {
    uint64_t n_bricks, n_tiles, first_brick, first_tile;
} fc_volume_frame_info;
int32_t fc_volume_build(fc_ctx* ctx, const fc_tape* tape, const fc_volume_cfg* cfg, const fc_mesh_frame* frames /* host */,
                        uint32_t n_frames, fc_volume_info* info /* may be NULL */,
                        fc_volume_frame_info* per_frame /* may be NULL */);
int32_t fc_volume_read(fc_ctx* ctx, fc_volume_brick* bricks, float* values, float* grads, fc_volume_tile* tiles);

/* ---- Ray casts: the first inside sample along each ray --------------------------------------------------------------
 * fc_raycast answers, for each of n_rays rays, where the ray first enters the shape (picking, line of sight, depth
 * sensors, placing a point on a surface).  Ray r has `steps` samples k = 0 .. steps - 1, each computed in f32 with one
 * round-to-nearest per operation, in model space (no transform):
 *     t_k = t0 + float(k) * dt,    x_k = origin + t_k * dir   (per axis)
 * With dt > 0 each of these steps is monotone in k (t_k non-decreasing; t * d non-decreasing or non-increasing in t by
 * the sign of d; o + s non-decreasing in s), so on every axis the samples of a segment [a, b] lie between x_a and x_b:
 * the box spanned by a segment's two end samples encloses every sample in it.  Which samples count is fixed by the
 * descent:
 *  - L = max(1, ceil(log2(steps) / 5)) interval levels l = 0 .. L - 1 of segments 32^(L - l) samples long, clipped to
 *    [0, steps): level 0 is the whole ray, and every ambiguous segment splits into 32 children (children that start at
 *    or past `steps` are not evaluated);
 *  - a segment is classified by the interval value over its box, with its own tape, as the tile renderers classify
 *    tiles: upper < 0 proves it inside, and its first sample is a candidate hit (FC_RAY_PROVEN); lower > 0 drops it;
 *    anything else, NaN included, splits it, and its children take the tape simplified by its choices when that tape is
 *    shorter (render/mod.rs:96-152);
 *  - every ambiguous segment of level L - 1 (32 samples) evaluates its samples with its tape: a value < 0 is a
 *    candidate hit.
 * The hit is the smallest candidate k.  Segments that start at or past a ray's best candidate so far are skipped, which
 * changes the speed only: the result depends on the descent alone, not on the launch grid, the passes or the order of
 * the work.  For tapes of IEEE operations an interval never contradicts a point value in its box, so k is the first
 * sample whose f32 value is < 0.  For each hit, value and grad are the ROOT tape at pos: value bit for bit what
 * fc_float_slice_eval gives there, grad (d/dx, d/dy, d/dz) what fc_grad_slice_eval gives.  A miss has k = FC_RAY_MISS
 * and every other field 0.
 *  - rays and hits: host or device.  cfg->var_values bind the tape's other inputs (ShapeVars), one binding per call.
 *  - info (may be NULL): hits, those proven by an interval, the segments evaluated per level, the samples evaluated by
 *    the leaf launch, the passes run, and with FC_FLAG_TIMING the device time summed over passes.
 *  - passes: rays run in passes; the first pass holds one ray, later ones are sized from the largest per-ray arena and
 *    job-list use seen so far, and a pass that overflows anyway is run again in halves: FC_ERR_ARENA or a work-list
 *    overflow comes back only where one ray alone gives it.
 *  - Checked before anything is allocated or launched (device rays are first read back, in the order of the context's
 *    stream): steps of 0 or above FC_RAY_MAX_STEPS, a ray with a non-finite
 *    origin, dir, t0 or dt, dt <= 0 or a non-finite t at its last sample, a multi-output tape, more than FC_MAX_VARS
 *    values or a missing value for a bound variable, NULL cfg, rays or hits with n_rays > 0: FC_ERR_INVALID; a tape
 *    with memory slots: FC_ERR_UNSUPPORTED.  n_rays == 0 launches nothing and returns FC_OK.
 *  - The cancel flag behaves as in fc_mesh_build.  A cancelled or failed call leaves every hit a miss, and the context
 *    stays usable. */
#define FC_RAY_MISS 0xFFFFFFFFu
#define FC_RAY_PROVEN 1u
#define FC_RAY_MAX_STEPS 16777216u   /* 2^24 */
typedef struct fc_ray {
    float origin[3], dir[3];        /* model space */
    float t0, dt;                   /* t_k = t0 + k dt, dt > 0 */
} fc_ray;
typedef struct fc_ray_hit {
    uint32_t k;                     /* index of the hit sample, FC_RAY_MISS if none */
    uint32_t flags;                 /* FC_RAY_PROVEN: the hit is the first sample of an interval-proven-inside segment */
    float t, pos[3];                /* t_k and x_k */
    float value, grad[3];           /* the root tape at pos: value, d/dx, d/dy, d/dz */
} fc_ray_hit;
typedef struct fc_raycast_cfg {
    uint32_t steps;                 /* samples per ray, 1 .. FC_RAY_MAX_STEPS */
    uint32_t flags;                 /* FC_FLAG_TIMING */
    uint32_t n_var_values;          /* ShapeVars, as fc_octree_cfg */
    float var_values[FC_MAX_VARS];
} fc_raycast_cfg;
typedef struct fc_raycast_info {
    uint64_t n_hits, n_proven;
    uint64_t evaluated[8];          /* segments evaluated per interval level */
    uint64_t leaf_samples;          /* samples evaluated by the leaf launch */
    uint32_t passes;
    float device_ms;                /* FC_FLAG_TIMING */
} fc_raycast_info;
int32_t fc_raycast(fc_ctx* ctx, const fc_tape* tape, const fc_raycast_cfg* cfg, const fc_ray* rays /* host or device */,
                   uint64_t n_rays, fc_ray_hit* hits /* host or device */, fc_raycast_info* info /* may be NULL */);

/* ---- 2D contours (libfive's Contours::render, on the quadtree the mesher's octree restricts to) -------------------
 * fc_contour_build extracts the contours of a 2D shape (a sketch, a cut profile, a Z slice of a 3D model) as closed or
 * open polylines, by dual contouring on a uniform quadtree of the [-1,1]^2 world square, the result staying in HBM until
 * it is read:
 *  1. the quadtree is descended by interval evaluation, with the tape simplified at every cell, exactly as
 *     fc_octree_sample does with Z fixed to [z, z]; cell bounds are float(i) * h - 1 with h = 2 / 2^depth, and a cell
 *     proven inside (upper < 0) or outside (lower > 0) is dropped;
 *  2. every remaining depth-level cell (ix, iy) gets a 4-bit corner mask (bit c = corner c inside, v < 0; bit 0 of c is
 *     +X, bit 1 is +Y); masks 0 and 15 are not surface leaves.  On every edge whose corners differ, the intersection is
 *     found by fc_octree_sample's 16-ary search, and the gradient there (dx, dy, v) in world coordinates;
 *  3. one vertex per connected group of inside corners (adjacent along cell edges: two diagonal inside corners give two
 *     vertices), placed by the 2D restriction of QuadraticErrorSolver::solve (fidget-mesh/src/qef.rs:67-168);
 *  4. one segment per sign-changing edge inside the domain, between the vertices owning it in its two cells, directed so
 *     that the inside lies on its left (counter-clockwise around inside regions, y up).  Edges on the domain boundary
 *     give no segment and are counted in n_open;
 *  5. segments are linked into polylines in a canonical order: an open polyline starts at its vertex without an incoming
 *     segment, a closed one at its smallest vertex key (iy, ix, group); polylines are ordered by the key of their first
 *     vertex.  The output is deterministic, bit for bit;
 *  6. with has_transform, unless world_to_model is the identity, vertices are mapped to model space through the matrix
 *     (f32, divided by the homogeneous term where that is not zero).  The direction of travel is the one in the world
 *     square: a mirroring matrix reverses it in model space.
 * world_to_model is a row-major 3x3, as the 2D renderers take it, applied to the world square (x, y, 1); Z is passed
 * through.  Errors: depth above FC_MAX_QUADTREE_DEPTH, a multi-output tape or n_var_values above FC_MAX_VARS give
 * FC_ERR_INVALID, a tape with memory slots FC_ERR_UNSUPPORTED.  The cancel flag (fc_ctx_set_cancel) stops the build; a
 * cancelled build leaves no contour (fc_contour_read copies nothing, every count is 0). */
#define FC_MAX_QUADTREE_DEPTH 14
typedef struct fc_contour_cfg {
    uint32_t depth;
    uint32_t has_transform;     /* 0: world_to_model is ignored */
    float world_to_model[9];    /* row-major 3x3 */
    float z;                    /* the Z slice */
    uint32_t flags;             /* FC_FLAG_TIMING: sampler_ms / contour_ms */
    uint32_t n_var_values;      /* ShapeVars, as in fc_render2d_cfg */
    float var_values[FC_MAX_VARS];
} fc_contour_cfg;
typedef struct fc_contour_info {
    uint64_t n_leaves, n_vertices, n_polylines, n_closed, n_open;
    float sampler_ms, contour_ms;   /* device time of the quadtree sampler / of vertices, segments and linking */
} fc_contour_info;
int32_t fc_contour_build(fc_ctx* ctx, const fc_tape* tape, const fc_contour_cfg* cfg, fc_contour_info* info);
/* Many slices of one tape contoured in one call: layers for a printer or a laser cutter, section drawings, a profile
 * swept through a ShapeVars parameter.  Slice k's polylines are bit for bit those of fc_contour_build called with cfg's
 * depth and flags plus slice k's z, has_transform, world_to_model and var_values (vertices, offsets relative to the
 * slice, closed flags, canonical order).  The slices of a pass share each launch of the pipeline: one tall quadtree grid
 * holds them, so every level launch holds the cells of all of them.
 *  - cfg supplies depth and flags; its z, has_transform, world_to_model and var_values are ignored.
 *  - fc_contour_read returns the whole stack: the slices in order, each slice's polylines in its canonical order, offsets
 *    global over the stack.  Whichever of fc_contour_build and fc_contour_build_slices ran last is what it returns.
 *  - per_slice (may be NULL, n_slices entries): slice k's n_leaves, n_vertices, n_polylines, n_closed and n_open; its
 *    timing fields are 0.  info: the sums of those counts, and with FC_FLAG_TIMING sampler_ms and contour_ms summed
 *    over passes.
 *  - passes: the first pass holds one slice, later ones are sized from the largest per-slice arena, job-list and leaf
 *    use seen so far (leaves and link scratch within FC_FRAMES_PASS_BYTES), and a pass that overflows anyway is run again
 *    in halves: FC_ERR_ARENA or a work-list overflow comes back only where one slice alone would give it.
 *  - Errors are fc_contour_build's, checked for every slice before anything is allocated or launched (depth, a
 *    multi-output tape, more than FC_MAX_VARS values or a slice without a value for a bound variable: FC_ERR_INVALID; a
 *    spilled tape: FC_ERR_UNSUPPORTED), and FC_ERR_INVALID for slices == NULL with n_slices > 0.  A stack of more than
 *    2^32 - 1 vertices in all gives FC_ERR_UNSUPPORTED.  A failed or cancelled call (the cancel flag behaves as in
 *    fc_contour_build) leaves no contour; n_slices == 0 launches nothing and leaves an empty contour. */
typedef struct fc_contour_slice {
    float z;                        /* as fc_contour_cfg.z */
    uint32_t has_transform;         /* as fc_contour_cfg.has_transform */
    float world_to_model[9];        /* as fc_contour_cfg.world_to_model */
    uint32_t n_var_values;          /* ShapeVars of this slice, as fc_contour_cfg */
    float var_values[FC_MAX_VARS];
} fc_contour_slice;
int32_t fc_contour_build_slices(fc_ctx* ctx, const fc_tape* tape, const fc_contour_cfg* cfg,
                                const fc_contour_slice* slices /* host */, uint32_t n_slices,
                                fc_contour_info* info /* totals */, fc_contour_info* per_slice /* may be NULL */);
/* The polylines of the last fc_contour_build or fc_contour_build_slices: vertices (2 floats each, in polyline order),
 * offsets (n_polylines + 1: polyline k is vertices offsets[k] .. offsets[k + 1] - 1) and closed (one byte per polyline,
 * 1 = the last vertex joins the first).  Host or device pointers; any may be NULL. */
int32_t fc_contour_read(fc_ctx* ctx, float* vertices, uint32_t* offsets, uint8_t* closed);

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
 * without memory slots; fc_solve_large_batch takes larger problems.  n_free == 0 is FC_ERR_INVALID (the reference
 * indexes an empty Jacobian).  Cancellable (fc_ctx_set_cancel): the solver stops claiming problems and stops each
 * problem in flight at its next iteration; a cancelled call returns FC_ERR_CANCELLED and copies nothing back to host
 * values / results, and a row in device memory is either untouched or fully solved. */
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
/* fc_solve_batch for larger problems: one problem per thread-block cluster of up to 16 CTAs, its matrices in a
 * context-owned device workspace (about 28 MiB per problem in flight at the limits; the problems in flight are capped
 * so that it stays within FC_FRAMES_PASS_BYTES, but a lone problem always gets its workspace).  Arguments, exits and
 * cancellation as in fc_solve_batch; it accepts every problem fc_solve_batch accepts, and its result is bit for bit
 * what fc_solve_batch gives there.  Limits (FC_ERR_UNSUPPORTED beyond them): n_free <= 1024, n_constraints <= 4096,
 * n_params <= 16384, constraint tapes without memory slots.  FC_ERR_CUDA if the workspace cannot be allocated. */
/* a cluster of up to 16 CTAs: 16 times fc_solve_batch's limits (1024, 4096, 16384) */
#define FC_SOLVE_LARGE_MAX_FREE (16 * FC_SOLVE_MAX_FREE)
#define FC_SOLVE_LARGE_MAX_CONSTRAINTS (16 * FC_SOLVE_MAX_CONSTRAINTS)
#define FC_SOLVE_LARGE_MAX_PARAMS (16 * FC_SOLVE_MAX_PARAMS)
int32_t fc_solve_large_batch(fc_ctx* ctx, const fc_tape* const* constraints, uint32_t n_constraints,
                             const int32_t* const* slot_param, const fc_solve_cfg* cfg, float* values,
                             uint64_t n_problems, fc_solve_result* results);

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
