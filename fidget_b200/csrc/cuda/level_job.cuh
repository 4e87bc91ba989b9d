// One unit of work of the interval levels: a parent tile (or, at level 0, a group of 32 root tiles)
// whose children are evaluated by the lanes of one warp, classified, simplified and queued.  Shared
// by k_interval_level (one launch per level) and by the fused 2D kernel of tail2d.cu, where jobs of
// every level are claimed from one dependency-ordered queue inside a single persistent launch
// (FUSED): there a job becomes visible through a ready mark written after its fields, child tapes
// occupy whole 128-byte lines of the arena, and `outstanding` counts the jobs not yet finished.
#pragma once
#include "interp.cuh"

namespace fdev {

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }

// Waits until job slot `j` carries this render's ready mark, then reads it from L2 (another SM wrote it
// during this launch; L1 may hold a stale copy of the line).  Bounded: a lost job raises error bit 2.
// A cancelled call leaves the wait with ok = false (and no error bit); the job is then skipped.
__device__ __forceinline__ TileJob load_job_ready(const TileJob* j, uint32_t epoch, Counters* ctr, const CancelRef& cancel,
                                                  bool& ok) {
    uint32_t spins = 0;
    ok = true;
    while (ld_volatile_u32(&j->pad) != epoch) {
        if (cancel_poll(cancel, CS_WAIT, ~0u)) { ok = false; return TileJob{}; }
        __nanosleep(64);
        if (++spins > (1u << 22)) { atomicOr(&ctr->error, 4u); break; }
    }
    __threadfence();
    TileJob o;
    const uint2* q = reinterpret_cast<const uint2*>(j);
    const uint2 a = __ldcg(q), b = __ldcg(q + 1), c = __ldcg(q + 2), d = __ldcg(q + 3), e = __ldcg(q + 4);
    o.x = a.x; o.y = a.y; o.z = b.x; o.pad = b.y;
    o.tape.ptr = reinterpret_cast<const uint2*>((unsigned long long)c.x | ((unsigned long long)c.y << 32));
    o.tape.n_ops = d.x; o.tape.ref_len = d.y; o.tape.n_choices = e.x; o.tape.pad = e.y;
    return o;
}
__device__ __forceinline__ void publish_job(TileJob* dst, TileJob o, uint32_t epoch) {
    o.pad = 0;
    *dst = o;
    __threadfence();
    *reinterpret_cast<volatile uint32_t*>(&dst->pad) = epoch;
}
__device__ __forceinline__ void store_fill(FillRec* dst, const FillRec& fr) {
    *reinterpret_cast<uint4*>(dst) = make_uint4(fr.x, fr.y, fr.value, fr.ready);
}

// fc_measure's sums of one lane (MeasureAcc's fields but the brick count), folded over a warp and into a frame's
// accumulator.  A cell of edge T at (x0, y0, z0) (depth-D cell indices) holds T^3 cells; along one axis its odd numbers
// 2i + 1 sum to (x0 + T)^2 - x0^2 and their squares to F(x0 + T) - F(x0), F(m) = m (4 m^2 - 1) / 3.  Every term fits
// u64 up to depth 12 (T <= 2^12, sums of one axis <= 2^24, F <= 2^36.5).
struct MeasureSums {
    unsigned long long n, s1[3], s2[6];
    uint32_t lo[3], hi[3];
    __device__ __forceinline__ void clear() {
        n = 0;
        for (int a = 0; a < 3; ++a) { s1[a] = 0; s2[a] = 0; s2[a + 3] = 0; lo[a] = 0xffffffffu; hi[a] = 0u; }
    }
    __device__ __forceinline__ static unsigned long long odd_sq(unsigned long long m) { return m * (4ull * m * m - 1ull) / 3ull; }
    __device__ __forceinline__ void add_block(uint32_t x0, uint32_t y0, uint32_t z0, uint32_t T) {
        const uint32_t c[3] = {x0, y0, z0};
        const unsigned long long t = T, t2 = t * t;
        unsigned long long a1[3];
        for (int a = 0; a < 3; ++a) {
            const unsigned long long e = c[a] + t;
            a1[a] = e * e - (unsigned long long)c[a] * c[a];
            s1[a] += t2 * a1[a];
            s2[a] += t2 * (odd_sq(e) - odd_sq(c[a]));
            lo[a] = min(lo[a], c[a]);
            hi[a] = max(hi[a], c[a] + T - 1u);
        }
        n += t2 * t;
        s2[3] += t * a1[0] * a1[1];
        s2[4] += t * a1[0] * a1[2];
        s2[5] += t * a1[1] * a1[2];
    }
    __device__ __forceinline__ void add_cell(uint32_t i, uint32_t j, uint32_t k) {
        const unsigned long long u = 2u * i + 1u, v = 2u * j + 1u, w = 2u * k + 1u;
        ++n;
        s1[0] += u; s1[1] += v; s1[2] += w;
        s2[0] += u * u; s2[1] += v * v; s2[2] += w * w;
        s2[3] += u * v; s2[4] += u * w; s2[5] += v * w;
        lo[0] = min(lo[0], i); lo[1] = min(lo[1], j); lo[2] = min(lo[2], k);
        hi[0] = max(hi[0], i); hi[1] = max(hi[1], j); hi[2] = max(hi[2], k);
    }
    // the sums of the whole warp, in every lane
    __device__ __forceinline__ void warp_fold() {
        for (int o = 16; o > 0; o >>= 1) {
            n += __shfl_xor_sync(FULL, n, o);
            for (int a = 0; a < 3; ++a) {
                s1[a] += __shfl_xor_sync(FULL, s1[a], o);
                lo[a] = min(lo[a], __shfl_xor_sync(FULL, lo[a], o));
                hi[a] = max(hi[a], __shfl_xor_sync(FULL, hi[a], o));
            }
            for (int a = 0; a < 6; ++a) s2[a] += __shfl_xor_sync(FULL, s2[a], o);
        }
    }
    // into a frame's accumulator (one thread): n inside cells, of which `proven` in proven-inside cells, and `undecided`
    // brick cells
    __device__ __forceinline__ void flush(MeasureAcc* acc, bool proven, unsigned long long undecided) const {
        if (undecided) atomicAdd(&acc->n_undecided, undecided);
        if (!n) return;
        atomicAdd(&acc->n_inside, n);
        if (proven) atomicAdd(&acc->n_proven, n);
        for (int a = 0; a < 3; ++a) {
            atomicAdd(&acc->s1[a], s1[a]);
            atomicMin(&acc->lo[a], lo[a]);
            atomicMax(&acc->hi[a], hi[a]);
        }
        for (int a = 0; a < 6; ++a) atomicAdd(&acc->s2[a], s2[a]);
    }
};

// The simplification of a warp's ambiguous children (render/mod.rs:96-152: keep the child only if it is shorter): the
// lanes whose choices (`pk`, packed at `cs` by the interval walk of `tr`) trace something claim one arena slot each and
// simplify `tr` into it.  Returns this lane's child tape, `tr` itself when it is not simplified or not shorter; `kept`
// says which.  An exhausted arena sets error bit 0 and keeps every parent tape.  Shared by level_job and the ray
// levels (ray.cu); the warp calls it together.
template <bool FUSED>
__device__ __forceinline__ TapeRef simplify_children(const LevelParams& p, const TapeRef& tr, bool amb, const ChoicePacker& pk,
                                                     uint32_t* cs, uint32_t (*live)[32], int lane, bool& kept) {
    TapeRef child = tr;
    kept = false;
    const bool need = amb && pk.any_nonboth;
    const uint32_t mneed = __ballot_sync(FULL, need);
    if (mneed) {
        const uint32_t total = __popc(mneed);
        // worst-case slot per child; in the fused kernel slots are whole 128-byte lines, so that a line
        // written for one tape is never one an SM may already hold in L1 for another
        const uint32_t slot_ops = FUSED ? ((tr.n_ops + 15u) & ~15u) : tr.n_ops;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(&p.ctr->arena_top, (unsigned long long)total * slot_ops + (FUSED ? 15u : 0u));
        base = __shfl_sync(FULL, base, 0);
        if (FUSED) base = (base + 15ull) & ~15ull;   // (the root level's tapes end anywhere)
        if (base + (unsigned long long)total * slot_ops > p.arena_cap) {
            if (lane == 0) atomicOr(&p.ctr->error, 1u);
        } else {
            const uint32_t rank = __popc(mneed & lanemask_lt());
            unsigned long long end = base + (unsigned long long)(rank + 1u) * slot_ops;
            ChoiceUnpacker cu;
            cu.base = cs;
            cu.ci = tr.n_choices;
            uint32_t n_dev, ref_len, nch;
            simplify_lane<!FUSED>(tr.ptr, tr.n_ops, need, live, lane, cu, p.arena + end, n_dev, ref_len, nch);
            bool keep = need && ref_len < tr.ref_len;
            kept = keep;
            if (keep) {
                child.ptr = p.arena + (end - n_dev);
                child.n_ops = n_dev;
                child.ref_len = ref_len;
                child.n_choices = nch;
            }
            if (p.stats) {
                uint32_t mk = __ballot_sync(FULL, keep);
                if (lane == 0 && mk) atomicAdd(&p.stats->simplified[p.level], (unsigned long long)__popc(mk));
            }
        }
    }
    return child;
}

// TREE: the samplers' trees whose cells read their view from a ContourSlice table (a MeshFrame is the same record, z
// unused), not from the render parameters.  DIM 2: the quadtree of
// fc_contour_build.  Coordinates are cells at the finest depth with world-square bounds coord * cell_h - 1, seen through
// `mat` when has_transform, at Z = [z2d, z2d]; classified tiles are dropped (no fills).  With FRAMES a contour slice
// stack: each cell's slice (`slices`, frame_rows rows each) supplies Z, the matrix, its has_transform and the vars, and
// the cell's rows are relative to its slice.  DIM 3 with FRAMES (octree mode 1): the stacked octree of a mesh frame
// batch, each cell's frame read the same way (its Z is the cell's own).  MEASURE (DIM 3, TREE, FRAMES: fc_measure): the
// block moments and box of the lanes' proven-inside cells go into their frame's accumulator, p.measure[cell row /
// frame_rows]; a warp's children share one frame, the root cells of level 0 each have their own.  VOLUME (DIM 3, TREE,
// FRAMES: fc_volume_build): cells are proven against -vol->band and vol->band instead of 0, and every proven cell is
// appended to vol's tile list, one atomic per warp.
template <int DIM, bool FUSED, bool FRAMES = false, bool SCENE = false, bool TREE = false, bool MEASURE = false,
          bool VOLUME = false>
__device__ __forceinline__ void level_job(const LevelParams& p, uint32_t j, uint32_t n_roots, itv* slots, uint32_t* cs,
                                          uint32_t (*live)[32], int lane, uint32_t epoch,
                                          const ContourSlice* slices = nullptr, const VolumeLevel* vol = nullptr) {
    const uint32_t T = p.tile;
    bool cull_open = false, cull_check = false;
    TapeRef tr;
    uint32_t px = 0, py = 0, pz = 0, nchild, ppl = 0;   // (SCENE: ppl = the parent's placement)
    if (p.root_mode) {
        tr = p.root_tape;
        nchild = min(32u, n_roots - j * 32u);
    } else {
        bool ok = true;
        const TileJob jb = FUSED ? load_job_ready(p.jobs_in + j, epoch, p.ctr, p.cancel, ok) : p.jobs_in[j];
        if (FUSED && __any_sync(FULL, !ok)) return;   // cancelled while waiting for the record
        px = jb.x;
        py = jb.y;
        pz = jb.z;
        tr = jb.tape;
        if (SCENE) ppl = jb.pad;
        nchild = p.n_axis * p.n_axis * (DIM == 3 ? p.n_axis : 1u);
        if (DIM == 3 && p.mode != 1u && p.cull) {
            // Every pixel under this parent already holds depth >= its top + 1 (tiles in front, proven inside by coarser
            // levels): nothing inside can show, so none of its children is evaluated.  The reference skips the same
            // tiles in its front-to-back walk (voxel.rs:283-293) -- and more, since it also knows the voxel hits in
            // front, which arrive last here.  One small read of the occlusion map per lane, not the heightmap itself.
            const uint32_t nb = (T * p.n_axis) / 16u, need = pz + T * p.n_axis + 1u;   // blocks per side of the parent
            const uint32_t fb0 = frame_of<FRAMES>(p, py).y0 / 16u;                      // (frame batch: its first block row)
            // (scene: every block must hold at least the rank of this placement's fill at top + 1: a greater depth, or
            //  that depth from this placement or a lower one -- a tie with a higher placement must still be evaluated)
            const unsigned long long need_rank = SCENE ? scene_rank(need, ppl, p.clamp_at, p.depth) : 0ull;
            for (uint32_t q = lane; q < nb * nb; q += 32u) {
                const uint32_t bx = px / 16u + q % nb, by = py / 16u + q / nb;
                if (bx < p.occl_w && by - fb0 < p.occl_h) {
                    if constexpr (SCENE) cull_open |= __ldcg(reinterpret_cast<const unsigned long long*>(p.occl) + size_t(by) * p.occl_w + bx) < need_rank;
                    else cull_open |= __ldcg(p.occl + size_t(by) * p.occl_w + bx) < need;
                }
            }
            cull_check = true;
        }
    }
    const uint2* tape = tr.ptr;

    for (uint32_t chunk = 0; chunk * 32u < nchild; ++chunk) {
        const uint32_t c = chunk * 32u + lane;
        bool valid = c < nchild;
        uint32_t cx, cy, cz = 0, pl = ppl;
        if (p.root_mode) {
            if (SCENE) pl = scene_root(p, j * 32u + (valid ? c : 0u), T, cx, cy, cz);
            else root_corner(p, j * 32u + (valid ? c : 0u), T, cx, cy, cz);
        } else {
            uint32_t cc = valid ? c : 0u;
            cx = px + (cc % p.n_axis) * T;
            cy = py + ((cc / p.n_axis) % p.n_axis) * T;
            if (DIM == 3) cz = pz + (cc / (p.n_axis * p.n_axis)) * T;
        }
        if constexpr (DIM == 2 && SCENE) {   // a tile under higher shapes' proven interiors is not evaluated (Scene2D)
            valid = valid && !scene2d_hidden(p.occl, p.occl_w, p.occl_h, p.cull, cx, cy, T, pl);
            if (!__any_sync(FULL, valid)) continue;
        }
        // Region in screen coordinates -> model space (pixel.rs:325-342, voxel.rs:291-306); in a frame batch a
        // tile's coordinates are relative to its frame (per lane at level 0, whose 32 roots may span frames)
        const FrameView fv = TREE ? quad_view<FRAMES>(p, slices, cy) : view_of<FRAMES, SCENE>(p, cy, pl);
        const Mat4& M = *fv.mat;
        const VarBind& vb = *fv.vb;
        itv X = iv(float(cx), float(cx) + float(T));
        itv Y = iv(float(cy - fv.y0), float(cy - fv.y0) + float(T));
        itv Z = DIM == 3 ? iv(float(cz), float(cz) + float(T)) : iv(fv.z, fv.z);
        itv vx, vy, vz;
        if (DIM == 3 && p.mode == 1u) {
            // octree cell bounds in world space (CellBounds::child, cell.rs:155-166): dyadic, exact in f32
            // (TREE: a mesh frame batch -- the rows are the frame's, and the frame supplies matrix and has_transform)
            const float h = p.cell_h;
            const uint32_t ry = TREE ? cy - fv.y0 : cy;
            X = iv(float(cx) * h - 1.0f, float(cx + T) * h - 1.0f);
            Y = iv(float(ry) * h - 1.0f, float(ry + T) * h - 1.0f);
            Z = iv(float(cz) * h - 1.0f, float(cz + T) * h - 1.0f);
            if (TREE ? quad_has_transform<FRAMES>(p, slices, cy) : p.has_transform) xform_iv(TREE ? M : p.mat, X, Y, Z, vx, vy, vz);
            else { vx = X; vy = Y; vz = Z; }
        } else if constexpr (TREE) {
            const float h = p.cell_h;
            const uint32_t ry = cy - fv.y0;
            X = iv(float(cx) * h - 1.0f, float(cx + T) * h - 1.0f);
            Y = iv(float(ry) * h - 1.0f, float(ry + T) * h - 1.0f);
            if (quad_has_transform<FRAMES>(p, slices, cy)) xform_iv(FRAMES ? M : p.mat, X, Y, Z, vx, vy, vz);
            else { vx = X; vy = Y; vz = Z; }
        } else {
            xform_iv(M, X, Y, Z, vx, vy, vz);
        }

        if (DIM == 3 && cull_check && chunk == 0) {
            if (!__any_sync(FULL, cull_open)) {
                if (p.stats && lane == 0) atomicAdd(&p.stats->culled[p.level], (unsigned long long)nchild);
                return;
            }
        }
        ChoicePacker pk;
        pk.base = cs;
        itv r = iv_nan();
        run_interval<!FUSED>(
            tape, tr.n_ops, slots,
            [&](uint32_t i) { return pick_input(vb, i, vx, vy, vz, [](float f) { return iv1(f); }); }, pk,
            [&](uint32_t oi, itv v) { if (oi == 0) r = v; });
        pk.finish();

        const float band = VOLUME ? vol->band : 0.0f;
        const bool fill_in = valid && !p.pixel_perfect && r.y < (VOLUME ? -band : 0.0f);
        const bool fill_out = valid && !p.pixel_perfect && !fill_in && r.x > band;
        const bool amb = valid && !fill_in && !fill_out;

        if constexpr (MEASURE) {
            static_assert(DIM == 3 && TREE && FRAMES, "fc_measure's levels are the stacked octree's");
            if (__any_sync(FULL, fill_in)) {
                MeasureSums ms;
                ms.clear();
                if (fill_in) ms.add_block(cx, cy - fv.y0, cz, T);
                if (p.root_mode) {
                    if (fill_in) ms.flush(p.measure + cy / p.frame_rows, true, 0);
                } else {
                    ms.warp_fold();
                    if (lane == 0) ms.flush(p.measure + cy / p.frame_rows, true, 0);
                }
            }
        }
        if constexpr (VOLUME) {
            static_assert(DIM == 3 && TREE && FRAMES, "fc_volume_build's levels are the stacked octree's");
            const bool proven = fill_in || fill_out;
            const uint32_t mp = __ballot_sync(FULL, proven);
            if (mp) {
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd(vol->n_tiles, uint32_t(__popc(mp)));
                base = __shfl_sync(FULL, base, 0);
                if (proven) {
                    const uint32_t slot = base + __popc(mp & lanemask_lt());
                    if (slot < vol->cap_tiles)
                        vol->tiles[slot] = volume_tile_key(cy / p.frame_rows, cx, cy - fv.y0, cz, uint32_t(__ffs(T) - 1), fill_in);
                    else atomicOr(&p.ctr->error, 2u);
                }
            }
        }
        if (DIM == 3) {
            // full tile: depth = max(depth, top + 1) over its footprint (voxel.rs:310-317)
            uint32_t m = p.mode == 1u ? 0u : __ballot_sync(FULL, fill_in);
            while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                const uint32_t fx = __shfl_sync(FULL, cx, src), fy = __shfl_sync(FULL, cy, src),
                               fz = __shfl_sync(FULL, cz, src);
                // (scene: the fill's rank, which carries its placement)
                const unsigned long long key = SCENE ? scene_rank(fz + T + 1u, __shfl_sync(FULL, pl, src), p.clamp_at, p.depth)
                                                     : (unsigned long long)(fz + T + 1u) << 32;
                // (frame batch: rows past the bottom of the tile's frame are its padding, not the next frame's image)
                const uint32_t fy0 = frame_of<FRAMES>(p, fy).y0;
                for (uint32_t q = lane; q < T * T; q += 32u) {
                    const uint32_t x = fx + q % T, y = fy + q / T;
                    if (x < p.width && y - fy0 < p.height) atomicMax(&p.heightmap[size_t(y) * p.width + x], key);
                }
                if (p.occl && T % 16u == 0u)   // the whole blocks this tile covers now hold its depth (the same value the heightmap gets)
                    for (uint32_t q = lane; q < (T / 16u) * (T / 16u); q += 32u) {
                        const uint32_t bx = fx / 16u + q % (T / 16u), by = fy / 16u + q / (T / 16u);
                        if (bx < p.occl_w && by - fy0 / 16u < p.occl_h) {
                            if (SCENE) atomicMax(reinterpret_cast<unsigned long long*>(p.occl) + size_t(by) * p.occl_w + bx, key);
                            else atomicMax(p.occl + size_t(by) * p.occl_w + bx, fz + T + 1u);
                        }
                    }
            }
            if (p.stats) {
                uint32_t mv = __ballot_sync(FULL, valid), mi = __ballot_sync(FULL, fill_in),
                         mo = __ballot_sync(FULL, fill_out), ma = __ballot_sync(FULL, amb);
                if (lane == 0) {
                    atomicAdd(&p.stats->evaluated[p.level], (unsigned long long)__popc(mv));
                    if (mi) atomicAdd(&p.stats->filled_inside[p.level], (unsigned long long)__popc(mi));
                    if (mo) atomicAdd(&p.stats->filled_outside[p.level], (unsigned long long)__popc(mo));
                    if (ma) atomicAdd(&p.stats->ambiguous[p.level], (unsigned long long)__popc(ma));
                }
            }
        } else {
            if constexpr (SCENE) {
                // 2D scene: an inside tile raises its blocks of the write cover map; nothing is painted
                uint32_t m = __ballot_sync(FULL, fill_in);
                uint32_t* const cover_out = p.occl + size_t(p.occl_w) * p.occl_h;
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    scene2d_cover(cover_out, p.occl_w, p.occl_h, p.cull, __shfl_sync(FULL, cx, src),
                                  __shfl_sync(FULL, cy, src), T, __shfl_sync(FULL, pl, src), lane, 32u);
                }
            } else if constexpr (!TREE) {
                uint32_t m = __ballot_sync(FULL, fill_in || fill_out);
                if (m) {
                    uint32_t base = 0;
                    if (lane == 0) base = atomicAdd(&p.ctr->n_fills[p.level], uint32_t(__popc(m)));
                    base = __shfl_sync(FULL, base, 0);
                    if (fill_in || fill_out) {
                        uint32_t slot = base + __popc(m & lanemask_lt());
                        if (slot < p.cap_fills) {
                            FillRec fr;
                            fr.x = cx;
                            fr.y = cy;
                            fr.value = 0x7FC00000u | (uint32_t(p.level & 0xff) << 1) | (fill_in ? 1u : 0u) | (0xF6u << 9);
                            fr.ready = epoch;
                            store_fill(p.fills + slot, fr);   // one 16-byte store: the ready mark travels with the record
                        } else {
                            atomicOr(&p.ctr->error, 2u);
                        }
                    }
                }
            }
            if (p.stats) {
                uint32_t mv = __ballot_sync(FULL, valid), mi = __ballot_sync(FULL, fill_in),
                         mo = __ballot_sync(FULL, fill_out), ma = __ballot_sync(FULL, amb);
                if (lane == 0) {
                    atomicAdd(&p.stats->evaluated[p.level], (unsigned long long)__popc(mv));
                    if (mi) atomicAdd(&p.stats->filled_inside[p.level], (unsigned long long)__popc(mi));
                    if (mo) atomicAdd(&p.stats->filled_outside[p.level], (unsigned long long)__popc(mo));
                    if (ma) atomicAdd(&p.stats->ambiguous[p.level], (unsigned long long)__popc(ma));
                }
            }
        }

        bool kept = false;
        const TapeRef child = simplify_children<FUSED>(p, tr, amb, pk, cs, live, lane, kept);

        if (DIM == 3 && p.census) {   // exact census: what this launch evaluated, judged later against the final heightmap
            const uint32_t mv = __ballot_sync(FULL, valid);
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(&p.ctr->n_census, uint32_t(__popc(mv)));
            base = __shfl_sync(FULL, base, 0);
            if (valid) {
                const uint32_t slot = base + __popc(mv & lanemask_lt());
                if (slot < p.cap_census) {
                    CensusRec r;
                    r.x = uint16_t(cx); r.y = uint16_t(cy); r.z = uint16_t(cz);
                    r.level = uint8_t(p.level);
                    r.flags = uint8_t((fill_in ? 1u : (fill_out ? 0u : 2u)) | (kept ? 4u : 0u));
                    p.census[slot] = r;
                } else atomicOr(&p.ctr->error, 2u);
            }
        }

        // queue ambiguous children for the next level
        const uint32_t mamb = __ballot_sync(FULL, amb);
        if (mamb) {
            uint32_t base = 0;
            if (lane == 0) {
                if (FUSED || p.fused_tail) {   // (only the fused kernel reads `outstanding`; it may consume a root launch's jobs)
                    atomicAdd(&p.ctr->outstanding, uint32_t(__popc(mamb)));   // before the jobs become claimable
                    if (FUSED) __threadfence();
                }
                base = atomicAdd(&p.ctr->n_jobs[p.level + 1], uint32_t(__popc(mamb)));
            }
            base = __shfl_sync(FULL, base, 0);
            if (amb) {
                uint32_t slot = base + __popc(mamb & lanemask_lt());
                if (slot < p.cap_out) {
                    TileJob o;
                    o.x = cx;
                    o.y = cy;
                    o.z = cz;
                    o.pad = 0;
                    o.tape = child;
                    if (FUSED) publish_job(p.jobs_out + slot, o, epoch);   // fields, fence, then the ready mark
                    else { o.pad = SCENE ? pl : epoch; p.jobs_out[slot] = o; }
                } else {
                    atomicOr(&p.ctr->error, 2u);
                    if (FUSED || p.fused_tail) atomicSub(&p.ctr->outstanding, 1u);   // never claimable: do not wait for it
                }
            }
        }
    }

}

}  // namespace fdev
