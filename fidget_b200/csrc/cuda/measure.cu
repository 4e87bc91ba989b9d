// fc_measure: volume, centre of mass, inertia and bounding box of a shape's voxel solid, from exact integer cell moments.
// The interval levels are the stacked octree's (k_tree_level with MEASURE folds the proven-inside cells); the brick kernel
// below classifies the cells of the ambiguous bricks by their centres; the host derives the float64 results.
#include <cmath>

#include "capi_internal.h"
#include "level_job.cuh"
#include "pass_plan.h"

namespace fdev {

// One warp per brick, claimed from the list.  A lane evaluates two of a 4^3 brick's cells at once (run_f32x2, one tape
// per brick); smaller bricks (depth < 2) leave lanes idle.  The sums stay in registers while the warp's bricks belong to
// one frame and are flushed, one set of atomics per warp, when the frame changes and at exit.
__global__ void __launch_bounds__(128) k_measure_brick(const __grid_constant__ MeasureBrickParams p, const MeshFrame* frames) {
    const int lane = threadIdx.x & 31;
    float2 slots[REG_SLOTS];
    const uint32_t n_jobs = min(p.ctr->n_jobs[p.list], p.cap_jobs);
    const uint32_t B = p.brick, nb = B * B * B;
    const float inv = 1.0f / float(1u << p.depth);   // 2^-D: the centre -1 + (2i + 1) 2^-D is exact in f32
    MeasureSums ms;
    ms.clear();
    uint32_t cur = ~0u;
    unsigned long long undecided = 0;
    auto flush = [&]() {
        ms.warp_fold();
        if (lane == 0) ms.flush(p.acc + cur, false, undecided);
        ms.clear();
        undecided = 0;
    };
    for (;;) {
        uint32_t j = 0;
        if (lane == 0) {
            j = atomicAdd(&p.ctr->cursor[p.cursor], 1u);
            if (j < n_jobs && cancel_poll(p.cancel, CS_MEASURE_BRICK, j)) j = ~0u;
        }
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_jobs) break;
        const TileJob* job = p.jobs + j;
        const uint32_t f = job->y / p.rows;
        if (f != cur) {
            if (cur != ~0u) flush();
            cur = f;
        }
        const uint32_t cx = job->x, cy = job->y - f * p.rows, cz = job->z;
        const TapeRef tr = job->tape;
        const MeshFrame& fr = frames[f];
        for (uint32_t q = 0; q < nb; q += 64u) {
            const uint32_t c0 = q + uint32_t(lane), c1 = c0 + 32u;
            const uint32_t e0 = c0 < nb ? c0 : 0u, e1 = c1 < nb ? c1 : 0u;
            const uint32_t i0 = cx + e0 % B, j0 = cy + (e0 / B) % B, k0 = cz + e0 / (B * B);
            const uint32_t i1 = cx + e1 % B, j1 = cy + (e1 / B) % B, k1 = cz + e1 / (B * B);
            float x0 = float(2u * i0 + 1u) * inv - 1.0f, y0 = float(2u * j0 + 1u) * inv - 1.0f,
                  z0 = float(2u * k0 + 1u) * inv - 1.0f;
            float x1 = float(2u * i1 + 1u) * inv - 1.0f, y1 = float(2u * j1 + 1u) * inv - 1.0f,
                  z1 = float(2u * k1 + 1u) * inv - 1.0f;
            if (fr.has_transform) {   // as the octree leaf's corners (k_octree_leaf)
                xform_f32(fr.mat, x0, y0, z0, x0, y0, z0);
                xform_f32(fr.mat, x1, y1, z1, x1, y1, z1);
            }
            const float2 X = make_float2(x0, x1), Y = make_float2(y0, y1), Z = make_float2(z0, z1);
            const float2 v = run_f32x2(tr.ptr, tr.n_ops, slots, [&](uint32_t i) {
                return pick_input(fr.vb, i, X, Y, Z, [](float s) { return make_float2(s, s); });
            });
            if (c0 < nb && v.x < 0.0f) ms.add_cell(i0, j0, k0);
            if (c1 < nb && v.y < 0.0f) ms.add_cell(i1, j1, k1);
        }
        undecided += nb;
    }
    if (cur != ~0u) flush();
}

void launch_measure_bricks(const MeasureBrickParams& p, const MeshFrame* frames, int blocks, cudaStream_t s) {
    k_measure_brick<<<blocks, 128, 0, s>>>(p, frames);
}

}  // namespace fdev

namespace {

// The float64 results of one frame from its integers (fc_measure_result's derived fields; see fidget_cuda.h)
void derive(const MeasureAcc& a, const fc_mesh_frame& fm, uint32_t D, fc_measure_result& r) {
    memset(&r, 0, sizeof r);
    r.n_inside = a.n_inside; r.n_proven = a.n_proven; r.n_undecided = a.n_undecided;
    for (int i = 0; i < 3; ++i) { r.s1[i] = a.s1[i]; r.lo[i] = a.lo[i]; r.hi[i] = a.hi[i]; }
    for (int i = 0; i < 6; ++i) r.s2[i] = a.s2[i];
    // the linear part A and translation t of world_to_model (the identity without a transform)
    double A[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}, t[3] = {0, 0, 0};
    if (fm.has_transform)
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) A[i][j] = fm.world_to_model[4 * i + j];
            t[i] = fm.world_to_model[4 * i + 3];
        }
    const double det = A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
                       A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
    const double scale = std::fabs(det), h3 = std::ldexp(1.0, 3 - 3 * int(D)), h = std::ldexp(1.0, 1 - int(D));
    r.volume_lo = double(a.n_proven) * h3 * scale;
    r.volume_hi = double(a.n_proven + a.n_undecided) * h3 * scale;
    const uint64_t N = a.n_inside;
    if (!N) {
        const double nan = std::nan("");
        for (int i = 0; i < 3; ++i) r.centroid[i] = r.bbox_min[i] = r.bbox_max[i] = nan;
        for (int i = 0; i < 6; ++i) r.inertia[i] = nan;
        return;
    }
    r.volume = double(N) * h3 * scale;
    // world centroid (s1 - N 2^D) / (N 2^D): the numerator is exact (|.| < 2^50), one rounding in the division
    const double n2d = std::ldexp(double(N), int(D));
    double c[3];
    for (int i = 0; i < 3; ++i) c[i] = double(int64_t(a.s1[i]) - int64_t(N << D)) / n2d;
    // world covariance: the numerators N s2 - s1 s1^T exactly in 128 bits (up to 2^98), then / N / N / 4^D
    static const int pair[6][2] = {{0, 0}, {1, 1}, {2, 2}, {0, 1}, {0, 2}, {1, 2}};
    double C[3][3];
    for (int k = 0; k < 6; ++k) {
        const int p = pair[k][0], q = pair[k][1];
        const __int128 num = (__int128)N * a.s2[k] - (__int128)a.s1[p] * a.s1[q];
        const double v = std::ldexp(double(num) / double(N) / double(N), -2 * int(D));
        C[p][q] = C[q][p] = v;
    }
    for (int i = 0; i < 3; ++i) C[i][i] += h * h / 12.0;
    // to model space: centroid A c + t, covariance A C A^T
    double cm[3], AC[3][3], Cm[3][3];
    for (int i = 0; i < 3; ++i) {
        cm[i] = t[i];
        for (int j = 0; j < 3; ++j) cm[i] += A[i][j] * c[j];
        for (int j = 0; j < 3; ++j) AC[i][j] = A[i][0] * C[0][j] + A[i][1] * C[1][j] + A[i][2] * C[2][j];
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Cm[i][j] = AC[i][0] * A[j][0] + AC[i][1] * A[j][1] + AC[i][2] * A[j][2];
    const double tr = Cm[0][0] + Cm[1][1] + Cm[2][2];
    for (int i = 0; i < 3; ++i) r.centroid[i] = cm[i];
    for (int k = 0; k < 6; ++k) {
        const int p = pair[k][0], q = pair[k][1];
        r.inertia[k] = r.volume * ((p == q ? tr : 0.0) - Cm[p][q]);
    }
    // the box of the 8 mapped corners of the world box
    double wlo[3], whi[3];
    for (int i = 0; i < 3; ++i) { wlo[i] = double(a.lo[i]) * h - 1.0; whi[i] = double(a.hi[i] + 1ull) * h - 1.0; }
    for (int i = 0; i < 3; ++i) { r.bbox_min[i] = INFINITY; r.bbox_max[i] = -INFINITY; }
    for (int k = 0; k < 8; ++k) {
        const double p[3] = {(k & 1) ? whi[0] : wlo[0], (k & 2) ? whi[1] : wlo[1], (k & 4) ? whi[2] : wlo[2]};
        for (int i = 0; i < 3; ++i) {
            const double m = t[i] + A[i][0] * p[0] + A[i][1] * p[1] + A[i][2] * p[2];
            r.bbox_min[i] = std::min(r.bbox_min[i], m);
            r.bbox_max[i] = std::max(r.bbox_max[i], m);
        }
    }
}

// The passes of a checked call: frame k's integers into acc[k].  The caller holds the context's lock.
int32_t measure_passes(fc_ctx* c, const fc_tape* tape, uint32_t D, bool timing, const std::vector<MeshFrame>& fr,
                       std::vector<MeasureAcc>& acc, float* device_ms, const CallCancel& cc) {
    const uint32_t N = uint32_t(fr.size());
    const uint32_t b = std::min<uint32_t>(D, 2), B = 1u << b;
    const int Lb = int(D - b) + 1;   // interval levels 0 .. D - b; the bricks are list Lb
    cudaStream_t s = c->stream;
    // a pass's cell rows must fit 32 bits
    PassPlan plan = tree_passes(c, N, uint32_t(std::min<uint64_t>({N, FC_MESH_MAX_PASS_FRAMES, 0xffffffffull >> D})), D, 3,
                                Lb, 0);
    MeasureAcc init{};
    for (int i = 0; i < 3; ++i) init.lo[i] = 0xffffffffu;
    std::vector<MeasureAcc> h_acc;
    while (plan.more()) {
        const PassPlan::Range r = plan.take();
        MeshFrame* d_fr = nullptr;
        MeasureAcc* d_acc = nullptr;
        CU(carve(c->mesh_frames, [&](Carve& cv) {
            cv.take(d_fr, size_t(r.n) * sizeof(MeshFrame));
            cv.take(d_acc, size_t(r.n) * sizeof(MeasureAcc));
        }));
        h_acc.assign(r.n, init);
        CU(cudaMemcpyAsync(d_fr, fr.data() + r.f0, size_t(r.n) * sizeof(MeshFrame), cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(d_acc, h_acc.data(), size_t(r.n) * sizeof(MeasureAcc), cudaMemcpyHostToDevice, s));
        TreeScratch t;
        if (int32_t trc = tree_scratch(c, tape, D, 3, r.n, 0, t)) return trc;
        if (timing) CU(cudaEventRecord(get_event(c, 0), s));
        for (int l = 0; l < Lb; ++l) {
            LevelParams p = tree_level(c, tape, t, l, fr[r.f0], cc);
            p.measure = d_acc;
            launch_tree_level_measure(p, d_fr, t.blocks(l), s);
        }
        MeasureBrickParams q{};
        q.jobs = c->jobs[Lb].as<TileJob>();
        q.cap_jobs = uint32_t(t.level_cap[Lb]);
        q.ctr = c->counters.as<Counters>();
        q.list = Lb; q.cursor = Lb;
        q.depth = D; q.brick = B; q.rows = 1u << D;
        q.acc = d_acc;
        q.cancel = cc.ref;
        launch_measure_bricks(q, d_fr, c->sm_count * 8, s);
        if (timing) CU(cudaEventRecord(get_event(c, 1), s));
        CU(cudaGetLastError());
        if (int32_t wrc = wait_read(c, s, cc, h_acc.data(), d_acc, size_t(r.n) * sizeof(MeasureAcc))) return wrc;
        Counters ctr;
        CU(cudaMemcpy(&ctr, c->counters.p, sizeof ctr, cudaMemcpyDeviceToHost));
        bool split = false;
        if (!plan.observe(ctr, 0, r, split)) return device_error(ctr.error);
        if (split) continue;
        if (timing && device_ms) {
            float ms = 0;
            cudaEventElapsedTime(&ms, get_event(c, 0), get_event(c, 1));
            *device_ms += ms;
        }
        std::copy(h_acc.begin(), h_acc.end(), acc.begin() + r.f0);
    }
    return FC_OK;
}

}  // namespace

extern "C" {

int32_t fc_measure(fc_ctx* c, const fc_tape* tape, const fc_octree_cfg* cfg, const fc_mesh_frame* frames, uint32_t n_frames,
                   fc_measure_result* out, float* device_ms) {
    static_assert(sizeof(fc_measure_result) == 264, "fc_measure_result layout");
    if (device_ms) *device_ms = 0;
    if (!c || !tape || !cfg) return fail(FC_ERR_INVALID, "null argument");
    if (n_frames && (!frames || !out)) return fail(FC_ERR_INVALID, "null frames or out");
    if (out && n_frames) memset(out, 0, size_t(n_frames) * sizeof *out);
    if (int32_t rc = check_tree_call(tape, 3, cfg->depth, frames, n_frames, "fc_measure")) return rc;
    std::vector<MeshFrame> fr(n_frames);
    for (uint32_t k = 0; k < n_frames; ++k) {
        const fc_mesh_frame& in = frames[k];
        if (in.has_transform && (in.world_to_model[12] != 0.0f || in.world_to_model[13] != 0.0f ||
                                 in.world_to_model[14] != 0.0f || in.world_to_model[15] != 1.0f))
            return fail(FC_ERR_UNSUPPORTED, "fc_measure needs an affine world_to_model (last row 0 0 0 1)");
        if (int32_t vrc = bind_frame(tape, in.has_transform, in.world_to_model, 0.0f, in.var_values, in.n_var_values, fr[k]))
            return vrc;
    }
    if (!n_frames) return FC_OK;
    const uint32_t D = cfg->depth;
    CallCancel cc;
    if (int32_t crc = begin_call(c, cc)) return crc;
    std::vector<MeasureAcc> acc(n_frames);
    int32_t rc;
    {
        std::lock_guard<std::mutex> guard(c->mu);
        CU(cudaSetDevice(c->device));
        rc = measure_passes(c, tape, D, (cfg->flags & FC_FLAG_TIMING) != 0, fr, acc, device_ms, cc);
    }
    if (rc) {
        memset(out, 0, size_t(n_frames) * sizeof *out);
        if (device_ms) *device_ms = 0;
        return rc;
    }
    for (uint32_t k = 0; k < n_frames; ++k) derive(acc[k], frames[k], D, out[k]);
    return FC_OK;
}

}  // extern "C"
