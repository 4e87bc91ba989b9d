// Persistent-CTA bulk evaluators for the trait-level slices (VmFloatSliceEval / VmGradSliceEval,
// fidget-core/src/vm/mod.rs:800-1085, 1097-1396) on short tapes, where the path is genuinely bound by
// HBM traffic (SURVEY.md section 8d: 16 B per point for f32, 64 B per point for gradients).
//
//  * one CTA per SM slot, looping over tiles of 256 float4 per variable (1024 points for f32 -- four
//    consecutive points per thread -- or 256 points for gradients);
//  * the tile's X/Y/Z/... slices arrive in shared memory through the TMA engine: one elected thread
//    issues `cp.async.bulk.shared::cluster.global` per variable against an mbarrier with an expected
//    byte count, three stages deep, so the loads of tiles t+1 and t+2 are in flight while tile t is
//    evaluated and no thread spends issue slots on address arithmetic or LDG;
//  * the tape itself is staged in shared memory once per CTA (bulk copy as well) and walked from there
//    with warp-uniform LDS;
//  * the tape's VM registers live in shared memory as [register][thread] float4 columns (conflict-free
//    128-bit accesses), nothing spills to local memory;
//  * results leave with one coalesced 128-bit store per thread and output.
// Tapes that do not fit the fast path (memory spills, many registers, unaligned slices) take the
// per-thread kernels of kernels.cu.
#include <algorithm>

#include "interp.cuh"

namespace fdev {

constexpr int TMA_THREADS = int(SLICE_TMA_TILE);   // one float4 per thread and variable
constexpr int TMA_STAGES = 3;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(b)), "r"(parity)
            : "memory");
    } while (!ok);
}

size_t slice_tma_smem(uint32_t n_ops, uint32_t n_vars, uint32_t n_regs) {
    return 128 + ((size_t(n_ops) * 8 + 127) & ~size_t(127)) + size_t(TMA_STAGES) * std::max(n_vars, 1u) * TMA_THREADS * 16 +
           size_t(std::max(n_regs, 1u)) * TMA_THREADS * 16;
}

template <bool GRAD>
__global__ void __launch_bounds__(TMA_THREADS) k_slice_tma(const __grid_constant__ SliceTmaParams p) {
    extern __shared__ __align__(128) unsigned char sm[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm);   // [TMA_STAGES] tile barriers, then the tape barrier
    uint2* tape_s = reinterpret_cast<uint2*>(sm + 128);
    const uint32_t nv = max(p.n_vars, 1u);
    float4* stage = reinterpret_cast<float4*>(sm + 128 + ((size_t(p.n_ops) * 8 + 127) & ~size_t(127)));
    float4* slots = stage + size_t(TMA_STAGES) * nv * TMA_THREADS;   // [register][thread]
    const uint32_t tid = threadIdx.x;
    constexpr uint32_t PTS = GRAD ? 1u : 4u;   // points per float4
    const uint64_t tiles = p.n / (uint64_t(TMA_THREADS) * PTS);   // full tiles; the ragged tail is handled below
    const uint32_t tile_bytes = TMA_THREADS * 16;

    if (tid == 0) {
        for (int s = 0; s <= TMA_STAGES; ++s) mbar_init(&bars[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](uint64_t tile, uint32_t s) {   // elected thread: one bulk copy per variable
        mbar_expect_tx(&bars[s], p.n_vars * tile_bytes);
        for (uint32_t k = 0; k < p.n_vars; ++k)
            bulk_g2s(stage + (size_t(s) * nv + k) * TMA_THREADS, p.vars[k] + tile * TMA_THREADS, tile_bytes, &bars[s]);
    };
    if (tid == 0) {
        const uint32_t even = (p.n_ops * 8u) & ~15u;   // bulk copies move multiples of 16 bytes
        mbar_expect_tx(&bars[TMA_STAGES], even);
        if (even) bulk_g2s(tape_s, p.tape, even, &bars[TMA_STAGES]);
        for (uint32_t s = 0; s < TMA_STAGES; ++s) {
            const uint64_t t = blockIdx.x + uint64_t(s) * gridDim.x;
            if (t < tiles) issue(t, s);
        }
    }
    if ((p.n_ops & 1u) && tid == 32) tape_s[p.n_ops - 1] = __ldg(p.tape + (p.n_ops - 1));   // odd tail clause
    mbar_wait(&bars[TMA_STAGES], 0);
    __syncthreads();

    auto run = [&](const float4* in /* [nv] strided by TMA_THREADS, already offset by tid */, uint32_t in_stride,
                   float4& res0, float4& res1) {
        float4* my = slots + tid;
        uint2 nxt = tape_s[0];
        for (uint32_t i = 0; i < p.n_ops; ++i) {
            const uint2 w = nxt;
            nxt = tape_s[i + 1 < p.n_ops ? i + 1 : i];   // the clause stream stays one LDS ahead of the arithmetic
            Dec d(w.x);
            const float imm = __uint_as_float(w.y);
            float4 r;
            bool handled = false;
            if (!GRAD) {
                // the CSG opcodes go through the per-(opcode, form) handlers of interp.cuh's dispatch table
                const uint32_t x = w.x;
                const float4 im = make_float4(imm, imm, imm, imm);
#define TMA_L my[size_t((x >> 16) & 0xffu) * TMA_THREADS]
#define TMA_R my[size_t(x >> 24) * TMA_THREADS]
#define TMA_BIN(H, EXPR)                                                                      \
    case H##_RR: { const float4 a = TMA_L, b = TMA_R; r = EXPR; handled = true; break; }      \
    case H##_RI: { const float4 a = TMA_L, b = im; r = EXPR; handled = true; break; }         \
    case H##_IR: { const float4 a = im, b = TMA_R; r = EXPR; handled = true; break; }
                switch (c_dop.h[x & 0xffu]) {
                    TMA_BIN(H_ADD, make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w))
                    TMA_BIN(H_SUB, make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w))
                    TMA_BIN(H_MUL, make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w))
                    TMA_BIN(H_MIN, make_float4(f_min(a.x, b.x), f_min(a.y, b.y), f_min(a.z, b.z), f_min(a.w, b.w)))
                    TMA_BIN(H_MAX, make_float4(f_max(a.x, b.x), f_max(a.y, b.y), f_max(a.z, b.z), f_max(a.w, b.w)))
                    case H_NEG: { const float4 a = TMA_L; r = make_float4(-a.x, -a.y, -a.z, -a.w); handled = true; break; }
                    case H_ABS: { const float4 a = TMA_L; r = make_float4(fabsf(a.x), fabsf(a.y), fabsf(a.z), fabsf(a.w)); handled = true; break; }
                    case H_SQRT: { const float4 a = TMA_L; r = make_float4(sqrtf(a.x), sqrtf(a.y), sqrtf(a.z), sqrtf(a.w)); handled = true; break; }
                    case H_SQUARE: { const float4 a = TMA_L; r = make_float4(a.x * a.x, a.y * a.y, a.z * a.z, a.w * a.w); handled = true; break; }
                    case H_COPY_REG: r = TMA_L; handled = true; break;
                    case H_COPY_IMM: r = im; handled = true; break;
                    default: break;
                }
#undef TMA_BIN
#undef TMA_L
#undef TMA_R
            }
            if (handled) {
            } else if (d.op == OP_INPUT) {
                r = in[size_t(w.y) * in_stride];
            } else if (d.op == OP_OUTPUT) {
                const float4 v = my[size_t(d.lhs) * TMA_THREADS];
                if (w.y & 1u) res1 = v; else res0 = v;
                continue;
            } else if (d.op == OP_COPY) {
                if (d.form == F_RI) r = GRAD ? gr1(imm) : make_float4(imm, imm, imm, imm);
                else r = my[size_t(d.lhs) * TMA_THREADS];
            } else if (d.op < OP_ADD) {
                const float4 sl = my[size_t(d.lhs) * TMA_THREADS];
                r = GRAD ? gr_unary(d.op, sl) : f32x4_unary(d.op, sl);
            } else {
                // an immediate operand has no register behind it (0xff): only touch the columns that exist
                const float4 im = GRAD ? gr1(imm) : make_float4(imm, imm, imm, imm);
                float4 a = im, b = im;
                if (d.form != F_IR) a = my[size_t(d.lhs) * TMA_THREADS];
                if (d.form != F_RI) b = my[size_t(d.rhs) * TMA_THREADS];
                if (GRAD) r = (d.op == OP_MUL && d.form == F_RI) ? gr_mul_f(a, imm) : gr_binary(d.op, a, b);
                else r = f32x4_binary(d.op, a, b);
            }
            my[size_t(d.out) * TMA_THREADS] = r;
        }
    };

    uint32_t it = 0;
    for (uint64_t t = blockIdx.x; t < tiles; t += gridDim.x, ++it) {
        const uint32_t s = it % TMA_STAGES, parity = (it / TMA_STAGES) & 1u;
        mbar_wait(&bars[s], parity);
        float4 res[2];
        run(stage + size_t(s) * nv * TMA_THREADS + tid, TMA_THREADS, res[0], res[1]);
        p.outs[0][t * TMA_THREADS + tid] = res[0];   // 128-bit, coalesced
        if (p.n_outputs > 1) p.outs[1][t * TMA_THREADS + tid] = res[1];
        __syncthreads();   // every thread has consumed stage s
        const uint64_t nt = t + uint64_t(TMA_STAGES) * gridDim.x;
        if (tid == 0 && nt < tiles) issue(nt, s);
    }

    // ragged tail (fewer points than a tile): the CTA that would own tile `tiles` reads it with guarded loads
    const uint64_t done = tiles * TMA_THREADS * PTS;
    if (done < p.n && blockIdx.x == tiles % gridDim.x) {
        __syncthreads();
        float4* tail = stage;   // stage 0 is free: all tiles of this CTA are consumed
        const uint64_t base = done + uint64_t(tid) * PTS;
        for (uint32_t k = 0; k < p.n_vars; ++k) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (GRAD) {
                if (base < p.n) v = p.vars[k][base];
            } else {
                const float* src = reinterpret_cast<const float*>(p.vars[k]);
                if (base + 0 < p.n) v.x = src[base + 0];
                if (base + 1 < p.n) v.y = src[base + 1];
                if (base + 2 < p.n) v.z = src[base + 2];
                if (base + 3 < p.n) v.w = src[base + 3];
            }
            tail[size_t(k) * TMA_THREADS + tid] = v;
        }
        float4 res[2];
        run(tail + tid, TMA_THREADS, res[0], res[1]);
#pragma unroll
        for (uint32_t o = 0; o < 2; ++o) {
            if (o >= p.n_outputs) break;
            if (GRAD) {
                if (base < p.n) p.outs[o][base] = res[o];
            } else {
                float* dst = reinterpret_cast<float*>(p.outs[o]);
                if (base + 0 < p.n) dst[base + 0] = res[o].x;
                if (base + 1 < p.n) dst[base + 1] = res[o].y;
                if (base + 2 < p.n) dst[base + 2] = res[o].z;
                if (base + 3 < p.n) dst[base + 3] = res[o].w;
            }
        }
    }
}

// Returns the number of CTAs launched, or 0 when the fast path does not apply (the caller then uses the per-thread
// kernel)
unsigned launch_slice_tma(const SliceTmaParams& p, bool grad, int sm_count, cudaStream_t s) {
    if (p.n_vars > 4 || p.n_outputs == 0 || p.n_outputs > 2 || p.n_regs > 40 || p.n_ops == 0 || p.n_ops > 2048) return 0;
    for (uint32_t k = 0; k < p.n_vars; ++k) if (reinterpret_cast<uintptr_t>(p.vars[k]) & 15u) return 0;
    for (uint32_t o = 0; o < p.n_outputs; ++o) if (reinterpret_cast<uintptr_t>(p.outs[o]) & 15u) return 0;
    if (reinterpret_cast<uintptr_t>(p.tape) & 15u) return 0;
    const size_t smem = slice_tma_smem(p.n_ops, p.n_vars, p.n_regs);
    if (smem > 220 * 1024) return 0;
    auto kern = grad ? k_slice_tma<true> : k_slice_tma<false>;
    static size_t configured[2] = {0, 0};
    if (smem > configured[grad]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) {
            cudaGetLastError();
            return 0;
        }
        configured[grad] = smem;
    }
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, TMA_THREADS, smem) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        return 0;
    }
    const uint64_t tiles = p.n / (uint64_t(TMA_THREADS) * (grad ? 1 : 4)) + 1;
    const unsigned grid = unsigned(std::min<uint64_t>(tiles, uint64_t(sm_count) * per_sm));
    kern<<<grid, TMA_THREADS, smem, s>>>(p);
    return grid;
}

}  // namespace fdev
