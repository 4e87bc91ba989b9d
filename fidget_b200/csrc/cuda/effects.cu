// Post-processing effects of fidget-raster (fidget-raster/src/effects.rs:13-547,
// GeometryPixel::to_color voxel.rs:136-153) as sm_90a kernels: one thread per pixel,
// images stay in HBM/L2 between the passes.
//
// Vector arithmetic keeps nalgebra's evaluation order for fixed 3-vectors
// (dot = (a0*b0 + a1*b1) + a2*b2; normalize divides by sqrt(dot); mat3*vec3 accumulates
// column by column) and the file is compiled with -fmad=false -prec-div -prec-sqrt, so that
// every IEEE result matches the CPU bit for bit.  Only to_rgba_distance (exp, cos) is
// within one 8-bit step instead.
#include <cuda_runtime.h>

#include <cstdint>

#include "effects.cuh"

namespace fdev {
namespace {

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3(float x, float y, float z) { return V3{x, y, z}; }
__device__ __forceinline__ V3 add(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 sub(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 mul(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ V3 divs(V3 a, float s) { return v3(a.x / s, a.y / s, a.z / s); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ V3 normalize(V3 a) { return divs(a, sqrtf(dot(a, a))); }
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
    return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// Rust `f as u8`: saturating, truncating, NaN -> 0
__device__ __forceinline__ uint8_t as_u8(float f) {
    if (!(f > 0.0f)) return 0;
    if (f >= 255.0f) return 255;
    return uint8_t(int(f));
}
// f32::clamp: NaN passes through
__device__ __forceinline__ float clampf(float x, float lo, float hi) {
    if (x < lo) x = lo;
    if (x > hi) x = hi;
    return x;
}
// ordered_float::OrderedFloat: NaN is the greatest value and equal to itself
__device__ __forceinline__ int ord_cmp(float a, float b) {
    const bool an = a != a, bn = b != b;
    if (an) return bn ? 0 : 1;
    if (bn) return -1;
    return a < b ? -1 : (a > b ? 1 : 0);
}
// fidget-core/src/rng/mod.rs:8-33
__device__ __forceinline__ uint32_t rng_hash(uint32_t v) {
    const uint32_t state = v * 747796405u + 2891336453u;
    const uint32_t word = ((state >> ((state >> 28) + 4)) ^ state) * 277803737u;
    return (word >> 22) ^ word;
}
__device__ __forceinline__ uint32_t rng_mix(uint32_t a, uint32_t b) { return rng_hash(a + rng_hash(b)); }

__device__ __forceinline__ GeoPixel load_geo(const GeoPixel* img, size_t i) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(img) + i);
    GeoPixel g;
    g.normal[0] = v.x; g.normal[1] = v.y; g.normal[2] = v.z; g.depth = __float_as_uint(v.w);
    return g;
}
__device__ __forceinline__ void store_geo(GeoPixel* img, size_t i, V3 n, uint32_t depth) {
    reinterpret_cast<float4*>(img)[i] = make_float4(n.x, n.y, n.z, __uint_as_float(depth));
}

constexpr uint32_t RAW_KEY = 0xF6u << 9, RAW_KEY_MASK = 0xFFu << 9;   // pixel.rs:180-181
__device__ __forceinline__ bool is_distance(float f) {               // pixel.rs:197-203
    return f == f || (__float_as_uint(f) & RAW_KEY_MASK) != RAW_KEY;
}

// ---- denoise_normals (effects.rs:17-36, 256-326) ---------------------------------------------
__global__ void __launch_bounds__(256) k_denoise_normals(const GeoPixel* __restrict__ img, int w, int h,
                                                         GeoPixel* __restrict__ out) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= w || y >= h) return;
    const size_t idx = size_t(y) * w + x;
    const GeoPixel g = load_geo(img, idx);
    if (g.depth == 0) { store_geo(out, idx, v3(0.0f, 0.0f, 0.0f), 0); return; }
    V3 best = v3(g.normal[0], g.normal[1], g.normal[2]);
    if (!(g.normal[2] > 0.0f)) {
        const int r = 2;
        bool have = false;
        float best_score = 0.0f;
#pragma unroll 1
        for (int k = 0; k < 4; ++k) {
            const int x0 = x - ((k & 1) ? r : 0), y0 = y - ((k & 2) ? r : 0);
            V3 sum = v3(0.0f, 0.0f, 0.0f);
            int count = 0;
            for (int i = 0; i <= r; ++i)
                for (int j = 0; j <= r; ++j) {
                    const int tx = x0 + i, ty = y0 + j;
                    if (tx >= 0 && ty >= 0 && tx < w && ty < h) {
                        const GeoPixel p = load_geo(img, size_t(ty) * w + tx);
                        if (p.depth != 0 && p.normal[2] > 0.0f) {
                            sum = add(sum, v3(p.normal[0], p.normal[1], p.normal[2]));
                            ++count;
                        }
                    }
                }
            if (!count) continue;
            const V3 mean = divs(sum, float(count));
            float score = 0.0f;
            for (int i = 0; i <= r; ++i)
                for (int j = 0; j <= r; ++j) {
                    const int tx = x0 + i, ty = y0 + j;
                    if (tx >= 0 && ty >= 0 && tx < w && ty < h) {
                        const GeoPixel p = load_geo(img, size_t(ty) * w + tx);
                        if (p.depth != 0) score += dot(v3(p.normal[0], p.normal[1], p.normal[2]), mean);
                    }
                }
            // Iterator::max_by_key keeps the last of several equal maxima
            if (!have || ord_cmp(best_score, score) <= 0) { best_score = score; best = mean; have = true; }
        }
    }
    store_geo(out, idx, best, g.depth);
}

// ---- compute_ssao (effects.rs:72-95, 159-253) -------------------------------------------------
__global__ void __launch_bounds__(256) k_compute_ssao(const GeoPixel* __restrict__ img, uint32_t w, uint32_t h,
                                                      uint32_t d, const float* __restrict__ kernel, uint32_t nk,
                                                      const float* __restrict__ noise, uint32_t nn,
                                                      float* __restrict__ out) {
    extern __shared__ float s_kernel[];   // 3 * nk
    for (uint32_t i = threadIdx.x; i < 3 * nk; i += blockDim.x) s_kernel[i] = kernel[i];
    __syncthreads();
    const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= w || y >= h) return;
    const size_t idx = size_t(y) * w + x;
    const GeoPixel g = load_geo(img, idx);
    if (g.depth == 0) { out[idx] = __uint_as_float(0x7FC00000u); return; }
    const float fw = float(w), fh = float(h), fd = float(d);
    const float scale_min = float(min(min(w, h), d));
    const float scale_x = scale_min / fw, scale_y = scale_min / fh, scale_z = scale_min / fd;
    const V3 p = v3((((float(x) + 0.5f) / fw) - 0.5f) * 2.0f, (((float(y) + 0.5f) / fh) - 0.5f) * 2.0f,
                    ((float(g.depth) / fd) - 0.5f) * 2.0f);
    const V3 n = normalize(v3(g.normal[0], g.normal[1], g.normal[2]));
    const uint32_t ri = rng_mix(y, x) % nn;
    const V3 rvec = v3(__ldg(noise + 2 * ri), __ldg(noise + 2 * ri + 1), 0.0f);
    const V3 tangent = normalize(sub(rvec, mul(n, dot(rvec, n))));
    const V3 bitangent = cross(n, tangent);
    const float RADIUS = 0.1f;
    float occlusion = 0.0f;
#pragma unroll 4
    for (uint32_t i = 0; i < nk; ++i) {
        const float k0 = s_kernel[3 * i], k1 = s_kernel[3 * i + 1], k2 = s_kernel[3 * i + 2];
        V3 off = v3(tangent.x * k0, tangent.y * k0, tangent.z * k0);
        off = v3(bitangent.x * k1 + off.x, bitangent.y * k1 + off.y, bitangent.z * k1 + off.z);
        off = v3(n.x * k2 + off.x, n.y * k2 + off.y, n.z * k2 + off.z);
        off = mul(off, RADIUS);
        off.x *= scale_x;
        off.y *= scale_y;
        off.z *= scale_z;
        const V3 sp = add(off, p);
        const float px = ((sp.x / 2.0f) + 0.5f) * fw;
        const float py = ((sp.y / 2.0f) + 0.5f) * fh;
        uint32_t actual_h = 0;
        if (px < fw && py < fh && px > 0.0f && py > 0.0f)
            actual_h = __ldg(&img[size_t(uint32_t(py)) * w + uint32_t(px)].depth);
        const float actual_z = ((float(actual_h) / fd) - 0.5f) * 2.0f;
        const float dz = sp.z - actual_z;
        if (dz < RADIUS) {
            occlusion += (sp.z <= actual_z) ? 1.0f : 0.0f;
        } else if (dz < RADIUS * 2.0f && sp.z <= actual_z) {
            const float t = (RADIUS - (dz - RADIUS)) / RADIUS;
            occlusion += t * t;
        }
    }
    out[idx] = 1.0f - (occlusion / float(nk));
}

// ---- blur_ssao (effects.rs:98-115, 329-381) -----------------------------------------------------
__device__ __forceinline__ float blur_pixel(const float* __restrict__ s, int w, int h, int x, int y, float self) {
    const int r = 2;
    bool have = false;
    float best_dev = 0.0f, best_mean = self;
#pragma unroll 1
    for (int k = 0; k < 4; ++k) {
        const int x0 = x - ((k & 1) ? r : 0), y0 = y - ((k & 2) ? r : 0);
        float v[9];
        float sum = 0.0f;
        int count = 0;
#pragma unroll
        for (int i = 0; i <= r; ++i)
#pragma unroll
            for (int j = 0; j <= r; ++j) {
                const int tx = x0 + i, ty = y0 + j;
                float t = __uint_as_float(0x7FC00000u);
                if (tx >= 0 && ty >= 0 && tx < w && ty < h) t = __ldg(s + size_t(ty) * w + tx);
                v[i * 3 + j] = t;
                if (t == t) { sum += t; ++count; }
            }
        if (!count) continue;
        const float mean = sum / float(count);
        float stdev = 0.0f;
#pragma unroll
        for (int q = 0; q < 9; ++q)
            if (v[q] == v[q]) { const float e = mean - v[q]; stdev += e * e; }
        const float dev = stdev / float(count);
        // Iterator::min_by_key keeps the first of several equal minima
        if (!have || ord_cmp(best_dev, dev) > 0) { best_dev = dev; best_mean = mean; have = true; }
    }
    return best_mean;
}

__global__ void __launch_bounds__(256) k_blur_ssao(const float* __restrict__ ssao, int w, int h,
                                                   float* __restrict__ out) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= w || y >= h) return;
    const size_t idx = size_t(y) * w + x;
    const float v = __ldg(ssao + idx);
    out[idx] = (v != v) ? __uint_as_float(0x7FC00000u) : blur_pixel(ssao, w, h, x, y, v);
}

// ---- apply_shading (effects.rs:42-66, 118-154) ----------------------------------------------------
// ssao: raw (unblurred) occlusion map or null; the blur of effects.rs:98-115 is applied on the fly
// when `blur` is set, so that the blurred map never goes through HBM.
__global__ void __launch_bounds__(256) k_apply_shading(const GeoPixel* __restrict__ img, uint32_t w, uint32_t h,
                                                       uint32_t d, const float* __restrict__ ssao, int blur,
                                                       uint8_t* __restrict__ out) {
    const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= w || y >= h) return;
    const size_t idx = size_t(y) * w + x;
    const GeoPixel g = load_geo(img, idx);
    uint8_t c = 0;
    if (g.depth > 0) {
        const V3 n = normalize(v3(g.normal[0], g.normal[1], g.normal[2]));
        const V3 p = v3(2.0f * (float(x) / float(w) - 0.5f), 2.0f * (float(y) / float(h) - 0.5f),
                        2.0f * (float(g.depth) / float(d) - 0.5f));
        const float lights[3][4] = {{5.0f, -5.0f, 10.0f, 0.5f}, {-5.0f, 0.0f, 10.0f, 0.15f}, {0.0f, -5.0f, 10.0f, 0.15f}};
        float accum = 0.2f;
#pragma unroll
        for (int l = 0; l < 3; ++l) {
            const V3 dir = normalize(sub(v3(lights[l][0], lights[l][1], lights[l][2]), p));
            accum += fmaxf(dot(dir, n), 0.0f) * lights[l][3];
        }
        if (ssao) {
            float s = __ldg(ssao + idx);
            if (blur && s == s) s = blur_pixel(ssao, int(w), int(h), int(x), int(y), s);
            accum *= s * 0.6f + 0.4f;
        }
        accum = clampf(accum, 0.0f, 1.0f);
        c = as_u8(accum * 255.0f);
    }
    out[idx * 3] = c;
    out[idx * 3 + 1] = c;
    out[idx * 3 + 2] = c;
}

// ---- GeometryPixel::to_color (voxel.rs:136-153) ---------------------------------------------------
__global__ void __launch_bounds__(256) k_normals_to_color(const GeoPixel* __restrict__ img, uint64_t n,
                                                          uint8_t* __restrict__ out) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const GeoPixel g = load_geo(img, i);
    const float dx = g.normal[0], dy = g.normal[1], dz = g.normal[2];
    const float s = sqrtf((dx * dx + dy * dy) + dz * dz);
    uint8_t r = 0, gg = 0, b = 0;
    if (s != 0.0f) {
        const float scale = 255.0f / s;
        r = as_u8(fabsf(dx) * scale);
        gg = as_u8(fabsf(dy) * scale);
        b = as_u8(fabsf(dz) * scale);
    }
    out[i * 3] = r; out[i * 3 + 1] = gg; out[i * 3 + 2] = b;
}

// ---- to_rgba_bitmap / to_debug_bitmap / to_rgba_distance (effects.rs:446-547) -----------------------
__device__ __forceinline__ uint32_t rgba(uint32_t r, uint32_t g, uint32_t b, uint32_t a) {
    return r | (g << 8) | (b << 16) | (a << 24);
}

__device__ __forceinline__ uint32_t px_bitmap(float f, int transparent) {
    const bool inside = is_distance(f) ? (f < 0.0f) : ((__float_as_uint(f) & 1u) == 1u);
    return inside ? 0xFFFFFFFFu : (transparent ? 0u : 0xFF000000u);
}

__device__ __forceinline__ uint32_t px_debug(float f) {
    if (is_distance(f)) return f < 0.0f ? 0xFFFFFFFFu : 0xFF000000u;
    const uint32_t bits = __float_as_uint(f);
    const uint32_t v = (bits & 1u) ? 255u : 50u, depth = (bits >> 1) & 0xFFu;
    return rgba((depth == 0 || depth > 2) ? v : 0, (depth == 1 || depth > 2) ? v : 0, depth == 2 ? v : 0, 255);
}

__device__ __forceinline__ float smoothstep(float e0, float e1, float x) {
    const float t = clampf((x - e0) / (e1 - e0), 0.0f, 1.0f);
    return t * t * (3.0f - 2.0f * t);
}

__device__ __forceinline__ uint32_t px_distance(float f) {
    if (!is_distance(f)) return (__float_as_uint(f) & 1u) ? rgba(184, 235, 255, 255) : rgba(217, 144, 72, 255);
    if (f != f) return rgba(255, 0, 0, 255);
    const float af = fabsf(f);
    const float dim = 1.0f - expf(-4.0f * af);
    const float bands = 0.8f + 0.2f * cosf(140.0f * f);
    const float a1 = 1.0f - smoothstep(0.0f, 0.015f, af), a2 = 1.0f - smoothstep(0.0f, 0.005f, af);
    const float base[3] = {0.1f, 0.4f, 0.7f};
    uint32_t c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float v = (1.0f - copysignf(base[k], f)) * dim * bands;
        v = v * (1.0f - a1) + 1.0f * a1;
        v = v * (1.0f - a2) + 1.0f * a2;
        c[k] = as_u8(clampf(v, 0.0f, 1.0f) * 255.0f);
    }
    return rgba(c[0], c[1], c[2], 255);
}

// mode 0: bitmap, 1: bitmap (transparent), 2: debug, 3: distance.  Four pixels per thread when
// the image is 16-byte aligned: 16 B in, 16 B out.
template <int MODE>
__device__ __forceinline__ uint32_t px_rgba(float f) {
    if (MODE == 0) return px_bitmap(f, 0);
    if (MODE == 1) return px_bitmap(f, 1);
    if (MODE == 2) return px_debug(f);
    return px_distance(f);
}

template <int MODE>
__global__ void __launch_bounds__(256) k_to_rgba(const float* __restrict__ img, uint64_t n, uint32_t* __restrict__ out,
                                                 int vec4) {
    const uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (vec4) {
        const uint64_t i = t * 4;
        if (i + 3 < n) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(img) + t);
            reinterpret_cast<uint4*>(out)[t] =
                make_uint4(px_rgba<MODE>(v.x), px_rgba<MODE>(v.y), px_rgba<MODE>(v.z), px_rgba<MODE>(v.w));
        } else {
            for (uint64_t j = i; j < n; ++j) out[j] = px_rgba<MODE>(img[j]);
        }
    } else if (t < n) {
        out[t] = px_rgba<MODE>(img[t]);
    }
}

inline dim3 grid2d(uint32_t w, uint32_t h) { return dim3((w + 31) / 32, (h + 7) / 8); }

}  // namespace

void launch_denoise_normals(const GeoPixel* img, uint32_t w, uint32_t h, GeoPixel* out, cudaStream_t s) {
    k_denoise_normals<<<grid2d(w, h), 256, 0, s>>>(img, int(w), int(h), out);
}
void launch_compute_ssao(const GeoPixel* img, uint32_t w, uint32_t h, uint32_t d, const float* kernel, uint32_t nk,
                         const float* noise, uint32_t nn, float* out, cudaStream_t s) {
    k_compute_ssao<<<grid2d(w, h), 256, size_t(nk) * 12, s>>>(img, w, h, d, kernel, nk, noise, nn, out);
}
void launch_blur_ssao(const float* ssao, uint32_t w, uint32_t h, float* out, cudaStream_t s) {
    k_blur_ssao<<<grid2d(w, h), 256, 0, s>>>(ssao, int(w), int(h), out);
}
void launch_apply_shading(const GeoPixel* img, uint32_t w, uint32_t h, uint32_t d, const float* ssao, int blur,
                          uint8_t* out, cudaStream_t s) {
    k_apply_shading<<<grid2d(w, h), 256, 0, s>>>(img, w, h, d, ssao, blur, out);
}
void launch_normals_to_color(const GeoPixel* img, uint64_t n, uint8_t* out, cudaStream_t s) {
    k_normals_to_color<<<unsigned((n + 255) / 256), 256, 0, s>>>(img, n, out);
}
// Inside/outside masks of a RawDistancePixel image (RawDistancePixel::inside, pixel.rs:177-183): one warp per
// 32 consecutive pixels of a row; the ballot IS the 1-bit packing (bit x%8 of byte x/8, LSB first).
__global__ void __launch_bounds__(256) k_to_mask(const float* __restrict__ img, uint32_t w, uint32_t h, uint8_t* __restrict__ out,
                                                 int one_bit, uint32_t stride) {
    const uint32_t words = (w + 31u) / 32u;
    const uint64_t warp = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (warp >= uint64_t(words) * h) return;
    const uint32_t y = uint32_t(warp / words), x = uint32_t(warp % words) * 32u + (threadIdx.x & 31u);
    bool inside = false;
    if (x < w) {
        const float f = __ldg(img + size_t(y) * w + x);
        inside = is_distance(f) ? (f < 0.0f) : ((__float_as_uint(f) & 1u) == 1u);
    }
    const uint32_t m = __ballot_sync(0xffffffffu, inside);
    if (one_bit) {
        const uint32_t lane = threadIdx.x & 31u;
        if (lane < 4u && x - lane + lane * 8u < w) out[size_t(y) * stride + (x - lane) / 8u + lane] = uint8_t(m >> (8u * lane));
    } else if (x < w) {
        out[size_t(y) * w + x] = inside ? 255 : 0;
    }
}
void launch_to_mask(const float* img, uint32_t w, uint32_t h, uint8_t* out, int one_bit, cudaStream_t s) {
    const uint64_t warps = uint64_t((w + 31u) / 32u) * h;
    if (!warps) return;
    k_to_mask<<<unsigned((warps * 32 + 255) / 256), 256, 0, s>>>(img, w, h, out, one_bit, (w + 7u) / 8u);
}

void launch_to_rgba(int mode, const float* img, uint64_t n, uint8_t* out, cudaStream_t s) {
    const int vec4 = (reinterpret_cast<uintptr_t>(img) % 16 == 0) && (reinterpret_cast<uintptr_t>(out) % 16 == 0);
    const uint64_t threads = vec4 ? (n + 3) / 4 : n;
    const unsigned blocks = unsigned((threads + 255) / 256);
    uint32_t* o = reinterpret_cast<uint32_t*>(out);
    switch (mode) {
        case 0: k_to_rgba<0><<<blocks, 256, 0, s>>>(img, n, o, vec4); break;
        case 1: k_to_rgba<1><<<blocks, 256, 0, s>>>(img, n, o, vec4); break;
        case 2: k_to_rgba<2><<<blocks, 256, 0, s>>>(img, n, o, vec4); break;
        default: k_to_rgba<3><<<blocks, 256, 0, s>>>(img, n, o, vec4); break;
    }
}

}  // namespace fdev
