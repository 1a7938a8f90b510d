// Device-side bodies of the weight-norm kernels, shared by the per-layer launches (weightnorm.cu) and the batched
// "all layers in one launch" variants (wn_batched.cu).
#pragma once
#include <cuda_bf16.h>
#include "common.cuh"

namespace dv3 {

// Output formats of the weight-norm pack: the (hi, lo) pairs of common.cuh (FMT_F16 forward operands, FMT_BF16
// gradients) or FMT_F32, w itself in one fp32 plane (the operands of the exact-fp32 kernels).
enum { FMT_F32 = 32 };

// NPL = 1: plane hi alone (single-pass mode), the same bits as plane 0 of the pair.
template <int FMT, int NPL = 2>
__device__ __forceinline__ void split_store(float v, void* __restrict__ base, size_t idx, size_t plane_stride) {
    if constexpr (FMT == FMT_F32) {
        static_cast<float*>(base)[idx] = v;
    } else if constexpr (NPL == 1) {
        static_cast<uint16_t*>(base)[idx] = split_hi<FMT>(v);
    } else {
        uint16_t h, l;
        split_pair<FMT>(v, h, l);
        static_cast<uint16_t*>(base)[idx] = h;
        static_cast<uint16_t*>(base)[plane_stride + idx] = l;
    }
}

// one warp per row r: inv_norm[r] = 1/||v[r,:]||, scale[r] = g[r]*inv_norm[r]
__device__ __forceinline__ void wn_norm_row(const float* __restrict__ v, const float* __restrict__ g,
                                            float* __restrict__ inv_norm, float* __restrict__ scale, int R, int L,
                                            int r, int lane) {
    if (r >= R) return;
    const float* row = v + (size_t)r * L;
    float s = 0.f;
    for (int e = lane; e < L; e += 32) { const float xx = row[e]; s = fmaf(xx, xx, s); }
    s = warp_sum(s);
    if (lane == 0) { const float inv = 1.f / sqrtf(s); inv_norm[r] = inv; scale[r] = g[r] * inv; }
}

// weight-norm pack of one 32(r) x 32(e) tile, block (32, 8): v [R][X][k] fp32, scale[R] = g/||v|| -> w = v * scale
// in two plane sets of format FMTA / FMTB with element (r,x,j) at r*s_r + x*s_x + j*s_j (either set may be null; the
// plane stride is unused for FMT_F32 and NPL = 1): outA is written with lanes along (x,j) (choose the set whose unit
// stride is s_x), outB with lanes along r (unit stride s_r).  NPL: 16-bit planes per set.
template <int FMTA, int FMTB, int NPL = 2>
__device__ __forceinline__ void wn_pack_split_tile(const float* __restrict__ v, const float* __restrict__ scale,
                                                   void* __restrict__ outA, long long a_r, long long a_x,
                                                   long long a_j, long long a_plane, void* __restrict__ outB,
                                                   long long b_r, long long b_x, long long b_j, long long b_plane,
                                                   int R, int X, int k, int bx, int by, float (*tile)[33]) {
    const int L = X * k;
    const int r0 = by * 32, e0 = bx * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + threadIdx.y + 8 * i, e = e0 + threadIdx.x;
        float w = 0.f;
        if (r < R && e < L) {
            w = v[(size_t)r * L + e] * scale[r];
            const int xx = e / k, j = e - xx * k;
            if (outA) split_store<FMTA, NPL>(w, outA, (size_t)(r * a_r + xx * a_x + j * a_j), (size_t)a_plane);
        }
        tile[threadIdx.y + 8 * i][threadIdx.x] = w;
    }
    __syncthreads();
    if (outB) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = e0 + threadIdx.y + 8 * i, r = r0 + threadIdx.x;
            if (r < R && e < L) {
                const int xx = e / k, j = e - xx * k;
                split_store<FMTB, NPL>(tile[threadIdx.x][threadIdx.y + 8 * i], outB,
                                  (size_t)(r * b_r + xx * b_x + j * b_j), (size_t)b_plane);
            }
        }
    }
}

// backward of one row r by one CTA of 256 threads:  dW = sum_s partial[s] ;  dot = <dW, v>
//   dg = dot * inv_norm ;  dv = scale*dW - scale*dot*inv_norm^2 * v
// (one warp per row left the big layers -- 1024 rows x 1536 x up to 16 partials -- at 0.4 TB/s.)
// Partials are either in v's own layout (jmajor_X == 0: element e of row r at r*L + e) or tap-major
// (jmajor_X = X > 0: element (r, x, j) at (j*R + r)*X + x -- what the tensor-core weight-gradient kernel writes with
// contiguous float4 stores).  The reduced dW is parked in partial slot 0 between the two passes, so dv / dg can be
// ACCUMULATED into (accumulate = 1: the flat gradient arena of the training step, no autograd add kernel afterwards).
__device__ __forceinline__ void wn_bwd_row(float* __restrict__ dw_partials, long long split_stride, int nsplit,
                                           int jmajor_X, const float* __restrict__ v, const float* __restrict__ g,
                                           const float* __restrict__ inv_norm, float* __restrict__ dv,
                                           float* __restrict__ dg, int R, int L, int accumulate, int r) {
    __shared__ float red[8];
    __shared__ float s_dot;
    const int tid = threadIdx.x;
    const size_t base = (size_t)r * L;
    const int X = jmajor_X > 0 ? jmajor_X : L, k = L / X;
    float dot = 0.f;
    const bool vec4 = jmajor_X > 0 && (X & 3) == 0 && (split_stride & 3) == 0;
    if (vec4) {                                          // tap-major partials: float4 along x, v gathered at stride k
        const int X4 = X >> 2;
        for (int q = tid; q < k * X4; q += 256) {
            const int j = q / X4, x = (q - j * X4) << 2;
            const size_t po = ((size_t)j * R + r) * X + x;
            float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int s = 0; s < nsplit; ++s) {
                const float4 t = *reinterpret_cast<const float4*>(&dw_partials[(size_t)s * split_stride + po]);
                d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
            }
            *reinterpret_cast<float4*>(&dw_partials[po]) = d;
            const float* vv = v + base + (size_t)x * k + j;
            dot = fmaf(d.x, vv[0], dot); dot = fmaf(d.y, vv[k], dot);
            dot = fmaf(d.z, vv[2 * k], dot); dot = fmaf(d.w, vv[3 * k], dot);
        }
    } else {
        for (int q = tid; q < L; q += 256) {             // q runs over the partial's own (coalesced) order
            size_t po; int e;
            if (jmajor_X > 0) { const int j = q / X, x = q - j * X; e = x * k + j; po = ((size_t)j * R + r) * X + x; }
            else { e = q; po = base + q; }
            float d = 0.f;
            for (int s = 0; s < nsplit; ++s) d += dw_partials[(size_t)s * split_stride + po];
            dw_partials[po] = d;
            dot = fmaf(d, v[base + e], dot);
        }
    }
    dot = warp_sum(dot);
    if ((tid & 31) == 0) red[tid >> 5] = dot;
    __syncthreads();
    if (tid < 32) {
        float t = tid < 8 ? red[tid] : 0.f;
        t = warp_sum(t);
        if (tid == 0) s_dot = t;
    }
    __syncthreads();
    dot = s_dot;
    const float inv = inv_norm[r], sc = g[r] * inv, c2 = sc * dot * inv * inv;
    for (int q = tid; q < L; q += 256) {                 // same thread -> same elements as in the first pass
        size_t po; int e;
        if (jmajor_X > 0) { const int j = q / X, x = q - j * X; e = x * k + j; po = ((size_t)j * R + r) * X + x; }
        else { e = q; po = base + q; }
        const float val = sc * dw_partials[po] - c2 * v[base + e];
        dv[base + e] = accumulate ? dv[base + e] + val : val;
    }
    if (tid == 0) dg[r] = accumulate ? dg[r] + dot * inv : dot * inv;
}

}  // namespace dv3
