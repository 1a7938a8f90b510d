// LWS phase recovery for every STFT frame audio.check_geometry accepts: lws.cu's algorithm with N = Q*R, K = N/2+1
// bins and Q in [2, 8] (lws.cu keeps the specialised 1024 / 256 kernels).  The frame shift turns into the phase factor
// e^{-2 pi i k'q/Q} (k' = k - d), which factors as e^{-2 pi i kq/Q} e^{2 pi i dq/Q}: the host folds the second factor
// into the weights in fp64 (audio._lws_tables), and each q's partial sum is rotated once by one of the Q roots
// e^{-2 pi i r/Q}, r = kq mod Q.  Weight table (float2): wf[(q + Q-1)*11 + d + 5] = beta_q(d) e^{2 pi i dq/Q} for
// |q| <= Q-1, |d| <= 5, then the Q roots.  Bins k' < 0 read conj X(m, -k'), bins k' > N/2 read conj X(m, N - k');
// frames outside the clip contribute 0; bins 0 and N/2 are projected onto the real axis, as in lws.cu.
//
//   lws_nofuture_any   one CTA per clip walks the frames in order; a ring of the Q-1 past frames in shared memory;
//                      each thread owns bins k, k + 1024, ... (K <= 2049).
//   lws_iterate_any    one batch (Jacobi) iteration: a CTA of 512 threads stages 8 frames x 64 bins plus a halo of
//                      +-(Q-1) frames and +-5 bins.
// Fixed summation orders and reads of a clip's own frames only: each clip of a ragged batch is bit-identical alone.
#include "common.cuh"

namespace dv3 {

constexpr int AL = 5, AND = 2 * AL + 1;
constexpr int AIT_F = 8, AIT_B = 64, AIT_THREADS = AIT_F * AIT_B, AIT_HB = AIT_B + 2 * AL;
constexpr int ANF_THREADS = 1024, ANF_BINS = 3;                   // bins per thread of the nofuture kernel (K <= 3072)

__device__ __forceinline__ float2 acmac(float2 acc, float2 a, float2 b) {     // acc + a*b
    acc.x = fmaf(a.x, b.x, fmaf(-a.y, b.y, acc.x));
    acc.y = fmaf(a.x, b.y, fmaf(a.y, b.x, acc.y));
    return acc;
}
__device__ __forceinline__ float2 acmul(float2 a, float2 b) {
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ int root_index(int k, int q, int Q) { return ((k * q) % Q + Q) % Q; }

__device__ __forceinline__ float2 any_mirrored(const float2* row, int kp, int K) {
    if (kp < 0) { const float2 v = row[-kp]; return make_float2(v.x, -v.y); }
    if (kp >= K) { const float2 v = row[2 * (K - 1) - kp]; return make_float2(v.x, -v.y); }
    return row[kp];
}

__device__ __forceinline__ float2 any_project(float a, float2 y, int k, int K) {
    if (k == 0 || k == K - 1) return make_float2(y.x < 0.f ? -a : a, 0.f);
    const float n = sqrtf(y.x * y.x + y.y * y.y);
    if (!(n > 0.f)) return make_float2(a, 0.f);
    const float s = a / n;
    return make_float2(y.x * s, y.y * s);
}

// grid (bin tiles, frame tiles, nclips); dynamic smem: tile (8 + 2(Q-1)) x 74, weights, roots
__global__ void __launch_bounds__(AIT_THREADS) lws_iterate_any_kernel(const float* __restrict__ mag,
                                                                      const float2* __restrict__ xin,
                                                                      float2* __restrict__ xout,
                                                                      const float2* __restrict__ wtab,
                                                                      const int* frames, long long frame_pitch, int K,
                                                                      int Q) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int H = Q - 1, HF = AIT_F + 2 * H, NW = (2 * H + 1) * AND;
    float2* tile = reinterpret_cast<float2*>(smem_raw);
    float2* w = tile + HF * AIT_HB;                                // NW weights, then Q roots
    const int clip = blockIdx.z, tid = threadIdx.x;
    const int T = frames[clip];
    const int m0 = blockIdx.y * AIT_F, k0 = blockIdx.x * AIT_B;
    if (m0 >= T) return;
    const size_t base = (size_t)clip * frame_pitch * K;
    xin += base; xout += base; mag += base;
    for (int j = tid; j < NW + Q; j += AIT_THREADS) w[j] = wtab[j];
    for (int j = tid; j < HF * AIT_HB; j += AIT_THREADS) {
        const int f = j / AIT_HB, b = j % AIT_HB, m = m0 - H + f, kp = k0 - AL + b;
        float2 v = make_float2(0.f, 0.f);
        if (m >= 0 && m < T && kp < K + AL) v = any_mirrored(xin + (size_t)m * K, kp, K);
        tile[f * AIT_HB + b] = v;
    }
    __syncthreads();
    const int b = tid % AIT_B, f = tid / AIT_B, k = k0 + b, m = m0 + f;
    if (k >= K || m >= T) return;
    float2 y = make_float2(0.f, 0.f);
    for (int q = -H; q <= H; ++q) {
        float2 s = make_float2(0.f, 0.f);
        const float2* wq = w + (q + H) * AND;
        const float2* row = tile + (f + H + q) * AIT_HB + b + AL;
#pragma unroll
        for (int d = -AL; d <= AL; ++d) {
            if (q == 0 && d == 0) continue;
            s = acmac(s, wq[d + AL], row[-d]);
        }
        const float2 r = acmul(s, w[NW + root_index(k, q, Q)]);
        y.x += r.x; y.y += r.y;
    }
    xout[(size_t)m * K + k] = any_project(mag[(size_t)m * K + k], y, k, K);
}

// one CTA per clip; ring[m % (Q-1)] holds frame m once it is final (zero before the clip)
__global__ void __launch_bounds__(ANF_THREADS) lws_nofuture_any_kernel(const float* __restrict__ mag,
                                                                       float2* __restrict__ spec,
                                                                       const float2* __restrict__ wtab,
                                                                       const int* frames, long long frame_pitch,
                                                                       int init_iters, int K, int Q) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int H = Q - 1, NW = (2 * H + 1) * AND;
    float2* ring = reinterpret_cast<float2*>(smem_raw);             // H rows of K
    float2* w = ring + H * K;
    const int clip = blockIdx.x, tid = threadIdx.x;
    const int T = frames[clip];
    const size_t base = (size_t)clip * frame_pitch * K;
    spec += base; mag += base;
    for (int j = tid; j < NW + Q; j += ANF_THREADS) w[j] = wtab[j];
    for (int j = tid; j < H * K; j += ANF_THREADS) ring[j] = make_float2(0.f, 0.f);
    __syncthreads();
    for (int m = 0; m < T; ++m) {
        float2 past[ANF_BINS], x[ANF_BINS];
        float a[ANF_BINS];
#pragma unroll
        for (int i = 0; i < ANF_BINS; ++i) {
            const int k = tid + i * ANF_THREADS;
            past[i] = x[i] = make_float2(0.f, 0.f);
            a[i] = 0.f;
            if (k >= K) continue;
            a[i] = mag[(size_t)m * K + k];
            for (int q = -H; q <= -1; ++q) {
                const float2* row = ring + ((m + q + H) % H) * K;
                const float2* wq = w + (q + H) * AND;
                float2 s = make_float2(0.f, 0.f);
#pragma unroll
                for (int d = -AL; d <= AL; ++d) s = acmac(s, wq[d + AL], any_mirrored(row, k - d, K));
                const float2 r = acmul(s, w[NW + root_index(k, q, Q)]);
                past[i].x += r.x; past[i].y += r.y;
            }
            x[i] = any_project(a[i], past[i], k, K);
        }
        float2* cur = ring + (m % H) * K;                       // frame m - (Q-1): no longer read
        __syncthreads();
#pragma unroll
        for (int i = 0; i < ANF_BINS; ++i)
            if (tid + i * ANF_THREADS < K) cur[tid + i * ANF_THREADS] = x[i];
        __syncthreads();
        for (int it = 0; it < init_iters; ++it) {
            const float2* w0 = w + H * AND;
#pragma unroll
            for (int i = 0; i < ANF_BINS; ++i) {
                const int k = tid + i * ANF_THREADS;
                if (k >= K) continue;
                float2 s = make_float2(0.f, 0.f);
#pragma unroll
                for (int d = -AL; d <= AL; ++d) {
                    if (d == 0) continue;
                    s = acmac(s, w0[d + AL], any_mirrored(cur, k - d, K));
                }
                x[i] = any_project(a[i], make_float2(past[i].x + s.x, past[i].y + s.y), k, K);
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < ANF_BINS; ++i)
                if (tid + i * ANF_THREADS < K) cur[tid + i * ANF_THREADS] = x[i];
            __syncthreads();
        }
#pragma unroll
        for (int i = 0; i < ANF_BINS; ++i)
            if (tid + i * ANF_THREADS < K) spec[(size_t)m * K + tid + i * ANF_THREADS] = x[i];
    }
}

static int lws_any_geometry(int N, int R, const char* what) {
    DV3_REQUIRE(N >= 256 && N <= 4096 && N % 2 == 0 && R >= 1 && N % R == 0 && N / R >= 2 && N / R <= 8,
                "%s: unsupported STFT geometry fft_size %d, hop %d", what, N, R);
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_lws_nofuture_geom(const float* mag, float* spec, const float* weights, const int* nframes, int max_frames,
                          int nclips, int init_iters, int n_fft, int hop, void* stream) {
    const char* what = "lws_nofuture_geom";
    if (lws_any_geometry(n_fft, hop, what)) return 1;
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nframes && weights && init_iters >= 0, "%s: bad shape", what);
    const int K = n_fft / 2 + 1, Q = n_fft / hop;
    const size_t smem = sizeof(float2) * ((size_t)(Q - 1) * K + (2 * Q - 1) * AND + Q);
    DV3_REQUIRE(cudaFuncSetAttribute(lws_nofuture_any_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                == cudaSuccess, "%s: cannot reserve %zu bytes of shared memory", what, smem);
    launch_k(lws_nofuture_any_kernel, nclips, ANF_THREADS, smem, (cudaStream_t)stream, mag, (float2*)spec,
             (const float2*)weights, nframes, (long long)max_frames, init_iters, K, Q);
    return check_launch(what);
}

int dv3_lws_iterate_geom(const float* mag, const float* spec_in, float* spec_out, const float* weights,
                         const int* nframes, int max_frames, int nclips, int n_fft, int hop, void* stream) {
    const char* what = "lws_iterate_geom";
    if (lws_any_geometry(n_fft, hop, what)) return 1;
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nclips <= 65535 && nframes && weights && spec_in != spec_out,
                "%s: bad shape or in-place call", what);
    DV3_REQUIRE(ceil_div(max_frames, AIT_F) <= 65535, "%s: too many frames", what);
    const int K = n_fft / 2 + 1, Q = n_fft / hop;
    const size_t smem = sizeof(float2) * ((size_t)(AIT_F + 2 * (Q - 1)) * AIT_HB + (2 * Q - 1) * AND + Q);
    launch_k(lws_iterate_any_kernel, dim3(ceil_div(K, AIT_B), ceil_div(max_frames, AIT_F), nclips), AIT_THREADS,
             smem, (cudaStream_t)stream, mag, (const float2*)spec_in, (float2*)spec_out, (const float2*)weights,
             nframes, (long long)max_frames, K, Q);
    return check_launch(what);
}

}  // extern "C"
