// LWS phase recovery: Local Weighted Sums (Le Roux et al., DAFx 2010), the algorithm of the reference's
// audio.inv_spectrogram (audio.py:37-43, `lws.run_lws`).  The `lws` package's source is absent, so this restates the
// published algorithm and parity with lws.run_lws is UNPINNED (like the forward STFT, DESIGN.md section 3).  The
// magnitude-threshold schedule of the package (it skips small bins to save CPU time) and online LWS are not done.
//
// Frame: the default one (N = 1024, hop R = 256, synthesis window = analysis window w, K = 513 bins).  X is a (T, 513)
// complex half spectrum, A the target magnitude.  Weights, computed once on the host in fp64 (audio._lws_weights):
//     beta_q(d) = (1/N) sum_n w(n) w(n - qR) e^{-2 pi i d n / N},   q in [-3, 3], d in [-5, 5]
// Local weighted sum (the complex-linear part of STFT(iSTFT(X)) minus the bin's own term):
//     Y(m,k) = sum_{(q,d) != (0,0)} beta_q(d) (-i)^{k'q} X(m+q, k'),   k' = k - d
// (-i)^{k'q} comes from hop = N/4.  It factors as (-i)^{kq} * i^{dq}: the kernels fold i^{dq} into the weights when they
// stage them and rotate each q's partial sum once -- a swap / negation of re and im, exact in fp32.  Bins k' < 0 read
// conj X(m, -k'), bins k' > 512 read conj X(m, 1024 - k').  Frames outside [0, T_c) contribute 0: exact away from the
// clip's ends, an approximation in its first and last 3 frames, where the inverse STFT crops the 768 padding samples.
// Update: X <- A Y / |Y| (A + 0i where Y == 0).  Bins 0 and 512 are set real, A sign(Re Y) (+A where Re Y == 0): their
// Y is real in exact arithmetic, and istft_any_kernel folds an imaginary part there into the waveform instead of dropping
// it.
//
//   lws_nofuture_kernel  one CTA per clip walks the frames in order: past = the q in {-3,-2,-1} terms from the last 3
//                        frames (a shared-memory ring, zero before the clip), X(m) <- A past/|past|, then init_iters
//                        in-frame Jacobi passes adding the beta_0(d) terms of the frame's own bins.  Latency-bound
//                        (nclips CTAs, 2 + 2*init_iters barriers per frame).
//   lws_iterate_kernel   one batch (Jacobi) iteration, spec_in -> spec_out: a CTA of 512 threads stages 8 frames x 64 bins plus the
//                        halo (+-3 frames, +-5 bins, conjugate mirror at both ends) in shared memory.
// Every sum runs in a fixed order and reads only its own clip's first frames[c] frames, so a clip in a ragged batch gets
// bit for bit what it gets alone, and two runs agree bit for bit.
#include "common.cuh"

namespace dv3 {

constexpr int LK = 513, LQ = 3, LL = 5, LNQ = 2 * LQ + 1, LND = 2 * LL + 1;
constexpr int IT_F = 8, IT_B = 64, IT_THREADS = IT_F * IT_B;      // lws_iterate_kernel tile: frames x bins
constexpr int IT_HF = IT_F + 2 * LQ, IT_HB = IT_B + 2 * LL;        // with the halo
constexpr int NF_THREADS = 544;                                    // lws_nofuture_kernel: one bin per thread (17 warps)

// v * (-i)^r, r in 0..3
__device__ __forceinline__ float2 rot_negi(float2 v, int r) {
    switch (r & 3) {
        case 0: return v;
        case 1: return make_float2(v.y, -v.x);
        case 2: return make_float2(-v.x, -v.y);
        default: return make_float2(-v.y, v.x);
    }
}

__device__ __forceinline__ float2 cmac(float2 acc, float2 a, float2 b) {      // acc + a*b
    acc.x = fmaf(a.x, b.x, fmaf(-a.y, b.y, acc.x));
    acc.y = fmaf(a.x, b.y, fmaf(a.y, b.x, acc.y));
    return acc;
}

// beta_q(d) * i^{dq} = beta_q(d) * (-i)^{-dq} into shared memory ([q+3][d+5])
__device__ __forceinline__ void stage_weights(const float2* __restrict__ beta, float2* w, int tid, int nthreads) {
    for (int j = tid; j < LNQ * LND; j += nthreads) {
        const int q = j / LND - LQ, d = j % LND - LL;
        w[j] = rot_negi(beta[j], -d * q);
    }
}

// X(m, k') of the full spectrum from the half spectrum row (k' in [-5, 517])
__device__ __forceinline__ float2 load_mirrored(const float2* __restrict__ row, int kp) {
    if (kp < 0) { const float2 v = row[-kp]; return make_float2(v.x, -v.y); }
    if (kp >= LK) { const float2 v = row[1024 - kp]; return make_float2(v.x, -v.y); }
    return row[kp];
}

__device__ __forceinline__ float2 project(float a, float2 y, int k) {
    if (k == 0 || k == LK - 1) return make_float2(y.x < 0.f ? -a : a, 0.f);
    const float n = sqrtf(y.x * y.x + y.y * y.y);
    if (!(n > 0.f)) return make_float2(a, 0.f);
    const float s = a / n;
    return make_float2(y.x * s, y.y * s);
}

// mag (nclips, T_max, 513), spec_in / spec_out (nclips, T_max, 513) float2; grid (9 bin tiles, frame tiles, nclips)
__global__ void __launch_bounds__(IT_THREADS) lws_iterate_kernel(const float* __restrict__ mag,
                                                                 const float2* __restrict__ xin,
                                                                 float2* __restrict__ xout,
                                                                 const float2* __restrict__ beta, int nframes0,
                                                                 const int* frames, long long frame_pitch) {
    pdl_trigger(); pdl_wait();
    __shared__ float2 tile[IT_HF][IT_HB];
    __shared__ float2 w[LNQ * LND];
    const int clip = blockIdx.z, tid = threadIdx.x;
    const int T = frames ? frames[clip] : nframes0;
    const int m0 = blockIdx.y * IT_F, k0 = blockIdx.x * IT_B;
    if (m0 >= T) return;
    const size_t base = (size_t)clip * frame_pitch * LK;
    xin += base; xout += base; mag += base;
    stage_weights(beta, w, tid, IT_THREADS);
    for (int j = tid; j < IT_HF * IT_HB; j += IT_THREADS) {
        const int f = j / IT_HB, b = j % IT_HB, m = m0 - LQ + f, kp = k0 - LL + b;
        float2 v = make_float2(0.f, 0.f);
        if (m >= 0 && m < T && kp < LK + LL) v = load_mirrored(xin + (size_t)m * LK, kp);
        tile[f][b] = v;
    }
    __syncthreads();
    const int b = tid % IT_B, f = tid / IT_B, k = k0 + b, m = m0 + f;      // one output bin per thread
    if (k >= LK || m >= T) return;
    float2 y = make_float2(0.f, 0.f);
#pragma unroll
    for (int q = -LQ; q <= LQ; ++q) {
        float2 s = make_float2(0.f, 0.f);
#pragma unroll
        for (int d = -LL; d <= LL; ++d) {
            if (q == 0 && d == 0) continue;
            s = cmac(s, w[(q + LQ) * LND + d + LL], tile[f + LQ + q][b + LL - d]);
        }
        const float2 r = rot_negi(s, k * q);
        y.x += r.x; y.y += r.y;
    }
    xout[(size_t)m * LK + k] = project(mag[(size_t)m * LK + k], y, k);
}

// One CTA per clip; thread k owns bin k.  ring[m % 3] holds frame m once it is final (zero before the clip).
__global__ void __launch_bounds__(NF_THREADS) lws_nofuture_kernel(const float* __restrict__ mag,
                                                                  float2* __restrict__ spec,
                                                                  const float2* __restrict__ beta, int nframes0,
                                                                  const int* frames, long long frame_pitch,
                                                                  int init_iters) {
    pdl_trigger(); pdl_wait();
    __shared__ float2 ring[LQ][LK];
    __shared__ float2 w[LNQ * LND];
    const int clip = blockIdx.x, k = threadIdx.x;
    const bool live = k < LK;
    const int T = frames ? frames[clip] : nframes0;
    const size_t base = (size_t)clip * frame_pitch * LK;
    spec += base; mag += base;
    stage_weights(beta, w, k, NF_THREADS);
    if (live) for (int s = 0; s < LQ; ++s) ring[s][k] = make_float2(0.f, 0.f);
    __syncthreads();
    for (int m = 0; m < T; ++m) {
        float2 past = make_float2(0.f, 0.f), x = past;
        float a = 0.f;
        if (live) {
            a = mag[(size_t)m * LK + k];
#pragma unroll
            for (int q = -LQ; q <= -1; ++q) {
                const float2* row = ring[(m + q + LQ) % LQ];
                float2 s = make_float2(0.f, 0.f);
#pragma unroll
                for (int d = -LL; d <= LL; ++d) s = cmac(s, w[(q + LQ) * LND + d + LL], load_mirrored(row, k - d));
                const float2 r = rot_negi(s, k * q);
                past.x += r.x; past.y += r.y;
            }
            x = project(a, past, k);
        }
        float2* cur = ring[m % LQ];                  // frame m - 3: no longer read
        __syncthreads();
        if (live) cur[k] = x;
        __syncthreads();
        for (int it = 0; it < init_iters; ++it) {
            if (live) {
                float2 s = make_float2(0.f, 0.f);
#pragma unroll
                for (int d = -LL; d <= LL; ++d) {
                    if (d == 0) continue;
                    s = cmac(s, w[LQ * LND + d + LL], load_mirrored(cur, k - d));
                }
                x = project(a, make_float2(past.x + s.x, past.y + s.y), k);
            }
            __syncthreads();
            if (live) cur[k] = x;
            __syncthreads();
        }
        if (live) spec[(size_t)m * LK + k] = x;
    }
}

}  // namespace dv3

using namespace dv3;

extern "C" {

static int lws_nofuture_launch(const float* mag, float* spec, const float* weights, int nframes0, const int* frames,
                               int max_frames, int nclips, int init_iters, cudaStream_t st) {
    launch_k(lws_nofuture_kernel, nclips, NF_THREADS, 0, st, mag, (float2*)spec, (const float2*)weights, nframes0,
             frames, (long long)max_frames, init_iters);
    return check_launch("lws_nofuture");
}

static int lws_iterate_launch(const float* mag, const float* spec_in, float* spec_out, const float* weights,
                              int nframes0, const int* frames, int max_frames, int nclips, cudaStream_t st) {
    launch_k(lws_iterate_kernel, dim3(ceil_div(LK, IT_B), ceil_div(max_frames, IT_F), nclips), IT_THREADS, 0, st, mag,
             (const float2*)spec_in, (float2*)spec_out, (const float2*)weights, nframes0, frames,
             (long long)max_frames);
    return check_launch("lws_iterate");
}

int dv3_lws_nofuture(const float* mag, float* spec, const float* weights, int nframes, int init_iters, void* stream) {
    DV3_REQUIRE(nframes >= 1 && init_iters >= 0, "lws_nofuture: bad shape");
    return lws_nofuture_launch(mag, spec, weights, nframes, nullptr, nframes, 1, init_iters, (cudaStream_t)stream);
}

int dv3_lws_iterate(const float* mag, const float* spec_in, float* spec_out, const float* weights, int nframes,
                    void* stream) {
    DV3_REQUIRE(nframes >= 1 && spec_in != spec_out, "lws_iterate: bad shape or in-place call");
    return lws_iterate_launch(mag, spec_in, spec_out, weights, nframes, nullptr, nframes, 1, (cudaStream_t)stream);
}

int dv3_lws_nofuture_batched(const float* mag, float* spec, const float* weights, const int* nframes, int max_frames,
                             int nclips, int init_iters, void* stream) {
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nframes && init_iters >= 0, "lws_nofuture_batched: bad shape");
    return lws_nofuture_launch(mag, spec, weights, 0, nframes, max_frames, nclips, init_iters, (cudaStream_t)stream);
}

int dv3_lws_iterate_batched(const float* mag, const float* spec_in, float* spec_out, const float* weights,
                            const int* nframes, int max_frames, int nclips, void* stream) {
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nclips <= 65535 && nframes && spec_in != spec_out,
                "lws_iterate_batched: bad shape or in-place call");
    DV3_REQUIRE(ceil_div(max_frames, IT_F) <= 65535, "lws_iterate_batched: too many frames");
    return lws_iterate_launch(mag, spec_in, spec_out, weights, 0, nframes, max_frames, nclips, (cudaStream_t)stream);
}

}  // extern "C"
