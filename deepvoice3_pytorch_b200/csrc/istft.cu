// Inverse audio path: reference audio.py:37-43 (inv_spectrogram) = _denormalize (:92-93) -> _db_to_amp (:84-85) ->
// ** power -> phase recovery -> inverse STFT -> inv_preemphasis (:26-28).
// The reference recovers the phase with the `lws` package (Local Weighted Sums), an un-vendored, unpinned dependency
// whose source is absent -- PARITY UNPINNED.  What is restated here is the published Griffin-Lim fixed-point iteration
// on the SAME STFT frame the forward path uses (sqrt-Hann window * sqrt(2*hop/fsize), 1024 / hop 256, 768 samples of
// zero padding on both sides = lws "perfectrec": sum of squared windows over the 4 overlapping frames == 1, so the
// synthesis window equals the analysis window and no normalisation pass is needed):
//     x <- istft(S * exp(i * angle(stft(x))))        (host loop in audio.py; each arrow below is one launch)
// Kernels (one CTA of 256 threads per frame, the shared-memory radix-2 transform of stft.cu):
//   spec_to_amp_kernel      normalised dB spectrogram -> linear magnitude ** power
//   stft_complex_kernel     waveform -> complex half spectrum (frames, 513) [optionally projected onto a magnitude]
//   stft_complex_momentum_kernel  the same transform with the fast Griffin-Lim epilogue
//                           (audio.griffin_lim_batch with momentum > 0, DESIGN.md section 7.3)
//   istft_kernel            complex half spectrum -> windowed frame, overlap-added into the waveform: frames f and f+4
//                           do not overlap (fsize = 4*hop), so one launch per residue class f mod 4 adds with plain
//                           loads and stores -- deterministic, each sample summed in the same order every run
// Both take a clip grid dimension (blockIdx.y): clip c has its own sample / frame counts (lens / frames arrays, or the
// scalar when the array is NULL) and pitches, so a ragged batch of clips runs in one launch and every clip gets exactly
// what it gets alone.
//   deemphasis_kernel       y[n] = x[n] + c*y[n-1] (a 1st-order IIR: one thread per clip, chunks staged through smem)
// The reference's own algorithm, LWS phase recovery on this frame, is csrc/lws.cu (audio.inv_spectrogram(method="lws")).
#include "common.cuh"

namespace dv3 {

constexpr int IFFT_N = 1024, IHOP = 256, INH = 512, INBINS = 513, IPAD = IFFT_N - IHOP;

__device__ __forceinline__ int ibitrev9(int x) { return (int)(__brev((unsigned)x) >> 23); }
__device__ __forceinline__ float frame_window(int i) {           // sqrt(hann(i) * 2*hop/N), hann = .5*(1-cos(2pi(i+.5)/N))
    const float hann = 0.5f - 0.5f * cospif((2 * i + 1) / (float)IFFT_N);
    return sqrtf(hann * (2.f * IHOP / IFFT_N));
}

// 512-point complex radix-2 DIT FFT in shared memory (input in bit-reversed order), 256 threads, forward sign
__device__ __forceinline__ void fft512(float* zr, float* zi, const float* twr, const float* twi, int tid) {
#pragma unroll
    for (int s = 0; s < 9; ++s) {
        const int half = 1 << s;
        const int pos = tid & (half - 1);
        const int i0 = ((tid >> s) << (s + 1)) + pos, i1 = i0 + half;
        const int tw = pos << (8 - s);
        const float wr = twr[tw], wi = twi[tw];
        const float ar = zr[i0], ai = zi[i0], br0 = zr[i1], bi0 = zi[i1];
        const float br = br0 * wr - bi0 * wi, bi = br0 * wi + bi0 * wr;
        zr[i0] = ar + br; zi[i0] = ai + bi;
        zr[i1] = ar - br; zi[i1] = ai - bi;
        __syncthreads();
    }
}

// S (n) in [0,1] (normalised dB, audio.py:88-89) -> amplitude ** power:  dB = S*(-min_db) + min_db + ref_db
__global__ void spec_to_amp_kernel(const float* __restrict__ s, float* __restrict__ amp, long long n, float min_db,
                                   float ref_db, float power) {
    pdl_trigger(); pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = fminf(fmaxf(s[i], 0.f), 1.f);
        const float db = v * -min_db + min_db + ref_db;                    // audio.py:92-93, :39
        amp[i] = powf(powf(10.f, db * 0.05f), power);                     // audio.py:84-85, :41
    }
}

// The forward transform of one frame: frame `frame` of the clip x (len samples), windowed, 512-point packed FFT, split
// into the half spectrum; epi(k, Re X_k, Im X_k) for k = 0..512 (k = tid, tid + 256, and 512 on thread 0).  No
// preemphasis here (the iteration runs on the pre-emphasised signal).
template <class Epi>
__device__ __forceinline__ void stft_frame_1024(const float* __restrict__ x, int len, int frame, Epi epi) {
    __shared__ float zr[INH], zi[INH], twr[INH / 2], twi[INH / 2];
    const int tid = threadIdx.x;
    { float s, c; sincospif(-(float)tid / 256.f, &s, &c); twr[tid] = c; twi[tid] = s; }
    const int base = frame * IHOP - IPAD;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = tid + h * 256;
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int i = 2 * n + e, sidx = base + i;
            v[e] = (sidx >= 0 && sidx < len) ? x[sidx] * frame_window(i) : 0.f;
        }
        const int r = ibitrev9(n);
        zr[r] = v[0]; zi[r] = v[1];
    }
    __syncthreads();
    fft512(zr, zi, twr, twi, tid);
    for (int k = tid; k <= INH; k += 256) {
        const int ka = k & (INH - 1), kb = (INH - k) & (INH - 1);
        const float ar = zr[ka], ai = zi[ka], br = zr[kb], bi = -zi[kb];
        const float er = 0.5f * (ar + br), ei = 0.5f * (ai + bi), dr = 0.5f * (ar - br), di = 0.5f * (ai - bi);
        const float orr = di, oi = -dr;
        float s, c;
        sincospif(-(float)k / 512.f, &s, &c);
        epi(k, er + c * orr - s * oi, ei + c * oi + s * orr);
    }
}

// mag X / |X| (X == 0 gives phase 0): the Griffin-Lim magnitude projection of both complex-STFT kernels
__device__ __forceinline__ void project_1024(float m, float& xr, float& xi) {
    const float a = sqrtf(fmaf(xr, xr, xi * xi));      // explicit: both kernels round |X|^2 the same way
    if (a > 0.f) { xr *= m / a; xi *= m / a; } else { xr = m; xi = 0.f; }
}

// wav (len) -> spec (nframes, 513, 2).  mag != null: the result is projected onto that magnitude (Griffin-Lim step):
// spec = mag * X / |X| (X == 0 keeps phase 0).
// Clip c = blockIdx.y: x + c*x_pitch, spec / mag + c*frame_pitch frames; len / nframes from lens / frames when given.
__global__ void __launch_bounds__(256) stft_complex_kernel(const float* __restrict__ x, int len0, const int* lens,
                                                           long long x_pitch, const float* __restrict__ mag,
                                                           float* __restrict__ spec, int nframes0, const int* frames,
                                                           long long frame_pitch) {
    pdl_trigger(); pdl_wait();
    const int frame = blockIdx.x, clip = blockIdx.y;
    const int nframes = frames ? frames[clip] : nframes0, len = lens ? lens[clip] : len0;
    if (frame >= nframes) return;
    x += clip * x_pitch;
    spec += clip * frame_pitch * INBINS * 2;
    if (mag) mag += clip * frame_pitch * INBINS;
    stft_frame_1024(x, len, frame, [&](int k, float xr, float xi) {
        const size_t o = ((size_t)frame * INBINS + k) * 2;
        if (mag) project_1024(mag[(size_t)frame * INBINS + k], xr, xi);
        spec[o] = xr; spec[o + 1] = xi;
    });
}

// The fast Griffin-Lim step (Perraudin, Balazs & Sondergaard, WASPAA 2013) on the same transform: per bin,
// C = X - beta * prev, prev <- X (read and written in place by the same thread), spec = mag * C / |C| (C == 0 gives
// (mag, 0)).  beta == 0 takes C = X itself, so the step is then stft_complex_kernel's projection bit for bit whatever
// prev holds.  Layout and ragged-clip rules as stft_complex_kernel (prev like spec); every clip is batched (lens and
// frames given).
__global__ void __launch_bounds__(256) stft_complex_momentum_kernel(const float* __restrict__ x, const int* lens,
                                                                    long long x_pitch, const float* __restrict__ mag,
                                                                    float2* __restrict__ prev,
                                                                    float2* __restrict__ spec, const int* frames,
                                                                    long long frame_pitch, float beta) {
    pdl_trigger(); pdl_wait();
    const int frame = blockIdx.x, clip = blockIdx.y;
    if (frame >= frames[clip]) return;
    const size_t row = ((size_t)clip * frame_pitch + frame) * INBINS;
    stft_frame_1024(x + clip * x_pitch, lens[clip], frame, [&](int k, float xr, float xi) {
        const float2 p = prev[row + k];
        prev[row + k] = make_float2(xr, xi);
        if (beta != 0.f) { xr = fmaf(-beta, p.x, xr); xi = fmaf(-beta, p.y, xi); }
        project_1024(mag[row + k], xr, xi);
        spec[row + k] = make_float2(xr, xi);
    });
}

// spec (nframes, 513, 2) -> y (len) += window * irfft(spec[frame]) placed at frame*hop - pad   (y zeroed by the caller)
// for the frames frame = 4*blockIdx.x + residue: no two of them overlap, so the add is a plain load and store.
// Inverse real FFT through the same 512-point complex transform: Z[k] = E[k] + i*O[k] with
// E = (X[k] + conj(X[512-k]))/2, O = (X[k] - conj(X[512-k]))/2 * conj(W1024^k); z = IFFT512(Z); x[2n] = Re z, x[2n+1] = Im z.
// IFFT via conjugation: ifft(Z) = conj(fft(conj(Z))) / 512.
__global__ void __launch_bounds__(256) istft_kernel(const float* __restrict__ spec, float* __restrict__ y, int len0,
                                                    const int* lens, long long y_pitch, int nframes0,
                                                    const int* frames, long long frame_pitch, int residue) {
    pdl_trigger(); pdl_wait();
    __shared__ float zr[INH], zi[INH], twr[INH / 2], twi[INH / 2];
    const int frame = 4 * blockIdx.x + residue, clip = blockIdx.y, tid = threadIdx.x;
    const int nframes = frames ? frames[clip] : nframes0, len = lens ? lens[clip] : len0;
    if (frame >= nframes) return;
    y += clip * y_pitch;
    { float s, c; sincospif(-(float)tid / 256.f, &s, &c); twr[tid] = c; twi[tid] = s; }
    const float* X = spec + (clip * frame_pitch + frame) * INBINS * 2;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int k = tid + h * 256;                                   // 0..511
        const float ar = X[2 * k], ai = X[2 * k + 1];
        const float br = X[2 * (INH - k)], bi = -X[2 * (INH - k) + 1];    // conj(X[512-k])
        const float er = 0.5f * (ar + br), ei = 0.5f * (ai + bi), dr = 0.5f * (ar - br), di = 0.5f * (ai - bi);
        float s, c;
        sincospif((float)k / 512.f, &s, &c);                           // conj(W1024^k) = exp(+2 pi i k / 1024)
        const float orr = dr * c - di * s, oi = dr * s + di * c;
        // Z = E + i*O ; feed conj(Z) to the forward transform
        const float Zr = er - oi, Zi = ei + orr;
        const int r = ibitrev9(k);
        zr[r] = Zr; zi[r] = -Zi;
    }
    __syncthreads();
    fft512(zr, zi, twr, twi, tid);
    const int base = frame * IHOP - IPAD;
    const float inv = 1.f / 512.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = tid + h * 256;
        const float v0 = zr[n] * inv, v1 = -zi[n] * inv;                 // conj back
        const int s0 = base + 2 * n, s1 = s0 + 1;
        if (s0 >= 0 && s0 < len) y[s0] += v0 * frame_window(2 * n);
        if (s1 >= 0 && s1 < len) y[s1] += v1 * frame_window(2 * n + 1);
    }
}

// y[n] = x[n] + c*y[n-1]  (audio.py:26-28: lfilter([1], [1, -c], x)).  One CTA per clip: the recurrence is serial, so
// thread 0 walks it while the whole block streams 1024-sample chunks through shared memory (coalesced HBM traffic).
__global__ void __launch_bounds__(256) deemphasis_kernel(const float* __restrict__ x, float* __restrict__ y, int len,
                                                         long long stride, float c) {
    pdl_trigger(); pdl_wait();
    __shared__ float buf[1024];
    const float* xi = x + blockIdx.x * stride;
    float* yo = y + blockIdx.x * stride;
    float prev = 0.f;
    for (int c0 = 0; c0 < len; c0 += 1024) {
        const int n = min(1024, len - c0);
        for (int i = threadIdx.x; i < n; i += 256) buf[i] = xi[c0 + i];
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int i = 0; i < n; ++i) { prev = fmaf(c, prev, buf[i]); buf[i] = prev; }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += 256) yo[c0 + i] = buf[i];
        __syncthreads();
    }
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_spec_to_amp(const float* spec_norm, float* amp, long long n, float min_level_db, float ref_level_db,
                    float power, void* stream) {
    long long blocks = (n + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    launch_k(spec_to_amp_kernel, (int)blocks, 256, 0, (cudaStream_t)stream, spec_norm, amp, n, min_level_db, ref_level_db,
             power);
    return check_launch("spec_to_amp");
}

static int stft_complex_launch(const float* wav, int len0, const int* lens, long long pitch, const float* mag,
                               float* spec, int nframes0, const int* frames, int max_frames, int nclips,
                               cudaStream_t st) {
    launch_k(stft_complex_kernel, dim3(max_frames, nclips), 256, 0, st, wav, len0, lens, pitch, mag, spec, nframes0,
             frames, (long long)max_frames);
    return check_launch("stft_complex");
}

// four ordered launches, one per residue class of the frame index (see istft_kernel)
static int istft_launch(const float* spec, float* wav, int len0, const int* lens, long long pitch, int nframes0,
                        const int* frames, int max_frames, int nclips, cudaStream_t st) {
    for (int r = 0; r < 4; ++r) {
        const int gx = (max_frames - r + 3) / 4;
        if (gx < 1) break;
        launch_k(istft_kernel, dim3(gx, nclips), 256, 0, st, spec, wav, len0, lens, pitch, nframes0, frames,
                 (long long)max_frames, r);
        if (int e = check_launch("istft")) return e;
    }
    return 0;
}

int dv3_stft_complex(const float* wav, int n_samples, const float* mag, float* spec, int nframes, void* stream) {
    DV3_REQUIRE(nframes >= 1 && n_samples >= 1, "stft_complex: empty input");
    return stft_complex_launch(wav, n_samples, nullptr, 0, mag, spec, nframes, nullptr, nframes, 1,
                               (cudaStream_t)stream);
}

int dv3_istft(const float* spec, float* wav, int n_samples, int nframes, void* stream) {
    DV3_REQUIRE(nframes >= 1 && n_samples >= 1, "istft: empty input");
    return istft_launch(spec, wav, n_samples, nullptr, 0, nframes, nullptr, nframes, 1, (cudaStream_t)stream);
}

int dv3_stft_complex_batched(const float* wav, const int* n_samples, long long wav_pitch, const float* mag,
                             float* spec, const int* nframes, int max_frames, int nclips, void* stream) {
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nclips <= 65535 && n_samples && nframes,
                "stft_complex_batched: bad shape");
    return stft_complex_launch(wav, 0, n_samples, wav_pitch, mag, spec, 0, nframes, max_frames, nclips,
                               (cudaStream_t)stream);
}

int dv3_stft_complex_momentum_batched(const float* wav, const int* n_samples, long long wav_pitch, const float* mag,
                                      float* prev, float* spec, const int* nframes, int max_frames, int nclips,
                                      float beta, void* stream) {
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nclips <= 65535 && n_samples && nframes && mag && prev,
                "stft_complex_momentum_batched: bad shape");
    DV3_REQUIRE(beta >= 0.f && beta < 1.f, "stft_complex_momentum_batched: beta %g outside [0, 1)", (double)beta);
    launch_k(stft_complex_momentum_kernel, dim3(max_frames, nclips), 256, 0, (cudaStream_t)stream, wav, n_samples,
             wav_pitch, mag, (float2*)prev, (float2*)spec, nframes, (long long)max_frames, beta);
    return check_launch("stft_complex_momentum");
}

int dv3_istft_batched(const float* spec, float* wav, const int* n_samples, long long wav_pitch, const int* nframes,
                      int max_frames, int nclips, void* stream) {
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nclips <= 65535 && n_samples && nframes,
                "istft_batched: bad shape");
    return istft_launch(spec, wav, 0, n_samples, wav_pitch, 0, nframes, max_frames, nclips, (cudaStream_t)stream);
}

int dv3_deemphasis(const float* x, float* y, int nclips, int n_samples, long long stride, float coef, void* stream) {
    DV3_REQUIRE(nclips >= 1 && n_samples >= 1, "deemphasis: empty input");
    launch_k(deemphasis_kernel, nclips, 256, 0, (cudaStream_t)stream, x, y, n_samples, stride, coef);
    return check_launch("deemphasis");
}

}  // extern "C"
