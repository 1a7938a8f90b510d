// The audio front-end and Griffin-Lim kernels for every STFT frame audio.check_geometry accepts (fft_size N even,
// 256 <= N <= 4096, N/2 with no prime factor above 5; hop R = N/Q with Q in [2, 8]).  stft.cu keeps the specialised
// 1024 / 256 forward kernel, so audio.py selects stft_any_kernel only for other frames; the complex STFT and inverse
// STFT kernels here run at every frame, 1024 / 256 included.  The transform is fft_any.cuh's
// mixed-radix Stockham FFT of length N/2 with the real-packing split; window, twiddles and split factors come from a
// per-geometry fp32 table the host builds in fp64 (audio._geometry_table).
//
//   stft_any_kernel     preemphasis -> window -> rfft -> |.| -> linear dB row and sparse mel dB row, for F consecutive
//                       frames of one clip per CTA.  The (F-1)*R + N samples they span are staged once in shared memory
//                       (converted from int16 and rescaled as they are staged); the first FFT pass reads its points
//                       from there with pre-emphasis and window applied.  The whole CTA runs one frame at a time: a
//                       pass per barrier, then the split writes the linear row (coalesced) and the magnitudes to
//                       shared memory, then one warp per mel filter sums its non-zero bins (lane-strided, then a fixed
//                       shuffle tree: deterministic).  Output descriptor and zero rows as stft.cu's StftParams.
//   stft_complex_any    waveform -> complex half spectrum, optionally projected onto a magnitude (Griffin-Lim step);
//                       one CTA per frame.
//   stft_complex_momentum_any  the same transform with the fast Griffin-Lim epilogue (DESIGN.md section 7.3).
//   istft_any           complex half spectrum -> windowed frame, overlap-added in Q ordered launches, one per residue
//                       class f mod Q: frames f and f+Q do not overlap (N = Q*R), so the adds are plain loads and
//                       stores and every sample is summed in the same order every run.
#include "common.cuh"
#include "fft_any.cuh"

namespace dv3 {

using namespace fftany;

constexpr int ANY_THREADS = 256, ANY_MAX_F = 32, ANY_MAX_MELS = 128;

struct AnyParams {
    const void* wav;           // (nclips, max_len) fp32 or int16 (kernel template)
    const int* lengths;
    const float* peak;         // rescale x / peak * gain (kernel template SCALE), or null
    const float* tab;          // fft_any.cuh table for (N, R)
    const float* mel_basis;    // (n_mels, K) dense
    const int* mel_start;
    const int* mel_len;
    float* linear;             // (nclips, lin_rows, K) or null
    float* mel;                // (nclips, mel_rows, n_mels) or null
    int max_len, max_frames, n_mels, lead, ds, lin_rows, mel_rows;
    int N, R, F;               // frame, hop, frames per CTA
    Plan plan;
    float gain, preemph, c2, c0, min_level;
};

// frames of a clip of n samples (lws "perfectrec" padding of N - R samples on both sides)
__host__ __device__ __forceinline__ int any_num_frames(int n, int N, int R) { return (n + N - 2 * R + R - 1) / R + 1; }

// frames per CTA: enough to stage max(2N, 4096) samples, at most ANY_MAX_F
static inline int any_frames_per_cta(int N, int R) {
    const int span = N > 2048 ? 2 * N : 4096;
    return max(1, min(ANY_MAX_F, (span - N) / R + 1));
}
static inline size_t any_smem(int N, int R, int F) {
    const int M = N / 2, raw = ((F - 1) * R + N + 2 + 1) & ~1;
    return sizeof(float) * raw + 2 * sizeof(c2) * M + sizeof(float) * (M + 2);
}

template <bool SCALE> __device__ __forceinline__ float any_rescale(float v, float peak, float gain) {
    return SCALE ? __fmul_rn(__fdiv_rn(v, peak), gain) : v;
}
template <typename In> __device__ __forceinline__ float any_sample(In v) {
    if constexpr (sizeof(In) == 2) return __fmul_rn((float)v, 3.0517578125e-05f);       // x / 32768
    else return v;
}

// the run of passes after the first: ping-pong between a and b; returns the buffer holding the result
__device__ __forceinline__ c2* any_passes(const Plan pl, c2* a, c2* b, const c2* tw, int tid) {
    int Ns = pl.radix(0);
    for (int s = 1; s < pl.npass; ++s) {
        const int p = pl.radix(s);
        __syncthreads();
        fft_pass(SmemLoad{a}, b, tw, pl.M, p, Ns, tid, ANY_THREADS);
        Ns *= p;
        c2* t = a; a = b; b = t;
    }
    __syncthreads();
    return a;
}

struct FrameLoad {             // first-pass points of a staged frame: pre-emphasis on clip samples, zero outside, window
    const float* raw;          // raw[j] = x[pos0 + j - 1]
    const float* win;
    int pos0, len;
    float c;
    __device__ __forceinline__ float e(int j) const {
        const int pos = pos0 + j;
        return (pos >= 0 && pos < len) ? fmaf(-c, raw[j], raw[j + 1]) : 0.f;
    }
    __device__ __forceinline__ c2 operator()(int i) const {
        return {e(2 * i) * __ldg(win + 2 * i), e(2 * i + 1) * __ldg(win + 2 * i + 1)};
    }
};

template <typename In, bool SCALE>
__global__ void __launch_bounds__(ANY_THREADS) stft_any_kernel(const __grid_constant__ AnyParams p) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int N = p.N, R = p.R, M = N / 2, K = M + 1, F = p.F, PAD = N - R;
    const int clip = blockIdx.y, f_begin = blockIdx.x * F, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int raw_n = ((F - 1) * R + N + 2 + 1) & ~1;
    float* raw = reinterpret_cast<float*>(smem_raw);
    c2* bufa = reinterpret_cast<c2*>(raw + raw_n);
    c2* bufb = bufa + M;
    float* mag = reinterpret_cast<float*>(bufb + M);
    const int len = p.lengths[clip];
    const int nframes = min(any_num_frames(len, N, R), p.max_frames);
    const int f_end = min(f_begin + F, p.max_frames);
    const int lead = p.lead, ds = p.ds;

    {   // zero rows: this chunk's frames past the clip's end, and the lead rows in front of frame 0 (first chunk)
        const int z0 = max(f_begin, nframes);
        const int zr[2][2] = {{lead + z0, lead + f_end}, {0, blockIdx.x == 0 ? lead : 0}};
#pragma unroll
        for (int z = 0; z < 2; ++z) {
            const int r0 = zr[z][0], r1 = zr[z][1];
            if (r0 >= r1) continue;
            if (p.linear) {
                float* o = p.linear + ((size_t)clip * p.lin_rows + r0) * K;
                for (int i = tid; i < (r1 - r0) * K; i += ANY_THREADS) o[i] = 0.f;
            }
            if (p.mel) {
                const int m0 = (r0 + ds - 1) / ds, m1 = (r1 + ds - 1) / ds;
                float* o = p.mel + ((size_t)clip * p.mel_rows + m0) * p.n_mels;
                for (int i = tid; i < (m1 - m0) * p.n_mels; i += ANY_THREADS) o[i] = 0.f;
            }
        }
    }
    if (f_begin >= nframes) return;
    const int nf = min(f_end, nframes) - f_begin;

    // stage x[s0 - 1 .. s0 + span) once for the nf frames, zero outside the clip
    const In* x = reinterpret_cast<const In*>(p.wav) + (size_t)clip * p.max_len;
    const float peak = SCALE ? p.peak[clip] : 1.f, gain = p.gain;
    const int s0 = f_begin * R - PAD, span = (nf - 1) * R + N;
    for (int i = tid; i <= span; i += ANY_THREADS) {
        const int s = s0 - 1 + i;
        raw[i] = (s >= 0 && s < len) ? any_rescale<SCALE>(any_sample(x[s]), peak, gain) : 0.f;
    }
    const float* win = p.tab;
    const c2* tw = reinterpret_cast<const c2*>(p.tab + tab_tw(N));
    const c2* sp = reinterpret_cast<const c2*>(p.tab + tab_sp(N));
    const float c2s = p.c2, c0 = p.c0, min_level = p.min_level;
    __syncthreads();

    for (int fl = 0; fl < nf; ++fl) {
        const int frame = f_begin + fl;
        const FrameLoad load{raw + fl * R, win, frame * R - PAD, len, p.preemph};
        fft_pass(load, bufa, tw, M, p.plan.radix(0), 1, tid, ANY_THREADS);
        const c2* Z = any_passes(p.plan, bufa, bufb, tw, tid);

        float* lin = p.linear ? p.linear + ((size_t)clip * p.lin_rows + lead + frame) * K : nullptr;
        for (int k = tid; k < K; k += ANY_THREADS) {
            const c2 X = split_bin(Z, M, k, sp[k]);
            const float a = sqrtf(fmaf(X.x, X.x, X.y * X.y));
            if (lin) lin[k] = __saturatef(fmaf(c2s, log2f(fmaxf(a, min_level)), c0));
            mag[k] = a;
        }
        __syncthreads();                                   // magnitudes complete; Z's buffer free for the next frame
        const int t = lead + frame;
        if (p.mel && t % ds == 0) {
            float* out = p.mel + ((size_t)clip * p.mel_rows + t / ds) * p.n_mels;
            for (int m = warp; m < p.n_mels; m += ANY_THREADS / 32) {
                const int s = __ldg(p.mel_start + m), l = __ldg(p.mel_len + m);
                const float* w = p.mel_basis + (size_t)m * K + s;
                float acc = 0.f;
                for (int j = lane; j < l; j += 32) acc = fmaf(__ldg(w + j), mag[s + j], acc);
#pragma unroll
                for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (lane == 0) out[m] = __saturatef(fmaf(c2s, log2f(fmaxf(acc, min_level)), c0));
            }
        }
        // the next frame's first pass writes bufa and its split writes mag only after at least one more barrier
    }
}

struct WaveLoad {              // first-pass points of a frame read straight from the waveform (no pre-emphasis)
    const float* x;
    const float* win;
    int pos0, len;
    __device__ __forceinline__ float s(int j) const {
        const int pos = pos0 + j;
        return (pos >= 0 && pos < len) ? x[pos] * __ldg(win + j) : 0.f;
    }
    __device__ __forceinline__ c2 operator()(int i) const { return {s(2 * i), s(2 * i + 1)}; }
};

// The forward transform of frame `frame` of clip `clip` into shared memory: -> the packed transform Z, whose bin k is
// split_bin(Z, M, k, sp[k]) with the split factors sp it sets.  Shared by both complex-STFT kernels.
__device__ __forceinline__ const c2* complex_any_frame(const float* x, const int* lens, long long x_pitch, int clip,
                                                       int frame, const float* tab, int N, int R, Plan plan,
                                                       const c2*& sp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int M = N / 2, tid = threadIdx.x;
    c2* bufa = reinterpret_cast<c2*>(smem_raw);
    c2* bufb = bufa + M;
    const c2* tw = reinterpret_cast<const c2*>(tab + tab_tw(N));
    sp = reinterpret_cast<const c2*>(tab + tab_sp(N));
    const WaveLoad load{x + clip * x_pitch, tab, frame * R - (N - R), lens[clip]};
    fft_pass(load, bufa, tw, M, plan.radix(0), 1, tid, ANY_THREADS);
    return any_passes(plan, bufa, bufb, tw, tid);
}

// mag X / |X| (X == 0 gives phase 0): the Griffin-Lim magnitude projection of both complex-STFT kernels
__device__ __forceinline__ void project_any(float m, c2& X) {
    const float a = sqrtf(fmaf(X.x, X.x, X.y * X.y));  // explicit: both kernels round |X|^2 the same way
    if (a > 0.f) { X.x *= m / a; X.y *= m / a; } else { X.x = m; X.y = 0.f; }
}

// wav -> spec (clip, frame, K) float2 [projected onto mag when given]; grid (max_frames, nclips)
__global__ void __launch_bounds__(ANY_THREADS) stft_complex_any_kernel(const float* __restrict__ x, const int* lens,
                                                                       long long x_pitch, const float* __restrict__ magp,
                                                                       float2* __restrict__ spec, const int* frames,
                                                                       long long frame_pitch, const float* tab, int N,
                                                                       int R, Plan plan) {
    pdl_trigger(); pdl_wait();
    const int M = N / 2, K = M + 1;
    const int frame = blockIdx.x, clip = blockIdx.y, tid = threadIdx.x;
    if (frame >= frames[clip]) return;
    const c2* sp;
    const c2* Z = complex_any_frame(x, lens, x_pitch, clip, frame, tab, N, R, plan, sp);
    const size_t row = ((size_t)clip * frame_pitch + frame) * K;
    for (int k = tid; k < K; k += ANY_THREADS) {
        c2 X = split_bin(Z, M, k, sp[k]);
        if (magp) project_any(magp[row + k], X);
        spec[row + k] = make_float2(X.x, X.y);
    }
}

// The fast Griffin-Lim step on the same transform (Perraudin, Balazs & Sondergaard, WASPAA 2013): per bin
// C = X - beta * prev, prev <- X in place (same thread, same element), spec = mag * C / |C|; beta == 0 takes C = X,
// the projection of stft_complex_any_kernel bit for bit.  grid (max_frames, nclips); frames past a clip's count are
// neither read nor written.
__global__ void __launch_bounds__(ANY_THREADS) stft_complex_momentum_any_kernel(
        const float* __restrict__ x, const int* lens, long long x_pitch, const float* __restrict__ magp,
        float2* __restrict__ prev, float2* __restrict__ spec, const int* frames, long long frame_pitch, float beta,
        const float* tab, int N, int R, Plan plan) {
    pdl_trigger(); pdl_wait();
    const int M = N / 2, K = M + 1;
    const int frame = blockIdx.x, clip = blockIdx.y, tid = threadIdx.x;
    if (frame >= frames[clip]) return;
    const c2* sp;
    const c2* Z = complex_any_frame(x, lens, x_pitch, clip, frame, tab, N, R, plan, sp);
    const size_t row = ((size_t)clip * frame_pitch + frame) * K;
    for (int k = tid; k < K; k += ANY_THREADS) {
        c2 X = split_bin(Z, M, k, sp[k]);
        const float2 p = prev[row + k];
        prev[row + k] = make_float2(X.x, X.y);
        if (beta != 0.f) { X.x = fmaf(-beta, p.x, X.x); X.y = fmaf(-beta, p.y, X.y); }
        project_any(magp[row + k], X);
        spec[row + k] = make_float2(X.x, X.y);
    }
}

struct SpecLoad {              // first-pass points of the inverse: conj Z[i] merged from the half spectrum
    const float2* X;
    const c2* sp;
    int M;
    __device__ __forceinline__ c2 operator()(int i) const {
        const float2 a = X[i], b = X[M - i];
        return merge_bin_conj(c2{a.x, a.y}, c2{b.x, b.y}, sp[i]);
    }
};

// y (clip) += window * irfft(spec[frame]) at frame*R - (N - R), frames frame = Q*blockIdx.x + residue
__global__ void __launch_bounds__(ANY_THREADS, 4) istft_any_kernel(const float2* __restrict__ spec, float* __restrict__ y,
                                                                const int* lens, long long y_pitch, const int* frames,
                                                                long long frame_pitch, int residue, const float* tab,
                                                                int N, int R, Plan plan) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int M = N / 2, K = M + 1, Q = N / R;
    const int frame = Q * blockIdx.x + residue, clip = blockIdx.y, tid = threadIdx.x;
    if (frame >= frames[clip]) return;
    c2* bufa = reinterpret_cast<c2*>(smem_raw);
    c2* bufb = bufa + M;
    const c2* tw = reinterpret_cast<const c2*>(tab + tab_tw(N));
    const c2* sp = reinterpret_cast<const c2*>(tab + tab_sp(N));
    const SpecLoad load{spec + ((size_t)clip * frame_pitch + frame) * K, sp, M};
    fft_pass(load, bufa, tw, M, plan.radix(0), 1, tid, ANY_THREADS);
    const c2* z = any_passes(plan, bufa, bufb, tw, tid);
    const int len = lens[clip], base = frame * R - (N - R);
    const float inv = 1.f / (float)M;
    y += clip * y_pitch;
    for (int n = tid; n < M; n += ANY_THREADS) {
        const int s0 = base + 2 * n, s1 = s0 + 1;
        if (s0 >= 0 && s0 < len) y[s0] += (z[n].x * inv) * __ldg(tab + 2 * n);
        if (s1 >= 0 && s1 < len) y[s1] += (-z[n].y * inv) * __ldg(tab + 2 * n + 1);
    }
}

static int any_geometry(int N, int R, Plan& plan, const char* what) {
    DV3_REQUIRE(N >= MIN_N && N <= MAX_N && N % 2 == 0 && R >= 1 && N % R == 0 && N / R >= 2 && N / R <= 8,
                "%s: unsupported STFT geometry fft_size %d, hop %d", what, N, R);
    plan = make_plan(N / 2);
    DV3_REQUIRE(plan.npass > 0, "%s: fft_size / 2 = %d has a prime factor above 5", what, N / 2);
    return 0;
}

template <typename Kern>
static int any_reserve(Kern k, size_t bytes, const char* what) {
    DV3_REQUIRE(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess,
                "%s: cannot reserve %zu bytes of shared memory", what, bytes);
    return 0;
}

template <typename In, bool SCALE>
static int launch_stft_any(const AnyParams& p, int nclips, cudaStream_t st, const char* what) {
    const size_t smem = any_smem(p.N, p.R, p.F);
    if (any_reserve(stft_any_kernel<In, SCALE>, smem, what)) return 1;
    launch_k(stft_any_kernel<In, SCALE>, dim3(ceil_div(p.max_frames, p.F), nclips), ANY_THREADS, smem, st, p);
    return check_launch(what);
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_stft_num_frames_geom(int n_samples, int n_fft, int hop) { return any_num_frames(n_samples, n_fft, hop); }

int dv3_stft_mel_geom(const void* wav, int wav_int16, const int* lengths, const float* peak, float rescaling_max,
                      const float* table, const float* mel_basis, const int* mel_start, const int* mel_len,
                      float* linear, float* mel, int nclips, int max_len, int T_lin, int lead, int downsample_step,
                      int n_mels, int n_fft, int hop, float preemph, float min_level_db, float ref_level_db,
                      void* stream) {
    const char* what = "stft_mel_geom";
    AnyParams p{};
    if (any_geometry(n_fft, hop, p.plan, what)) return 1;
    DV3_REQUIRE(nclips >= 1 && nclips <= 65535, "%s: nclips %d out of range", what, nclips);
    DV3_REQUIRE(lead >= 0 && lead < T_lin, "%s: lead %d must lie in [0, T_lin = %d)", what, lead, T_lin);
    DV3_REQUIRE(downsample_step >= 1, "%s: bad downsample_step %d", what, downsample_step);
    DV3_REQUIRE(n_mels >= 0 && n_mels <= ANY_MAX_MELS, "%s: n_mels %d > %d", what, n_mels, ANY_MAX_MELS);
    DV3_REQUIRE(min_level_db < 0.f, "%s: min_level_db must be negative (got %g)", what, (double)min_level_db);
    DV3_REQUIRE(table && lengths, "%s: missing table or lengths", what);
    const double inv = 1.0 / -(double)min_level_db, c2 = 20.0 * 0.30102999566398120 * inv;
    p.wav = wav; p.lengths = lengths; p.peak = peak; p.tab = table;
    p.mel_basis = mel_basis; p.mel_start = mel_start; p.mel_len = mel_len; p.linear = linear; p.mel = mel;
    p.max_len = max_len; p.max_frames = T_lin - lead; p.n_mels = n_mels; p.lead = lead; p.ds = downsample_step;
    p.lin_rows = T_lin; p.mel_rows = (T_lin + downsample_step - 1) / downsample_step;
    p.N = n_fft; p.R = hop; p.F = any_frames_per_cta(n_fft, hop);
    p.gain = rescaling_max; p.preemph = preemph; p.c2 = (float)c2; p.c0 = (float)(1.0 - (double)ref_level_db * inv);
    p.min_level = (float)pow(10.0, (double)min_level_db / 20.0);
    const cudaStream_t st = (cudaStream_t)stream;
    if (wav_int16) return peak ? launch_stft_any<short, true>(p, nclips, st, what)
                               : launch_stft_any<short, false>(p, nclips, st, what);
    return peak ? launch_stft_any<float, true>(p, nclips, st, what) : launch_stft_any<float, false>(p, nclips, st, what);
}

int dv3_stft_complex_geom(const float* wav, const int* n_samples, long long wav_pitch, const float* mag, float* spec,
                          const int* nframes, int max_frames, int nclips, const float* table, int n_fft, int hop,
                          void* stream) {
    const char* what = "stft_complex_geom";
    Plan plan;
    if (any_geometry(n_fft, hop, plan, what)) return 1;
    DV3_REQUIRE(max_frames >= 1 && max_frames <= 2147483647 && nclips >= 1 && nclips <= 65535 && n_samples && nframes
                && table, "%s: bad shape", what);
    const size_t smem = 2 * sizeof(c2) * (n_fft / 2);
    if (any_reserve(stft_complex_any_kernel, smem, what)) return 1;
    launch_k(stft_complex_any_kernel, dim3(max_frames, nclips), ANY_THREADS, smem, (cudaStream_t)stream, wav,
             n_samples, wav_pitch, mag, (float2*)spec, nframes, (long long)max_frames, table, n_fft, hop, plan);
    return check_launch(what);
}

int dv3_stft_complex_momentum_geom(const float* wav, const int* n_samples, long long wav_pitch, const float* mag,
                                   float* prev, float* spec, const int* nframes, int max_frames, int nclips,
                                   float beta, const float* table, int n_fft, int hop, void* stream) {
    const char* what = "stft_complex_momentum_geom";
    Plan plan;
    if (any_geometry(n_fft, hop, plan, what)) return 1;
    DV3_REQUIRE(max_frames >= 1 && max_frames <= 2147483647 && nclips >= 1 && nclips <= 65535 && n_samples && nframes
                && table && mag && prev, "%s: bad shape", what);
    DV3_REQUIRE(beta >= 0.f && beta < 1.f, "%s: beta %g outside [0, 1)", what, (double)beta);
    const size_t smem = 2 * sizeof(c2) * (n_fft / 2);
    if (any_reserve(stft_complex_momentum_any_kernel, smem, what)) return 1;
    launch_k(stft_complex_momentum_any_kernel, dim3(max_frames, nclips), ANY_THREADS, smem, (cudaStream_t)stream, wav,
             n_samples, wav_pitch, mag, (float2*)prev, (float2*)spec, nframes, (long long)max_frames, beta, table,
             n_fft, hop, plan);
    return check_launch(what);
}

// Q = n_fft / hop ordered launches, one per residue class of the frame index (see istft_any_kernel)
int dv3_istft_geom(const float* spec, float* wav, const int* n_samples, long long wav_pitch, const int* nframes,
                   int max_frames, int nclips, const float* table, int n_fft, int hop, void* stream) {
    const char* what = "istft_geom";
    Plan plan;
    if (any_geometry(n_fft, hop, plan, what)) return 1;
    DV3_REQUIRE(max_frames >= 1 && nclips >= 1 && nclips <= 65535 && n_samples && nframes && table, "%s: bad shape",
                what);
    const size_t smem = 2 * sizeof(c2) * (n_fft / 2);
    if (any_reserve(istft_any_kernel, smem, what)) return 1;
    const int Q = n_fft / hop;
    for (int r = 0; r < Q; ++r) {
        const int gx = (max_frames - r + Q - 1) / Q;
        if (gx < 1) break;
        launch_k(istft_any_kernel, dim3(gx, nclips), ANY_THREADS, smem, (cudaStream_t)stream,
                 (const float2*)spec, wav, n_samples, wav_pitch, nframes, (long long)max_frames, r, table, n_fft, hop,
                 plan);
        if (int e = check_launch(what)) return e;
    }
    return 0;
}

}  // extern "C"
