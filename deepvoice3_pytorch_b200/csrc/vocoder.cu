// Neural vocoder kernels (DESIGN.md section 2.23): the multi-resolution STFT loss of Parallel WaveGAN (Yamamoto et
// al., 2020), the training-segment gather and the stride-s time interleave of the k = s transposed convolutions.
//
// Loss.  For one resolution (N, R), X = STFT(y) of the generated waveform and Y = STFT(x) of the target come from
// dv3_stft_complex_geom.  With A = sqrt(max(re^2 + im^2, 1e-7)), clip c's three sums over its frames and bins are
//   num = sum (A_Y - A_X)^2,  den = sum A_Y^2,  lg = sum |log A_Y - log A_X|,
// each formed in fp64: mrstft_partials_kernel sums VOC_CHUNK frames per CTA in a fixed thread order and a fixed tree,
// mrstft_clip_kernel adds the chunks of a clip in chunk order.  No atomics, and a clip's sums depend on its own frames
// alone.  mrstft_total_kernel forms clip_loss[c] = (1/M) sum_m (sqrt(num / den) + lg / (F_c K)) and the loss
// (1/B) sum_c clip_loss[c].  A clip whose length lies outside [1, n] or whose sums are not finite sets *err_flag and
// counts 0 in the loss and in the gradient.
//
// Gradient.  mrstft_bwd_kernel writes, per bin, dL/dX = dL/dA * X / A (0 where the clamp is active) with
//   dL/dA = w ((A_X - A_Y) / (sqrt(num) sqrt(den)) + sign(log A_X - log A_Y) / (F_c K A_X)),  w = d_loss / (M B),
// the first term 0 when num == 0.  adjoint = 1 writes the spectrum whose dv3_istft_geom is dL/dy instead: the inverse
// STFT computes w(n) irfft(S)(n) with irfft's 1/N, and the STFT's adjoint is w(n) sum_k Re(G_k e^{2 pi i k n / N}),
// so S_k = N G_k / 2 for 0 < k < N/2 and S_k = N Re(G_k) at k = 0 and N/2 (DESIGN.md section 2.23 derives it).
#include "common.cuh"
#include "../../include/dv3b200.h"

namespace dv3 {

constexpr int VOC_THREADS = 256, VOC_CHUNK = 8;
constexpr double VOC_FLOOR = 1e-7;

__host__ __device__ __forceinline__ int voc_num_frames(int n, int N, int R) { return (n + N - 2 * R + R - 1) / R + 1; }

__device__ __forceinline__ double voc_mag(float2 z) {
    const double re = z.x, im = z.y;
    return sqrt(fmax(re * re + im * im, VOC_FLOOR));
}

// grid (G, B): chunk g of clip c -> ws[(c G + g) * 3 + {0, 1, 2}]
__global__ void __launch_bounds__(VOC_THREADS) mrstft_partials_kernel(const float2* __restrict__ X,
                                                                      const float2* __restrict__ Y,
                                                                      const int* __restrict__ lengths, int n,
                                                                      int max_frames, int N, int R,
                                                                      double* __restrict__ ws) {
    pdl_trigger(); pdl_wait();
    __shared__ double red[3][VOC_THREADS];
    const int g = blockIdx.x, c = blockIdx.y, G = gridDim.x, K = N / 2 + 1, tid = threadIdx.x;
    const int len = lengths[c];
    const int F = (len >= 1 && len <= n) ? min(voc_num_frames(len, N, R), max_frames) : 0;
    const int f0 = g * VOC_CHUNK, f1 = min(f0 + VOC_CHUNK, F);
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    bool finite = true;                    // fmax drops a NaN, so non-finite bins are caught here
    const size_t base = (size_t)c * max_frames * K;
    for (int i = f0 * K + tid; i < f1 * K; i += VOC_THREADS) {
        const float2 zx = X[base + i], zy = Y[base + i];
        finite &= isfinite(zx.x) && isfinite(zx.y) && isfinite(zy.x) && isfinite(zy.y);
        const double a = voc_mag(zx), b = voc_mag(zy);
        const double d = b - a;
        s0 += d * d;
        s1 += b * b;
        s2 += fabs(log(b) - log(a));
    }
    if (!finite) s0 = __longlong_as_double(0x7ff8000000000000LL);      // NaN: the clip kernel flags the clip
    red[0][tid] = s0; red[1][tid] = s1; red[2][tid] = s2;
    for (int w = VOC_THREADS / 2; w > 0; w >>= 1) {
        __syncthreads();
        if (tid < w) {
#pragma unroll
            for (int j = 0; j < 3; ++j) red[j][tid] += red[j][tid + w];
        }
    }
    __syncthreads();                       // the last pass's sums (thread 0's writes) before threads 0..2 read them
    if (tid < 3) ws[((size_t)c * G + g) * 3 + tid] = red[tid][0];
}

// one thread per clip: stats[c] = (num, den, lg, F_c K), or zeros and *err_flag for an invalid clip
__global__ void mrstft_clip_kernel(const double* __restrict__ ws, int G, const int* __restrict__ lengths, int n,
                                   int max_frames, int N, int R, int B, double* __restrict__ stats,
                                   int* __restrict__ err_flag) {
    pdl_trigger(); pdl_wait();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= B) return;
    const int len = lengths[c];
    double s[3] = {0.0, 0.0, 0.0};
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int j = 0; j < 3; ++j) s[j] += ws[((size_t)c * G + g) * 3 + j];
    const bool ok = len >= 1 && len <= n && voc_num_frames(len, N, R) <= max_frames && isfinite(s[0]) &&
                    isfinite(s[1]) && isfinite(s[2]);
    double* o = stats + (size_t)c * 4;
    if (!ok) *err_flag = 1;
    o[0] = ok ? s[0] : 0.0;
    o[1] = ok ? s[1] : 0.0;
    o[2] = ok ? s[2] : 0.0;
    o[3] = ok ? (double)voc_num_frames(len, N, R) * (N / 2 + 1) : 0.0;
}

__device__ __forceinline__ double voc_clip_term(const double* o) {
    return o[3] > 0.0 ? sqrt(o[0] / o[1]) + o[2] / o[3] : 0.0;
}

// one thread: clip_loss[c] = (1/M) sum_m term(m, c) in m order, *loss = (1/B) sum_c clip_loss[c] in c order
__global__ void mrstft_total_kernel(const double* __restrict__ stats, int M, int B, double* __restrict__ clip_loss,
                                    float* __restrict__ loss) {
    pdl_trigger(); pdl_wait();
    double tot = 0.0;
    for (int c = 0; c < B; ++c) {
        double s = 0.0;
        for (int m = 0; m < M; ++m) s += voc_clip_term(stats + ((size_t)m * B + c) * 4);
        s /= M;
        if (clip_loss) clip_loss[c] = s;
        tot += s;
    }
    *loss = (float)(tot / B);
}

// grid (ceil(max_frames K / 256), B): dL/dX per bin (0 past the clip's frames and for invalid clips)
__global__ void __launch_bounds__(VOC_THREADS) mrstft_bwd_kernel(const float2* __restrict__ X,
                                                                 const float2* __restrict__ Y,
                                                                 const double* __restrict__ stats, int max_frames,
                                                                 int N, int M, int B, const float* __restrict__ d_loss,
                                                                 int adjoint, float2* __restrict__ dX) {
    pdl_trigger(); pdl_wait();
    const int c = blockIdx.y, K = N / 2 + 1;
    const int i = blockIdx.x * VOC_THREADS + threadIdx.x;
    if (i >= max_frames * K) return;
    const size_t at = (size_t)c * max_frames * K + i;
    const double* o = stats + (size_t)c * 4;
    const int k = i % K;
    float2 out = make_float2(0.f, 0.f);
    if (o[3] > 0.0 && i < (int)o[3]) {
        const float2 z = X[at];
        const double re = z.x, im = z.y, p = re * re + im * im;
        if (p > VOC_FLOOR) {
            const double a = sqrt(p), b = voc_mag(Y[at]);
            const double w = (double)d_loss[0] / ((double)M * B);
            const double nrm = sqrt(o[0]) * sqrt(o[1]);
            const double la = log(a), lb = log(b);
            double da = (o[0] > 0.0 ? (a - b) / nrm : 0.0) + (la > lb ? 1.0 : la < lb ? -1.0 : 0.0) / (o[3] * a);
            da *= w / a;
            double gr = da * re, gi = da * im;
            if (adjoint) {
                const bool edge = k == 0 || k == K - 1;
                const double s = edge ? (double)N : 0.5 * N;
                gr *= s;
                gi = edge ? 0.0 : gi * s;
            }
            out = make_float2((float)gr, (float)gi);
        }
    }
    dX[at] = out;
}

// Segment gather, grid (tiles + ceil(S R / 256), B), 32 x 8 threads.  The first tiles = ceil(S/32) ceil(K/32) CTAs move
// one 32 x 32 tile each through shared memory, so that both the spectrogram reads (along k) and the cond writes (along
// s) are coalesced:
//   cond[b, k, s] = lin[b, f0_b + s, k]                       (s < S, k < K)
// the remaining CTAs write 256 target samples each:
//   target[b, u]  = fp32(x[p] - c x[p - 1]) at p = f0_b R - (N - R) / 2 + u, x = 0 outside [0, len_b)   (u < S R)
// A start outside [0, frames_b - S] sets *err_flag and writes zeros.
__global__ void __launch_bounds__(VOC_THREADS) voc_gather_kernel(const float* __restrict__ lin, int lin_rows,
                                                                 const int* __restrict__ frames,
                                                                 const float* __restrict__ wav, long long pitch,
                                                                 const int* __restrict__ lengths,
                                                                 const int* __restrict__ starts, int S, int N, int R,
                                                                 double preemph, float* __restrict__ cond,
                                                                 float* __restrict__ target, int* __restrict__ err_flag) {
    pdl_trigger(); pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.y, K = N / 2 + 1, tx = threadIdx.x, ty = threadIdx.y;
    const int ns = (S + 31) / 32, tiles = ns * ((K + 31) / 32);
    const int f0 = starts[b], len = lengths[b];
    const bool ok = f0 >= 0 && f0 + S <= frames[b] && frames[b] <= lin_rows && len >= 0 && len <= pitch;
    if (!ok && blockIdx.x == 0 && tx == 0 && ty == 0) *err_flag = 1;
    if ((int)blockIdx.x < tiles) {                         // uniform per CTA: the barrier below is reached by all
        const int s0 = (blockIdx.x % ns) * 32, k0 = (blockIdx.x / ns) * 32;
        for (int r = ty; r < 32; r += 8) {
            const int s = s0 + r, k = k0 + tx;
            tile[r][tx] = (ok && s < S && k < K) ? lin[((size_t)b * lin_rows + f0 + s) * K + k] : 0.f;
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) {
            const int k = k0 + r, s = s0 + tx;
            if (k < K && s < S) cond[((size_t)b * K + k) * S + s] = tile[tx][r];
        }
        return;
    }
    const int i = ((int)blockIdx.x - tiles) * VOC_THREADS + ty * 32 + tx;
    if (i < S * R) {
        const long long p = (long long)f0 * R - (N - R) / 2 + i;
        const float* x = wav + b * pitch;
        double v = 0.0;
        if (ok && p >= 0 && p < len) v = p >= 1 ? fma(-preemph, (double)x[p - 1], (double)x[p]) : (double)x[p];
        target[(size_t)b * S * R + i] = (float)v;
    }
}

// out[b, c, s t + j] = in[b, j C + c, t]; inverse = 1 undoes it
__global__ void __launch_bounds__(VOC_THREADS) interleave_s_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                                   int B, int C, int T, int s, int inverse) {
    pdl_trigger(); pdl_wait();
    const long long total = (long long)B * C * s * T;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(i % ((long long)s * T));
        const long long bc = i / ((long long)s * T);
        const int c = (int)(bc % C), b = (int)(bc / C);
        const int t = u / s, j = u % s;
        const size_t packed = ((size_t)b * s * C + (size_t)j * C + c) * T + t;
        if (!inverse) out[i] = in[packed];
        else out[packed] = in[i];
    }
}

static int voc_geometry(int N, int R, const char* what) {
    DV3_REQUIRE(N >= 256 && N <= 4096 && N % 2 == 0 && R >= 1 && N % R == 0 && N / R >= 2 && N / R <= 8,
                "%s: unsupported STFT geometry fft_size %d, hop %d", what, N, R);
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

long long dv3_mrstft_ws_doubles(int B, int max_frames) {
    return (long long)B * ((max_frames + VOC_CHUNK - 1) / VOC_CHUNK) * 3;
}

int dv3_mrstft_loss_fwd(const float* spec_y, const float* spec_x, const int* lengths, int n, int B, int max_frames,
                        int n_fft, int hop, double* ws, double* stats, int* err_flag, void* stream) {
    const char* what = "mrstft_loss_fwd";
    if (voc_geometry(n_fft, hop, what)) return 1;
    DV3_REQUIRE(spec_y && spec_x && lengths && ws && stats && err_flag, "%s: null operand", what);
    DV3_REQUIRE(B >= 1 && B <= 65535 && n >= 1 && max_frames >= 1 &&
                (long long)B * max_frames * (n_fft / 2 + 1) < 2147483647LL, "%s: B=%d, n=%d, max_frames=%d", what, B,
                n, max_frames);
    const int G = (max_frames + VOC_CHUNK - 1) / VOC_CHUNK;
    cudaStream_t st = (cudaStream_t)stream;
    launch_k(mrstft_partials_kernel, dim3(G, B), VOC_THREADS, 0, st, (const float2*)spec_y, (const float2*)spec_x,
             lengths, n, max_frames, n_fft, hop, ws);
    if (int e = check_launch(what)) return e;
    launch_k(mrstft_clip_kernel, ceil_div(B, 128), 128, 0, st, (const double*)ws, G, lengths, n, max_frames, n_fft, hop,
             B, stats, err_flag);
    return check_launch(what);
}

int dv3_mrstft_loss_total(const double* stats, int M, int B, double* clip_loss, float* loss, void* stream) {
    DV3_REQUIRE(stats && loss && M >= 1 && B >= 1 && B <= 65535, "mrstft_loss_total: M=%d, B=%d", M, B);
    launch_k(mrstft_total_kernel, 1, 1, 0, (cudaStream_t)stream, stats, M, B, clip_loss, loss);
    return check_launch("mrstft_loss_total");
}

int dv3_mrstft_loss_bwd(const float* spec_y, const float* spec_x, const double* stats, int B, int max_frames,
                        int n_fft, int hop, int M, const float* d_loss, int adjoint, float* dspec, void* stream) {
    const char* what = "mrstft_loss_bwd";
    if (voc_geometry(n_fft, hop, what)) return 1;
    DV3_REQUIRE(spec_y && spec_x && stats && d_loss && dspec && M >= 1, "%s: null operand or M=%d", what, M);
    const long long bins = (long long)max_frames * (n_fft / 2 + 1);
    DV3_REQUIRE(B >= 1 && B <= 65535 && max_frames >= 1 && bins * B < 2147483647LL, "%s: B=%d, max_frames=%d", what, B,
                max_frames);
    launch_k(mrstft_bwd_kernel, dim3((unsigned)((bins + VOC_THREADS - 1) / VOC_THREADS), B), VOC_THREADS, 0,
             (cudaStream_t)stream, (const float2*)spec_y, (const float2*)spec_x, stats, max_frames, n_fft, M, B, d_loss,
             adjoint, (float2*)dspec);
    return check_launch(what);
}

int dv3_vocoder_gather(const float* lin, int lin_rows, const int* frames, const float* wav, long long pitch,
                       const int* lengths, const int* starts, int B, int S, int n_fft, int hop, double preemph,
                       float* cond, float* target, int* err_flag, void* stream) {
    const char* what = "vocoder_gather";
    if (voc_geometry(n_fft, hop, what)) return 1;
    DV3_REQUIRE(lin && frames && wav && lengths && starts && cond && target && err_flag, "%s: null operand", what);
    const int K = n_fft / 2 + 1;
    DV3_REQUIRE(B >= 1 && B <= 65535 && S >= 1 && lin_rows >= S && pitch >= 1 && (long long)S * hop < 2147483647LL &&
                (long long)B * lin_rows * K < 2147483647LL, "%s: B=%d, S=%d, lin_rows=%d", what, B, S, lin_rows);
    const int tiles = ceil_div(S, 32) * ceil_div(K, 32);
    launch_k(voc_gather_kernel, dim3(tiles + ceil_div(S * hop, VOC_THREADS), B), dim3(32, 8), 0, (cudaStream_t)stream, lin,
             lin_rows, frames, wav, pitch, lengths, starts, S, n_fft, hop, preemph, cond, target, err_flag);
    return check_launch(what);
}

int dv3_interleave(const float* in, float* out, int B, int C, int T, int stride, int inverse, void* stream) {
    DV3_REQUIRE(in && out && B >= 1 && C >= 1 && T >= 1 && stride >= 2 && stride <= 8 &&
                (long long)B * C * stride * T < 2147483647LL, "interleave: B=%d, C=%d, T=%d, stride=%d", B, C, T,
                stride);
    const long long total = (long long)B * C * stride * T;
    const long long want = (total + VOC_THREADS - 1) / VOC_THREADS, cap = 64LL * config().sms;
    const int blocks = (int)(want < cap ? want : cap);
    launch_k(interleave_s_kernel, blocks, VOC_THREADS, 0, (cudaStream_t)stream, in, out, B, C, T, stride, inverse);
    return check_launch("interleave");
}

}  // extern "C"
