// Intelligibility of speech (intelligibility.py, DESIGN.md section 2.20): STOI (Taal et al. 2011) and ESTOI (Jensen &
// Taal 2016) of clips already resampled to 10 kHz, in four entry points that follow the measure's stages.
//
// Clip descriptor: int64 rows (wav_off, n, frame_off, ola_off, mask_clip).  Clip c is n samples at wav + wav_off.  It
// has F0 = len(range(0, n - 256, 128)) analysis frames, whose per-frame values sit at frame_off .. frame_off + F0 - 1;
// its band envelopes take 15 F0 floats from 15 frame_off on (band i, frame t at i F0 + t).  Its compacted signal takes
// the (F0 - 1) 128 + 256 samples (0 when F0 = 0) from ola_off on.  mask_clip is the clip whose keep mask it uses: itself
// for the warped measure, the clean clip of the pair (of the same n) for the aligned one.
//
//   frames    one CTA per clip.  e_t = 20 log10(||w x_t||_2 + eps), w(m) = 0.5 - 0.5 cos(2 pi (m + 1) / 257) in fp64,
//             the squares summed in fp64 (lane l sums m = l + 32 q in q order, then a fixed shfl_down tree); keep_t =
//             e_t > max_t e_t - 40; kept_idx = the kept frames in order (a ballot / popc scan, integers only) and
//             kept[c] = their count K.
//   ola       elementwise over the compacted signal of (K - 1) 128 + 256 samples, K the mask clip's count: sample s is
//             w(r) x[128 kept_idx[k] + r] of kept frame k = s / 128 (r = s % 128), added after the one of frame k - 1
//             (r + 128), each product rounded to fp32.  frames[c] = max(K - 1, 0), the frames of the compacted signal.
//   bands     one warp per frame t < frames[c] of the compacted signal: the fp32 512-point real transform of fft_any.cuh
//             (M = 256: four radix-4 Stockham passes and the split) of w y_t zero-padded to 512; X[i, t] = sqrt of the
//             |X(k)|^2 of bins lo_i <= k < hi_i summed in bin order.  feat (optional) gets the DTW features
//             10 log10(max(X[i, t]^2, 1e-10)) as (frame, 15) rows at frame_off.
//   segments  one warp per segment s < J = L - 29 of a pair's path of L = steps[p] steps (pairs: int64 rows (clean
//             clip, processed clip, path_off, seg_off); path: int32 (i, j) frame pairs from path_off on).  The two
//             15 x 30 matrices are staged in fp64 and everything after is fp64: STOI's clipped, centred correlation of
//             each band row (lane i owns band i, 30 steps in order), summed over the bands in order; ESTOI's row then
//             column normalisation and (1/30) sum X^ Y^ (lane t owns column t, the bands in order, then t in order).
//             A second launch, one thread per pair, sums its J segments in order: stoi = sum / (15 J), estoi = sum / J,
//             NaN when J = 0.
// No atomics anywhere and every sum has a fixed order, so a pair's bits depend on its own clips alone.
#include <math_constants.h>

#include "fft_any.cuh"
#include "common.cuh"

namespace dv3 {

constexpr int ST_FRAME = 256, ST_HOP = 128, ST_NFFT = 512, ST_M = ST_NFFT / 2;
constexpr int ST_BANDS = 15, ST_SEG = 30;
constexpr int ST_CLIP = 5, ST_PAIR = 4;            // int64 fields of a clip / pair descriptor
constexpr int ST_THREADS = 256;                     // frames and ola kernels
constexpr int ST_OLA_TILE = 1024;                   // compacted samples per ola CTA
constexpr int ST_BAND_WARPS = 8;                    // frames per bands CTA
constexpr int ST_SEG_WARPS = 4;                     // segments per segments CTA
constexpr int ST_MAX_BIN = 256;                     // bands use bins below this
constexpr double ST_EPS = 2.220446049250313e-16;
constexpr double ST_RANGE_DB = 40.0;
constexpr double ST_CLIP_Y = 6.623413251903491;       // 1 + 10^(-beta / 20), beta = -15 dB

static __host__ __device__ inline long long st_frames(long long n) {
    return n > ST_FRAME ? (n - ST_FRAME + ST_HOP - 1) / ST_HOP : 0;
}

__global__ void __launch_bounds__(ST_THREADS)
stoi_frames_kernel(const float* __restrict__ wav, const long long* __restrict__ clips, const double* __restrict__ win,
                   double* __restrict__ energy, int* __restrict__ keep, int* __restrict__ kept_idx,
                   int* __restrict__ kept) {
    pdl_trigger(); pdl_wait();
    __shared__ double s_max[ST_THREADS / 32];
    __shared__ int s_cnt[ST_THREADS / 32];
    const long long* d = clips + (long long)ST_CLIP * blockIdx.x;
    const float* x = wav + d[0];
    const long long F0 = st_frames(d[1]), fo = d[2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double mx = -INFINITY;
    for (long long t = warp; t < F0; t += ST_THREADS / 32) {
        const float* xt = x + t * ST_HOP;
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < ST_FRAME / 32; ++q) {
            const int m = lane + 32 * q;
            const double v = win[m] * (double)xt[m];
            acc = fma(v, v, acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            const double e = 20.0 * log10(sqrt(acc) + ST_EPS);
            energy[fo + t] = e;
            mx = fmax(mx, e);
        }
    }
    if (lane == 0) s_max[warp] = mx;
    __syncthreads();                                 // also makes this CTA's energy stores visible to all its threads
    mx = s_max[0];
#pragma unroll
    for (int w = 1; w < ST_THREADS / 32; ++w) mx = fmax(mx, s_max[w]);
    const double thr = mx - ST_RANGE_DB;
    int base = 0;
    for (long long t0 = 0; t0 < F0; t0 += ST_THREADS) {
        const long long t = t0 + threadIdx.x;
        const bool k = t < F0 && energy[fo + t] > thr;
        const unsigned b = __ballot_sync(0xffffffffu, k);
        if (lane == 0) s_cnt[warp] = __popc(b);
        __syncthreads();
        int pos = base + __popc(b & ((1u << lane) - 1u));
        for (int w = 0; w < warp; ++w) pos += s_cnt[w];
        if (t < F0) {
            keep[fo + t] = k;
            if (k) kept_idx[fo + pos] = (int)t;
        }
        for (int w = 0; w < ST_THREADS / 32; ++w) base += s_cnt[w];
        __syncthreads();
    }
    if (threadIdx.x == 0) kept[blockIdx.x] = base;
}

__global__ void __launch_bounds__(ST_THREADS)
stoi_ola_kernel(const float* __restrict__ wav, const long long* __restrict__ clips, const float* __restrict__ win,
                const int* __restrict__ kept_idx, const int* __restrict__ kept, float* __restrict__ ola,
                int* __restrict__ frames) {
    pdl_trigger(); pdl_wait();
    const int c = blockIdx.y;
    const long long* d = clips + (long long)ST_CLIP * c;
    const long long m = d[4];
    const int K = kept[m];
    if (blockIdx.x == 0 && threadIdx.x == 0) frames[c] = K > 0 ? K - 1 : 0;
    const long long L = K > 0 ? (long long)(K - 1) * ST_HOP + ST_FRAME : 0;
    const float* x = wav + d[0];
    const int* idx = kept_idx + clips[(long long)ST_CLIP * m + 2];
    float* y = ola + d[3];
    const long long s1 = min(L, (long long)(blockIdx.x + 1) * ST_OLA_TILE);
    for (long long s = (long long)blockIdx.x * ST_OLA_TILE + threadIdx.x; s < s1; s += ST_THREADS) {
        const long long k = s / ST_HOP;
        const int r = (int)(s - k * ST_HOP);
        float acc = 0.f;
        if (k >= 1) acc = __fmul_rn(win[r + ST_HOP], x[(long long)idx[k - 1] * ST_HOP + r + ST_HOP]);
        if (k < K) acc = __fadd_rn(acc, __fmul_rn(win[r], x[(long long)idx[k] * ST_HOP + r]));
        y[s] = acc;
    }
}

// blocks: int32 (clip, t0) rows; warp w of a CTA takes frame t0 + w.
__global__ void __launch_bounds__(32 * ST_BAND_WARPS)
stoi_bands_kernel(const float* __restrict__ ola, const long long* __restrict__ clips, const int* __restrict__ blocks,
                  const float* __restrict__ table, const int* __restrict__ bands, const int* __restrict__ frames,
                  float* __restrict__ env, float* __restrict__ feat) {
    using namespace fftany;
    pdl_trigger(); pdl_wait();
    __shared__ c2 s_buf[ST_BAND_WARPS][2][ST_M];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blocks[2 * blockIdx.x];
    const long long t = blocks[2 * blockIdx.x + 1] + warp;
    if (t >= frames[c]) return;                      // warp-uniform; no block barrier below
    const long long* d = clips + (long long)ST_CLIP * c;
    const long long F0 = st_frames(d[1]), fo = d[2];
    const float* y = ola + d[3] + t * ST_HOP;
    c2* A = s_buf[warp][0];
    c2* B = s_buf[warp][1];
    const float* win = table + tab_win(ST_NFFT);
    const c2* tw = reinterpret_cast<const c2*>(table + tab_tw(ST_NFFT));
    const c2* sp = reinterpret_cast<const c2*>(table + tab_sp(ST_NFFT));
    for (int q = lane; q < ST_M; q += 32)           // z[q] = (w y)[2q] + i (w y)[2q + 1]; zero past the 256 samples
        A[q] = q < ST_FRAME / 2 ? c2{__fmul_rn(win[2 * q], y[2 * q]), __fmul_rn(win[2 * q + 1], y[2 * q + 1])}
                                : c2{0.f, 0.f};
    __syncwarp();
    c2* in = A;
    c2* out = B;
    for (int Ns = 1; Ns < ST_M; Ns *= 4) {           // four radix-4 passes
        fft_pass(SmemLoad{in}, out, tw, ST_M, 4, Ns, lane, 32);
        __syncwarp();
        c2* tmp = in; in = out; out = tmp;
    }
    float* pw = reinterpret_cast<float*>(out);       // |X(k)|^2, k < ST_MAX_BIN
    for (int k = lane; k < ST_MAX_BIN; k += 32) {
        const c2 X = split_bin(in, ST_M, k, sp[k]);
        pw[k] = fmaf(X.x, X.x, __fmul_rn(X.y, X.y));
    }
    __syncwarp();
    if (lane < ST_BANDS) {
        float s = 0.f;
        for (int k = bands[lane]; k < bands[ST_BANDS + lane]; ++k) s = __fadd_rn(s, pw[k]);
        env[ST_BANDS * fo + lane * F0 + t] = sqrtf(s);
        if (feat) feat[(fo + t) * ST_BANDS + lane] = __fmul_rn(10.f, log10f(fmaxf(s, 1e-10f)));
    }
}

// blocks: int32 (pair, s0) rows; warp w of a CTA takes segment s0 + w.
__global__ void __launch_bounds__(32 * ST_SEG_WARPS)
stoi_segment_kernel(const float* __restrict__ env, const long long* __restrict__ clips,
                    const long long* __restrict__ pairs, const int* __restrict__ blocks, const int* __restrict__ path,
                    const int* __restrict__ steps, double* __restrict__ seg) {
    pdl_trigger(); pdl_wait();
    __shared__ double s_x[ST_SEG_WARPS][ST_BANDS][ST_SEG];
    __shared__ double s_y[ST_SEG_WARPS][ST_BANDS][ST_SEG];
    __shared__ double s_r[ST_SEG_WARPS][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int p = blocks[2 * blockIdx.x];
    const int s = blocks[2 * blockIdx.x + 1] + warp;
    if (s > steps[p] - ST_SEG) return;               // warp-uniform; no block barrier below
    const long long* pr = pairs + (long long)ST_PAIR * p;
    const long long* dx = clips + (long long)ST_CLIP * pr[0];
    const long long* dy = clips + (long long)ST_CLIP * pr[1];
    const float* ex = env + ST_BANDS * dx[2];
    const float* ey = env + ST_BANDS * dy[2];
    const long long Fx = st_frames(dx[1]), Fy = st_frames(dy[1]);
    const int* ph = path + 2 * (pr[2] + s);
    double (*x)[ST_SEG] = s_x[warp];
    double (*y)[ST_SEG] = s_y[warp];
    double* r = s_r[warp];
    for (int e = lane; e < ST_BANDS * ST_SEG; e += 32) {
        const int i = e / ST_SEG, tt = e - i * ST_SEG;
        x[i][tt] = (double)ex[i * Fx + ph[2 * tt]];
        y[i][tt] = (double)ey[i * Fy + ph[2 * tt + 1]];
    }
    __syncwarp();

    // STOI: band row i on lane i
    if (lane < ST_BANDS) {
        const double* xr = x[lane];
        const double* yr = y[lane];
        double sxx = 0.0, syy = 0.0;
        for (int tt = 0; tt < ST_SEG; ++tt) { sxx = fma(xr[tt], xr[tt], sxx); syy = fma(yr[tt], yr[tt], syy); }
        const double alpha = sqrt(sxx) / (sqrt(syy) + ST_EPS);
        double mx = 0.0, my = 0.0;
        for (int tt = 0; tt < ST_SEG; ++tt) { mx += xr[tt]; my += fmin(alpha * yr[tt], ST_CLIP_Y * xr[tt]); }
        mx /= ST_SEG; my /= ST_SEG;
        double cxx = 0.0, cyy = 0.0, cxy = 0.0;
        for (int tt = 0; tt < ST_SEG; ++tt) {
            const double a = xr[tt] - mx, b = fmin(alpha * yr[tt], ST_CLIP_Y * xr[tt]) - my;
            cxx = fma(a, a, cxx); cyy = fma(b, b, cyy); cxy = fma(a, b, cxy);
        }
        r[lane] = cxy / ((sqrt(cxx) + ST_EPS) * (sqrt(cyy) + ST_EPS));
    }
    __syncwarp();
    double d_stoi = 0.0;
    if (lane == 0)
        for (int i = 0; i < ST_BANDS; ++i) d_stoi += r[i];
    __syncwarp();

    // ESTOI: rows (x on lanes 0-14, y on lanes 15-29), then columns (lane tt), in place
    if (lane < 2 * ST_BANDS) {
        double* row = lane < ST_BANDS ? x[lane] : y[lane - ST_BANDS];
        double mu = 0.0;
        for (int tt = 0; tt < ST_SEG; ++tt) mu += row[tt];
        mu /= ST_SEG;
        double ss = 0.0;
        for (int tt = 0; tt < ST_SEG; ++tt) { row[tt] -= mu; ss = fma(row[tt], row[tt], ss); }
        const double nrm = sqrt(ss) + ST_EPS;
        for (int tt = 0; tt < ST_SEG; ++tt) row[tt] /= nrm;
    }
    __syncwarp();
    if (lane < ST_SEG) {
        double mux = 0.0, muy = 0.0;
        for (int i = 0; i < ST_BANDS; ++i) { mux += x[i][lane]; muy += y[i][lane]; }
        mux /= ST_BANDS; muy /= ST_BANDS;
        double sx = 0.0, sy = 0.0, sxy = 0.0;
        for (int i = 0; i < ST_BANDS; ++i) {
            const double a = x[i][lane] - mux, b = y[i][lane] - muy;
            sx = fma(a, a, sx); sy = fma(b, b, sy); sxy = fma(a, b, sxy);
        }
        r[lane] = sxy / ((sqrt(sx) + ST_EPS) * (sqrt(sy) + ST_EPS));
    }
    __syncwarp();
    if (lane == 0) {
        double d_e = 0.0;
        for (int tt = 0; tt < ST_SEG; ++tt) d_e += r[tt];
        double* o = seg + 2 * (pr[3] + s);
        o[0] = d_stoi;
        o[1] = d_e / ST_SEG;
    }
}

__global__ void __launch_bounds__(128)
stoi_reduce_kernel(const double* __restrict__ seg, const long long* __restrict__ pairs, const int* __restrict__ steps,
                   const int* __restrict__ kept, int P, double* __restrict__ result, int* __restrict__ counts) {
    pdl_trigger(); pdl_wait();
    const int p = blockIdx.x * 128 + threadIdx.x;
    if (p >= P) return;
    const long long* pr = pairs + (long long)ST_PAIR * p;
    const int J = max(steps[p] - ST_SEG + 1, 0);
    const double* v = seg + 2 * pr[3];
    double a = 0.0, b = 0.0;
    for (int s = 0; s < J; ++s) { a += v[2 * s]; b += v[2 * s + 1]; }
    result[2 * p] = J ? a / (ST_BANDS * (double)J) : CUDART_NAN;
    result[2 * p + 1] = J ? b / (double)J : CUDART_NAN;
    counts[2 * p] = J;
    counts[2 * p + 1] = kept[pr[0]];
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_stoi_frames(const float* wav, const long long* clips, int n_clips, const double* win, double* energy, int* keep,
                    int* kept_idx, int* kept, void* stream) {
    DV3_REQUIRE(wav && clips && win && energy && keep && kept_idx && kept, "stoi_frames: null operand");
    DV3_REQUIRE(n_clips >= 1 && n_clips <= 65535, "stoi_frames: n_clips=%d outside [1, 65535]", n_clips);
    launch_k(stoi_frames_kernel, (unsigned)n_clips, ST_THREADS, 0, (cudaStream_t)stream, wav, clips, win, energy, keep,
             kept_idx, kept);
    return check_launch("stoi_frames");
}

int dv3_stoi_overlap_add(const float* wav, const long long* clips, int n_clips, long long max_samples,
                         const float* table, const int* kept_idx, const int* kept, float* ola, int* frames,
                         void* stream) {
    DV3_REQUIRE(wav && clips && table && kept_idx && kept && ola && frames, "stoi_overlap_add: null operand");
    DV3_REQUIRE(n_clips >= 1 && n_clips <= 65535, "stoi_overlap_add: n_clips=%d outside [1, 65535]", n_clips);
    DV3_REQUIRE(max_samples >= 0 && max_samples < (1LL << 40), "stoi_overlap_add: max_samples=%lld", max_samples);
    const long long tiles = max_samples > 0 ? (max_samples + ST_OLA_TILE - 1) / ST_OLA_TILE : 1;
    DV3_REQUIRE(tiles < (1LL << 31), "stoi_overlap_add: %lld tiles", tiles);
    launch_k(stoi_ola_kernel, dim3((unsigned)tiles, (unsigned)n_clips), ST_THREADS, 0, (cudaStream_t)stream, wav, clips,
             table + fftany::tab_win(ST_NFFT), kept_idx, kept, ola, frames);
    return check_launch("stoi_overlap_add");
}

int dv3_stoi_bands(const float* ola, const long long* clips, const int* blocks, int n_blocks, const float* table,
                   const int* bands, const int* frames, float* env, float* feat, void* stream) {
    DV3_REQUIRE(n_blocks >= 0, "stoi_bands: n_blocks=%d", n_blocks);
    if (n_blocks == 0) return 0;
    DV3_REQUIRE(ola && clips && blocks && table && bands && frames && env, "stoi_bands: null operand");
    launch_k(stoi_bands_kernel, (unsigned)n_blocks, 32 * ST_BAND_WARPS, 0, (cudaStream_t)stream, ola, clips, blocks,
             table, bands, frames, env, feat);
    return check_launch("stoi_bands");
}

int dv3_stoi_segments(const float* env, const long long* clips, const long long* pairs, int n_pairs, const int* blocks,
                      int n_blocks, const int* path, const int* steps, const int* kept, double* seg, double* result,
                      int* counts, void* stream) {
    DV3_REQUIRE(pairs && steps && kept && result && counts, "stoi_segments: null operand");
    DV3_REQUIRE(n_pairs >= 1 && n_blocks >= 0, "stoi_segments: n_pairs=%d, n_blocks=%d", n_pairs, n_blocks);
    const cudaStream_t st = (cudaStream_t)stream;
    if (n_blocks > 0) {
        DV3_REQUIRE(env && clips && blocks && path && seg, "stoi_segments: null operand");
        launch_k(stoi_segment_kernel, (unsigned)n_blocks, 32 * ST_SEG_WARPS, 0, st, env, clips, pairs, blocks, path,
                 steps, seg);
        if (int rc = check_launch("stoi_segments")) return rc;
    }
    launch_k(stoi_reduce_kernel, (unsigned)ceil_div(n_pairs, 128), 128, 0, st, (const double*)seg, pairs, steps, kept,
             n_pairs, result, counts);
    return check_launch("stoi_reduce");
}

}  // extern "C"
