// Pitch of synthesized speech against recordings (pitch.py, DESIGN.md section 2.18): a batched YIN F0 tracker and the
// DTW warping path.
//
// YIN (de Cheveigne & Kawahara 2002, steps 1-5).  Frame t of a clip is centred on the sample c_t = t R + R - N/2 of the
// STFT frame t (N = fft_size = W, R = hop_size) and reads x[a_t + m], a_t = c_t - floor((W + tau_max) / 2), samples
// outside [0, n) reading as zero.
//   d(tau)  = sum_{j < W} (x[a_t + j] - x[a_t + j + tau])^2, tau = 1 .. tau_max: one fma chain over j in order
//   S(tau)  = d(1) + ... + d(tau), summed sequentially;  d'(tau) = tau d(tau) / S(tau), or 1 where S(tau) = 0
//   tau*    = the first tau in [tau_min, tau_max] with d' < threshold, walked forward while d' keeps decreasing
//             (voiced); else the argmin of d' over the range, ties to the smallest tau (unvoiced)
//   delta   = (y0 - y2) / (2 ((y0 + y2) - 2 y1)) of y = d'(tau* - 1, tau*, tau* + 1) when both neighbours lie in the
//             range and the curvature is > 0, clamped to [-1, 1], else 0;  f0 = sr / (tau* + delta) when voiced, else 0
//   aperiodicity = d'(tau*);  energy = sum_{j < W} x[a_t + j]^2 (one fma chain)
// Silence gate (second launch): f0 = 0 where energy < gate * (the clip's largest frame energy), gate =
// 10^(silence_db / 10).  No atomics: a clip's bits depend on its own samples alone.
//
// Kernel.  One CTA per YIN_FRAMES_PER_CTA(tau_max) consecutive frames of one clip stages their common sample span in
// shared memory (consecutive frames overlap by W + tau_max - R samples).  Each frame gets ceil(tau_max / (32 T)) warps;
// lane l of warp w owns the T consecutive lags tau = 1 + (32 w + l) T + k, k < T, and keeps their sums in registers.  T
// is odd, so the 32 lanes' lag windows start on 32 different banks.  Per block of J steps of j a lane loads J samples
// x[a + j] (a broadcast) and the J + T - 1 samples of its lag window, then does J T subtract + fma pairs: 2 J T FP32
// instructions for 2 J + T - 1 shared loads.  sm_90 has no packed f32x2 arithmetic, so every term costs two issue
// slots.  Lane 0 of the frame's first warp then sums S sequentially, the warp forms d', finds the first crossing
// by ballot (or the argmin by a reduction), and lane 0 walks forward from it.
//
// DTW path (csrc/dtw.cuh with PATH = true) and its backtrace: one thread per pair walks the direction words from (N, M)
// to (1, 1) and writes the 0-based (i, j) pairs in reverse order.
#include "dtw.cuh"

namespace dv3 {

constexpr int YIN_T = 13;                  // lags per lane (odd: conflict-free lag windows)
constexpr int YIN_J = 16;                  // j steps per register block
constexpr int YIN_WARPS = 8;               // warps per CTA (at most)
constexpr int YIN_THREADS = 32 * YIN_WARPS;
constexpr int YIN_MAX_TAU = 1024;
constexpr int YIN_MAX_W = 4096;            // audio.check_geometry's largest fft_size
constexpr int BT_THREADS = 128;

static __host__ __device__ inline int yin_warps_per_frame(int tau_max) { return (tau_max + 32 * YIN_T - 1) / (32 * YIN_T); }
static inline int yin_frames_per_cta(int tau_max) { return YIN_WARPS / yin_warps_per_frame(tau_max); }

// blocks: rows (sample_off, n_samples, out0, t0, nf) -- frames t0 .. t0 + nf - 1 of the clip at wav + sample_off, written
// at out0 ..; smem: span samples, then FB x tau_max floats (d, then d'), then FB x tau_max prefix sums S.
__global__ void __launch_bounds__(YIN_THREADS)
yin_kernel(const float* __restrict__ wav, const long long* __restrict__ blocks, float* __restrict__ f0,
           float* __restrict__ aper, float* __restrict__ energy, float* __restrict__ diff, int W, int R, int tau_min,
           int tau_max, float threshold, float sr) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    extern __shared__ float smem[];
    const int wpf = yin_warps_per_frame(tau_max), FB = YIN_WARPS / wpf;
    const int tau_cover = wpf * 32 * YIN_T;
    const int span = (FB - 1) * R + W + tau_cover;
    float* s_x = smem;
    float* s_d = smem + span;
    float* s_S = s_d + FB * tau_max;
    const long long* blk = blocks + 5LL * blockIdx.x;
    const long long soff = blk[0], out0 = blk[2];
    const int n = (int)blk[1], t0 = (int)blk[3], nf = min((int)blk[4], FB);
    const long long a0 = (long long)t0 * R + R - W / 2 - (W + tau_max) / 2;       // a_{t0}
    for (int m = threadIdx.x; m < span; m += blockDim.x) {     // wpf * FB warps: 192 threads at wpf = 3
        const long long g = a0 + m;
        s_x[m] = g >= 0 && g < n ? wav[soff + g] : 0.f;
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = warp / wpf, wf = warp - f * wpf;          // frame in the CTA, warp within the frame
    const bool active = f < nf;                             // warp-uniform
    float e = 0.f;
    if (active) {
        const int tau0 = 1 + (wf * 32 + lane) * YIN_T;
        const float* xs = s_x + f * R;
        const float* ys = xs + tau0;
        float acc[YIN_T];
#pragma unroll
        for (int k = 0; k < YIN_T; ++k) acc[k] = 0.f;
        const int Wj = W - W % YIN_J;
        for (int j0 = 0; j0 < Wj; j0 += YIN_J) {
            float xv[YIN_J], yv[YIN_J + YIN_T - 1];
#pragma unroll
            for (int q = 0; q < YIN_J; ++q) xv[q] = xs[j0 + q];
#pragma unroll
            for (int q = 0; q < YIN_J + YIN_T - 1; ++q) yv[q] = ys[j0 + q];
#pragma unroll
            for (int q = 0; q < YIN_J; ++q) {
                e = fmaf(xv[q], xv[q], e);
#pragma unroll
                for (int k = 0; k < YIN_T; ++k) {
                    const float t = xv[q] - yv[q + k];
                    acc[k] = fmaf(t, t, acc[k]);
                }
            }
        }
        for (int j = Wj; j < W; ++j) {                       // W % J steps (fft sizes that are not multiples of 16)
            const float x = xs[j];
            e = fmaf(x, x, e);
#pragma unroll
            for (int k = 0; k < YIN_T; ++k) {
                const float t = x - ys[j + k];
                acc[k] = fmaf(t, t, acc[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < YIN_T; ++k)
            if (tau0 + k <= tau_max) s_d[f * tau_max + tau0 + k - 1] = acc[k];
    }
    __syncthreads();
    if (!active || wf != 0) return;

    float* d = s_d + f * tau_max;
    float* S = s_S + f * tau_max;
    if (lane == 0) {                               // sequential prefix; 8 loads in flight ahead of the adds
        float s = 0.f;
        int tau = 0;
        for (; tau + 8 <= tau_max; tau += 8) {
            float v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = d[tau + q];
#pragma unroll
            for (int q = 0; q < 8; ++q) { s += v[q]; S[tau + q] = s; }
        }
        for (; tau < tau_max; ++tau) { s += d[tau]; S[tau] = s; }
    }
    __syncwarp();
    const long long out = out0 + f;
    for (int tau = lane + 1; tau <= tau_max; tau += 32) {
        const float dv = d[tau - 1], sv = S[tau - 1];
        const float dp = sv == 0.f ? 1.f : __fdiv_rn(__fmul_rn((float)tau, dv), sv);
        if (diff) {
            diff[(2 * out) * tau_max + tau - 1] = dv;
            diff[(2 * out + 1) * tau_max + tau - 1] = dp;
        }
        d[tau - 1] = dp;
    }
    __syncwarp();
    // the decision, warp-parallel with the sequential rule's result: the first crossing by ballot over 32 lags at a
    // time; without one, the argmin by a (value, lag) reduction that keeps the smaller lag on ties (min is exact)
    int best = 0;
    for (int base = tau_min; base <= tau_max && best == 0; base += 32) {
        const int tau = base + lane;
        const unsigned hit = __ballot_sync(0xffffffffu, tau <= tau_max && d[tau - 1] < threshold);
        if (hit) best = base + __ffs(hit) - 1;
    }
    const bool voiced = best != 0;
    if (voiced) {
        if (lane != 0) return;
        while (best < tau_max && d[best] < d[best - 1]) ++best;
    } else {
        float v = d[tau_min - 1];
        best = tau_min;
        for (int tau = tau_min + lane; tau <= tau_max; tau += 32)
            if (d[tau - 1] < v || (d[tau - 1] == v && tau < best)) { v = d[tau - 1]; best = tau; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, v, o);
            const int ot = __shfl_xor_sync(0xffffffffu, best, o);
            if (ov < v || (ov == v && ot < best)) { v = ov; best = ot; }
        }
        if (lane != 0) return;
    }
    float hz = 0.f;
    if (voiced) {
        float delta = 0.f;
        if (best - 1 >= tau_min && best + 1 <= tau_max) {
            const float y0 = d[best - 2], y1 = d[best - 1], y2 = d[best];
            const float c = __fsub_rn(__fadd_rn(y0, y2), __fmul_rn(2.f, y1));
            if (c > 0.f) delta = fminf(1.f, fmaxf(-1.f, __fdiv_rn(__fsub_rn(y0, y2), __fmul_rn(2.f, c))));
        }
        hz = __fdiv_rn(sr, __fadd_rn((float)best, delta));
    }
    f0[out] = hz;
    aper[out] = d[best - 1];
    energy[out] = e;
}

// One warp per clip row (out_off, n_frames): the clip's largest frame energy (max is exact in any order), then
// f0 = 0 where energy < gate * max.
__global__ void __launch_bounds__(32)
yin_gate_kernel(const long long* __restrict__ clips, float* __restrict__ f0, const float* __restrict__ energy,
                float gate) {
    pdl_trigger(); pdl_wait();
    const long long off = clips[2LL * blockIdx.x];
    const int nfr = (int)clips[2LL * blockIdx.x + 1];
    float m = 0.f;
    for (int t = threadIdx.x; t < nfr; t += 32) m = fmaxf(m, energy[off + t]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float thr = __fmul_rn(gate, m);
    for (int t = threadIdx.x; t < nfr; t += 32)
        if (energy[off + t] < thr) f0[off + t] = 0.f;
}

// One thread per work row: walk the direction words from (N, M) back to (1, 1); row k of the pair's path slot (N + M - 1
// rows of int32 (i, j), 0-based) is the k-th cell from the end.  The slot of row r starts at path_work[2r + 1] rows, and
// path_rows[pair] receives the cells written.  On row 1 the walk moves left and on column 1 up, whatever the code says:
// for finite costs those are the codes the recursion stores there, and where D is not finite (NaN or overflowing
// features: every comparison fails and the code is 0) the walk still stays in the grid and ends at (1, 1).
__global__ void __launch_bounds__(BT_THREADS)
dtw_backtrace_kernel(const long long* __restrict__ work, const long long* __restrict__ path_work,
                     const unsigned* __restrict__ dirs, int* __restrict__ path, int* __restrict__ path_rows, int P) {
    pdl_trigger(); pdl_wait();
    const int r = blockIdx.x * BT_THREADS + threadIdx.x;
    if (r >= P) return;
    const long long* w = work + 6LL * r;
    const int N = (int)w[2], M = (int)w[4];
    const int M16 = (M + 15) >> 4;
    const unsigned* dir = dirs + path_work[2LL * r];
    int* out = path + 2 * path_work[2LL * r + 1];
    int i = N, j = M, k = 0;
    long long wi = -1;
    unsigned word = 0;
    for (;;) {                                       // each step lowers i + j, so at most N + M - 1 cells
        out[2 * k] = i - 1;
        out[2 * k + 1] = j - 1;
        ++k;
        if (i == 1 && j == 1) break;
        if (i == 1) { --j; continue; }
        if (j == 1) { --i; continue; }
        const long long x = (long long)(i - 1) * M16 + ((j - 1) >> 4);
        if (x != wi) { word = dir[x]; wi = x; }
        const unsigned code = (word >> (2 * ((j - 1) & 15))) & 3u;
        if (code == 0) { --i; --j; }
        else if (code == 1) --i;
        else --j;
    }
    path_rows[w[0]] = k;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_yin_frames_per_cta(int tau_max) {
    return tau_max >= 1 && tau_max <= YIN_MAX_TAU ? yin_frames_per_cta(tau_max) : 0;
}

int dv3_yin_f0(const float* wav, const long long* blocks, int n_blocks, const long long* clips, int n_clips, float* f0,
               float* aperiodicity, float* energy, float* diff, int W, int R, int tau_min, int tau_max, float threshold,
               float gate, float sample_rate, void* stream) {
    DV3_REQUIRE(wav && blocks && clips && f0 && aperiodicity && energy, "yin_f0: null operand");
    DV3_REQUIRE(n_blocks >= 1 && n_clips >= 1 && n_clips <= n_blocks, "yin_f0: n_blocks=%d, n_clips=%d", n_blocks,
                n_clips);
    DV3_REQUIRE(W >= 2 && W <= YIN_MAX_W, "yin_f0: W=%d outside [2, %d]", W, YIN_MAX_W);
    DV3_REQUIRE(R >= 1 && R <= W, "yin_f0: R=%d outside [1, W=%d]", R, W);
    DV3_REQUIRE(tau_min >= 2 && tau_min <= tau_max && tau_max <= YIN_MAX_TAU,
                "yin_f0: tau range [%d, %d] outside [2, %d]", tau_min, tau_max, YIN_MAX_TAU);
    DV3_REQUIRE(threshold > 0.f && threshold <= 1.f, "yin_f0: threshold=%g outside (0, 1]", (double)threshold);
    DV3_REQUIRE(gate >= 0.f && gate <= 1.f, "yin_f0: gate=%g outside [0, 1]", (double)gate);
    DV3_REQUIRE(sample_rate > 0.f, "yin_f0: sample_rate=%g", (double)sample_rate);
    const int wpf = yin_warps_per_frame(tau_max), FB = YIN_WARPS / wpf;
    const size_t span = (size_t)(FB - 1) * R + W + wpf * 32 * YIN_T;
    const size_t smem = (span + 2 * (size_t)FB * tau_max) * sizeof(float);     // <= 100 KB (W = 4096, R = 2048, tau_max <= 416)
    if (cudaFuncSetAttribute(yin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return check_launch("yin smem attribute");
    const cudaStream_t st = (cudaStream_t)stream;
    launch_k(yin_kernel, (unsigned)n_blocks, wpf * FB * 32, smem, st, wav, blocks, f0, aperiodicity, energy, diff, W, R,
             tau_min, tau_max, threshold, sample_rate);
    if (int rc = check_launch("yin")) return rc;
    launch_k(yin_gate_kernel, (unsigned)n_clips, 32, 0, st, clips, f0, (const float*)energy, gate);
    return check_launch("yin_gate");
}

int dv3_dtw_path(const float* cep, int K, const long long* work, const long long* path_work, float* workspace,
                 unsigned* dirs, float* cost, int* path_len, int P, void* stream) {
    DV3_REQUIRE(cep && work && path_work && workspace && dirs && cost && path_len, "dtw_path: null operand");
    DV3_REQUIRE(P >= 1, "dtw_path: P=%d", P);
    DV3_REQUIRE(K >= 1 && K <= MC_MAX_K, "dtw_path: K=%d outside [1, %d]", K, MC_MAX_K);
    return dtw_dispatch<true>(cep, K, work, workspace, cost, path_len, P, path_work, dirs, (cudaStream_t)stream);
}

int dv3_dtw_backtrace(const long long* work, const long long* path_work, const unsigned* dirs, int* path, int* path_rows,
                      int P, void* stream) {
    DV3_REQUIRE(work && path_work && dirs && path && path_rows, "dtw_backtrace: null operand");
    DV3_REQUIRE(P >= 1, "dtw_backtrace: P=%d", P);
    launch_k(dtw_backtrace_kernel, (unsigned)ceil_div(P, BT_THREADS), BT_THREADS, 0, (cudaStream_t)stream, work,
             path_work, dirs, path, path_rows, P);
    return check_launch("dtw_backtrace");
}

}  // extern "C"
