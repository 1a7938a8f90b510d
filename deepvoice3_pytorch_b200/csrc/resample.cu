// Corpus front-end ahead of the STFT: polyphase resampling and silence-trim bounds, both per clip of a ragged batch.
//
// Resampler (dv3_resample_poly_batched): scipy.signal.resample_poly(x.astype(float64), up, down) cast to fp32, with
// scipy's default ('kaiser', 5.0) window and zero padding.  The host designs the zero-padded filter h once per
// (up, down) in fp64 (audio.resample_filter_bank) and hands over its polyphase bank, bank[j * up + p] = h[p + j * up]
// (j < ntaps; zero past h's end).  Output m of a clip is upfirdn's sample k = m + pre_remove:
//     t = k * down,  p = t % up,  b = t / up,   y[m] = sum_{j < ntaps} bank[j * up + p] * x[b - j]   (x = 0 outside)
// summed in fp64, j ascending, then rounded to fp32.  One CTA computes OUT_TILE consecutive outputs of one clip: the
// bank (52.5 KB at 48 kHz -> 22.05 kHz) and the input window those outputs read are staged in shared memory once, the
// window as fp32 (int16 read as x / 32768 and fp32 input are both exact in fp32, and exact again in fp64).  Every
// output reads only its own clip in a fixed order, so a clip is bit-identical alone and inside any batch.
// dv3_resample_segments_batched runs the same kernel on part of each clip's output: columns [0, seg_len) of a row get
// outputs [seg_start, seg_start + seg_len) of the whole clip, from a row that holds only the input span those outputs
// read (audio.input_span).  It is the training-time resampler of data.WavDataset.from_vctk.
// Per output: ntaps fp64 FMAs against about 4.4 bytes of int16 input and 4 bytes of output at 48 -> 22.05 kHz, so the
// kernel sits near the ridge of the H100's fp64 (34 TFLOP/s) and HBM (3.35 TB/s) roofs.
//
// Trim bounds (dv3_trim_bounds_batched): librosa.effects.trim(y, top_db) of the 0.6-0.9 era (frame 2048, hop 512,
// ref = max, centred frames with reflect padding) on y = clip[offset : offset + len], in fp64.  One CTA per clip, one
// warp per frame: frame f's mean square runs over padded[512 f : 512 f + 2048], padded = y reflected by 1024 on each
// side (numpy's repeated reflection when len <= 1024); the lanes stride the frame by 32 (coalesced) and fold their sums
// in a fixed tree.  Pass 1 takes the largest mean square, pass 2 recomputes each frame and marks it non-silent when
// 10 log10(max(1e-10, mse)) - 10 log10(max(1e-10, max mse)) > -top_db; first / last come from integer min / max, so
// the result does not depend on the warp schedule.  Each sample is read four times (the frames overlap 4x), from L1/L2.
#include <type_traits>

#include "common.cuh"

namespace dv3 {

constexpr int RS_THREADS = 256, RS_TILE = 4096;             // outputs per CTA
constexpr int RS_DESC = 6;                                  // ints per clip of a segment descriptor
constexpr int TRIM_WARPS = 8, TRIM_FRAME = 2048, TRIM_HOP = 512, TRIM_PAD = TRIM_FRAME / 2;

template <typename In> __device__ __forceinline__ float pcm(In v) {
    return std::is_same<In, float>::value ? (float)v : __fmul_rn((float)v, 3.0517578125e-05f);     // int16: / 32768
}

__host__ __device__ inline long long rs_out_len(long long n, int up, int down) { return (n * up + down - 1) / down; }

// window samples the tile [m0, m0 + RS_TILE) reads: base(m_last) - base(m0) + ntaps
__host__ __device__ inline int rs_window(int up, int down, int ntaps) {
    return (int)(((long long)(RS_TILE - 1) * down) / up) + 2 + ntaps;
}

// seg == NULL: clip c is row c, its whole output (lengths[c] input samples from row position 0).  Otherwise seg holds
// RS_DESC ints per clip, {row, n_in, in_start, in_len, seg_start, seg_len}: the row (input and output) holds source
// samples [in_start, in_start + in_len) of a clip of n_in samples, and output column k is the clip's output
// seg_start + k for k < seg_len.  Either way an output column reads the same bank entries and input values in the same
// order as the same absolute output of the whole clip, so its bits are those of the whole-clip output.
template <typename In>
__global__ void __launch_bounds__(RS_THREADS) resample_poly_kernel(const In* wav, const int* lengths, const int* seg,
                                                                   int pitch_in, float* out, int pitch_out,
                                                                   const double* bank, int up, int down, int ntaps,
                                                                   int pre_remove) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* sb = reinterpret_cast<double*>(smem_raw);
    float* win = reinterpret_cast<float*>(sb + (size_t)up * ntaps);
    const int clip = blockIdx.y, tid = threadIdx.x;
    int row = clip, n, in_start = 0, in_len;
    long long seg_start = 0, n_out;
    if (seg) {
        const int* d = seg + RS_DESC * clip;
        row = d[0]; n = d[1]; in_start = d[2]; in_len = d[3]; seg_start = d[4]; n_out = d[5];
    } else {
        n = lengths[clip];
        in_len = n;
        n_out = min(rs_out_len(n, up, down), (long long)pitch_out);
    }
    const long long k0 = (long long)blockIdx.x * RS_TILE;   // first output column of the tile
    float* o = out + (size_t)row * pitch_out;
    const long long k_end = min(k0 + RS_TILE, (long long)pitch_out);
    if (k0 >= n_out) {                                      // uniform: the tile lies past the clip's output
        for (long long k = k0 + tid; k < k_end; k += RS_THREADS) o[k] = 0.f;
        return;
    }
    const In* x = wav + (size_t)row * pitch_in;             // x[s - in_start] = source sample s
    const long long s_lo = max(in_start, 0), s_hi = min((long long)n, (long long)in_start + in_len);
    const long long m0 = seg_start + k0;
    const long long lo = ((m0 + pre_remove) * down) / up - (ntaps - 1);
    const int nwin = rs_window(up, down, ntaps);
    for (int i = tid; i < up * ntaps; i += RS_THREADS) sb[i] = bank[i];
    for (int i = tid; i < nwin; i += RS_THREADS) {
        const long long s = lo + i;
        win[i] = (s >= s_lo && s < s_hi) ? pcm(x[s - in_start]) : 0.f;
    }
    __syncthreads();
    for (long long k = k0 + tid; k < k_end; k += RS_THREADS) {
        if (k >= n_out) { o[k] = 0.f; continue; }
        const long long t = (seg_start + k + pre_remove) * down;
        const int p = (int)(t % up);
        const float* xw = win + (t / up - lo);               // xw[-j] = x[b - j]
        double acc = 0.0;
#pragma unroll 4
        for (int j = 0; j < ntaps; ++j) acc = fma(sb[j * up + p], (double)xw[-j], acc);
        o[k] = (float)acc;
    }
}

// index into y (length L >= 1) of position q of the reflect-padded signal: period 2 (L - 1), mirrored about 0 and L-1
__device__ __forceinline__ int reflect_index(int q, int L) {
    if (L == 1) return 0;
    const int period = 2 * (L - 1);
    int r = q % period;
    if (r < 0) r += period;
    return r >= L ? period - r : r;
}

template <typename In>
__device__ __forceinline__ double frame_sumsq(const In* y, int L, int f, int lane) {
    double acc = 0.0;
    const int q0 = f * TRIM_HOP - TRIM_PAD + lane;
#pragma unroll 4
    for (int i = 0; i < TRIM_FRAME / 32; ++i) {
        const double v = (double)pcm(y[reflect_index(q0 + 32 * i, L)]);
        acc = fma(v, v, acc);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    return __shfl_sync(0xffffffffu, acc, 0);
}

__device__ __forceinline__ double power_db(double mse) { return 10.0 * log10(fmax(1e-10, mse)); }

template <typename In>
__global__ void __launch_bounds__(TRIM_WARPS * 32) trim_bounds_kernel(const In* wav, const int* lengths,
                                                                      const int* offsets, int pitch,
                                                                      const double* top_db, int* bounds) {
    pdl_trigger(); pdl_wait();
    __shared__ double wmax[TRIM_WARPS];
    __shared__ int first, last;
    const int clip = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int L = lengths[clip];
    if (L <= 0) {
        if (tid == 0) { bounds[2 * clip] = 0; bounds[2 * clip + 1] = 0; }
        return;
    }
    const In* y = wav + (size_t)clip * pitch + (offsets ? offsets[clip] : 0);
    const int nfr = L / TRIM_HOP + 1;
    double mx = 0.0;
    for (int f = warp; f < nfr; f += TRIM_WARPS) mx = fmax(mx, frame_sumsq(y, L, f, lane) / TRIM_FRAME);
    if (lane == 0) wmax[warp] = mx;
    if (tid == 0) { first = nfr; last = -1; }
    __syncthreads();
    mx = wmax[0];
#pragma unroll
    for (int w = 1; w < TRIM_WARPS; ++w) mx = fmax(mx, wmax[w]);
    const double ref_db = power_db(mx), thr = -top_db[clip];
    for (int f = warp; f < nfr; f += TRIM_WARPS) {
        const double mse = frame_sumsq(y, L, f, lane) / TRIM_FRAME;
        if (lane == 0 && power_db(mse) - ref_db > thr) { atomicMin(&first, f); atomicMax(&last, f); }
    }
    __syncthreads();
    if (tid == 0) {
        const bool any = last >= 0;
        bounds[2 * clip] = any ? TRIM_HOP * first : 0;
        bounds[2 * clip + 1] = any ? min(L, TRIM_HOP * (last + 1)) : 0;
    }
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_resample_out_len(int n_samples, int up, int down) {
    return (int)rs_out_len(n_samples, up, down);
}

static int resample_launch(const char* what, const void* wav, int wav_int16, const int* lengths, const int* seg,
                           int pitch_in, float* out, int pitch_out, int nclips, const double* bank, int up, int down,
                           int ntaps, int pre_remove, void* stream) {
    DV3_REQUIRE(nclips >= 1 && nclips <= 65535, "%s: nclips %d out of range", what, nclips);
    DV3_REQUIRE(up >= 1 && down >= 1 && ntaps >= 1 && pre_remove >= 0, "%s: bad filter (up %d, down %d, ntaps %d)",
                what, up, down, ntaps);
    DV3_REQUIRE(pitch_in >= 0 && pitch_out >= 1, "%s: bad pitches %d, %d", what, pitch_in, pitch_out);
    const size_t smem = (size_t)up * ntaps * sizeof(double) + (size_t)rs_window(up, down, ntaps) * sizeof(float);
    int dev = 0, optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    DV3_REQUIRE(smem <= (size_t)optin, "%s: the %d x %d filter bank and its window need %zu bytes of shared memory "
                "(at most %d)", what, up, ntaps, smem, optin);
    const dim3 grid((unsigned)((pitch_out + RS_TILE - 1) / RS_TILE), nclips);
    const cudaStream_t st = (cudaStream_t)stream;
    if (wav_int16) {
        cudaFuncSetAttribute(resample_poly_kernel<short>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        launch_k(resample_poly_kernel<short>, grid, RS_THREADS, smem, st, reinterpret_cast<const short*>(wav),
                 lengths, seg, pitch_in, out, pitch_out, bank, up, down, ntaps, pre_remove);
    } else {
        cudaFuncSetAttribute(resample_poly_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        launch_k(resample_poly_kernel<float>, grid, RS_THREADS, smem, st, reinterpret_cast<const float*>(wav),
                 lengths, seg, pitch_in, out, pitch_out, bank, up, down, ntaps, pre_remove);
    }
    return check_launch(what);
}

int dv3_resample_poly_batched(const void* wav, int wav_int16, const int* lengths, int pitch_in, float* out,
                              int pitch_out, int nclips, const double* bank, int up, int down, int ntaps,
                              int pre_remove, void* stream) {
    return resample_launch("resample_poly", wav, wav_int16, lengths, nullptr, pitch_in, out, pitch_out, nclips, bank,
                           up, down, ntaps, pre_remove, stream);
}

int dv3_resample_segments_batched(const void* wav, int wav_int16, int pitch_in, const int* seg, int nclips, float* out,
                                  int pitch_out, const double* bank, int up, int down, int ntaps, int pre_remove,
                                  void* stream) {
    DV3_REQUIRE(seg != nullptr, "resample_segments: no segment descriptors");
    return resample_launch("resample_segments", wav, wav_int16, nullptr, seg, pitch_in, out, pitch_out, nclips, bank,
                           up, down, ntaps, pre_remove, stream);
}

int dv3_trim_bounds_batched(const void* wav, int wav_int16, const int* lengths, const int* offsets, int pitch,
                            int nclips, const double* top_db, int* bounds, void* stream) {
    DV3_REQUIRE(nclips >= 1, "trim_bounds: nclips %d out of range", nclips);
    const cudaStream_t st = (cudaStream_t)stream;
    if (wav_int16)
        launch_k(trim_bounds_kernel<short>, dim3(nclips), TRIM_WARPS * 32, 0, st, reinterpret_cast<const short*>(wav),
                 lengths, offsets, pitch, top_db, bounds);
    else
        launch_k(trim_bounds_kernel<float>, dim3(nclips), TRIM_WARPS * 32, 0, st, reinterpret_cast<const float*>(wav),
                 lengths, offsets, pitch, top_db, bounds);
    return check_launch("trim_bounds");
}

}  // extern "C"
