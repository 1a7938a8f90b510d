// The element-wise ends of the inverse audio path, reference audio.py:37-43 (inv_spectrogram) = _denormalize
// (:92-93) -> _db_to_amp (:84-85) -> ** power -> phase recovery -> inverse STFT -> inv_preemphasis (:26-28):
//   spec_to_amp_kernel      normalised dB spectrogram -> linear magnitude ** power
//   deemphasis_kernel       y[n] = x[n] + c*y[n-1] (a 1st-order IIR: one CTA per clip, chunks staged through smem)
// The phase recovery and the inverse STFT between them run for every STFT frame, 1024 / 256 included, in
// csrc/stft_any.cu (Griffin-Lim and fast Griffin-Lim) and csrc/lws_any.cu (LWS).
#include "common.cuh"

namespace dv3 {

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

int dv3_deemphasis(const float* x, float* y, int nclips, int n_samples, long long stride, float coef, void* stream) {
    DV3_REQUIRE(nclips >= 1 && n_samples >= 1, "deemphasis: empty input");
    launch_k(deemphasis_kernel, nclips, 256, 0, (cudaStream_t)stream, x, y, n_samples, stride, coef);
    return check_launch("deemphasis");
}

}  // extern "C"
