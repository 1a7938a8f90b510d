// Mel-cepstral distortion after dynamic time warping (mcd.py, DESIGN.md section 2.17).
//
// Cepstra.  c[t, k-1] = sum_m basis[k-1, m] mel[t, m] for k = 1..K: basis is the orthonormal DCT-II row k of the
// natural-log amplitude, scaled by -min_level_db ln10 / 20 (built in fp64 on the host, rounded once).  The affine
// offset of the denormalisation only reaches c_0, which is dropped, so the kernel reads the normalised mels as they
// are.  One CTA per MC_ROWS frames of one sequence stages those rows and the table in shared memory; every output is
// one fma chain over m in order.  Frames at or past a sequence's count are not read and their outputs are zero.
//
// DTW.  The recursion of csrc/dtw.cuh without the warping path (PATH = false): cost D(N, M) and path length L only.
// The instantiations that also record the path live in csrc/pitch.cu.
#include "dtw.cuh"

namespace dv3 {

constexpr int MC_ROWS = 32;               // frames per CTA of the cepstra kernel
constexpr int MC_THREADS = 128;
constexpr int MC_MAX_MELS = 128;          // the filterbank's limit (audio.check_geometry)

// smem: MC_ROWS mel rows, then the K table rows, both at the odd stride LD = M | 1 (conflict-free for distinct rows)
__global__ void __launch_bounds__(MC_THREADS)
mcd_cepstra_kernel(const float* __restrict__ mels, const int* __restrict__ lengths, const float* __restrict__ basis,
                   float* __restrict__ cep, int T_max, int M, int K) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    extern __shared__ float smem[];
    const int LD = M | 1;
    float* s_mel = smem;
    float* s_w = smem + MC_ROWS * LD;
    const int q = blockIdx.y, t0 = blockIdx.x * MC_ROWS, tid = threadIdx.x;
    const int n = lengths[q];
    const long long base = (long long)q * T_max;
    for (int i = tid; i < MC_ROWS * M; i += MC_THREADS) {
        const int r = i / M, m = i - r * M;
        s_mel[r * LD + m] = t0 + r < n && t0 + r < T_max ? mels[(base + t0 + r) * M + m] : 0.f;
    }
    for (int i = tid; i < K * M; i += MC_THREADS) {
        const int k = i / M, m = i - k * M;
        s_w[k * LD + m] = basis[i];
    }
    __syncthreads();
    for (int i = tid; i < MC_ROWS * K; i += MC_THREADS) {
        const int r = i / K, k = i - r * K, t = t0 + r;
        if (t >= T_max) continue;
        float acc = 0.f;
        if (t < n) {
            const float* w = s_w + k * LD;
            const float* x = s_mel + r * LD;
            for (int m = 0; m < M; ++m) acc = fmaf(w[m], x[m], acc);
        }
        cep[(base + t) * K + k] = acc;
    }
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_mcd_max_frames(void) { return MC_MAX_FRAMES; }

int dv3_mel_cepstra(const float* mels, const int* lengths, const float* basis, float* cep, int n_seq, int T_max, int M,
                    int K, void* stream) {
    DV3_REQUIRE(mels && lengths && basis && cep, "mel_cepstra: null operand");
    DV3_REQUIRE(n_seq >= 1 && n_seq <= 65535, "mel_cepstra: n_seq=%d outside [1, 65535]", n_seq);
    DV3_REQUIRE(T_max >= 1 && T_max <= MC_MAX_FRAMES, "mel_cepstra: T_max=%d outside [1, %d]", T_max, MC_MAX_FRAMES);
    DV3_REQUIRE(M >= 2 && M <= MC_MAX_MELS, "mel_cepstra: M=%d outside [2, %d]", M, MC_MAX_MELS);
    DV3_REQUIRE(K >= 1 && K <= M - 1 && K <= MC_MAX_K, "mel_cepstra: K=%d outside [1, min(M - 1, %d)]", K, MC_MAX_K);
    const dim3 grid((unsigned)ceil_div(T_max, MC_ROWS), (unsigned)n_seq);
    const size_t smem = (size_t)(MC_ROWS + K) * (M | 1) * sizeof(float);     // up to 49.5 KB at M = 128, K = 64
    if (cudaFuncSetAttribute(mcd_cepstra_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return check_launch("mcd_cepstra smem attribute");
    launch_k(mcd_cepstra_kernel, grid, MC_THREADS, smem, (cudaStream_t)stream, mels, lengths, basis, cep, T_max, M, K);
    return check_launch("mcd_cepstra");
}

int dv3_dtw_mcd(const float* cep, int K, const long long* work, float* workspace, float* cost, int* path_len, int P,
                void* stream) {
    DV3_REQUIRE(cep && work && workspace && cost && path_len, "dtw_mcd: null operand");
    DV3_REQUIRE(P >= 1, "dtw_mcd: P=%d", P);
    DV3_REQUIRE(K >= 1 && K <= MC_MAX_K, "dtw_mcd: K=%d outside [1, %d]", K, MC_MAX_K);
    return dtw_dispatch<false>(cep, K, work, workspace, cost, path_len, P, nullptr, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
