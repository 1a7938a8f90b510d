// Mel-cepstral distortion after dynamic time warping (mcd.py, DESIGN.md section 2.17).
//
// Cepstra.  c[t, k-1] = sum_m basis[k-1, m] mel[t, m] for k = 1..K: basis is the orthonormal DCT-II row k of the
// natural-log amplitude, scaled by -min_level_db ln10 / 20 (built in fp64 on the host, rounded once).  The affine
// offset of the denormalisation only reaches c_0, which is dropped, so the kernel reads the normalised mels as they
// are.  One CTA per MC_ROWS frames of one sequence stages those rows and the table in shared memory; every output is
// one fma chain over m in order.  Frames at or past a sequence's count are not read and their outputs are zero.
//
// DTW.  D(0,0) = 0, D(i,0) = D(0,j) = +inf, D(i,j) = d(i,j) + min(D(i-1,j-1), D(i-1,j), D(i,j-1)) with ties to the
// diagonal, then (i-1,j), then (i,j-1); the path length L (cells on the chosen path) rides along with the chosen
// predecessor.  One warp per pair, a systolic array over strips of 32 rows: lane l owns row i0 + l + 1 and keeps its
// cepstrum in registers; at step s it computes column j = s - l + 1.  D(i-1,j) arrives from lane l-1 by __shfl_up_sync,
// D(i-1,j-1) is the value that arrived one step earlier, D(i,j-1) is the lane's own last value.  Lane 0 reads row i0
// of the strip above from a per-pair boundary buffer in global memory, which lane 31 rewrites in place with row
// i0 + 32 (column j is read at step j - 1 and rewritten at step j + 30).  The b frames are staged by cp.async in
// 32-row chunks into a three-chunk shared-memory ring, one chunk ahead; the ring's row stride KP + 1 is odd, so the
// 32 lanes, each reading a different row, hit 32 different banks.  d(i,j) = sqrt of one fma chain over k in order
// (padding k >= K adds exact zeros).  No atomics, no block barriers: a pair's bits depend on its own lengths alone.
#include "common.cuh"

namespace dv3 {

constexpr int MC_ROWS = 32;               // frames per CTA of the cepstra kernel
constexpr int MC_THREADS = 128;
constexpr int MC_MAX_MELS = 128;          // the filterbank's limit (audio.check_geometry)
constexpr int MC_MAX_K = 64;
constexpr int MC_MAX_FRAMES = 16384;      // per sequence: about 190 s at 22 050 Hz / hop 256
constexpr int DTW_RING = 3;               // b chunks of 32 rows: the two being read and the one landing

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

__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
                 : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
                 "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_0() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// One warp per work row (pair, a_row, N, b_row, M, ws_off); ws holds per pair roundup(M, 32) boundary costs, then as
// many path lengths (int bits), 32-float aligned.  KP: K rounded up to a multiple of 8.
template <int KP>
__global__ void __launch_bounds__(32)
mcd_dtw_kernel(const float* __restrict__ cep, const long long* __restrict__ work, float* __restrict__ ws,
               float* __restrict__ cost, int* __restrict__ path_len, int K) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    constexpr int S = KP + 1;                     // odd ring row stride: conflict-free reads of 32 different rows
    extern __shared__ float smem[];
    float* ring = smem;                                              // DTW_RING x 32 rows x S
    float* ringD = smem + DTW_RING * 32 * S;                         // DTW_RING x 32 boundary costs
    int* ringL = reinterpret_cast<int*>(ringD + DTW_RING * 32);      // DTW_RING x 32 boundary path lengths
    const int lane = threadIdx.x;
    const long long* w = work + 6LL * blockIdx.x;
    const long long pair = w[0], a_row = w[1], b_row = w[3], ws_off = w[5];
    const int N = (int)w[2], M = (int)w[4];
    const int M32 = (M + 31) & ~31;
    float* bufD = ws + ws_off;
    int* bufL = reinterpret_cast<int*>(ws + ws_off + M32);
    const float INF = __int_as_float(0x7f800000);
    for (int i = lane; i < DTW_RING * 32 * S; i += 32) ring[i] = 0.f;     // columns K..KP-1 stay zero
    __syncwarp();

    for (int i0 = 0; i0 < N; i0 += 32) {
        const int i = i0 + lane + 1;
        const bool row_ok = i <= N;
        const bool has_above = i0 > 0, has_below = i0 + 32 < N;
        float a[KP];
#pragma unroll
        for (int k = 0; k < KP; ++k) a[k] = row_ok && k < K ? cep[(a_row + i - 1) * K + k] : 0.f;
        // chunk c: b rows 32c .. 32c + 31 (0-based) and, below the first strip, boundary columns 32c + 1 .. 32c + 32
        auto issue = [&](int c) {
            if (32 * c < M) {
                float* dst = ring + (c % DTW_RING) * 32 * S;
                const int nrow = min(32, M - 32 * c);
                const float* src = cep + (b_row + 32LL * c) * K;
                for (int e = lane; e < nrow * K; e += 32) {
                    const int r = e / K, k = e - r * K;
                    cp_async4(dst + r * S + k, src + e);
                }
                if (has_above && lane < 16) {
                    const int slot = (c % DTW_RING) * 32, part = (lane & 7) * 4;
                    if (lane < 8) cp_async16(ringD + slot + part, bufD + 32 * c + part);
                    else cp_async16(ringL + slot + part, bufL + 32 * c + part);
                }
            }
            cp_async_commit();
        };
        __syncwarp();
        issue(0);
        float up = has_above ? INF : 0.f;          // lane 0: D(i0, 0), the diagonal of its first column
        int upL = 0;
        float left = INF, sh = INF;                // D(i, j-1); the value lane l-1 passed up
        int leftL = 0, shL = 0;
        const int steps = M + min(32, N - i0) - 1;
        for (int s = 0; s < steps; ++s) {
            if ((s & 31) == 0) {
                issue((s >> 5) + 1);
                cp_async_wait_1();
                __syncwarp();
            }
            const int j = s - lane + 1;
            const float dg = up;
            const int dgL = upL;
            if (lane == 0) {
                if (!has_above || j > M) { up = INF; upL = 0; }
                else { const int x = ((j - 1) >> 5) % DTW_RING * 32 + ((j - 1) & 31); up = ringD[x]; upL = ringL[x]; }
            } else { up = sh; upL = shL; }
            if (row_ok && j >= 1 && j <= M) {
                const float* b = ring + (((j - 1) >> 5) % DTW_RING * 32 + ((j - 1) & 31)) * S;
                float acc = 0.f;
#pragma unroll
                for (int k = 0; k < KP; ++k) {
                    const float t = a[k] - b[k];
                    acc = fmaf(t, t, acc);
                }
                float best = dg;
                int bl = dgL;
                if (up < best) { best = up; bl = upL; }
                if (left < best) { best = left; bl = leftL; }
                left = sqrtf(acc) + best;
                leftL = bl + 1;
                if (i == N && j == M) { cost[pair] = left; path_len[pair] = leftL; }
                if (lane == 31 && has_below) { bufD[j - 1] = left; bufL[j - 1] = leftL; }
            }
            sh = __shfl_up_sync(0xffffffffu, left, 1);
            shL = __shfl_up_sync(0xffffffffu, leftL, 1);
        }
        cp_async_wait_0();
        __threadfence_block();                     // lane 31's boundary row before the next strip's cp.async reads it
        __syncwarp();
    }
}

static size_t dtw_smem_bytes(int KP) { return (size_t)DTW_RING * 32 * (KP + 1) * 4 + (size_t)DTW_RING * 32 * 8; }

template <int KP>
static int dtw_launch(const float* cep, const long long* work, float* ws, float* cost, int* path_len, int K, int P,
                      cudaStream_t st) {
    const size_t smem = dtw_smem_bytes(KP);
    launch_k(mcd_dtw_kernel<KP>, (unsigned)P, 32, smem, st, cep, work, ws, cost, path_len, K);
    return check_launch("mcd_dtw");
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
    const cudaStream_t st = (cudaStream_t)stream;
    switch ((K + 7) / 8) {
        case 1: return dtw_launch<8>(cep, work, workspace, cost, path_len, K, P, st);
        case 2: return dtw_launch<16>(cep, work, workspace, cost, path_len, K, P, st);
        case 3: return dtw_launch<24>(cep, work, workspace, cost, path_len, K, P, st);
        case 4: return dtw_launch<32>(cep, work, workspace, cost, path_len, K, P, st);
        case 5: return dtw_launch<40>(cep, work, workspace, cost, path_len, K, P, st);
        case 6: return dtw_launch<48>(cep, work, workspace, cost, path_len, K, P, st);
        case 7: return dtw_launch<56>(cep, work, workspace, cost, path_len, K, P, st);
        default: return dtw_launch<64>(cep, work, workspace, cost, path_len, K, P, st);
    }
}

}  // extern "C"
