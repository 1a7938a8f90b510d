// The DTW recursion of MCD-DTW (mcd.py, DESIGN.md sections 2.17 and 2.18), shared by csrc/mcd.cu (cost and path length
// only, PATH = false) and csrc/pitch.cu (PATH = true: also the predecessor of every cell, for the warping path).
//
// D(0,0) = 0, D(i,0) = D(0,j) = +inf, D(i,j) = d(i,j) + min(D(i-1,j-1), D(i-1,j), D(i,j-1)) with ties to the
// diagonal, then (i-1,j), then (i,j-1); the path length L (cells on the chosen path) rides along with the chosen
// predecessor.  One warp per pair, a systolic array over strips of 32 rows: lane l owns row i0 + l + 1 and keeps its
// cepstrum in registers; at step s it computes column j = s - l + 1.  D(i-1,j) arrives from lane l-1 by __shfl_up_sync,
// D(i-1,j-1) is the value that arrived one step earlier, D(i,j-1) is the lane's own last value.  Lane 0 reads row i0
// of the strip above from a per-pair boundary buffer in global memory, which lane 31 rewrites in place with row
// i0 + 32 (column j is read at step j - 1 and rewritten at step j + 30).  The b frames are staged by cp.async in
// 32-row chunks into a three-chunk shared-memory ring, one chunk ahead; the ring's row stride KP + 1 is odd, so the
// 32 lanes, each reading a different row, hit 32 different banks.  d(i,j) = sqrt of one fma chain over k in order
// (padding k >= K adds exact zeros).  No atomics, no block barriers: a pair's bits depend on its own lengths alone.
//
// PATH: each lane also packs the 2-bit code of every cell's chosen predecessor (0 diagonal, 1 up = (i-1,j), 2 left =
// (i,j-1)) into a register, 16 columns a word, and stores the word when its 16th column (or column M) is done: row i's
// words are dirs[path_work[2 * row] + (i-1)*ceil(M/16) + (j-1)/16].  The arithmetic of D and L is the same code in both variants,
// so cost and L are bit-identical.
#pragma once
#include "common.cuh"

namespace dv3 {

constexpr int MC_MAX_K = 64;
constexpr int MC_MAX_FRAMES = 16384;      // per sequence: about 190 s at 22 050 Hz / hop 256
constexpr int DTW_RING = 3;               // b chunks of 32 rows: the two being read and the one landing

static __device__ __forceinline__ void cp_async4(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
                 : "memory");
}
static __device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
                 "l"(src) : "memory");
}
static __device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
static __device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;\n" ::: "memory"); }
static __device__ __forceinline__ void cp_async_wait_0() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }
template <int N>
static __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// One warp per work row (pair, a_row, N, b_row, M, ws_off); ws holds per pair roundup(M, 32) boundary costs, then as
// many path lengths (int bits), 32-float aligned.  KP: K rounded up to a multiple of 8.  PATH: path_work[2 * row] is
// the word offset of the row's N * ceil(M/16) direction words in dirs (both unused without PATH).
template <int KP, bool PATH>
__global__ void __launch_bounds__(32)
mcd_dtw_kernel(const float* __restrict__ cep, const long long* __restrict__ work, float* __restrict__ ws,
               float* __restrict__ cost, int* __restrict__ path_len, int K, const long long* __restrict__ path_work,
               unsigned* __restrict__ dirs) {
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
    const int M16 = (M + 15) >> 4;
    unsigned* dir = nullptr;
    if (PATH) dir = dirs + path_work[2LL * blockIdx.x];
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
        unsigned word = 0;                         // PATH: the codes of this row's current 16 columns
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
                unsigned code = 0;
                if (up < best) { best = up; bl = upL; code = 1; }
                if (left < best) { best = left; bl = leftL; code = 2; }
                left = sqrtf(acc) + best;
                leftL = bl + 1;
                if (i == N && j == M) { cost[pair] = left; path_len[pair] = leftL; }
                if (lane == 31 && has_below) { bufD[j - 1] = left; bufL[j - 1] = leftL; }
                if (PATH) {
                    const int c = (j - 1) & 15;
                    word |= code << (2 * c);
                    if (c == 15 || j == M) {
                        dir[(long long)(i - 1) * M16 + ((j - 1) >> 4)] = word;
                        word = 0;
                    }
                }
            }
            sh = __shfl_up_sync(0xffffffffu, left, 1);
            shL = __shfl_up_sync(0xffffffffu, leftL, 1);
        }
        cp_async_wait_0();
        __threadfence_block();                     // lane 31's boundary row before the next strip's cp.async reads it
        __syncwarp();
    }
}

static inline size_t dtw_smem_bytes(int KP) { return (size_t)DTW_RING * 32 * (KP + 1) * 4 + (size_t)DTW_RING * 32 * 8; }

template <int KP, bool PATH>
static int dtw_launch(const float* cep, const long long* work, float* ws, float* cost, int* path_len, int K, int P,
                      const long long* path_work, unsigned* dirs, cudaStream_t st) {
    const size_t smem = dtw_smem_bytes(KP);
    launch_k(mcd_dtw_kernel<KP, PATH>, (unsigned)P, 32, smem, st, cep, work, ws, cost, path_len, K, path_work, dirs);
    return check_launch(PATH ? "dtw_path" : "mcd_dtw");
}

// KP = K rounded up to 8 -> the instantiation
template <bool PATH>
static int dtw_dispatch(const float* cep, int K, const long long* work, float* ws, float* cost, int* path_len, int P,
                        const long long* path_work, unsigned* dirs, cudaStream_t st) {
    switch ((K + 7) / 8) {
        case 1: return dtw_launch<8, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        case 2: return dtw_launch<16, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        case 3: return dtw_launch<24, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        case 4: return dtw_launch<32, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        case 5: return dtw_launch<40, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        case 6: return dtw_launch<48, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        case 7: return dtw_launch<56, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
        default: return dtw_launch<64, PATH>(cep, work, ws, cost, path_len, K, P, path_work, dirs, st);
    }
}

}  // namespace dv3
