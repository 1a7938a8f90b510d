// Speaker classification head (speaker_classifier.SpeakerClassifier, DESIGN.md section 2.15): logits z = h W^T + c of
// pooled features h (R, C) over K speaker classes (W (K, C)), the row-wise log-sum-exp and argmax, the mean softmax
// cross-entropy over the rows, and its gradients.
//
// Forward.  A grid of 32 x 32 (row, class) tiles computes the logits; the operands are staged through shared memory in
// 64-channel chunks and every logit is one fma chain over c in order.  Then one CTA per row: the max, the log-sum-exp
// (each thread walks k = tid, tid + 256, ...; a fixed butterfly and the warps in order: a partition fixed by K alone),
// the argmax (ties to the lowest index) and, with labels, the loss partial lse - z[label].
//
// Backward.  G[r,k] = d_logits[r,k] (nullable) + d_loss[0] * loss_scale * (exp(z[r,k] - lse[r]) - [k == label[r]]),
// formed in shared memory while the tiles are staged, never written out.  d_h = G W (R, C) runs as (row, channel) tiles
// summed over k in index order; d_W = G^T h and d_c = sum_r G as (class, channel) tiles summed over r in index order
// (d_c by the first channel tile), written directly: no per-row partial rows, no second reduce, no atomics.
//
// A label outside [0, K) sets *err_flag; its row adds 0 to the loss and nothing to the onehot, and is never used as
// an index.
#include "common.cuh"

namespace dv3 {

constexpr int SC_THREADS = 256;
constexpr int SC_TILE = 32;                 // (row, class), (row, channel) and (class, channel) tiles
constexpr int SC_CHUNK = 64;                // channels staged per pass of the logits tile
constexpr int SC_MAX_C = 256;
constexpr int SC_MIN_K = 2;
constexpr int SC_MAX_K = 8192;

__device__ __forceinline__ bool label_ok(long long lab, int K) { return lab >= 0 && lab < K; }

// G[r,k] of the backward (see the file comment); onehot only for a label inside [0, K)
__device__ __forceinline__ float spkcls_grad(const float* __restrict__ logits, const float* __restrict__ d_logits,
                                             long long idx, int k, float lse, long long lab, bool loss, float dls) {
    float g = d_logits != nullptr ? d_logits[idx] : 0.f;
    if (loss) g += dls * (expf(logits[idx] - lse) - (k == lab ? 1.f : 0.f));
    return g;
}

// ---- forward ------------------------------------------------------------------------------------------------------
// one CTA per 32 x 32 (row, class) tile; thread (rows ty, ty + 16; classes tx, tx + 16), ty = tid / 16, tx = tid % 16
__global__ void __launch_bounds__(SC_THREADS)
spkcls_logits_kernel(const float* __restrict__ h, long long ld, const float* __restrict__ w,
                     const float* __restrict__ bias, float* __restrict__ logits, int R, int C, int K) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sh[SC_TILE * (SC_CHUNK + 1)], sw[SC_TILE * (SC_CHUNK + 1)];
    constexpr int LD = SC_CHUNK + 1;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const long long r0 = (long long)blockIdx.x * SC_TILE;
    const int k0 = blockIdx.y * SC_TILE;
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (int c0 = 0; c0 < C; c0 += SC_CHUNK) {
        const int n = min(SC_CHUNK, C - c0);
        __syncthreads();
        for (int i = tid; i < SC_TILE * SC_CHUNK; i += SC_THREADS) {
            const int t = i / SC_CHUNK, c = i % SC_CHUNK;
            const bool in = c < n;
            sh[t * LD + c] = in && r0 + t < R ? h[(r0 + t) * ld + c0 + c] : 0.f;
            sw[t * LD + c] = in && k0 + t < K ? w[(long long)(k0 + t) * C + c0 + c] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int c = 0; c < SC_CHUNK; ++c) {            // zeros past n: adding 0 keeps every sum as it is
            const float a0 = sh[ty * LD + c], a1 = sh[(ty + 16) * LD + c];
            const float b0 = sw[tx * LD + c], b1 = sw[(tx + 16) * LD + c];
            acc[0][0] = fmaf(a0, b0, acc[0][0]);
            acc[0][1] = fmaf(a0, b1, acc[0][1]);
            acc[1][0] = fmaf(a1, b0, acc[1][0]);
            acc[1][1] = fmaf(a1, b1, acc[1][1]);
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const long long r = r0 + ty + 16 * i;
            const int k = k0 + tx + 16 * j;
            if (r < R && k < K) logits[r * K + k] = acc[i][j] + bias[k];
        }
}

// (value, index) of the larger logit, ties to the lower index
__device__ __forceinline__ void argmax_pair(float& v, int& i, float v2, int i2) {
    if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

// one CTA per row
__global__ void __launch_bounds__(SC_THREADS)
spkcls_rows_kernel(const float* __restrict__ logits, const long long* __restrict__ labels, float* __restrict__ lse,
                   int* __restrict__ pred, float* __restrict__ loss_partials, int* __restrict__ err_flag, int K) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float s_v[SC_THREADS / 32];
    __shared__ int s_i[SC_THREADS / 32];
    __shared__ float s_max;
    const long long r = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* z = logits + r * K;
    float v = -INFINITY;
    int vi = K;
    for (int k = tid; k < K; k += SC_THREADS) argmax_pair(v, vi, z[k], k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) argmax_pair(v, vi, __shfl_xor_sync(0xffffffffu, v, o),
                                                 __shfl_xor_sync(0xffffffffu, vi, o));
    if (lane == 0) { s_v[warp] = v; s_i[warp] = vi; }
    __syncthreads();
    if (tid == 0) {
        for (int q = 1; q < SC_THREADS / 32; ++q) argmax_pair(v, vi, s_v[q], s_i[q]);
        s_max = v;
        pred[r] = vi;
    }
    __syncthreads();
    const float m = s_max;
    float s = 0.f;
    for (int k = tid; k < K; k += SC_THREADS) s += expf(z[k] - m);
    s = warp_sum(s);
    if (lane == 0) s_v[warp] = s;          // tid 0 read s_v before the barrier above
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int q = 0; q < SC_THREADS / 32; ++q) t += s_v[q];
        const float l = m + logf(t);
        lse[r] = l;
        if (labels != nullptr) {
            const long long lab = labels[r];
            const bool ok = label_ok(lab, K);
            if (!ok) *err_flag = 1;
            loss_partials[r] = ok ? l - z[lab] : 0.f;
        }
    }
}

// ---- backward -----------------------------------------------------------------------------------------------------
// d_h: one CTA per 32 x 32 (row, channel) tile, k in chunks of 32; thread (rows ty, ty + 16; channels tx, tx + 16)
__global__ void __launch_bounds__(SC_THREADS)
spkcls_dh_kernel(const float* __restrict__ w, const float* __restrict__ logits, const float* __restrict__ lse,
                 const long long* __restrict__ labels, const float* __restrict__ d_logits,
                 const float* __restrict__ d_loss, float loss_scale, float* __restrict__ d_h,
                 int* __restrict__ err_flag, int R, int C, int K) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    constexpr int LD = SC_TILE + 1;
    __shared__ float sg[SC_TILE * LD], sw[SC_TILE * LD];
    __shared__ float s_lse[SC_TILE];
    __shared__ long long s_lab[SC_TILE];
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const long long r0 = (long long)blockIdx.x * SC_TILE;
    const int c0 = blockIdx.y * SC_TILE;
    const bool loss = labels != nullptr && d_loss != nullptr;
    const float dls = loss ? d_loss[0] * loss_scale : 0.f;
    if (tid < SC_TILE) {
        const long long r = r0 + tid;
        s_lse[tid] = r < R ? lse[r] : 0.f;
        long long lab = -1;
        if (labels != nullptr && r < R) {
            lab = labels[r];
            if (!label_ok(lab, K)) {
                if (blockIdx.y == 0) *err_flag = 1;
                lab = -1;
            }
        }
        s_lab[tid] = lab;
    }
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (int k0 = 0; k0 < K; k0 += SC_TILE) {
        __syncthreads();
        for (int i = tid; i < SC_TILE * SC_TILE; i += SC_THREADS) {
            const int t = i / SC_TILE, j = i % SC_TILE;
            const long long r = r0 + t;
            const int k = k0 + j;
            sg[t * LD + j] = r < R && k < K ? spkcls_grad(logits, d_logits, r * K + k, k, s_lse[t], s_lab[t], loss, dls)
                                            : 0.f;
            sw[t * LD + j] = k0 + t < K && c0 + j < C ? w[(long long)(k0 + t) * C + c0 + j] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int j = 0; j < SC_TILE; ++j) {             // zeros past K
            const float g0 = sg[ty * LD + j], g1 = sg[(ty + 16) * LD + j];
            const float w0 = sw[j * LD + tx], w1 = sw[j * LD + tx + 16];
            acc[0][0] = fmaf(g0, w0, acc[0][0]);
            acc[0][1] = fmaf(g0, w1, acc[0][1]);
            acc[1][0] = fmaf(g1, w0, acc[1][0]);
            acc[1][1] = fmaf(g1, w1, acc[1][1]);
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const long long r = r0 + ty + 16 * i;
            const int c = c0 + tx + 16 * j;
            if (r < R && c < C) d_h[r * C + c] = acc[i][j];
        }
}

// d_W, d_c: one CTA per 32 x 32 (class, channel) tile, r in chunks of 32; thread (classes ty, ty + 16; channels tx,
// tx + 16); the first channel tile's first 32 threads also sum d_c of the tile's classes
__global__ void __launch_bounds__(SC_THREADS)
spkcls_dw_kernel(const float* __restrict__ h, long long ld, const float* __restrict__ logits,
                 const float* __restrict__ lse, const long long* __restrict__ labels,
                 const float* __restrict__ d_logits, const float* __restrict__ d_loss, float loss_scale,
                 float* __restrict__ d_w, float* __restrict__ d_bias, int R, int C, int K) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    constexpr int LD = SC_TILE + 1;
    __shared__ float sg[SC_TILE * LD], sh[SC_TILE * LD];
    __shared__ float s_lse[SC_TILE];
    __shared__ long long s_lab[SC_TILE];
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int c0 = blockIdx.x * SC_TILE, k0 = blockIdx.y * SC_TILE;
    const bool loss = labels != nullptr && d_loss != nullptr;
    const float dls = loss ? d_loss[0] * loss_scale : 0.f;
    const bool bias_tile = blockIdx.x == 0;
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    float db = 0.f;
    for (long long r0 = 0; r0 < R; r0 += SC_TILE) {
        __syncthreads();
        if (tid < SC_TILE) {
            const long long r = r0 + tid;
            s_lse[tid] = r < R ? lse[r] : 0.f;
            long long lab = labels != nullptr && r < R ? labels[r] : -1;
            s_lab[tid] = label_ok(lab, K) ? lab : -1;
        }
        __syncthreads();
        for (int i = tid; i < SC_TILE * SC_TILE; i += SC_THREADS) {
            const int t = i / SC_TILE, j = i % SC_TILE;
            const long long r = r0 + t;
            const int k = k0 + j;
            sg[t * LD + j] = r < R && k < K ? spkcls_grad(logits, d_logits, r * K + k, k, s_lse[t], s_lab[t], loss, dls)
                                            : 0.f;
            sh[t * LD + j] = r < R && c0 + j < C ? h[r * ld + c0 + j] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int t = 0; t < SC_TILE; ++t) {             // zeros past R
            const float g0 = sg[t * LD + ty], g1 = sg[t * LD + ty + 16];
            const float h0 = sh[t * LD + tx], h1 = sh[t * LD + tx + 16];
            acc[0][0] = fmaf(g0, h0, acc[0][0]);
            acc[0][1] = fmaf(g0, h1, acc[0][1]);
            acc[1][0] = fmaf(g1, h0, acc[1][0]);
            acc[1][1] = fmaf(g1, h1, acc[1][1]);
        }
        if (bias_tile && tid < SC_TILE)
            for (int t = 0; t < SC_TILE; ++t) db += sg[t * LD + tid];
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int k = k0 + ty + 16 * i, c = c0 + tx + 16 * j;
            if (k < K && c < C) d_w[(long long)k * C + c] = acc[i][j];
        }
    if (bias_tile && tid < SC_TILE && k0 + tid < K) d_bias[k0 + tid] = db;
}

static int spkcls_check(const char* what, int R, int C, int K, long long ld) {
    DV3_REQUIRE(R >= 1, "%s: R=%d", what, R);
    DV3_REQUIRE(C >= 1 && C <= SC_MAX_C, "%s: C=%d outside [1, %d]", what, C, SC_MAX_C);
    DV3_REQUIRE(K >= SC_MIN_K && K <= SC_MAX_K, "%s: K=%d outside [%d, %d]", what, K, SC_MIN_K, SC_MAX_K);
    DV3_REQUIRE((long long)R * K < (1LL << 31), "%s: R*K = %lld past 2^31", what, (long long)R * K);
    DV3_REQUIRE(ld >= C, "%s: row stride %lld below C = %d", what, ld, C);
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_spkcls_fwd(const float* h, long long ld, const float* w, const float* bias, const long long* labels,
                   float* logits, float* lse, int* pred, float* loss_partials, int* err_flag, int R, int C, int K,
                   void* stream) {
    if (spkcls_check("spkcls_fwd", R, C, K, ld)) return 1;
    DV3_REQUIRE(h && w && bias && logits && lse && pred && err_flag, "spkcls_fwd: null operand");
    DV3_REQUIRE((labels == nullptr) == (loss_partials == nullptr), "spkcls_fwd: labels and loss_partials go together");
    const dim3 grid((unsigned)((R + SC_TILE - 1) / SC_TILE), (unsigned)((K + SC_TILE - 1) / SC_TILE));
    launch_k(spkcls_logits_kernel, grid, SC_THREADS, 0, (cudaStream_t)stream, h, ld, w, bias, logits, R, C, K);
    if (check_launch("spkcls_logits")) return 1;
    launch_k(spkcls_rows_kernel, (unsigned)R, SC_THREADS, 0, (cudaStream_t)stream, logits, labels, lse, pred,
             loss_partials, err_flag, K);
    return check_launch("spkcls_rows");
}

int dv3_spkcls_bwd(const float* h, long long ld, const float* w, const float* logits, const float* lse,
                   const long long* labels, const float* d_logits, const float* d_loss, float loss_scale, float* d_h,
                   float* d_w, float* d_bias, int* err_flag, int R, int C, int K, void* stream) {
    if (spkcls_check("spkcls_bwd", R, C, K, ld)) return 1;
    DV3_REQUIRE(h && w && logits && lse && d_h && d_w && d_bias && err_flag, "spkcls_bwd: null operand");
    const dim3 g_dh((unsigned)((R + SC_TILE - 1) / SC_TILE), (unsigned)((C + SC_TILE - 1) / SC_TILE));
    launch_k(spkcls_dh_kernel, g_dh, SC_THREADS, 0, (cudaStream_t)stream, w, logits, lse, labels, d_logits, d_loss,
             loss_scale, d_h, err_flag, R, C, K);
    if (check_launch("spkcls_dh")) return 1;
    const dim3 g_dw((unsigned)((C + SC_TILE - 1) / SC_TILE), (unsigned)((K + SC_TILE - 1) / SC_TILE));
    launch_k(spkcls_dw_kernel, g_dw, SC_THREADS, 0, (cudaStream_t)stream, h, ld, logits, lse, labels, d_logits, d_loss,
             loss_scale, d_w, d_bias, R, C, K);
    return check_launch("spkcls_dw");
}

}  // extern "C"
