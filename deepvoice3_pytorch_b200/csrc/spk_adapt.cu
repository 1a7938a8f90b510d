// Speaker adaptation (train_step.TrainStep(adapt_speakers=...)): the gradient of the speaker embedding with every
// weight frozen.
//
// A speaker-conditioned site adds softsign(z) to its stream, z(b,c,t) = sum_s W[c,s] e~(b,t,s) + bias[c], where
// e~ = the time-expanded embedding after the counter-based dropout of its stack (mask m(b,t,s) / (1-p), regenerated
// here from the forward's seed and salt at element index (b*T + t)*S + s of the (B,T,S) tensor).  With W frozen the
// embedding gradient of the site collapses to (summed over the sites of a pass)
//
//     d_e(b,s) = sum_t m(b,t,s)/(1-p) * sum_c W[c,s] * G(b,c,t) * (1 - |y(b,c,t)|)^2,     y = softsign(z)
//
// G is the gradient reaching the addend, read in the form the backward already has it: the bf16 operand planes of
// the tensor-core gate split (hi + lo * 2^-11), the fp32 gate gradient of the exact path, or a (B,T,C) fp32
// residual-stream gradient.  Nothing of size (B,C,T) or (B,T,S) is written; no dW, no dbias.
//
// Order: row b gets SPK_SPLITS blocks.  The row's work items are (32-frame tile, 32-channel chunk) pairs, tiles below
// the row's logical extent only, numbered tile-major; block k takes items k, k + SPK_SPLITS, ... in ascending order.
// Per item it stages G and y of 32 channels x 32 frames together, thread (lane = frame, warp) accumulates
// u(t,s) = sum_c W[c,s] G (1-|y|)^2 over the chunk's channels in ascending order, and the masked u are summed over the
// frames by a fixed butterfly into the block's running total (the mask depends on (t,s) only, so the sum splits over
// channels).  Block k writes its total to partials[(k*B + b)*S + s] -- idle blocks write 0 -- and
// dv3_spk_grad_reduce later sums the partials of every site of the pass in index order.  No atomics; a row's bits
// depend neither on the other rows nor on the padding of the batch (nor on the schedule).
#include "common.cuh"

namespace dv3 {

constexpr int SPK_TT = 32;                       // frames per tile (one per lane)
constexpr int SPK_CC = 32;                       // channels per chunk
constexpr int SPK_THREADS = 256;
constexpr int SPK_GROUPS = SPK_THREADS / 32;     // speaker-dim groups: warp g owns s = g, g + 8, ...
constexpr int SPK_MAX_S = 64;
constexpr int SPK_J = SPK_MAX_S / SPK_GROUPS;
constexpr int SPK_SPLITS = 64;                   // blocks per row

struct SpkOperand {          // element (b, c, t) at b*sb + c*sc + t*st (elements)
    const void* p;
    long long sb, sc, st;
    long long plane;         // offset of the lo plane (PLANES only)
    int npl;
};

template <bool PLANES>
__device__ __forceinline__ float spk_load_g(const SpkOperand& g, long long off) {
    if (PLANES) {
        const bf16* q = static_cast<const bf16*>(g.p) + off;
        float v = __bfloat162float(q[0]);
        if (g.npl == 2) v += __bfloat162float(q[g.plane]) * LO_INV;
        return v;
    }
    return static_cast<const float*>(g.p)[off];
}

template <bool PLANES>
__global__ void __launch_bounds__(SPK_THREADS)
spk_grad_kernel(SpkOperand g, SpkOperand y, const float* __restrict__ w, float* __restrict__ partials, int B, int C,
                int T, int S, const long long* __restrict__ ext, int ext_mult, float p,
                const unsigned long long* __restrict__ seed, unsigned salt) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sG[SPK_CC][SPK_TT + 1];
    __shared__ float sY[SPK_CC][SPK_TT + 1];
    __shared__ float sW[SPK_CC][SPK_MAX_S];
    const int k = blockIdx.x, b = blockIdx.y;
    const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
    int tend = T;
    if (ext != nullptr) {
        const long long e = ext[0] * (long long)ext_mult;
        tend = (int)(e < 0 ? 0 : (e < T ? e : T));
    }
    const int nchunk = (C + SPK_CC - 1) / SPK_CC, nitems = ((tend + SPK_TT - 1) / SPK_TT) * nchunk;
    const DropCfg dc = make_drop(p, seed, salt);
    float tot[SPK_J];
#pragma unroll
    for (int j = 0; j < SPK_J; ++j) tot[j] = 0.f;
    for (int item = k; item < nitems; item += SPK_SPLITS) {
        const int t0 = (item / nchunk) * SPK_TT, c0 = (item % nchunk) * SPK_CC;
        __syncthreads();
        // G, y and the chunk's W rows -> shared memory; lanes along whichever axis is contiguous
        for (int i = threadIdx.x; i < SPK_CC * SPK_TT; i += SPK_THREADS) {
            const int a = i & 31, r = i >> 5;
            {
                const int cc = g.sc == 1 ? a : r, tt = g.sc == 1 ? r : a, c = c0 + cc, t = t0 + tt;
                sG[cc][tt] = (c < C && t < tend) ? spk_load_g<PLANES>(g, b * g.sb + c * g.sc + t * g.st) : 0.f;
            }
            {
                const int cc = y.sc == 1 ? a : r, tt = y.sc == 1 ? r : a, c = c0 + cc, t = t0 + tt;
                sY[cc][tt] = (c < C && t < tend) ? static_cast<const float*>(y.p)[b * y.sb + c * y.sc + t * y.st]
                                                 : 0.f;
            }
        }
        for (int i = threadIdx.x; i < SPK_CC * S; i += SPK_THREADS) {
            const int cc = i / S, s = i % S, c = c0 + cc;
            sW[cc][s] = c < C ? w[(long long)c * S + s] : 0.f;
        }
        __syncthreads();
        float u[SPK_J];
#pragma unroll
        for (int j = 0; j < SPK_J; ++j) u[j] = 0.f;
#pragma unroll 16
        for (int cc = 0; cc < SPK_CC; ++cc) {
            const float d = 1.f - fabsf(sY[cc][lane]);
            const float h = sG[cc][lane] * (d * d);              // H = G (1 - |y|)^2 = G / (1 + |z|)^2
#pragma unroll
            for (int j = 0; j < SPK_J; ++j)
                if (grp + j * SPK_GROUPS < S) u[j] = fmaf(sW[cc][grp + j * SPK_GROUPS], h, u[j]);
        }
        const int t = t0 + lane;
#pragma unroll
        for (int j = 0; j < SPK_J; ++j) {
            const int s = grp + j * SPK_GROUPS;
            if (j * SPK_GROUPS < S) {                      // uniform over the warp
                float v = 0.f;
                if (t < tend && s < S) v = u[j] * drop_scale(dc, (uint32_t)(((long long)b * T + t) * S + s));
                tot[j] += warp_sum(v);
            }
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < SPK_J; ++j) {
            const int s = grp + j * SPK_GROUPS;
            if (s < S) partials[((long long)k * B + b) * S + s] = tot[j];
        }
    }
}

// d_e[b,s] = sum_{i < nparts} partials[(i*B + b)*S + s]: one warp per (b,s), lane l takes parts l, l+32, ... in
// order, then a fixed butterfly.
__global__ void spk_grad_reduce_kernel(const float* __restrict__ partials, long long nparts, float* __restrict__ d_e,
                                       int B, int S) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int pair = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (pair >= B * S) return;
    float acc = 0.f;
    for (long long i = lane; i < nparts; i += 32) acc += partials[i * B * S + pair];
    acc = warp_sum(acc);
    if (lane == 0) d_e[pair] = acc;
}

// grad[j, s] = sum over batch rows b with ids[b] == lo + j, in row order, of d_e[b,s] (+ d_e2[b,s]); a row whose id
// lies outside [lo, lo + n) contributes nothing and sets *err_flag = 1.
__global__ void spk_rows_grad_kernel(const float* __restrict__ d_e, const float* __restrict__ d_e2,
                                     const long long* __restrict__ ids, long long lo, int n, float* __restrict__ grad,
                                     int* __restrict__ err_flag, int B, int S) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    for (int i = threadIdx.x; i < n * S; i += blockDim.x) {
        const int j = i / S, s = i % S;
        float acc = 0.f;
        for (int b = 0; b < B; ++b) {
            if (ids[b] != lo + j) continue;
            float v = d_e[(long long)b * S + s];
            if (d_e2 != nullptr) v += d_e2[(long long)b * S + s];
            acc += v;
        }
        grad[i] = acc;
    }
    if (threadIdx.x == 0 && err_flag != nullptr) {
        for (int b = 0; b < B; ++b)
            if (ids[b] < lo || ids[b] >= lo + n) *err_flag = 1;
    }
}

static int spk_grad_launch(bool planes, const SpkOperand& g, const SpkOperand& y, const float* w, float* partials,
                           int B, int C, int T, int S, const long long* ext, int ext_mult, float p,
                           const unsigned long long* seed, unsigned salt, void* stream) {
    DV3_REQUIRE(g.p && y.p && w && partials, "spk_grad: null operand");
    DV3_REQUIRE(B > 0 && C > 0 && T > 0 && S > 0 && S <= SPK_MAX_S, "spk_grad: bad shape B=%d C=%d T=%d S=%d (S <= %d)",
                B, C, T, S, SPK_MAX_S);
    DV3_REQUIRE((long long)B * C * T < (1LL << 31) && (long long)B * T * S < (1LL << 32),
                "spk_grad: B*C*T past 32-bit indexing");
    DV3_REQUIRE(B <= 65535, "spk_grad: B=%d > 65535", B);
    DV3_REQUIRE(ext_mult >= 1, "spk_grad: ext_mult=%d < 1", ext_mult);
    DV3_REQUIRE(p >= 0.f && p < 1.f, "spk_grad: p=%g outside [0, 1)", p);
    const dim3 grid(SPK_SPLITS, B);
    cudaStream_t st = (cudaStream_t)stream;
    if (planes)
        launch_k(spk_grad_kernel<true>, grid, SPK_THREADS, 0, st, g, y, w, partials, B, C, T, S, ext, ext_mult, p,
                 seed, salt);
    else
        launch_k(spk_grad_kernel<false>, grid, SPK_THREADS, 0, st, g, y, w, partials, B, C, T, S, ext, ext_mult, p,
                 seed, salt);
    return check_launch("spk_grad");
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_spk_grad_splits(void) { return SPK_SPLITS; }

int dv3_spk_grad_reduce(const float* partials, long long nparts, float* d_e, int B, int S, void* stream) {
    DV3_REQUIRE(partials && d_e && nparts > 0 && B > 0 && S > 0, "spk_grad_reduce: bad arguments");
    const int warps = 8, pairs = B * S;
    launch_k(spk_grad_reduce_kernel, ceil_div(pairs, warps), 32 * warps, 0, (cudaStream_t)stream, partials, nparts,
             d_e, B, S);
    return check_launch("spk_grad_reduce");
}

int dv3_spk_grad_planes(const void* g_planes, int npl, long long plane_stride, int ldg, const float* y_bct,
                        const float* w, float* partials, int B, int C, int T, int S, const long long* ext,
                        int ext_mult, float p, const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    DV3_REQUIRE(npl == 1 || npl == 2, "spk_grad_planes: npl=%d", npl);
    DV3_REQUIRE(ldg >= C, "spk_grad_planes: ldg=%d < C=%d", ldg, C);
    const SpkOperand g = {g_planes, (long long)T * ldg, 1, ldg, plane_stride, npl};
    const SpkOperand y = {y_bct, (long long)C * T, T, 1, 0, 1};
    return spk_grad_launch(true, g, y, w, partials, B, C, T, S, ext, ext_mult, p, seed_ptr, salt, stream);
}

int dv3_spk_grad_bct(const float* g_bct, long long g_bstride, const float* y_bct, const float* w, float* partials,
                     int B, int C, int T, int S, const long long* ext, int ext_mult, float p,
                     const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    DV3_REQUIRE(g_bstride >= (long long)C * T, "spk_grad_bct: batch stride %lld < C*T", g_bstride);
    const SpkOperand g = {g_bct, g_bstride, T, 1, 0, 1};
    const SpkOperand y = {y_bct, (long long)C * T, T, 1, 0, 1};
    return spk_grad_launch(false, g, y, w, partials, B, C, T, S, ext, ext_mult, p, seed_ptr, salt, stream);
}

int dv3_spk_grad_btc(const float* g_btc, const float* y_btc, const float* w, float* partials, int B, int C,
                     int T, int S, const long long* ext, int ext_mult, float p, const unsigned long long* seed_ptr,
                     unsigned salt, void* stream) {
    const SpkOperand g = {g_btc, (long long)T * C, 1, C, 0, 1};
    const SpkOperand y = {y_btc, (long long)T * C, 1, C, 0, 1};
    return spk_grad_launch(false, g, y, w, partials, B, C, T, S, ext, ext_mult, p, seed_ptr, salt, stream);
}

int dv3_spk_rows_grad(const float* d_e, const float* d_e2, const long long* ids, long long lo, int n, float* grad,
                      int* err_flag, int B, int S, void* stream) {
    DV3_REQUIRE(d_e && ids && grad, "spk_rows_grad: null operand");
    DV3_REQUIRE(B > 0 && n > 0 && S > 0, "spk_rows_grad: bad shape B=%d n=%d S=%d", B, n, S);
    launch_k(spk_rows_grad_kernel, 1, 256, 0, (cudaStream_t)stream, d_e, d_e2, ids, lo, n, grad, err_flag, B, S);
    return check_launch("spk_rows_grad");
}

}  // extern "C"
