// Speaker verification head (speaker_verifier.SpeakerVerifier, DESIGN.md section 2.14): the embeddings of enrollment
// sets and test utterances, the PLDA-like score of every (enrollment, test) pair and the class-balanced binary
// cross-entropy over the pairs of a training batch.
//
// Embed.  For row b over its n = counts[b] <= N valid rows h_{b,i} (C): hbar = (sum_{i<n} h_{b,i}) / n (sum in i
// order), out_b = W hbar + c (W (D, C)); one CTA per row, one warp per output d (lanes stride c, then a fixed
// butterfly).  Backward: d h_{b,i} = W^T d(out_b) / n for i < n, 0 past it, and one partial gradient row per input row:
// [d W = d(out_b) hbar^T (D*C), d c = d(out_b) (D)].  A count outside [1, N] sets *err_flag and yields 0.
//
// Score.  L[e,t] = x_e.y_t - x_e^T S x_e - y_t^T S y_t + b.  The quadratic terms are computed once per row (one CTA per
// row of x and of y), then a grid of 32 x 32 pair tiles spreads the dot products over the SMs.  Every pair's dot runs
// over d in order, so a pair's score depends only on its own two rows.  With speaker ids, pair (e, t) is "same" when
// ids_e[e] == ids_t[t]; its loss is w_same softplus(-L) (same) or w_diff softplus(L) (different), w_same = 1/(2 n_same),
// w_diff = 1/(2 n_diff) over the whole batch, counted on the device; each tile writes one partial per row (its 32
// columns in order), and dv3_spkenc_reduce sums the partials in index order.
// Backward, one CTA per row of x and of y: G[e,t] = d_scores[e,t] + d_loss * dLoss/dL[e,t];
//     dx_e = sum_t G[e,t] y_t - g_e (S + S^T) x_e,   g_e = sum_t G[e,t]      (and symmetrically dy_t, g_t = sum_e G)
// and one partial row [d S = -g_r z_r z_r^T (D*D), d b] per row r of x then y (d b: g_e on x rows, 0 on y rows).
// No atomics anywhere.
#include "common.cuh"

namespace dv3 {

constexpr int SV_THREADS = 256;
constexpr int SV_MAX_N = 32;
constexpr int SV_MAX_C = 256;
constexpr int SV_MAX_D = 128;
constexpr int SV_TILE = 32;                 // pair tile: SV_TILE enrollment rows x SV_TILE test rows
constexpr int SV_LD = SV_MAX_D + 1;         // padded shared row: the 8 test rows a warp reads fall in distinct banks

// ---- embed --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SV_THREADS)
spkver_embed_fwd_kernel(const float* __restrict__ h, long long ld, const int* __restrict__ counts,
                        const float* __restrict__ w, const float* __restrict__ c, float* __restrict__ hbar,
                        float* __restrict__ out, int* __restrict__ err_flag, int N, int C, int D) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sm[SV_MAX_C];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = counts[b];
    if (n < 1 || n > N) {
        if (tid == 0) *err_flag = 1;
        for (int k = tid; k < C; k += SV_THREADS) hbar[(long long)b * C + k] = 0.f;
        for (int d = tid; d < D; d += SV_THREADS) out[(long long)b * D + d] = 0.f;
        return;
    }
    const float* hb = h + (long long)b * ld;
    for (int k = tid; k < C; k += SV_THREADS) {
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc += hb[(long long)i * C + k];
        acc /= (float)n;
        sm[k] = acc;
        hbar[(long long)b * C + k] = acc;
    }
    __syncthreads();
    for (int d = warp; d < D; d += SV_THREADS / 32) {
        float acc = 0.f;
        for (int k = lane; k < C; k += 32) acc = fmaf(w[(long long)d * C + k], sm[k], acc);
        acc = warp_sum(acc);
        if (lane == 0) out[(long long)b * D + d] = acc + c[d];
    }
}

__global__ void __launch_bounds__(SV_THREADS)
spkver_embed_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ hbar,
                        const int* __restrict__ counts, const float* __restrict__ w, float* __restrict__ d_h,
                        long long ld, float* __restrict__ partials, int* __restrict__ err_flag, int N, int C, int D) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sg[SV_MAX_D];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = counts[b];
    const bool ok = n >= 1 && n <= N;
    const long long P = (long long)D * C + D;
    float* part = partials + (long long)b * P;
    float* dhb = d_h + (long long)b * ld;
    if (!ok) {
        if (tid == 0) *err_flag = 1;
        for (long long i = tid; i < P; i += SV_THREADS) part[i] = 0.f;
        for (int i = tid; i < N * C; i += SV_THREADS) dhb[i] = 0.f;
        return;
    }
    for (int d = tid; d < D; d += SV_THREADS) sg[d] = d_out[(long long)b * D + d];
    __syncthreads();
    for (int k = tid; k < C; k += SV_THREADS) {
        float acc = 0.f;
        for (int d = 0; d < D; ++d) acc = fmaf(w[(long long)d * C + k], sg[d], acc);
        acc /= (float)n;
        for (int i = 0; i < N; ++i) dhb[(long long)i * C + k] = i < n ? acc : 0.f;
    }
    const float* hb = hbar + (long long)b * C;
    for (long long idx = tid; idx < (long long)D * C; idx += SV_THREADS) {
        const int d = (int)(idx / C), k = (int)(idx % C);
        part[idx] = sg[d] * hb[k];
    }
    for (int d = tid; d < D; d += SV_THREADS) part[(long long)D * C + d] = sg[d];
}

// ---- score --------------------------------------------------------------------------------------------------------
// q[r] = z_r^T S z_r for the rows of x (r < B_e) then of y: u_j = sum_i z_i S[i, j] (coalesced over j), then
// q = sum_j z_j u_j in j order by one thread.
__global__ void __launch_bounds__(SV_MAX_D)
spkver_quad_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ S,
                   float* __restrict__ qx, float* __restrict__ qy, int B_e, int D) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sz[SV_MAX_D], su[SV_MAX_D];
    const int r = blockIdx.x, j = threadIdx.x;
    const float* z = r < B_e ? x + (long long)r * D : y + (long long)(r - B_e) * D;
    if (j < D) sz[j] = z[j];
    __syncthreads();
    if (j < D) {
        float acc = 0.f;
        for (int i = 0; i < D; ++i) acc = fmaf(sz[i], S[(long long)i * D + j], acc);
        su[j] = sz[j] * acc;
    }
    __syncthreads();
    if (j == 0) {
        float acc = 0.f;
        for (int i = 0; i < D; ++i) acc += su[i];
        if (r < B_e) qx[r] = acc; else qy[r - B_e] = acc;
    }
}

// the class weights of the balanced loss: 1 / (2 n_same), 1 / (2 n_diff) (0 for an empty class); integer counts, so the
// order of the block-wide count does not matter
__device__ inline void spkver_weights(const long long* __restrict__ ids_e, const long long* __restrict__ ids_t,
                                      int B_e, int B_t, float& w_same, float& w_diff) {
    const long long pairs = (long long)B_e * B_t;
    long long same = 0;
    for (long long base = 0; base < pairs; base += blockDim.x) {
        const long long p = base + threadIdx.x;
        same += __syncthreads_count(p < pairs && ids_e[p / B_t] == ids_t[p % B_t]);
    }
    const long long diff = pairs - same;
    w_same = same > 0 ? 0.5f / (float)same : 0.f;
    w_diff = diff > 0 ? 0.5f / (float)diff : 0.f;
}

__device__ __forceinline__ float softplus(float z) { return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))); }
__device__ __forceinline__ float sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

// one CTA per 32 x 32 pair tile; thread (e = tid / 8, t = tid % 8 + 8 k), k < 4
__global__ void __launch_bounds__(SV_THREADS)
spkver_score_fwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ qx,
                        const float* __restrict__ qy, const float* __restrict__ bias,
                        const long long* __restrict__ ids_e, const long long* __restrict__ ids_t,
                        float* __restrict__ scores, float* __restrict__ loss_partials, int B_e, int B_t, int D) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sx[SV_TILE * SV_LD], sy[SV_TILE * SV_LD];
    __shared__ float sl[SV_TILE * (SV_TILE + 1)];
    const int tid = threadIdx.x;
    const int e0 = blockIdx.y * SV_TILE, t0 = blockIdx.x * SV_TILE;
    for (int i = tid; i < SV_TILE * D; i += SV_THREADS) {
        const int r = i / D, d = i % D;
        sx[r * SV_LD + d] = e0 + r < B_e ? x[(long long)(e0 + r) * D + d] : 0.f;
        sy[r * SV_LD + d] = t0 + r < B_t ? y[(long long)(t0 + r) * D + d] : 0.f;
    }
    float w_same = 0.f, w_diff = 0.f;
    if (ids_e != nullptr) spkver_weights(ids_e, ids_t, B_e, B_t, w_same, w_diff);
    __syncthreads();
    const float b = bias[0];
    const int el = tid >> 3;
    const int e = e0 + el;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int tl = (tid & 7) + 8 * k, t = t0 + tl;
        float l = 0.f;
        if (e < B_e && t < B_t) {
            float dot = 0.f;
            for (int d = 0; d < D; ++d) dot = fmaf(sx[el * SV_LD + d], sy[tl * SV_LD + d], dot);
            const float L = ((dot - qx[e]) - qy[t]) + b;
            scores[(long long)e * B_t + t] = L;
            if (ids_e != nullptr) l = ids_e[e] == ids_t[t] ? w_same * softplus(-L) : w_diff * softplus(L);
        }
        sl[el * (SV_TILE + 1) + tl] = l;
    }
    if (ids_e == nullptr) return;
    __syncthreads();
    if (tid < SV_TILE && e0 + tid < B_e) {
        float acc = 0.f;
        for (int tl = 0; tl < SV_TILE && t0 + tl < B_t; ++tl) acc += sl[tid * (SV_TILE + 1) + tl];
        loss_partials[(long long)(e0 + tid) * gridDim.x + blockIdx.x] = acc;
    }
}

// one CTA per row r of x (r < B_e) and of y, one thread per d
__global__ void __launch_bounds__(SV_MAX_D)
spkver_score_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ S,
                        const float* __restrict__ scores, const long long* __restrict__ ids_e,
                        const long long* __restrict__ ids_t, const float* __restrict__ d_scores,
                        const float* __restrict__ d_loss, float* __restrict__ dx, float* __restrict__ dy,
                        float* __restrict__ partials, int B_e, int B_t, int D) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sG[SV_MAX_D], sz[SV_MAX_D];
    const int r = blockIdx.x, j = threadIdx.x;
    const bool is_x = r < B_e;
    const int row = is_x ? r : r - B_e;
    const int n_other = is_x ? B_t : B_e;
    const float* z = is_x ? x + (long long)row * D : y + (long long)row * D;
    const float* other = is_x ? y : x;
    const bool loss = ids_e != nullptr && d_loss != nullptr;
    float w_same = 0.f, w_diff = 0.f;
    if (loss) spkver_weights(ids_e, ids_t, B_e, B_t, w_same, w_diff);
    const float dl = loss ? d_loss[0] : 0.f;
    if (j < D) sz[j] = z[j];
    float acc = 0.f, g = 0.f;
    for (int base = 0; base < n_other; base += SV_MAX_D) {
        __syncthreads();
        const int o = base + j;
        if (o < n_other) {
            const long long p = is_x ? (long long)row * B_t + o : (long long)o * B_t + row;
            float G = d_scores != nullptr ? d_scores[p] : 0.f;
            if (loss) {
                const float L = scores[p];
                const bool same = ids_e[is_x ? row : o] == ids_t[is_x ? o : row];
                G += dl * (same ? -w_same * sigmoid(-L) : w_diff * sigmoid(L));
            }
            sG[j] = G;
        }
        __syncthreads();
        const int m = min(SV_MAX_D, n_other - base);
        for (int i = 0; i < m; ++i) {
            g += sG[i];
            if (j < D) acc = fmaf(sG[i], other[(long long)(base + i) * D + j], acc);
        }
    }
    const long long P = (long long)D * D + 1;
    float* part = partials + (long long)r * P;
    if (j < D) {
        float s2 = 0.f;
        for (int i = 0; i < D; ++i) s2 = fmaf(S[(long long)j * D + i] + S[(long long)i * D + j], sz[i], s2);
        (is_x ? dx : dy)[(long long)row * D + j] = acc - g * s2;
        const float gz = -g * sz[j];
        for (int i = 0; i < D; ++i) part[(long long)j * D + i] = gz * sz[i];
    }
    if (j == 0) part[(long long)D * D] = is_x ? g : 0.f;
}

static int spkver_embed_check(const char* what, int B, int N, int C, int D, long long ld) {
    DV3_REQUIRE(B >= 1 && B <= (1 << 30), "%s: B=%d outside [1, 2^30]", what, B);
    DV3_REQUIRE(N >= 1 && N <= SV_MAX_N, "%s: N=%d outside [1, %d]", what, N, SV_MAX_N);
    DV3_REQUIRE(C >= 1 && C <= SV_MAX_C, "%s: C=%d outside [1, %d]", what, C, SV_MAX_C);
    DV3_REQUIRE(D >= 1 && D <= SV_MAX_D, "%s: D=%d outside [1, %d]", what, D, SV_MAX_D);
    DV3_REQUIRE(ld >= (long long)N * C, "%s: row stride %lld below N*C = %d", what, ld, N * C);
    return 0;
}

static int spkver_score_check(const char* what, int B_e, int B_t, int D) {
    DV3_REQUIRE(B_e >= 1 && B_t >= 1 && (long long)B_e + B_t <= (1LL << 30), "%s: B_e=%d, B_t=%d", what, B_e, B_t);
    DV3_REQUIRE(D >= 1 && D <= SV_MAX_D, "%s: D=%d outside [1, %d]", what, D, SV_MAX_D);
    DV3_REQUIRE((B_e + SV_TILE - 1) / SV_TILE <= 65535, "%s: B_e=%d past the tile grid", what, B_e);
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

long long dv3_spkver_loss_floats(int B_e, int B_t) { return (long long)B_e * ((B_t + SV_TILE - 1) / SV_TILE); }

int dv3_spkver_embed_fwd(const float* h, long long ld, const int* counts, const float* w, const float* c, float* hbar,
                         float* out, int* err_flag, int B, int N, int C, int D, void* stream) {
    if (spkver_embed_check("spkver_embed_fwd", B, N, C, D, ld)) return 1;
    DV3_REQUIRE(h && counts && w && c && hbar && out && err_flag, "spkver_embed_fwd: null operand");
    launch_k(spkver_embed_fwd_kernel, B, SV_THREADS, 0, (cudaStream_t)stream, h, ld, counts, w, c, hbar, out,
             err_flag, N, C, D);
    return check_launch("spkver_embed_fwd");
}

int dv3_spkver_embed_bwd(const float* d_out, const float* hbar, const int* counts, const float* w, float* d_h,
                         long long ld, float* partials, int* err_flag, int B, int N, int C, int D, void* stream) {
    if (spkver_embed_check("spkver_embed_bwd", B, N, C, D, ld)) return 1;
    DV3_REQUIRE(d_out && hbar && counts && w && d_h && partials && err_flag, "spkver_embed_bwd: null operand");
    launch_k(spkver_embed_bwd_kernel, B, SV_THREADS, 0, (cudaStream_t)stream, d_out, hbar, counts, w, d_h, ld,
             partials, err_flag, N, C, D);
    return check_launch("spkver_embed_bwd");
}

int dv3_spkver_score_fwd(const float* x, const float* y, const float* S, const float* bias, const long long* ids_e,
                         const long long* ids_t, float* qx, float* qy, float* scores, float* loss_partials, int B_e,
                         int B_t, int D, void* stream) {
    if (spkver_score_check("spkver_score_fwd", B_e, B_t, D)) return 1;
    DV3_REQUIRE(x && y && S && bias && qx && qy && scores, "spkver_score_fwd: null operand");
    DV3_REQUIRE((ids_e == nullptr) == (ids_t == nullptr) && (ids_e == nullptr) == (loss_partials == nullptr),
                "spkver_score_fwd: ids_e, ids_t and loss_partials go together");
    launch_k(spkver_quad_kernel, B_e + B_t, SV_MAX_D, 0, (cudaStream_t)stream, x, y, S, qx, qy, B_e, D);
    if (check_launch("spkver_quad")) return 1;
    const dim3 grid((B_t + SV_TILE - 1) / SV_TILE, (B_e + SV_TILE - 1) / SV_TILE);
    launch_k(spkver_score_fwd_kernel, grid, SV_THREADS, 0, (cudaStream_t)stream, x, y, qx, qy, bias, ids_e, ids_t,
             scores, loss_partials, B_e, B_t, D);
    return check_launch("spkver_score_fwd");
}

int dv3_spkver_score_bwd(const float* x, const float* y, const float* S, const float* scores, const long long* ids_e,
                         const long long* ids_t, const float* d_scores, const float* d_loss, float* dx, float* dy,
                         float* partials, int B_e, int B_t, int D, void* stream) {
    if (spkver_score_check("spkver_score_bwd", B_e, B_t, D)) return 1;
    DV3_REQUIRE(x && y && S && scores && dx && dy && partials, "spkver_score_bwd: null operand");
    DV3_REQUIRE((ids_e == nullptr) == (ids_t == nullptr), "spkver_score_bwd: ids_e and ids_t go together");
    launch_k(spkver_score_bwd_kernel, B_e + B_t, SV_MAX_D, 0, (cudaStream_t)stream, x, y, S, scores, ids_e, ids_t,
             d_scores, d_loss, dx, dy, partials, B_e, B_t, D);
    return check_launch("spkver_score_bwd");
}

}  // extern "C"
