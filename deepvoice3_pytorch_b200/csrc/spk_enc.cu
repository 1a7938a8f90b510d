// Speaker encoder (speaker_encoder.SpeakerEncoder, DESIGN.md section 2.13): the masked temporal mean of each cloning
// sample's features and the cloning-sample attention that turns B speakers x N samples of pooled features into B
// speaker embeddings, with the L1 loss against target rows fused in.
//
// Pool.  y[r,c] = (sum_{t < len[r]} x[r,c,t]) / len[r]: one warp per (r,c), lane l adds t = l, l+32, ... in order,
// then a fixed butterfly -- the order depends on len[r] alone (not on R, T or the other rows).  Backward: dx[r,c,t] =
// dy[r,c] / len[r] for t < len[r], 0 past it.  A length outside [1, T] sets *err_flag and yields 0.
//
// Attention, one CTA per speaker b, over its n = counts[b] <= N valid samples h_i (C):
//     q_i, k_i, v_i = W_{q,k,v} h_i + b_{q,k,v}                          (C x C each)
//     o_i[head]     = sum_{j<n} P[head,i,j] v_j[head],  P = softmax_j(q_i[head].k_j[head] / sqrt(C/heads))
//     s_i = w_s.o_i + b_s,  a = softmax_{i<n}(s),  e_i = W_e h_i + b_e   (S x C),  out = sum_{i<n} a_i e_i
// and, with a target, the per-row L1 partial sum_s |out[s] - target[s]|.  The backward CTA writes d(h) (rows >= n: 0)
// and one partial parameter-gradient row per speaker (layout: spkenc_param_offsets), which dv3_spkenc_reduce sums over
// the speakers in index order.  Every sum runs in a fixed order over i < n, j < n, c, d or s: a speaker's results
// depend on neither N nor the other speakers.  No atomics anywhere.
#include "common.cuh"

namespace dv3 {

constexpr int SE_THREADS = 256;
constexpr int SE_MAX_N = 32;
constexpr int SE_MAX_C = 256;
constexpr int SE_MAX_S = 64;
constexpr int SE_MAX_H = 8;

struct SeParams {
    const float *wq, *bq, *wk, *bk, *wv, *bv, *ws, *bs, *we, *be;
};

// per-speaker workspace: what the forward saves for the backward, and the backward's own scratch
struct SeWs {
    float *q, *k, *v, *o, *dq, *dk, *dv, *dO, *P, *dZ, *e, *a, *out;
};

__host__ __device__ inline long long se_ws_floats(int N, int C, int S, int H) {
    return 8LL * N * C + 2LL * H * N * N + (long long)N * S + N + S;
}

__device__ inline SeWs se_ws(float* base, int N, int C, int S, int H) {
    SeWs w;
    const long long nc = (long long)N * C, hnn = (long long)H * N * N;
    w.q = base; w.k = w.q + nc; w.v = w.k + nc; w.o = w.v + nc;
    w.dq = w.o + nc; w.dk = w.dq + nc; w.dv = w.dk + nc; w.dO = w.dv + nc;
    w.P = w.dO + nc; w.dZ = w.P + hnn; w.e = w.dZ + hnn; w.a = w.e + (long long)N * S;
    w.out = w.a + N;
    return w;
}

// offsets of the parameter gradients in a partial row (and in the reduced gradient)
struct SeOffsets {
    long long wq, wk, wv, bq, bk, bv, ws, bs, we, be, total;
};
__host__ __device__ inline SeOffsets spkenc_param_offsets(int C, int S) {
    SeOffsets o;
    const long long cc = (long long)C * C;
    o.wq = 0; o.wk = cc; o.wv = 2 * cc; o.bq = 3 * cc; o.bk = o.bq + C; o.bv = o.bk + C; o.ws = o.bv + C;
    o.bs = o.ws + C; o.we = o.bs + 1; o.be = o.we + (long long)S * C; o.total = o.be + S;
    return o;
}

// ---- pool ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SE_THREADS)
spkenc_pool_fwd_kernel(const float* __restrict__ x, const int* __restrict__ lengths, float* __restrict__ y,
                       int* __restrict__ err_flag, int R, int C, int T) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int lane = threadIdx.x & 31;
    const long long rc = (long long)blockIdx.x * (SE_THREADS / 32) + (threadIdx.x >> 5);
    if (rc >= (long long)R * C) return;
    const int len = lengths[rc / C];
    if (len < 1 || len > T) {
        if (lane == 0) { *err_flag = 1; y[rc] = 0.f; }
        return;
    }
    const float* row = x + rc * T;
    float acc = 0.f;
    for (int t = lane; t < len; t += 32) acc += row[t];
    acc = warp_sum(acc);
    if (lane == 0) y[rc] = acc / (float)len;
}

__global__ void __launch_bounds__(SE_THREADS)
spkenc_pool_bwd_kernel(const float* __restrict__ dy, const int* __restrict__ lengths, float* __restrict__ dx,
                       int* __restrict__ err_flag, int R, int C, int T) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const long long n = (long long)R * C * T;
    for (long long i = blockIdx.x * (long long)SE_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * SE_THREADS) {
        const long long rc = i / T;
        const int t = (int)(i - rc * T);
        const int len = lengths[rc / C];
        const bool ok = len >= 1 && len <= T;
        if (!ok && t == 0) *err_flag = 1;
        dx[i] = (ok && t < len) ? dy[rc] / (float)len : 0.f;
    }
}

// ---- attention forward --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SE_THREADS)
spkenc_attn_fwd_kernel(const float* __restrict__ h, const int* __restrict__ counts, SeParams pr,
                       const float* __restrict__ target, float* __restrict__ out, float* ws_all,
                       float* __restrict__ loss_part, int* __restrict__ err_flag, int N, int C, int S, int H) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sh[SE_MAX_N * SE_MAX_C];
    __shared__ float sc[SE_MAX_N];
    __shared__ float sa[SE_MAX_N];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = counts[b];
    if (n < 1 || n > N) {
        if (tid == 0) *err_flag = 1;
        for (int s = tid; s < S; s += SE_THREADS) out[(long long)b * S + s] = 0.f;
        if (tid == 0 && loss_part != nullptr) loss_part[b] = 0.f;
        return;
    }
    const SeWs w = se_ws(ws_all + (long long)b * se_ws_floats(N, C, S, H), N, C, S, H);
    const float* hb = h + (long long)b * N * C;
    for (int i = tid; i < n * C; i += SE_THREADS) sh[i] = hb[i];
    __syncthreads();

    // q, k, v: one thread per (matrix, output channel), all n rows at once
    for (int item = tid; item < 3 * C; item += SE_THREADS) {
        const int m = item / C, c = item % C;
        const float* W = m == 0 ? pr.wq : (m == 1 ? pr.wk : pr.wv);
        const float bias = (m == 0 ? pr.bq : (m == 1 ? pr.bk : pr.bv))[c];
        float* dst = m == 0 ? w.q : (m == 1 ? w.k : w.v);
        float acc[SE_MAX_N];
#pragma unroll
        for (int i = 0; i < SE_MAX_N; ++i) acc[i] = bias;
        for (int d = 0; d < C; ++d) {
            const float wv = W[(long long)c * C + d];
#pragma unroll
            for (int i = 0; i < SE_MAX_N; ++i)
                if (i < n) acc[i] = fmaf(wv, sh[i * C + d], acc[i]);
        }
#pragma unroll
        for (int i = 0; i < SE_MAX_N; ++i)
            if (i < N) dst[i * C + c] = i < n ? acc[i] : 0.f;
    }
    __syncthreads();

    // P = softmax over the valid keys, one thread per (head, query row)
    const int dh = C / H;
    const float scale = 1.f / sqrtf((float)dh);
    for (int item = tid; item < H * N; item += SE_THREADS) {
        const int hh = item / N, i = item % N;
        float* Pr = w.P + ((long long)hh * N + i) * N;
        if (i >= n) {
            for (int j = 0; j < N; ++j) Pr[j] = 0.f;
            continue;
        }
        const float* qi = w.q + i * C + hh * dh;
        float mx = -INFINITY;
        for (int j = 0; j < n; ++j) {
            const float* kj = w.k + j * C + hh * dh;
            float z = 0.f;
            for (int dd = 0; dd < dh; ++dd) z = fmaf(qi[dd], kj[dd], z);
            z *= scale;
            Pr[j] = z;
            mx = fmaxf(mx, z);
        }
        float sum = 0.f;
        for (int j = 0; j < n; ++j) {
            const float p = expf(Pr[j] - mx);
            Pr[j] = p;
            sum += p;
        }
        for (int j = 0; j < N; ++j) Pr[j] = j < n ? Pr[j] / sum : 0.f;
    }
    __syncthreads();

    // o = P v
    for (int item = tid; item < N * C; item += SE_THREADS) {
        const int i = item / C, c = item % C;
        float acc = 0.f;
        if (i < n) {
            const float* Pr = w.P + ((long long)(c / dh) * N + i) * N;
            for (int j = 0; j < n; ++j) acc = fmaf(Pr[j], w.v[j * C + c], acc);
        }
        w.o[item] = acc;
    }
    __syncthreads();

    // scores s_i = w_s.o_i + b_s, one warp per row
    const int lane = tid & 31, warp = tid >> 5;
    for (int i = warp; i < n; i += SE_THREADS / 32) {
        float acc = 0.f;
        for (int c = lane; c < C; c += 32) acc = fmaf(pr.ws[c], w.o[i * C + c], acc);
        acc = warp_sum(acc);
        if (lane == 0) sc[i] = acc + pr.bs[0];
    }
    // sample embeddings e_i = W_e h_i + b_e, one thread per (i, s)
    for (int item = tid; item < N * S; item += SE_THREADS) {
        const int i = item / S, s = item % S;
        float acc = 0.f;
        if (i < n) {
            acc = pr.be[s];
            for (int d = 0; d < C; ++d) acc = fmaf(pr.we[(long long)s * C + d], sh[i * C + d], acc);
        }
        w.e[item] = acc;
    }
    __syncthreads();
    if (tid == 0) {
        float mx = -INFINITY;
        for (int i = 0; i < n; ++i) mx = fmaxf(mx, sc[i]);
        float sum = 0.f;
        for (int i = 0; i < n; ++i) {
            sa[i] = expf(sc[i] - mx);
            sum += sa[i];
        }
        for (int i = 0; i < n; ++i) {
            sa[i] = sa[i] / sum;
            w.a[i] = sa[i];
        }
    }
    __syncthreads();
    for (int s = tid; s < S; s += SE_THREADS) {
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc = fmaf(sa[i], w.e[i * S + s], acc);
        out[(long long)b * S + s] = acc;
        w.out[s] = acc;
    }
    if (loss_part != nullptr) {
        __syncthreads();
        if (tid == 0) {
            float acc = 0.f;
            for (int s = 0; s < S; ++s) acc += fabsf(w.out[s] - target[(long long)b * S + s]);
            loss_part[b] = acc;
        }
    }
}

// ---- attention backward -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SE_THREADS)
spkenc_attn_bwd_kernel(const float* __restrict__ h, const int* __restrict__ counts, SeParams pr,
                       const float* __restrict__ target, const float* __restrict__ d_out,
                       const float* __restrict__ d_loss, float loss_scale, float* ws_all, float* __restrict__ d_h,
                       float* __restrict__ partials, int* __restrict__ err_flag, int N, int C, int S, int H) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sh[SE_MAX_N * SE_MAX_C];
    __shared__ float shbar[SE_MAX_C];
    __shared__ float sdout[SE_MAX_S];
    __shared__ float sa[SE_MAX_N], sda[SE_MAX_N], sds[SE_MAX_N];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = counts[b];
    const SeOffsets off = spkenc_param_offsets(C, S);
    float* part = partials + (long long)b * off.total;
    float* dhb = d_h + (long long)b * N * C;
    if (n < 1 || n > N) {
        if (tid == 0) *err_flag = 1;
        for (long long i = tid; i < off.total; i += SE_THREADS) part[i] = 0.f;
        for (int i = tid; i < N * C; i += SE_THREADS) dhb[i] = 0.f;
        return;
    }
    const SeWs w = se_ws(ws_all + (long long)b * se_ws_floats(N, C, S, H), N, C, S, H);
    const float* hb = h + (long long)b * N * C;
    for (int i = tid; i < n * C; i += SE_THREADS) sh[i] = hb[i];
    // d(out) = the incoming gradient + d(loss) * loss_scale * sign(out - target)
    for (int s = tid; s < S; s += SE_THREADS) {
        float g = d_out != nullptr ? d_out[(long long)b * S + s] : 0.f;
        if (target != nullptr && d_loss != nullptr) {
            const float diff = w.out[s] - target[(long long)b * S + s];
            const float sg = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
            g += d_loss[0] * loss_scale * sg;
        }
        sdout[s] = g;
    }
    for (int i = tid; i < n; i += SE_THREADS) sa[i] = w.a[i];
    __syncthreads();
    // d a_i = e_i . d(out);  hbar = sum_i a_i h_i (dW_e = d(out) hbar^T)
    for (int i = tid; i < n; i += SE_THREADS) {
        float acc = 0.f;
        for (int s = 0; s < S; ++s) acc = fmaf(w.e[i * S + s], sdout[s], acc);
        sda[i] = acc;
    }
    for (int d = tid; d < C; d += SE_THREADS) {
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc = fmaf(sa[i], sh[i * C + d], acc);
        shbar[d] = acc;
    }
    __syncthreads();
    if (tid == 0) {
        float dot = 0.f;
        for (int i = 0; i < n; ++i) dot = fmaf(sa[i], sda[i], dot);
        float dbs = 0.f;
        for (int i = 0; i < n; ++i) {
            sds[i] = sa[i] * (sda[i] - dot);
            dbs += sds[i];
        }
        part[off.bs] = dbs;
    }
    __syncthreads();
    // d o_i = ds_i w_s;  d w_s = sum_i ds_i o_i;  d W_e, d b_e
    for (int item = tid; item < N * C; item += SE_THREADS) {
        const int i = item / C, c = item % C;
        w.dO[item] = i < n ? sds[i] * pr.ws[c] : 0.f;
    }
    for (int c = tid; c < C; c += SE_THREADS) {
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc = fmaf(sds[i], w.o[i * C + c], acc);
        part[off.ws + c] = acc;
    }
    for (int item = tid; item < S * C; item += SE_THREADS) {
        const int s = item / C, d = item % C;
        part[off.we + item] = sdout[s] * shbar[d];
    }
    for (int s = tid; s < S; s += SE_THREADS) {
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc = fmaf(sa[i], sdout[s], acc);
        part[off.be + s] = acc;
    }
    __syncthreads();
    // dZ = P (dP - rowsum(P dP)), dP[head,i,j] = dO_i[head].v_j[head]; one thread per (head, query row)
    const int dh = C / H;
    const float scale = 1.f / sqrtf((float)dh);
    for (int item = tid; item < H * n; item += SE_THREADS) {
        const int hh = item / n, i = item % n;
        const float* Pr = w.P + ((long long)hh * N + i) * N;
        float* Zr = w.dZ + ((long long)hh * N + i) * N;
        const float* doi = w.dO + i * C + hh * dh;
        float rs = 0.f;
        for (int j = 0; j < n; ++j) {
            const float* vj = w.v + j * C + hh * dh;
            float dp = 0.f;
            for (int dd = 0; dd < dh; ++dd) dp = fmaf(doi[dd], vj[dd], dp);
            Zr[j] = dp;
            rs = fmaf(Pr[j], dp, rs);
        }
        for (int j = 0; j < n; ++j) Zr[j] = Pr[j] * (Zr[j] - rs);
    }
    __syncthreads();
    // d q, d k, d v (rows >= n: 0)
    for (int item = tid; item < N * C; item += SE_THREADS) {
        const int i = item / C, c = item % C, hh = c / dh;
        float gq = 0.f, gk = 0.f, gv = 0.f;
        if (i < n) {
            const float* Pc = w.P + (long long)hh * N * N;
            const float* Zc = w.dZ + (long long)hh * N * N;
            for (int j = 0; j < n; ++j) {
                gv = fmaf(Pc[j * N + i], w.dO[j * C + c], gv);
                gq = fmaf(Zc[i * N + j], w.k[j * C + c], gq);
                gk = fmaf(Zc[j * N + i], w.q[j * C + c], gk);
            }
            gq *= scale;
            gk *= scale;
        }
        w.dq[item] = gq;
        w.dk[item] = gk;
        w.dv[item] = gv;
    }
    __syncthreads();
    // partial dW_{q,k,v}[c,d] = sum_i d{q,k,v}_i[c] h_i[d], d b = sum_i d{q,k,v}_i
    const long long cc = (long long)C * C;
    for (long long item = tid; item < 3 * cc; item += SE_THREADS) {
        const int m = (int)(item / cc);
        const int c = (int)((item % cc) / C), d = (int)(item % C);
        const float* G = m == 0 ? w.dq : (m == 1 ? w.dk : w.dv);
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc = fmaf(G[i * C + c], sh[i * C + d], acc);
        part[item] = acc;           // wq, wk, wv are the first 3 C^2 floats of the row
    }
    for (int item = tid; item < 3 * C; item += SE_THREADS) {
        const int m = item / C, c = item % C;
        const float* G = m == 0 ? w.dq : (m == 1 ? w.dk : w.dv);
        float acc = 0.f;
        for (int i = 0; i < n; ++i) acc += G[i * C + c];
        part[off.bq + item] = acc;  // bq, bk, bv follow one another
    }
    // d h_i[d] = sum_c (W_q[c,d] dq_i[c] + W_k[c,d] dk_i[c] + W_v[c,d] dv_i[c]) + sum_s W_e[s,d] a_i d(out)[s]
    for (int d = tid; d < C; d += SE_THREADS) {
        float acc[SE_MAX_N];
#pragma unroll
        for (int i = 0; i < SE_MAX_N; ++i) acc[i] = 0.f;
        for (int c = 0; c < C; ++c) {
            const float a = pr.wq[(long long)c * C + d], bk = pr.wk[(long long)c * C + d],
                        bv = pr.wv[(long long)c * C + d];
#pragma unroll
            for (int i = 0; i < SE_MAX_N; ++i)
                if (i < n) {
                    acc[i] = fmaf(a, w.dq[i * C + c], acc[i]);
                    acc[i] = fmaf(bk, w.dk[i * C + c], acc[i]);
                    acc[i] = fmaf(bv, w.dv[i * C + c], acc[i]);
                }
        }
        for (int s = 0; s < S; ++s) {
            const float we = pr.we[(long long)s * C + d], g = sdout[s];
#pragma unroll
            for (int i = 0; i < SE_MAX_N; ++i)
                if (i < n) acc[i] = fmaf(we, sa[i] * g, acc[i]);
        }
#pragma unroll
        for (int i = 0; i < SE_MAX_N; ++i)
            if (i < N) dhb[i * C + d] = i < n ? acc[i] : 0.f;
    }
}

// grad[p] = sum_{b < B} partials[b*P + p] in index order; loss[0] = loss_scale * sum_b loss_partials[b] in order
__global__ void __launch_bounds__(SE_THREADS)
spkenc_reduce_kernel(const float* __restrict__ partials, long long P, const float* __restrict__ loss_partials,
                     float loss_scale, float* __restrict__ grad, float* __restrict__ loss, int B) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const long long p = blockIdx.x * (long long)SE_THREADS + threadIdx.x;
    if (partials != nullptr && p < P) {
        float acc = 0.f;
        for (int b = 0; b < B; ++b) acc += partials[(long long)b * P + p];
        grad[p] = acc;
    }
    if (loss != nullptr && p == 0) {
        float acc = 0.f;
        for (int b = 0; b < B; ++b) acc += loss_partials[b];
        loss[0] = acc * loss_scale;
    }
}

static int spkenc_check(const char* what, int B, int N, int C, int S, int H) {
    DV3_REQUIRE(B >= 1 && B <= 65535, "%s: B=%d outside [1, 65535]", what, B);
    DV3_REQUIRE(N >= 1 && N <= SE_MAX_N, "%s: N=%d outside [1, %d]", what, N, SE_MAX_N);
    DV3_REQUIRE(C >= 1 && C <= SE_MAX_C, "%s: C=%d outside [1, %d]", what, C, SE_MAX_C);
    DV3_REQUIRE(S >= 1 && S <= SE_MAX_S, "%s: S=%d outside [1, %d]", what, S, SE_MAX_S);
    DV3_REQUIRE(H >= 1 && H <= SE_MAX_H && C % H == 0, "%s: heads=%d must divide C=%d and be <= %d", what, H, C,
                SE_MAX_H);
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

long long dv3_spkenc_ws_floats(int N, int C, int S, int heads) { return se_ws_floats(N, C, S, heads); }

long long dv3_spkenc_param_floats(int C, int S) { return spkenc_param_offsets(C, S).total; }

int dv3_spkenc_pool_fwd(const float* x, const int* lengths, float* y, int* err_flag, int R, int C, int T,
                        void* stream) {
    DV3_REQUIRE(x && lengths && y && err_flag, "spkenc_pool_fwd: null operand");
    DV3_REQUIRE(R > 0 && C > 0 && T > 0 && (long long)R * C * T < (1LL << 40), "spkenc_pool_fwd: bad shape");
    const long long warps = (long long)R * C, per = SE_THREADS / 32;
    DV3_REQUIRE((warps + per - 1) / per < (1LL << 31), "spkenc_pool_fwd: R*C too large");
    launch_k(spkenc_pool_fwd_kernel, (unsigned)((warps + per - 1) / per), SE_THREADS, 0, (cudaStream_t)stream, x,
             lengths, y, err_flag, R, C, T);
    return check_launch("spkenc_pool_fwd");
}

int dv3_spkenc_pool_bwd(const float* dy, const int* lengths, float* dx, int* err_flag, int R, int C, int T,
                        void* stream) {
    DV3_REQUIRE(dy && lengths && dx && err_flag, "spkenc_pool_bwd: null operand");
    DV3_REQUIRE(R > 0 && C > 0 && T > 0 && (long long)R * C * T < (1LL << 40), "spkenc_pool_bwd: bad shape");
    const long long n = (long long)R * C * T;
    const long long blocks = (n + SE_THREADS - 1) / SE_THREADS;
    launch_k(spkenc_pool_bwd_kernel, (unsigned)(blocks < 8192 ? blocks : 8192), SE_THREADS, 0, (cudaStream_t)stream,
             dy, lengths, dx, err_flag, R, C, T);
    return check_launch("spkenc_pool_bwd");
}

int dv3_spkenc_attn_fwd(const float* h, const int* counts, const float* w_q, const float* b_q, const float* w_k,
                        const float* b_k, const float* w_v, const float* b_v, const float* w_s, const float* b_s,
                        const float* w_e, const float* b_e, const float* target, float* out, float* ws,
                        float* loss_partials, int* err_flag, int B, int N, int C, int S, int heads, void* stream) {
    if (spkenc_check("spkenc_attn_fwd", B, N, C, S, heads)) return 1;
    DV3_REQUIRE(h && counts && w_q && b_q && w_k && b_k && w_v && b_v && w_s && b_s && w_e && b_e && out && ws &&
                err_flag, "spkenc_attn_fwd: null operand");
    DV3_REQUIRE((target == nullptr) == (loss_partials == nullptr),
                "spkenc_attn_fwd: target and loss_partials go together");
    const SeParams pr = {w_q, b_q, w_k, b_k, w_v, b_v, w_s, b_s, w_e, b_e};
    launch_k(spkenc_attn_fwd_kernel, B, SE_THREADS, 0, (cudaStream_t)stream, h, counts, pr, target, out, ws,
             loss_partials, err_flag, N, C, S, heads);
    return check_launch("spkenc_attn_fwd");
}

int dv3_spkenc_attn_bwd(const float* h, const int* counts, const float* w_q, const float* b_q, const float* w_k,
                        const float* b_k, const float* w_v, const float* b_v, const float* w_s, const float* b_s,
                        const float* w_e, const float* b_e, const float* target, const float* d_out,
                        const float* d_loss, float loss_scale, float* ws, float* d_h, float* partials,
                        int* err_flag, int B, int N, int C, int S, int heads, void* stream) {
    if (spkenc_check("spkenc_attn_bwd", B, N, C, S, heads)) return 1;
    DV3_REQUIRE(h && counts && w_q && b_q && w_k && b_k && w_v && b_v && w_s && b_s && w_e && b_e && ws && d_h &&
                partials && err_flag, "spkenc_attn_bwd: null operand");
    const SeParams pr = {w_q, b_q, w_k, b_k, w_v, b_v, w_s, b_s, w_e, b_e};
    launch_k(spkenc_attn_bwd_kernel, B, SE_THREADS, 0, (cudaStream_t)stream, h, counts, pr, target, d_out, d_loss,
             loss_scale, ws, d_h, partials, err_flag, N, C, S, heads);
    return check_launch("spkenc_attn_bwd");
}

int dv3_spkenc_reduce(const float* partials, long long P, const float* loss_partials, float loss_scale, float* grad,
                      float* loss, int B, void* stream) {
    DV3_REQUIRE(B >= 1, "spkenc_reduce: B=%d", B);
    DV3_REQUIRE(partials == nullptr || (grad != nullptr && P > 0), "spkenc_reduce: partials without a gradient");
    DV3_REQUIRE(loss == nullptr || loss_partials != nullptr, "spkenc_reduce: loss without loss partials");
    const long long n = partials != nullptr ? P : 1;
    launch_k(spkenc_reduce_kernel, (unsigned)((n + SE_THREADS - 1) / SE_THREADS), SE_THREADS, 0,
             (cudaStream_t)stream, partials, P, loss_partials, loss_scale, grad, loss, B);
    return check_launch("spkenc_reduce");
}

}  // extern "C"
