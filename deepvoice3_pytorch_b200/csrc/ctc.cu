// CTC loss, its gradient, greedy CTC decoding and batched edit distance for the token recognizer (recognition.py,
// DESIGN.md section 2.21).
//
// Logits z (B, V, T) as the recognizer's final 1x1 conv writes them: z[b*stride_b + v*stride_v + t].  Class 0 is the
// CTC blank (and the TTS padding id); targets are ids in [1, V).  Row b has T_b frames and L_b target tokens; frames
// t >= T_b are never read.  The extended label sequence l' has S_b = 2 L_b + 1 states: blanks at even s, label k at
// s = 2k + 1.
//
// Forward.  ctc_lse_kernel: per (b, t) the fp64 log-sum-exp lse[b, t] of z over V (one CTA per 32 frames of a row, 8
// class groups of 32 frames each summed in v order, then the groups in order).  ctc_alpha_kernel: one CTA per row.
// Thread k owns states 2k + 1 (label k) and 2k + 2 (the blank after it); thread 0 also owns state 0.  So a row takes
// max(L_b, 1) threads, at most 1024.  Per frame, in fp64 with e_t(s) = z[l'_s, t] - lse[t]:
//   alpha_t(s) = e_t(s) + logsumexp(alpha_{t-1}(s), alpha_{t-1}(s-1), alpha_{t-1}(s-2) if l'_s != l'_{s-2} != blank).
// alpha_{t-1}(2k) and alpha_{t-1}(2k-1) come from thread k-1 by __shfl_up_sync, or for lane 0 from lane 31 of the
// warp before through a double-buffered shared slot (the layout of align.cu); one named barrier per frame over the
// row's own warps.  Every alpha is stored in the workspace for the backward.  Each frame's operands are loaded into
// registers one frame ahead.  log p = logsumexp(alpha_{T-1}(S-1), alpha_{T-1}(S-2)); nll[b] = -log p and
// partials[b] = -log p / max(L_b, 1).  A row with no feasible path (T_b < L_b + repeated adjacent labels) gets
// nll = partial = 0 and infeasible[b] = 1 (torch's zero_infinity); so does a row whose log p is -inf.
//
// Backward.  One CTA per row of roundup(max(L_b, V), 32) live threads; thread k owns the states of the forward and
// thread v owns class v.  With beta_t(s) the log-sum over the path suffixes after frame t, walking t = T_b - 1 .. 0:
//   beta_t(s) = logsumexp(q_{t+1}(s), q_{t+1}(s+1), q_{t+1}(s+2) if l'_{s+2} != blank, l'_s),  q_t(s) = beta_t(s) + e_t(s)
// (the neighbour's q by __shfl_down_sync and the shared slot), then gamma_t(s) = exp(alpha_t(s) + beta_t(s) - log p)
// and, after the frame's one barrier,
//   dz[b, v, t] = w_b (exp(z[v, t] - lse[t]) - sum_{s: l'_s = v} gamma_t(s)),  w_b = d_loss[0] scale / max(L_b, 1).
// Class v walks its target positions in index order: a per-row list of positions sorted stably by label, built in
// shared memory from the targets (rank of k = #{j: l_j < l_k} + #{j < k: l_j = l_k}).  The blank's sum runs over the
// even states as a fixed butterfly within each warp, then the warps in order.  dz = 0 for t >= T_b and for the whole
// row when the forward flagged it.
//
// Greedy decoding.  ctc_argmax_kernel: per (b, t < T_b) the first class of largest logit (NaN never wins), written to
// hyps[b, t].  ctc_collapse_kernel: one warp per row compacts hyps[b] in place, in chunks of 32 frames: keep a frame
// whose class is not the blank and differs from the frame before (__ballot_sync, then the rank among kept lanes).
//
// Edit distance.  One warp per (hypothesis, reference) pair, the systolic array of dtw.cuh: lane l owns reference row
// i = i0 + l + 1 of a strip of 32 rows and at step s computes hypothesis column j = s - l + 1; D(i-1, j) arrives from
// lane l-1 by __shfl_up_sync, D(i-1, j-1) is the value that arrived one step earlier, D(i, j-1) is the lane's own last
// value; lane 0 reads row i0 from a per-pair boundary buffer in global memory that lane 31 of the strip above wrote.
//   D(i, j) = min(D(i-1, j-1) + [r_i != h_j], D(i-1, j) + 1, D(i, j-1) + 1)
// with ties to the diagonal (match or substitution), then the deletion (i-1, j) (a reference token the hypothesis
// lacks), then the insertion (i, j-1).  The substitution and deletion counts ride along with the chosen predecessor,
// packed S | D << 16 in one int beside the cost; insertions are cost - S - D.  Integer arithmetic: exact.
//
// No atomics anywhere and every sum has a fixed order: a row's (a pair's) bits depend on its own data and lengths.
// An out-of-range length or target id sets *err_flag; the row is then left out (zero loss and gradient, empty
// hypothesis, zero counts) and the value is never used as an index.
#include "common.cuh"

namespace dv3 {

constexpr int CTC_MAX_VOCAB = 1024;
constexpr int CTC_MAX_TARGET = 1024;         // one thread per label state pair: the largest max_positions
constexpr int CTC_MAX_HYP = 65535;
constexpr int CTC_LSE_GROUPS = 8;            // class groups of ctc_lse_kernel / ctc_argmax_kernel
constexpr int CTC_COLLAPSE_WARPS = 4;
constexpr int CTC_PAIRS = 2;                 // target positions per thread of the alpha and beta kernels
constexpr int CTC_THREADS = CTC_MAX_TARGET / CTC_PAIRS;

// threads that own the states of a row of L_b target tokens
__host__ __device__ __forceinline__ int ctc_row_threads(int Lb) { return (max(Lb, 1) + CTC_PAIRS - 1) / CTC_PAIRS; }

enum { CTC_OK = 0, CTC_INFEASIBLE = 1, CTC_INVALID = 2 };

// workspace: lse (B*T doubles), log p (B doubles), status (B long longs), alpha (B*T*(2L+1) doubles)
static inline long long ctc_ws_doubles(int B, int T, int L) {
    return (long long)B * T + 2LL * B + (long long)B * T * (2LL * L + 1);
}

__device__ __forceinline__ double neg_inf() { return __longlong_as_double(0xfff0000000000000LL); }

__device__ __forceinline__ double lse2(double a, double b) {
    const double m = fmax(a, b);
    if (m == neg_inf()) return m;
    return m + log(exp(a - m) + exp(b - m));
}
__device__ __forceinline__ double lse3(double a, double b, double c) {
    const double m = fmax(fmax(a, b), c);
    if (m == neg_inf()) return m;
    return m + log(exp(a - m) + exp(b - m) + exp(c - m));
}

// 1 / max(n, 1) for a count n <= 1024: the fp32 reciprocal refined by two Newton steps in fp64 (no division
// subroutine, whose call would cap the register budget)
__device__ __forceinline__ double inv_count(int n) {
    const double d = (double)max(n, 1);
    double r = (double)__frcp_rn((float)d);
    r = fma(r, fma(-d, r, 1.0), r);
    return fma(r, fma(-d, r, 1.0), r);
}

__device__ __forceinline__ void named_barrier(int nthr) { asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory"); }

// ---- per-frame log-sum-exp ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * CTC_LSE_GROUPS)
ctc_lse_kernel(const float* __restrict__ z, long long sb, long long sv, const int* __restrict__ frames, int T, int V,
               double* __restrict__ lse) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float s_m[CTC_LSE_GROUPS][32];
    __shared__ double s_s[CTC_LSE_GROUPS][32];
    const int b = blockIdx.y, lane = threadIdx.x & 31, g = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + lane;
    const int Tb = frames[b];
    const bool on = Tb >= 1 && Tb <= T && t < Tb;
    const float* zt = z + b * sb + t;
    float m = -INFINITY;
    if (on)
#pragma unroll 1
        for (int v = g; v < V; v += CTC_LSE_GROUPS) m = fmaxf(m, zt[v * sv]);
    s_m[g][lane] = m;
    __syncthreads();
    m = s_m[0][lane];
#pragma unroll
    for (int q = 1; q < CTC_LSE_GROUPS; ++q) m = fmaxf(m, s_m[q][lane]);
    double s = 0.0;
    if (on)
#pragma unroll 1
        for (int v = g; v < V; v += CTC_LSE_GROUPS) s += exp((double)zt[v * sv] - (double)m);
    s_s[g][lane] = s;
    __syncthreads();
    if (g == 0 && on) {
        double tot = s_s[0][lane];
#pragma unroll
        for (int q = 1; q < CTC_LSE_GROUPS; ++q) tot += s_s[q][lane];
        lse[(long long)b * T + t] = (double)m + log(tot);
    }
}

// ---- alpha recursion ----------------------------------------------------------------------------------------------
// Thread k owns target positions m = 2k + j, j < CTC_PAIRS: states 2m + 1 (label m) and 2m + 2 (the blank after it);
// thread 0 also owns state 0.
__global__ void __launch_bounds__(CTC_THREADS, 1)
ctc_alpha_kernel(const float* __restrict__ z, long long sb, long long sv, const int* __restrict__ frames,
                 const int* __restrict__ targets, long long ld, const int* __restrict__ tlen, int T, int V, int L,
                 double* __restrict__ ws, float* __restrict__ nll, float* __restrict__ partials,
                 int* __restrict__ infeasible, int* __restrict__ err_flag, int B) {
    pdl_trigger(); pdl_wait();
    __shared__ double edge[2][32][2];                 // lane 31 of each warp: alpha of its last (label, blank)
    const int b = blockIdx.x, k = threadIdx.x, lane = k & 31, warp = k >> 5;
    const long long S = 2LL * L + 1;
    double* lse = ws;
    double* logp = ws + (long long)B * T;
    long long* status = reinterpret_cast<long long*>(logp + B);
    double* alpha = reinterpret_cast<double*>(status + B) + (long long)b * T * S;
    const int Tb = frames[b];
    int Lb = tlen[b];
    const bool len_ok = Tb >= 1 && Tb <= T && Lb >= 0 && Lb <= L;
    if (!len_ok) Lb = 0;
    bool hasl[CTC_PAIRS], skip[CTC_PAIRS];
    int lab[CTC_PAIRS];
    int badl = 0, rep = 0;
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j) {
        const int m = CTC_PAIRS * k + j;
        hasl[j] = m < Lb;
        lab[j] = hasl[j] ? targets[b * ld + m] : 0;
        const int prv = hasl[j] && m > 0 ? targets[b * ld + m - 1] : -1;
        badl |= hasl[j] && (lab[j] < 1 || lab[j] >= V);
        rep += hasl[j] && m > 0 && lab[j] == prv;
        skip[j] = hasl[j] && m > 0 && lab[j] != prv;
    }
    const int bad = __syncthreads_or(!len_ok || badl);
    const int reps = __syncthreads_count(rep > 0) + __syncthreads_count(rep > 1);
    if (bad || Tb < Lb + reps) {
        if (k == 0) {
            if (bad) *err_flag = 1;
            nll[b] = 0.f;
            partials[b] = 0.f;
            infeasible[b] = 1;
            status[b] = bad ? CTC_INVALID : CTC_INFEASIBLE;
        }
        return;
    }
    const int nw = (ctc_row_threads(Lb) + 31) >> 5;
    if (warp >= nw) return;
    const int nthr = nw * 32;
    const float* zb = z + b * sb;
    const float* zl[CTC_PAIRS];
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j) zl[j] = zb + (long long)lab[j] * sv;
    const double* lse_b = lse + (long long)b * T;
    const double NEG = neg_inf();
    // frame 0: alpha_0(0) = e(blank), alpha_0(1) = e(label 0)
    double l_t = lse_b[0];
    const double eb0 = (double)zb[0] - l_t;
    double a0 = k == 0 ? eb0 : NEG;
    double aL[CTC_PAIRS], aB[CTC_PAIRS];
    float nzl[CTC_PAIRS];
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j) {
        aL[j] = k == 0 && j == 0 && hasl[0] ? (double)zl[0][0] - l_t : NEG;
        aB[j] = NEG;
        nzl[j] = Tb > 1 ? zl[j][1] : 0.f;
    }
    float nzb = Tb > 1 ? zb[1] : 0.f;
    double nl = Tb > 1 ? lse_b[1] : 0.0;
    if (k == 0) alpha[0] = a0;
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j)
        if (hasl[j]) { const int m = CTC_PAIRS * k + j; alpha[2 * m + 1] = aL[j]; alpha[2 * m + 2] = aB[j]; }
    if (lane == 31) { edge[0][warp][0] = aL[CTC_PAIRS - 1]; edge[0][warp][1] = aB[CTC_PAIRS - 1]; }
    named_barrier(nthr);
    for (int t = 1; t < Tb; ++t) {
        l_t = nl;
        const double eb = (double)nzb - l_t;
        double el[CTC_PAIRS];
#pragma unroll
        for (int j = 0; j < CTC_PAIRS; ++j) el[j] = (double)nzl[j] - l_t;
        if (t + 1 < Tb) {
            nzb = zb[t + 1];
            nl = lse_b[t + 1];
#pragma unroll
            for (int j = 0; j < CTC_PAIRS; ++j) nzl[j] = zl[j][t + 1];
        }
        const int buf = t & 1;
        double pL = __shfl_up_sync(0xffffffffu, aL[CTC_PAIRS - 1], 1);     // alpha_{t-1}(2m - 1), m = 2k
        double pB = __shfl_up_sync(0xffffffffu, aB[CTC_PAIRS - 1], 1);     // alpha_{t-1}(2m)
        if (lane == 0) {
            if (warp > 0) { pL = edge[buf ^ 1][warp - 1][0]; pB = edge[buf ^ 1][warp - 1][1]; }
            else { pL = NEG; pB = a0; }
        }
        double nL[CTC_PAIRS], nB[CTC_PAIRS];
#pragma unroll
        for (int j = 0; j < CTC_PAIRS; ++j) {
            const double qL = j == 0 ? pL : aL[j - 1], qB = j == 0 ? pB : aB[j - 1];
            nL[j] = hasl[j] ? el[j] + lse3(aL[j], qB, skip[j] ? qL : NEG) : NEG;
            nB[j] = hasl[j] ? eb + lse2(aB[j], aL[j]) : NEG;
        }
        if (k == 0) a0 = eb + a0;
        double* at = alpha + (long long)t * S;
        if (k == 0) at[0] = a0;
#pragma unroll
        for (int j = 0; j < CTC_PAIRS; ++j) {
            aL[j] = nL[j];
            aB[j] = nB[j];
            if (hasl[j]) { const int m = CTC_PAIRS * k + j; at[2 * m + 1] = aL[j]; at[2 * m + 2] = aB[j]; }
        }
        if (lane == 31) { edge[buf][warp][0] = aL[CTC_PAIRS - 1]; edge[buf][warp][1] = aB[CTC_PAIRS - 1]; }
        named_barrier(nthr);
    }
    const int last = max(Lb, 1) - 1;                  // the thread and pair that own the final states
    if (k == last / CTC_PAIRS) {
        const int j = last % CTC_PAIRS;
        const double lp = Lb == 0 ? a0 : lse2(j == 0 ? aL[0] : aL[CTC_PAIRS - 1], j == 0 ? aB[0] : aB[CTC_PAIRS - 1]);
        const bool fin = lp > NEG;
        logp[b] = lp;
        status[b] = fin ? CTC_OK : CTC_INFEASIBLE;
        nll[b] = fin ? (float)(-lp) : 0.f;
        partials[b] = fin ? (float)(-lp * inv_count(Lb)) : 0.f;
        infeasible[b] = fin ? 0 : 1;
    }
}

// ---- beta recursion fused with the gradient -----------------------------------------------------------------------
__global__ void __launch_bounds__(CTC_THREADS, 1)
ctc_beta_grad_kernel(const float* __restrict__ z, long long sb, long long sv, const int* __restrict__ frames,
                     const int* __restrict__ targets, long long ld, const int* __restrict__ tlen, int T, int V, int L,
                     const double* __restrict__ ws, const float* __restrict__ d_loss, float scale,
                     float* __restrict__ dz, int B) {
    pdl_trigger(); pdl_wait();
    __shared__ int s_lab[CTC_MAX_TARGET];
    __shared__ int s_pos[CTC_MAX_TARGET];
    __shared__ int s_start[CTC_MAX_VOCAB + 1];
    __shared__ double s_gam[2][CTC_MAX_TARGET];       // gamma of the label states, by target position
    __shared__ double s_bsum[2][CTC_THREADS / 32];    // each warp's blank gamma
    __shared__ double s_edge[2][CTC_THREADS / 32];    // q of each warp's lane 0 first label state
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long S = 2LL * L + 1;
    const double* lse_b = ws + (long long)b * T;
    const double lp = ws[(long long)B * T + b];
    const long long st = reinterpret_cast<const long long*>(ws + (long long)B * T + B)[b];
    const double* alpha = ws + (long long)B * T + 2LL * B + (long long)b * T * S;
    float* dzb = dz + (long long)b * V * T;
    int Tb = frames[b];
    const int Lb = st == CTC_OK ? tlen[b] : 0;
    if (st != CTC_OK) Tb = 0;                         // the status covers out-of-range lengths too
    // frames t >= T_b (every frame of a flagged row): zero
    const int tail = T - Tb;
    for (long long i = tid; i < (long long)V * tail; i += blockDim.x) {
        const int v = (int)(i / tail), t = Tb + (int)(i - (long long)v * tail);
        dzb[(long long)v * T + t] = 0.f;
    }
    if (Tb == 0) return;
    const int nw = (max(ctc_row_threads(Lb), min(V, CTC_THREADS)) + 31) >> 5;
    if (warp >= nw) return;
    const int nthr = nw * 32;
    const int nws = (ctc_row_threads(Lb) + 31) >> 5;  // warps that own states
    // stable sort of the target positions by label
    for (int m = tid; m < Lb; m += nthr) s_lab[m] = targets[b * ld + m];
    named_barrier(nthr);
    for (int m = tid; m < Lb; m += nthr) {
        const int lm = s_lab[m];
        int r = 0;
        for (int j = 0; j < Lb; ++j) {
            const int lj = s_lab[j];
            r += lj < lm || (lj == lm && j < m);
        }
        s_pos[r] = m;
    }
    for (int v = tid; v <= V; v += nthr) {
        int c = 0;
        for (int j = 0; j < Lb; ++j) c += s_lab[j] < v;
        s_start[v] = c;
    }
    bool hasl[CTC_PAIRS], nskip[CTC_PAIRS], nlab[CTC_PAIRS];
    int lab[CTC_PAIRS];
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j) {
        const int m = CTC_PAIRS * tid + j;
        hasl[j] = m < Lb;
        lab[j] = hasl[j] ? s_lab[m] : 0;
        nlab[j] = m + 1 < Lb;                         // label m -> label m + 1
        nskip[j] = nlab[j] && s_lab[m + 1] != lab[j];
    }
    named_barrier(nthr);
    const double wgt = (double)d_loss[0] * (double)scale * inv_count(Lb);
    const float* zb = z + b * sb;
    const float* zl[CTC_PAIRS];
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j) zl[j] = zb + (long long)lab[j] * sv;
    const double NEG = neg_inf();
    // z and lse one frame ahead; alpha of the frame at its top, ahead of the frame's beta
    int t = Tb - 1;
    double l_t = lse_b[t];
    float cz_b = zb[t], cz_l[CTC_PAIRS];
    double bL[CTC_PAIRS], bB[CTC_PAIRS], qL[CTC_PAIRS], qB[CTC_PAIRS];
    const int last = max(Lb, 1) - 1;
#pragma unroll
    for (int j = 0; j < CTC_PAIRS; ++j) {
        cz_l[j] = zl[j][t];
        bL[j] = bB[j] = Lb > 0 && CTC_PAIRS * tid + j == last ? 0.0 : NEG;
        qL[j] = qB[j] = NEG;
    }
    double b0 = Lb == 0 && tid == 0 ? 0.0 : NEG, q0 = NEG;
    for (; t >= 0; --t) {
        const double* at = alpha + (long long)t * S;
        const double A0 = tid == 0 ? at[0] : NEG;
        double AL[CTC_PAIRS], AB[CTC_PAIRS];
        float z_l[CTC_PAIRS];
#pragma unroll
        for (int j = 0; j < CTC_PAIRS; ++j) {
            const int m = CTC_PAIRS * tid + j;
            AL[j] = hasl[j] ? at[2 * m + 1] : NEG;
            AB[j] = hasl[j] ? at[2 * m + 2] : NEG;
            z_l[j] = cz_l[j];
        }
        const double l_c = l_t;
        const float z_b = cz_b;
        if (t > 0) {
            l_t = lse_b[t - 1];
            cz_b = zb[t - 1];
#pragma unroll
            for (int j = 0; j < CTC_PAIRS; ++j) cz_l[j] = zl[j][t - 1];
        }
        const int buf = t & 1;
        if (t < Tb - 1) {
            double qn = __shfl_down_sync(0xffffffffu, qL[0], 1);         // q_{t+1}(2m + 3), m = 2k + 1
            if (lane == 31) qn = warp + 1 < nw ? s_edge[buf ^ 1][warp + 1] : NEG;
            if (tid == 0) b0 = Lb > 0 ? lse2(q0, qL[0]) : q0;
#pragma unroll
            for (int j = 0; j < CTC_PAIRS; ++j) {
                const double qx = !nlab[j] ? NEG : j + 1 < CTC_PAIRS ? qL[j + 1] : qn;
                bL[j] = hasl[j] ? lse3(qL[j], qB[j], nskip[j] ? qx : NEG) : NEG;
                bB[j] = hasl[j] ? lse2(qB[j], qx) : NEG;
            }
        }
        const double eb = (double)z_b - l_c;
        double gb = tid == 0 ? exp(A0 + b0 - lp) : 0.0;
        if (tid == 0) q0 = b0 + eb;
#pragma unroll
        for (int j = 0; j < CTC_PAIRS; ++j) {
            qL[j] = bL[j] + ((double)z_l[j] - l_c);
            qB[j] = bB[j] + eb;
            if (hasl[j]) {
                s_gam[buf][CTC_PAIRS * tid + j] = exp(AL[j] + bL[j] - lp);
                gb += exp(AB[j] + bB[j] - lp);
            }
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) gb += __shfl_xor_sync(0xffffffffu, gb, o);
        if (lane == 0) { s_bsum[buf][warp] = gb; s_edge[buf][warp] = qL[0]; }
        named_barrier(nthr);
        for (int v = tid; v < V; v += nthr) {
            double occ = 0.0;
            if (v == 0) {
                for (int w = 0; w < nws; ++w) occ += s_bsum[buf][w];
            } else {
                const int e = s_start[v + 1];
                for (int i = s_start[v]; i < e; ++i) occ += s_gam[buf][s_pos[i]];
            }
            dzb[(long long)v * T + t] = (float)(wgt * (exp((double)zb[(long long)v * sv + t] - l_c) - occ));
        }
    }
}

// ---- greedy decoding ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * CTC_LSE_GROUPS)
ctc_argmax_kernel(const float* __restrict__ z, long long sb, long long sv, const int* __restrict__ frames, int T,
                  int V, int* __restrict__ hyps) {
    pdl_trigger(); pdl_wait();
    __shared__ float s_v[CTC_LSE_GROUPS][32];
    __shared__ int s_i[CTC_LSE_GROUPS][32];
    const int b = blockIdx.y, lane = threadIdx.x & 31, g = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + lane;
    const int Tb = frames[b];
    const bool on = Tb >= 1 && Tb <= T && t < Tb;
    const float* zt = z + b * sb + t;
    float m = -INFINITY;
    int mi = V;                                        // NaN and -inf never win: a row of them decodes to the blank
    if (on)
        for (int v = g; v < V; v += CTC_LSE_GROUPS) {
            const float x = zt[v * sv];
            if (x > m) { m = x; mi = v; }
        }
    s_v[g][lane] = m;
    s_i[g][lane] = mi;
    __syncthreads();
    if (g == 0 && on) {
#pragma unroll
        for (int q = 1; q < CTC_LSE_GROUPS; ++q) {
            const float x = s_v[q][lane];
            const int xi = s_i[q][lane];
            if (x > m || (x == m && xi < mi)) { m = x; mi = xi; }
        }
        hyps[(long long)b * T + t] = mi == V ? 0 : mi;
    }
}

__global__ void __launch_bounds__(32 * CTC_COLLAPSE_WARPS)
ctc_collapse_kernel(const int* __restrict__ frames, int B, int T, int* __restrict__ hyps, int* __restrict__ lengths,
                    int* __restrict__ err_flag) {
    pdl_trigger(); pdl_wait();
    const int b = blockIdx.x * CTC_COLLAPSE_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    const int Tb = frames[b];
    if (Tb < 1 || Tb > T) {
        if (lane == 0) { *err_flag = 1; lengths[b] = 0; }
        return;
    }
    int* h = hyps + (long long)b * T;
    int out = 0, carry = -1;
    for (int t0 = 0; t0 < Tb; t0 += 32) {
        const int t = t0 + lane;
        const int a = t < Tb ? h[t] : 0;
        int prev = __shfl_up_sync(0xffffffffu, a, 1);
        if (lane == 0) prev = carry;
        const bool keep = t < Tb && a != 0 && a != prev;
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (keep) h[out + __popc(mask & ((1u << lane) - 1u))] = a;
        out += __popc(mask);
        carry = __shfl_sync(0xffffffffu, a, 31);
        __syncwarp();
    }
    if (lane == 0) lengths[b] = out;
}

// ---- edit distance ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
edit_distance_kernel(const int* __restrict__ hyp, long long hs, const int* __restrict__ hyp_len,
                     const int* __restrict__ ref, long long rs, const int* __restrict__ ref_len, int M_max, int N_max,
                     int* __restrict__ ws, long long ws_stride, int* __restrict__ out, int* __restrict__ err_flag) {
    pdl_trigger(); pdl_wait();
    const long long p = blockIdx.x;
    const int lane = threadIdx.x;
    const int M = hyp_len[p], N = ref_len[p];
    int* o = out + 4 * p;
    if (M < 0 || M > M_max || N < 0 || N > N_max) {
        if (lane == 0) { *err_flag = 1; o[0] = o[1] = o[2] = o[3] = 0; }
        return;
    }
    if (M == 0 || N == 0) {                           // all deletions or all insertions
        if (lane == 0) { o[0] = M + N; o[1] = 0; o[2] = N; o[3] = M; }
        return;
    }
    const int* h = hyp + p * hs;
    const int* r = ref + p * rs;
    int* bufC = ws + p * ws_stride;                   // row i0 of the strip: cost, then S | D << 16
    int* bufS = bufC + ((M + 31) & ~31);
    constexpr int DEL = 1 << 16;
    for (int i0 = 0; i0 < N; i0 += 32) {
        const int i = i0 + lane + 1;
        const bool row_ok = i <= N;
        const bool has_above = i0 > 0, has_below = i0 + 32 < N;
        const int rt = row_ok ? r[i - 1] : 0;
        int upC = i0, upS = i0 * DEL;                 // lane 0: D(i0, 0), the diagonal of its first column
        int leftC = i, leftS = i * DEL;               // D(i, 0): i deletions
        int shC = i - 1, shS = (i - 1) * DEL;         // D(i-1, 0): what lane l-1 passes before its first column
        const int steps = M + min(32, N - i0) - 1;
        for (int s = 0; s < steps; ++s) {
            const int j = s - lane + 1;
            const int dgC = upC, dgS = upS;
            if (lane == 0) {
                if (j > M) { upC = 0; upS = 0; }
                else if (has_above) { upC = bufC[j - 1]; upS = bufS[j - 1]; }
                else { upC = j; upS = 0; }             // row 0: j insertions
            } else { upC = shC; upS = shS; }
            if (row_ok && j >= 1 && j <= M) {
                const int mis = h[j - 1] != rt;
                int bC = dgC + mis, bS = dgS + mis;
                if (upC + 1 < bC) { bC = upC + 1; bS = upS + DEL; }
                if (leftC + 1 < bC) { bC = leftC + 1; bS = leftS; }
                leftC = bC;
                leftS = bS;
                if (i == N && j == M) {
                    const int sub = bS & (DEL - 1), del = bS >> 16;
                    o[0] = bC; o[1] = sub; o[2] = del; o[3] = bC - sub - del;
                }
                if (lane == 31 && has_below) { bufC[j - 1] = bC; bufS[j - 1] = bS; }
            }
            shC = __shfl_up_sync(0xffffffffu, leftC, 1);
            shS = __shfl_up_sync(0xffffffffu, leftS, 1);
        }
        __syncwarp();                                  // lane 31's boundary row before the next strip's lane 0 reads it
    }
}

static int ctc_check(const char* what, const float* z, long long sb, long long sv, int B, int V, int T, int L) {
    DV3_REQUIRE(z != nullptr, "%s: null logits", what);
    DV3_REQUIRE(B >= 1 && T >= 1, "%s: B=%d, T=%d", what, B, T);
    DV3_REQUIRE(V >= 2 && V <= CTC_MAX_VOCAB, "%s: V=%d outside [2, %d]", what, V, CTC_MAX_VOCAB);
    DV3_REQUIRE(L >= 1 && L <= CTC_MAX_TARGET, "%s: L=%d outside [1, %d]", what, L, CTC_MAX_TARGET);
    DV3_REQUIRE(sv >= T && (B == 1 || sb >= (long long)(V - 1) * sv + T), "%s: strides (%lld, %lld) for V=%d, T=%d",
                what, sb, sv, V, T);
    DV3_REQUIRE((long long)(B - 1) * sb + (long long)(V - 1) * sv + T < (1LL << 31) && (long long)B * V * T < (1LL << 31),
                "%s: B*V*T past 2^31", what);
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_ctc_max_vocab(void) { return CTC_MAX_VOCAB; }

long long dv3_ctc_ws_bytes(int B, int T, int L) {
    if (B < 1 || T < 1 || L < 1 || L > CTC_MAX_TARGET) return 0;
    return 8 * ctc_ws_doubles(B, T, L);
}

int dv3_ctc_fwd(const float* z, long long stride_b, long long stride_v, const int* frames, const int* targets,
                long long tgt_stride, const int* target_lengths, int B, int V, int T, int L, void* ws, float* nll,
                float* partials, int* infeasible, int* err_flag, void* stream) {
    if (ctc_check("ctc_fwd", z, stride_b, stride_v, B, V, T, L)) return 1;
    DV3_REQUIRE(frames && targets && target_lengths && ws && nll && partials && infeasible && err_flag,
                "ctc_fwd: null operand");
    DV3_REQUIRE(tgt_stride >= L, "ctc_fwd: target stride %lld below L=%d", tgt_stride, L);
    double* w = static_cast<double*>(ws);
    const dim3 g_lse((unsigned)ceil_div(T, 32), (unsigned)B);
    launch_k(ctc_lse_kernel, g_lse, 32 * CTC_LSE_GROUPS, 0, (cudaStream_t)stream, z, stride_b, stride_v, frames, T, V,
             w);
    if (check_launch("ctc_lse")) return 1;
    launch_k(ctc_alpha_kernel, (unsigned)B, (ctc_row_threads(L) + 31) / 32 * 32, 0, (cudaStream_t)stream, z, stride_b, stride_v, frames,
             targets, tgt_stride, target_lengths, T, V, L, w, nll, partials, infeasible, err_flag, B);
    return check_launch("ctc_alpha");
}

int dv3_ctc_bwd(const float* z, long long stride_b, long long stride_v, const int* frames, const int* targets,
                long long tgt_stride, const int* target_lengths, int B, int V, int T, int L, const void* ws,
                const float* d_loss, float scale, float* dz, void* stream) {
    if (ctc_check("ctc_bwd", z, stride_b, stride_v, B, V, T, L)) return 1;
    DV3_REQUIRE(frames && targets && target_lengths && ws && d_loss && dz, "ctc_bwd: null operand");
    DV3_REQUIRE(tgt_stride >= L, "ctc_bwd: target stride %lld below L=%d", tgt_stride, L);
    const int threads = (max(ctc_row_threads(L), min(V, CTC_THREADS)) + 31) / 32 * 32;
    launch_k(ctc_beta_grad_kernel, (unsigned)B, threads, 0, (cudaStream_t)stream, z, stride_b, stride_v, frames,
             targets, tgt_stride, target_lengths, T, V, L, static_cast<const double*>(ws), d_loss, scale, dz, B);
    return check_launch("ctc_beta_grad");
}

int dv3_ctc_greedy(const float* z, long long stride_b, long long stride_v, const int* frames, int B, int V, int T,
                   int* hyps, int* hyp_lengths, int* err_flag, void* stream) {
    if (ctc_check("ctc_greedy", z, stride_b, stride_v, B, V, T, 1)) return 1;
    DV3_REQUIRE(frames && hyps && hyp_lengths && err_flag, "ctc_greedy: null operand");
    const dim3 g((unsigned)ceil_div(T, 32), (unsigned)B);
    launch_k(ctc_argmax_kernel, g, 32 * CTC_LSE_GROUPS, 0, (cudaStream_t)stream, z, stride_b, stride_v, frames, T, V,
             hyps);
    if (check_launch("ctc_argmax")) return 1;
    launch_k(ctc_collapse_kernel, (unsigned)ceil_div(B, CTC_COLLAPSE_WARPS), 32 * CTC_COLLAPSE_WARPS, 0,
             (cudaStream_t)stream, frames, B, T, hyps, hyp_lengths, err_flag);
    return check_launch("ctc_collapse");
}

long long dv3_edit_ws_ints(int P, int M_max) {
    if (P < 1 || M_max < 0 || M_max > CTC_MAX_HYP) return 0;
    return (long long)P * 2 * ((M_max + 31) / 32 * 32 + 32);
}

int dv3_edit_distance(const int* hyp, long long hyp_stride, const int* hyp_len, const int* ref, long long ref_stride,
                      const int* ref_len, int P, int M_max, int N_max, int* ws, int* out, int* err_flag,
                      void* stream) {
    DV3_REQUIRE(hyp && hyp_len && ref && ref_len && ws && out && err_flag, "edit_distance: null operand");
    DV3_REQUIRE(P >= 1 && M_max >= 0 && M_max <= CTC_MAX_HYP && N_max >= 0 && N_max <= CTC_MAX_TARGET,
                "edit_distance: P=%d, M_max=%d (<= %d), N_max=%d (<= %d)", P, M_max, CTC_MAX_HYP, N_max,
                CTC_MAX_TARGET);
    DV3_REQUIRE(hyp_stride >= M_max && ref_stride >= N_max && hyp_stride >= 0 && ref_stride >= 0,
                "edit_distance: strides (%lld, %lld) for lengths (%d, %d)", hyp_stride, ref_stride, M_max, N_max);
    const long long ws_stride = dv3_edit_ws_ints(1, M_max);
    launch_k(edit_distance_kernel, (unsigned)P, 32, 0, (cudaStream_t)stream, hyp, hyp_stride, hyp_len, ref, ref_stride,
             ref_len, M_max, N_max, ws, ws_stride, out, err_flag);
    return check_launch("edit_distance");
}

}  // extern "C"
