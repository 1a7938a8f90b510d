// Fused training losses + their gradients in one pass each (reference train.py:537-601, 665-740): masked-L1 +
// binary-divergence spectrogram loss (mel and linear), BCE on the done flag, guided-attention loss with the soft
// mask W[b,t,n] = 1 - exp(-(n/N_b - t/T_b)^2 / 2g^2) generated on the fly (the reference builds W with numba on the
// host and uploads it every step).  Each kernel adds its already-normalised contribution to ONE device scalar and
// writes dLoss/dPrediction, so the autograd graph of ~60 elementwise ATen kernels over (16,800,513) tensors
// collapses to 3 launches.  HBM-bound: 8 B read + 4 B written per spectrogram element.
#include "common.cuh"

namespace dv3 {

__device__ __forceinline__ float block_sum_256(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 32) {
        t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        t = warp_sum(t);
    }
    __syncthreads();
    return t;            // valid in thread 0 (and lanes of warp 0)
}

// ---- deterministic mode (ops.deterministic): fixed-order sums instead of one float atomic per block ----------------
// Every block stores its (up to) three partial sums at scratch[3 * blockIdx.x ..]; the block that draws the last
// ticket adds them in a fixed order -- warp j owns sum j, lane l adds the partials of blocks l, l + 32, ... in ascending
// order, then the xor-shuffle tree of warp_sum -- and adds the totals to loss / terms.  The order depends on the grid
// alone, and the grid on the tensor shapes alone.  No block waits for another: the last one to arrive does the tail.
// scratch: LOSS_DET_SCRATCH floats, zero-filled once by the caller; its last word is the ticket, left at zero.
constexpr int LOSS_MAX_BLOCKS = 132 * 8;
constexpr int LOSS_DET_SCRATCH = 3 * LOSS_MAX_BLOCKS + 1;

template <bool TERMS>
__device__ __forceinline__ void det_loss_tail(float s, float s1, float s2, float* __restrict__ loss,
                                              float* __restrict__ terms, float* __restrict__ scratch) {
    __shared__ bool last;
    if (threadIdx.x == 0) {
        scratch[3 * blockIdx.x] = s;
        if (TERMS) { scratch[3 * blockIdx.x + 1] = s1; scratch[3 * blockIdx.x + 2] = s2; }
        __threadfence();
        unsigned* ticket = reinterpret_cast<unsigned*>(scratch + LOSS_DET_SCRATCH - 1);
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    const int j = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (j < (TERMS ? 3 : 1)) {
        float t = 0.f;
        for (int i = lane; i < (int)gridDim.x; i += 32) t += __ldcg(&scratch[3 * i + j]);
        t = warp_sum(t);
        if (lane == 0) {
            if (j == 0) loss[0] += t; else terms[j - 1] += t;
        }
    }
    if (threadIdx.x == 0) *reinterpret_cast<unsigned*>(scratch + LOSS_DET_SCRATCH - 1) = 0u;
}

// y_hat (B, T, D) predictions, y (B, T, D) targets; pairs (y_hat[b,t], y[b,t+r]) for t < T-r; lengths int64 [B]
// (valid target frames per utterance, in this tensor's time units); grad (B, T, D) fully written.
//   loss += sum (1-bw)*coef1*|d| + bw*coef*z,  coef = w*m/Sm + (1-w)/N,  m = (t+r < len_b)
// priority bins (train.py:559-567): the L1 term becomes (1-pw)*L1(all bins) + pw*L1(bins < pbin), i.e.
//   coef1 = (1-pw)*coef + [d < pbin]*pw*coef*(D/pbin)     (the same masked/plain means over the pbin-wide slice)
// t_log (int64 in device memory, or null = T): the logical time extent of a batch padded to a larger bucket.  Pairs
// t >= t_log - r are left out of the loss and its means, and their gradient is written as 0.
// TERMS: also add the two parts of the loss to terms[0] (the L1 part, priority bins combined) and terms[1] (the
// binary-divergence part) -- the l1_loss / binary_div pair reference spec_loss returns.  loss and grad are unchanged.
// DET: the block sums go through det_loss_tail (scratch) instead of the atomics; everything else is the same code.
template <bool TERMS, bool DET>
__device__ __forceinline__ void spec_loss_body(const float* __restrict__ y_hat, const float* __restrict__ y,
                                               const long long* __restrict__ lengths,
                                               const long long* __restrict__ t_log, float* __restrict__ grad,
                                               float* __restrict__ loss, int B, int T, int D, int r, float w, float bw,
                                               float eps, int pbin, float pw, float* __restrict__ terms,
                                               float* __restrict__ scratch) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float red[8];
    __shared__ float s_inv_sm;
    const int TL = t_log ? (int)min((long long)T, max((long long)r + 1, *t_log)) : T;
    if (threadIdx.x == 0) {
        double sm = 0.0;
        for (int b = 0; b < B; ++b) {
            long long v = lengths[b] - r;
            if (v < 0) v = 0;
            if (v > TL - r) v = TL - r;
            sm += (double)v;
        }
        s_inv_sm = sm > 0 ? (float)(1.0 / (sm * D)) : 0.f;
    }
    __syncthreads();
    const float inv_sm = s_inv_sm;
    const float inv_n = 1.f / ((float)B * (float)(TL - r) * (float)D);
    const long long total = (long long)B * T * D;
    const long long shift = (long long)r * D;
    const bool prio = pbin > 0 && pw > 0.f;
    const float prio_gain = prio ? pw * ((float)D / (float)pbin) : 0.f;
    float acc = 0.f, acc_l1 = 0.f, acc_bd = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long bt = i / D;
        const int t = (int)(bt % T), b = (int)(bt / T);
        float g = 0.f;
        if (t < TL - r) {
            const float p = y_hat[i], tg = y[i + shift];
            const float m = (t + r < lengths[b]) ? 1.f : 0.f;
            const float coef = w * m * inv_sm + (1.f - w) * inv_n;
            const float d = p - tg;
            float c1 = 1.f;                                   // L1 weight relative to coef
            if (prio) c1 = (1.f - pw) + ((int)(i - bt * D) < pbin ? prio_gain : 0.f);
            float e = c1 * (1.f - bw) * fabsf(d);
            float de = c1 * (1.f - bw) * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
            if (TERMS) acc_l1 += coef * (c1 * fabsf(d));
            if (bw > 0.f) {
                const float L = logf(p + eps) - logf(1.f - p + eps);
                const float u = expf(L);
                const float z = -tg * L + log1pf(u);
                e += bw * z;
                de += bw * (u / (1.f + u) - tg) * (1.f / (p + eps) + 1.f / (1.f - p + eps));
                if (TERMS) acc_bd += coef * z;
            }
            acc += coef * e;
            g = coef * de;
        }
        grad[i] = g;
    }
    const float s = block_sum_256(acc, red);
    if (DET) {
        const float s1 = TERMS ? block_sum_256(acc_l1, red) : 0.f, s2 = TERMS ? block_sum_256(acc_bd, red) : 0.f;
        det_loss_tail<TERMS>(s, s1, s2, loss, terms, scratch);
        return;
    }
    if (threadIdx.x == 0) atomicAdd(loss, s);
    if (TERMS) {
        const float s1 = block_sum_256(acc_l1, red);
        if (threadIdx.x == 0) atomicAdd(&terms[0], s1);
        const float s2 = block_sum_256(acc_bd, red);
        if (threadIdx.x == 0) atomicAdd(&terms[1], s2);
    }
}

template <bool TERMS>
__global__ void spec_loss_kernel(const float* __restrict__ y_hat, const float* __restrict__ y,
                                 const long long* __restrict__ lengths, const long long* __restrict__ t_log,
                                 float* __restrict__ grad, float* __restrict__ loss, int B, int T, int D, int r,
                                 float w, float bw, float eps, int pbin, float pw, float* __restrict__ terms) {
    spec_loss_body<TERMS, false>(y_hat, y, lengths, t_log, grad, loss, B, T, D, r, w, bw, eps, pbin, pw, terms, nullptr);
}

template <bool TERMS>
__global__ void spec_loss_det_kernel(const float* __restrict__ y_hat, const float* __restrict__ y,
                                     const long long* __restrict__ lengths, const long long* __restrict__ t_log,
                                     float* __restrict__ grad, float* __restrict__ loss, int B, int T, int D, int r,
                                     float w, float bw, float eps, int pbin, float pw, float* __restrict__ terms,
                                     float* __restrict__ scratch) {
    spec_loss_body<TERMS, true>(y_hat, y, lengths, t_log, grad, loss, B, T, D, r, w, bw, eps, pbin, pw, terms, scratch);
}

// done BCE (mean) + guided attention (mean of attn*W):
//   done_hat, done (n_done);  attn (A, B, Td, Ts), in_len / dec_len int64 [B];  grads written in full.
// ext (int64 [2] in device memory, or null): logical (decoder steps, text positions) of a batch padded to a larger
// bucket -- done_hat is then (B, Td); steps >= ext[0] and text positions >= ext[1] are left out of both means and
// their gradient is written as 0.
// TERMS: also add the done BCE to terms[0] and the guided-attention term to terms[1].
template <bool TERMS, bool DET>
__device__ __forceinline__ void aux_loss_body(const float* __restrict__ done_hat, const float* __restrict__ done,
                                              float* __restrict__ d_done, long long n_done,
                                              const float* __restrict__ attn, float* __restrict__ d_attn,
                                              const long long* __restrict__ in_len,
                                              const long long* __restrict__ dec_len, const long long* __restrict__ ext,
                                              int A, int B, int Td, int Ts, float sigma, int use_attn,
                                              float* __restrict__ loss, float* __restrict__ terms,
                                              float* __restrict__ scratch) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float red[8];
    float acc = 0.f, acc_done = 0.f, acc_attn = 0.f;
    const long long stride = (long long)gridDim.x * blockDim.x, start = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const int TdL = ext ? (int)min((long long)Td, max(1LL, ext[0])) : Td;
    const int TsL = ext ? (int)min((long long)Ts, max(1LL, ext[1])) : Ts;
    const float inv_nd = 1.f / (float)(ext ? (long long)B * TdL : n_done);
    for (long long i = start; i < n_done; i += stride) {
        if (ext && (int)(i % Td) >= TdL) { d_done[i] = 0.f; continue; }
        const float p = done_hat[i], t = done[i];
        acc -= inv_nd * (t * fmaxf(logf(p), -100.f) + (1.f - t) * fmaxf(logf(1.f - p), -100.f));
        d_done[i] = inv_nd * (p - t) / fmaxf((1.f - p) * p, 1e-12f);
    }
    if (TERMS) acc_done = acc;
    if (use_attn) {
        const long long n_attn = (long long)A * B * Td * Ts;
        const float inv_na = 1.f / (float)((long long)A * B * TdL * TsL);
        const double inv2g2 = 1.0 / (2.0 * (double)sigma * (double)sigma);
        for (long long i = start; i < n_attn; i += stride) {
            const int n = (int)(i % Ts);
            const int t = (int)((i / Ts) % Td);
            const int b = (int)((i / ((long long)Ts * Td)) % B);
            const long long N = in_len[b], Tl = dec_len[b];
            float wv = 0.f;
            if (n < N && t < Tl && n < TsL && t < TdL) {
                const double q = (double)n / (double)N - (double)t / (double)Tl;
                wv = (float)(1.0 - exp(-q * q * inv2g2));
            }
            acc += inv_na * attn[i] * wv;
            if (TERMS) acc_attn += inv_na * attn[i] * wv;
            d_attn[i] = inv_na * wv;
        }
    } else if (d_attn) {
        const long long n_attn = (long long)A * B * Td * Ts;
        for (long long i = start; i < n_attn; i += stride) d_attn[i] = 0.f;
    }
    const float s = block_sum_256(acc, red);
    if (DET) {
        const float s1 = TERMS ? block_sum_256(acc_done, red) : 0.f, s2 = TERMS ? block_sum_256(acc_attn, red) : 0.f;
        det_loss_tail<TERMS>(s, s1, s2, loss, terms, scratch);
        return;
    }
    if (threadIdx.x == 0) atomicAdd(loss, s);
    if (TERMS) {
        const float s1 = block_sum_256(acc_done, red);
        if (threadIdx.x == 0) atomicAdd(&terms[0], s1);
        const float s2 = block_sum_256(acc_attn, red);
        if (threadIdx.x == 0) atomicAdd(&terms[1], s2);
    }
}

template <bool TERMS>
__global__ void aux_loss_kernel(const float* __restrict__ done_hat, const float* __restrict__ done,
                                float* __restrict__ d_done, long long n_done, const float* __restrict__ attn,
                                float* __restrict__ d_attn, const long long* __restrict__ in_len,
                                const long long* __restrict__ dec_len, const long long* __restrict__ ext, int A,
                                int B, int Td, int Ts, float sigma, int use_attn, float* __restrict__ loss,
                                float* __restrict__ terms) {
    aux_loss_body<TERMS, false>(done_hat, done, d_done, n_done, attn, d_attn, in_len, dec_len, ext, A, B, Td, Ts, sigma,
                                use_attn, loss, terms, nullptr);
}

template <bool TERMS>
__global__ void aux_loss_det_kernel(const float* __restrict__ done_hat, const float* __restrict__ done,
                                    float* __restrict__ d_done, long long n_done, const float* __restrict__ attn,
                                    float* __restrict__ d_attn, const long long* __restrict__ in_len,
                                    const long long* __restrict__ dec_len, const long long* __restrict__ ext, int A,
                                    int B, int Td, int Ts, float sigma, int use_attn, float* __restrict__ loss,
                                    float* __restrict__ terms, float* __restrict__ scratch) {
    aux_loss_body<TERMS, true>(done_hat, done, d_done, n_done, attn, d_attn, in_len, dec_len, ext, A, B, Td, Ts, sigma,
                               use_attn, loss, terms, scratch);
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_spec_loss_terms(const float* y_hat, const float* y, const long long* lengths, const long long* t_log,
                        float* grad, float* loss, float* terms, int B, int T, int D, int r, float masked_loss_weight,
                        float binary_divergence_weight, int priority_bin, float priority_weight, void* stream) {
    DV3_REQUIRE(T > r && r >= 0, "spec_loss: need T > r");
    DV3_REQUIRE(priority_bin >= 0 && priority_bin <= D && priority_weight >= 0.f && priority_weight <= 1.f,
                "spec_loss: priority_bin=%d (D=%d) priority_weight=%g out of range", priority_bin, D, priority_weight);
    long long blocks = ((long long)B * T * D + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (terms)
        launch_k(spec_loss_kernel<true>, (int)blocks, 256, 0, (cudaStream_t)stream, y_hat, y, lengths, t_log, grad,
                 loss, B, T, D, r, masked_loss_weight, binary_divergence_weight, 1e-8f, priority_bin, priority_weight,
                 terms);
    else
        launch_k(spec_loss_kernel<false>, (int)blocks, 256, 0, (cudaStream_t)stream, y_hat, y, lengths, t_log, grad,
                 loss, B, T, D, r, masked_loss_weight, binary_divergence_weight, 1e-8f, priority_bin, priority_weight,
                 terms);
    return check_launch("spec_loss");
}

int dv3_spec_loss(const float* y_hat, const float* y, const long long* lengths, float* grad, float* loss, int B,
                  int T, int D, int r, float masked_loss_weight, float binary_divergence_weight, int priority_bin,
                  float priority_weight, void* stream) {
    return dv3_spec_loss_terms(y_hat, y, lengths, nullptr, grad, loss, nullptr, B, T, D, r, masked_loss_weight,
                               binary_divergence_weight, priority_bin, priority_weight, stream);
}

int dv3_spec_loss_ext(const float* y_hat, const float* y, const long long* lengths, const long long* t_log,
                      float* grad, float* loss, int B, int T, int D, int r, float masked_loss_weight,
                      float binary_divergence_weight, int priority_bin, float priority_weight, void* stream) {
    DV3_REQUIRE(t_log != nullptr, "spec_loss_ext: t_log is NULL");
    return dv3_spec_loss_terms(y_hat, y, lengths, t_log, grad, loss, nullptr, B, T, D, r, masked_loss_weight,
                               binary_divergence_weight, priority_bin, priority_weight, stream);
}

int dv3_aux_loss_terms(const float* done_hat, const float* done, float* d_done, long long n_done, const float* attn,
                       float* d_attn, const long long* in_len, const long long* dec_len, const long long* ext, int A,
                       int B, int Td, int Ts, float sigma, int use_attn, float* loss, float* terms, void* stream) {
    DV3_REQUIRE(ext == nullptr || n_done == (long long)B * Td, "aux_loss: with extents done_hat must be (B, Td)");
    if (terms)
        launch_k(aux_loss_kernel<true>, 132 * 2, 256, 0, (cudaStream_t)stream, done_hat, done, d_done, n_done, attn,
                 d_attn, in_len, dec_len, ext, A, B, Td, Ts, sigma, use_attn, loss, terms);
    else
        launch_k(aux_loss_kernel<false>, 132 * 2, 256, 0, (cudaStream_t)stream, done_hat, done, d_done, n_done, attn,
                 d_attn, in_len, dec_len, ext, A, B, Td, Ts, sigma, use_attn, loss, terms);
    return check_launch("aux_loss");
}

int dv3_aux_loss(const float* done_hat, const float* done, float* d_done, long long n_done, const float* attn,
                 float* d_attn, const long long* in_len, const long long* dec_len, int A, int B, int Td, int Ts,
                 float sigma, int use_attn, float* loss, void* stream) {
    return dv3_aux_loss_terms(done_hat, done, d_done, n_done, attn, d_attn, in_len, dec_len, nullptr, A, B, Td, Ts,
                              sigma, use_attn, loss, nullptr, stream);
}

int dv3_aux_loss_ext(const float* done_hat, const float* done, float* d_done, const float* attn, float* d_attn,
                     const long long* in_len, const long long* dec_len, const long long* ext, int A, int B, int Td,
                     int Ts, float sigma, int use_attn, float* loss, void* stream) {
    DV3_REQUIRE(ext != nullptr, "aux_loss_ext: ext is NULL");
    return dv3_aux_loss_terms(done_hat, done, d_done, (long long)B * Td, attn, d_attn, in_len, dec_len, ext, A, B, Td,
                              Ts, sigma, use_attn, loss, nullptr, stream);
}

// ---- deterministic forms (see det_loss_tail): the same grids, arithmetic and gradients; t_log / ext / terms nullable, so
// each covers the plain, _ext and _terms forms of its atomic twin.  scratch: dv3_loss_det_scratch_floats() floats.
int dv3_loss_det_scratch_floats(void) { return LOSS_DET_SCRATCH; }

int dv3_spec_loss_det(const float* y_hat, const float* y, const long long* lengths, const long long* t_log,
                      float* grad, float* loss, float* terms, float* scratch, int B, int T, int D, int r,
                      float masked_loss_weight, float binary_divergence_weight, int priority_bin,
                      float priority_weight, void* stream) {
    DV3_REQUIRE(T > r && r >= 0, "spec_loss_det: need T > r");
    DV3_REQUIRE(priority_bin >= 0 && priority_bin <= D && priority_weight >= 0.f && priority_weight <= 1.f,
                "spec_loss_det: priority_bin=%d (D=%d) priority_weight=%g out of range", priority_bin, D,
                priority_weight);
    DV3_REQUIRE(scratch != nullptr, "spec_loss_det: scratch buffer required");
    long long blocks = ((long long)B * T * D + 255) / 256;
    if (blocks > LOSS_MAX_BLOCKS) blocks = LOSS_MAX_BLOCKS;
    if (terms)
        launch_k(spec_loss_det_kernel<true>, (int)blocks, 256, 0, (cudaStream_t)stream, y_hat, y, lengths, t_log,
                 grad, loss, B, T, D, r, masked_loss_weight, binary_divergence_weight, 1e-8f, priority_bin,
                 priority_weight, terms, scratch);
    else
        launch_k(spec_loss_det_kernel<false>, (int)blocks, 256, 0, (cudaStream_t)stream, y_hat, y, lengths, t_log,
                 grad, loss, B, T, D, r, masked_loss_weight, binary_divergence_weight, 1e-8f, priority_bin,
                 priority_weight, terms, scratch);
    return check_launch("spec_loss_det");
}

int dv3_aux_loss_det(const float* done_hat, const float* done, float* d_done, long long n_done, const float* attn,
                     float* d_attn, const long long* in_len, const long long* dec_len, const long long* ext, int A,
                     int B, int Td, int Ts, float sigma, int use_attn, float* loss, float* terms, float* scratch,
                     void* stream) {
    DV3_REQUIRE(ext == nullptr || n_done == (long long)B * Td, "aux_loss_det: with extents done_hat must be (B, Td)");
    DV3_REQUIRE(scratch != nullptr, "aux_loss_det: scratch buffer required");
    if (terms)
        launch_k(aux_loss_det_kernel<true>, 132 * 2, 256, 0, (cudaStream_t)stream, done_hat, done, d_done, n_done,
                 attn, d_attn, in_len, dec_len, ext, A, B, Td, Ts, sigma, use_attn, loss, terms, scratch);
    else
        launch_k(aux_loss_det_kernel<false>, 132 * 2, 256, 0, (cudaStream_t)stream, done_hat, done, d_done, n_done,
                 attn, d_attn, in_len, dec_len, ext, A, B, Td, Ts, sigma, use_attn, loss, terms, scratch);
    return check_launch("aux_loss_det");
}

}  // extern "C"
