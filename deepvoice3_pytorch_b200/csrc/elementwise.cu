// Memory-bound glue kernels of the hot path: layout changes, lookups, position encodings, dropout,
// masked softmax.  All are coalesced along the fastest axis and vectorised where alignment allows.
#include "common.cuh"

namespace dv3 {

// ---- (B, R, C) -> (B, C, R) -------------------------------------------------------------------
// reference: every x.transpose(1, 2) between the (B,T,C) attention layout and the (B,C,T) conv layout
// (deepvoice3.py:86,93,318,324,340-345,355,359,592,602; nyanko.py:66,206,214-217,230,234,402).
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int C) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float tile[32][33];
    const int b = blockIdx.z, r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    const float* src = in + (size_t)b * R * C;
    float* dst = out + (size_t)b * R * C;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + threadIdx.y + 8 * i, c = c0 + threadIdx.x;
        if (r < R && c < C) tile[threadIdx.y + 8 * i][threadIdx.x] = src[(size_t)r * C + c];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = c0 + threadIdx.y + 8 * i, r = r0 + threadIdx.x;
        if (r < R && c < C) dst[(size_t)c * R + r] = tile[threadIdx.x][threadIdx.y + 8 * i];
    }
}

// ---- embedding lookup: reference deepvoice3.py:74, nyanko.py:64,201-203 (F.embedding) ---------------
// ids int64 (N) -> out (N, D).  One warp per row; ids are validated (bit-exact indexing).
__global__ void embedding_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ table,
                                     float* __restrict__ out, int N, int D, int V, int* __restrict__ err) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (n >= N) return;
    const long long id = ids[n];
    if (id < 0 || id >= V) { if (lane == 0) atomicExch(err, 1); return; }
    const float* src = table + (size_t)id * D;
    float* dst = out + (size_t)n * D;
    for (int d = lane; d < D; d += 32) dst[d] = src[d];
}
// dtable[ids[n]] += dy[n] unless ids[n] == padding_idx (padding_idx < 0: none)
__global__ void embedding_bwd_kernel(const long long* __restrict__ ids, const float* __restrict__ dy,
                                     float* __restrict__ dtable, int N, int D, int V, long long padding_idx) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (n >= N) return;
    const long long id = ids[n];
    if (id == padding_idx || id < 0 || id >= V) return;
    for (int d = lane; d < D; d += 32) atomicAdd(&dtable[(size_t)id * D + d], dy[(size_t)n * D + d]);
}

// ---- sinusoidal position encoding: reference modules.py:27-31,45-64 ---------------------------------
// out[b,t,i] = pos==0 ? 0 : (i even ? sin : cos)(w_b * table[pos,i]);  w per batch row (nw==B) or shared (nw==1).
// Same fp32 operation order as the reference: fp32 product, then fp32 sin/cos (full-range, not fast-math).
__global__ void sinusoid_fwd_kernel(const long long* __restrict__ pos, const float* __restrict__ table,
                                    const float* __restrict__ w, int nw, float* __restrict__ out, int B,
                                    int T, int D, int P, int* __restrict__ err) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (n >= B * T) return;
    const long long ps = pos[n];
    if (ps < 0 || ps >= P) { if (lane == 0) atomicExch(err, 1); return; }
    const float wb = w[nw == 1 ? 0 : n / T];
    float* dst = out + (size_t)n * D;
    const float* row = table + (size_t)ps * D;
    for (int i = lane; i < D; i += 32) {
        float y = 0.f;
        if (ps != 0) { const float a = wb * row[i]; y = (i & 1) ? cosf(a) : sinf(a); }
        dst[i] = y;
    }
}
// dtable[pos,i] += dy * d/da * w ; dw[b] += sum dy * d/da * table   (row 0 / padding gets nothing)
__global__ void sinusoid_bwd_kernel(const long long* __restrict__ pos, const float* __restrict__ table,
                                    const float* __restrict__ w, int nw, const float* __restrict__ dy,
                                    float* __restrict__ dtable, int B, int T, int D, int P) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (n >= B * T) return;
    const long long ps = pos[n];
    if (ps <= 0 || ps >= P) return;
    const float wb = w[nw == 1 ? 0 : n / T];
    const float* row = table + (size_t)ps * D;
    for (int i = lane; i < D; i += 32) {
        const float a = wb * row[i];
        const float da = dy[(size_t)n * D + i] * ((i & 1) ? -sinf(a) : cosf(a));
        atomicAdd(&dtable[(size_t)ps * D + i], da * wb);
    }
}

// ---- deterministic mode: the two table gradients without atomics -----------------------------------------------------
// One CTA (256 threads) per table row.  The CTA scans the id list 256 entries at a time and compacts the entries that
// name its row into shared memory IN INDEX ORDER (warp ballots + a prefix over the 8 warp counts); every thread then
// walks that list and accumulates its columns (d = tid, tid + 256, ...: D <= TABLE_DET_MAX_D) in registers, and the row
// is stored once, coalesced: dtable[row] += sum.  Each element is therefore the sum of its tokens in ascending token
// index, whatever order blocks run in.  SINUSOID = false: dtable[ids[n]] += dy[n] (row padding_idx gets nothing);
// SINUSOID = true: the position-table gradient of sinusoid_bwd_kernel, term for term (row 0 gets nothing).
constexpr int TABLE_DET_MAX_D = 1024;
template <bool SINUSOID>
__global__ void __launch_bounds__(256) table_bwd_det_kernel(const long long* __restrict__ ids,
                                                            const float* __restrict__ table,
                                                            const float* __restrict__ w, int nw, int T,
                                                            const float* __restrict__ dy, float* __restrict__ dtable,
                                                            int N, int D, long long padding_idx) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ int s_list[256];
    __shared__ int s_cnt[8];
    const int row = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (row == padding_idx) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, tv[4] = {0.f, 0.f, 0.f, 0.f};
    if (SINUSOID) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (tid + 256 * q < D) tv[q] = table[(size_t)row * D + tid + 256 * q];
    }
    bool any = false;
    for (int base = 0; base < N; base += 256) {
        const int n = base + tid;
        const bool match = n < N && ids[n] == row;
        const unsigned bal = __ballot_sync(0xffffffffu, match);
        if (lane == 0) s_cnt[warp] = __popc(bal);
        __syncthreads();
        int off = 0, total = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) { if (i < warp) off += s_cnt[i]; total += s_cnt[i]; }
        if (match) s_list[off + __popc(bal & ((1u << lane) - 1u))] = n;
        __syncthreads();
        for (int j = 0; j < total; ++j) {
            const int m = s_list[j];
            const float wb = SINUSOID ? w[nw == 1 ? 0 : m / T] : 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int d = tid + 256 * q;
                if (d < D) {
                    const float g = dy[(size_t)m * D + d];
                    if (SINUSOID) {
                        const float a = wb * tv[q];
                        const float da = g * ((d & 1) ? -sinf(a) : cosf(a));
                        acc[q] += __fmul_rn(da, wb);      // the rounded product the atomic kernel adds: no fma
                    } else {
                        acc[q] += g;
                    }
                }
            }
        }
        any |= total > 0;
        __syncthreads();
    }
    if (!any) return;
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (tid + 256 * q < D) dtable[(size_t)row * D + tid + 256 * q] += acc[q];
}

// d(loss)/d(position rate): dw[wi] = sum over the rows of utterance wi (all rows if nw == 1) of <dy * d(enc)/d(a), table>.
// The sum cancels heavily (its terms are O(1), the result often 1e-4 of that), so it is accumulated in double by ONE
// CTA per rate, in a fixed order: deterministic, and as accurate as the fp32 CPU reference (float atomics over the
// rows gave 4e-2 relative error on the multi-speaker position-rate projections).
__global__ void __launch_bounds__(256) sinusoid_dw_kernel(const long long* __restrict__ pos,
                                                          const float* __restrict__ table,
                                                          const float* __restrict__ w, int nw,
                                                          const float* __restrict__ dy, float* __restrict__ dw, int B,
                                                          int T, int D, int P) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ double red[8];
    const int wi = blockIdx.x;
    const int r0 = nw == 1 ? 0 : wi * T, r1 = nw == 1 ? B * T : (wi + 1) * T;
    const float wb = w[wi];
    double acc = 0.0;
    const long long total = (long long)(r1 - r0) * D;
    for (long long q = threadIdx.x; q < total; q += blockDim.x) {
        const int n = r0 + (int)(q / D), i = (int)(q % D);
        const long long ps = pos[n];
        if (ps <= 0 || ps >= P) continue;
        const float tv = table[(size_t)ps * D + i], a = wb * tv;
        acc += (double)(dy[(size_t)n * D + i] * ((i & 1) ? -sinf(a) : cosf(a))) * (double)tv;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += red[i];
        dw[wi] += (float)t;
    }
}

// ---- standalone dropout (inputs / embeddings / speaker embeddings): reference F.dropout call sites
// deepvoice3.py:75,80,294,321,588,597 ; same call with the same (seed, salt) is its own backward.
__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float p,
                               const unsigned long long* __restrict__ seed_ptr, unsigned salt) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const DropCfg d = make_drop(p, seed_ptr, salt);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        y[i] = x[i] * drop_scale(d, (uint32_t)i);
}

// ---- masked row softmax (+ dropout): reference deepvoice3.py:145-148,161-165 ------------------------
// s (rows, L) scores; mask (B, L) bytes (1 = padding -> -inf) or null, row r belongs to batch r / rows_per_b.
// probs = softmax(s) (returned to the caller as the alignment), pd = dropout(probs) (fed to P.V).
__global__ void softmax_fwd_kernel(const float* __restrict__ s, const unsigned char* __restrict__ mask,
                                   float* __restrict__ probs, float* __restrict__ pd, int rows, int L,
                                   int rows_per_b, float p, const unsigned long long* __restrict__ seed_ptr,
                                   unsigned salt) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (r >= rows) return;
    const DropCfg d = make_drop(p, seed_ptr, salt);
    const float* row = s + (size_t)r * L;
    const unsigned char* mrow = mask ? mask + (size_t)(r / rows_per_b) * L : nullptr;
    float mx = -INFINITY;
    for (int i = lane; i < L; i += 32) {
        const float v = (mrow && mrow[i]) ? -INFINITY : row[i];
        mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int i = lane; i < L; i += 32) {
        const float v = (mrow && mrow[i]) ? -INFINITY : row[i];
        sum += expf(v - mx);
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int i = lane; i < L; i += 32) {
        const float v = (mrow && mrow[i]) ? -INFINITY : row[i];
        const float pr = expf(v - mx) * inv;
        const size_t idx = (size_t)r * L + i;
        probs[idx] = pr;
        if (pd) pd[idx] = pr * drop_scale(d, (uint32_t)idx);
    }
}
// ds = P * (dPt - sum(dPt*P)),  dPt = dpd * dropmask + dprobs_ext (gradient arriving at the returned alignment)
__global__ void softmax_bwd_kernel(const float* __restrict__ probs, const float* __restrict__ dpd,
                                   const float* __restrict__ dprobs_ext, float* __restrict__ ds, int rows,
                                   int L, float p, const unsigned long long* __restrict__ seed_ptr,
                                   unsigned salt) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (r >= rows) return;
    const DropCfg d = make_drop(p, seed_ptr, salt);
    float dot = 0.f;
    for (int i = lane; i < L; i += 32) {
        const size_t idx = (size_t)r * L + i;
        float g = dpd ? dpd[idx] * drop_scale(d, (uint32_t)idx) : 0.f;
        if (dprobs_ext) g += dprobs_ext[idx];
        dot = fmaf(g, probs[idx], dot);
    }
    dot = warp_sum(dot);
    for (int i = lane; i < L; i += 32) {
        const size_t idx = (size_t)r * L + i;
        float g = dpd ? dpd[idx] * drop_scale(d, (uint32_t)idx) : 0.f;
        if (dprobs_ext) g += dprobs_ext[idx];
        ds[idx] = probs[idx] * (g - dot);
    }
}

// ---- ConvTranspose1d(k=2, s=2) time interleave: reference deepvoice3.py:519,527 ; nyanko.py:372,377 ----
// in (B, 2*C, T) rows ordered (j, co)  <->  out (B, C, 2T) with out[b,co,2t+j] = in[b, j*C+co, t]
__global__ void interleave2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int T,
                                   int inverse) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const long long total = (long long)B * C * 2 * T;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(i % (2 * T));
        const long long bc = i / (2 * T);
        const int c = (int)(bc % C), b = (int)(bc / C);
        const int t = u >> 1, j = u & 1;
        const size_t packed = ((size_t)b * 2 * C + (size_t)j * C + c) * T + t;
        if (!inverse) out[i] = in[packed];
        else out[packed] = in[i];
    }
}

// y = x with y[b,:,t] = 0 for t >= mult*lengths[b * len_stride]   (B,C,T); x == y allowed.  len_stride 0: one length
// for every row (the logical extent of a batch padded to a bucket).
__global__ void mask_time_kernel(const float* x, float* y, const long long* __restrict__ lengths, int len_stride,
                                 int mult, int C, int T, long long total) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const int b = (int)(i / ((long long)C * T));
        y[i] = (long long)t < (long long)mult * lengths[(long long)b * len_stride] ? x[i] : 0.f;
    }
}

}  // namespace dv3

using namespace dv3;

static inline int ew_blocks(long long n, int threads) {
    long long b = (n + threads - 1) / threads;
    return (int)(b > 132 * 16 ? 132 * 16 : (b < 1 ? 1 : b));
}

extern "C" {

int dv3_transpose(const float* in, float* out, int B, int R, int C, void* stream) {
    DV3_REQUIRE(B <= 65535, "transpose: batch %d > 65535", B);
    launch_k(transpose_kernel, dim3(ceil_div(C, 32), ceil_div(R, 32), B), dim3(32, 8), 0, (cudaStream_t)stream, 
        in, out, R, C);
    return check_launch("transpose");
}

int dv3_embedding_fwd(const long long* ids, const float* table, float* out, int N, int D, int V, int* err_flag,
                      void* stream) {
    launch_k(embedding_fwd_kernel, ceil_div(N * 32, 256), 256, 0, (cudaStream_t)stream, ids, table, out, N, D, V,
                                                                                 err_flag);
    return check_launch("embedding_fwd");
}
int dv3_embedding_bwd(const long long* ids, const float* dy, float* dtable, int N, int D, int V,
                      long long padding_idx, void* stream) {
    launch_k(embedding_bwd_kernel, ceil_div(N * 32, 256), 256, 0, (cudaStream_t)stream, ids, dy, dtable, N, D, V,
                                                                                 padding_idx);
    return check_launch("embedding_bwd");
}

int dv3_sinusoid_fwd(const long long* pos, const float* table, const float* w, int nw, float* out, int B, int T,
                     int D, int P, int* err_flag, void* stream) {
    DV3_REQUIRE(nw == 1 || nw == B, "sinusoid_fwd: need 1 or B position rates, got %d", nw);
    launch_k(sinusoid_fwd_kernel, ceil_div(B * T * 32, 256), 256, 0, (cudaStream_t)stream, pos, table, w, nw, out, B,
                                                                                    T, D, P, err_flag);
    return check_launch("sinusoid_fwd");
}
int dv3_sinusoid_bwd(const long long* pos, const float* table, const float* w, int nw, const float* dy,
                     float* dtable, float* dw, int B, int T, int D, int P, void* stream) {
    if (dtable) {
        launch_k(sinusoid_bwd_kernel, ceil_div(B * T * 32, 256), 256, 0, (cudaStream_t)stream, pos, table, w, nw, dy,
                 dtable, B, T, D, P);
        if (int e = check_launch("sinusoid_bwd(table)")) return e;
    }
    if (dw) {
        launch_k(sinusoid_dw_kernel, nw, 256, 0, (cudaStream_t)stream, pos, table, w, nw, dy, dw, B, T, D, P);
        if (int e = check_launch("sinusoid_bwd(rate)")) return e;
    }
    return 0;
}

// Deterministic forms of the two table gradients (table_bwd_det_kernel): same values term for term, summed in token order.
int dv3_embedding_bwd_det(const long long* ids, const float* dy, float* dtable, int N, int D, int V,
                          long long padding_idx, void* stream) {
    DV3_REQUIRE(D >= 1 && D <= TABLE_DET_MAX_D && V >= 1, "embedding_bwd_det: D=%d not in [1,%d]", D, TABLE_DET_MAX_D);
    launch_k(table_bwd_det_kernel<false>, V, 256, 0, (cudaStream_t)stream, ids, (const float*)nullptr,
             (const float*)nullptr, 1, 1, dy, dtable, N, D, padding_idx);
    return check_launch("embedding_bwd_det");
}
int dv3_sinusoid_bwd_det(const long long* pos, const float* table, const float* w, int nw, const float* dy,
                         float* dtable, float* dw, int B, int T, int D, int P, void* stream) {
    DV3_REQUIRE(nw == 1 || nw == B, "sinusoid_bwd_det: need 1 or B position rates, got %d", nw);
    if (dtable) {
        DV3_REQUIRE(D >= 1 && D <= TABLE_DET_MAX_D && P >= 1, "sinusoid_bwd_det: D=%d not in [1,%d]", D, TABLE_DET_MAX_D);
        launch_k(table_bwd_det_kernel<true>, P, 256, 0, (cudaStream_t)stream, pos, table, w, nw, T, dy, dtable, B * T,
                 D, 0LL);
        if (int e = check_launch("sinusoid_bwd_det(table)")) return e;
    }
    if (dw) {       // already a fixed-order, one-CTA reduction
        launch_k(sinusoid_dw_kernel, nw, 256, 0, (cudaStream_t)stream, pos, table, w, nw, dy, dw, B, T, D, P);
        if (int e = check_launch("sinusoid_bwd_det(rate)")) return e;
    }
    return 0;
}

int dv3_dropout(const float* x, float* y, long long n, float p, const unsigned long long* seed_ptr, unsigned salt,
                void* stream) {
    DV3_REQUIRE(n < (1LL << 32), "dropout: tensor too large");
    launch_k(dropout_kernel, ew_blocks(n, 256), 256, 0, (cudaStream_t)stream, x, y, n, p, seed_ptr, salt);
    return check_launch("dropout");
}

int dv3_softmax_fwd(const float* s, const unsigned char* mask, float* probs, float* pd, int rows, int L,
                    int rows_per_b, float p, const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    launch_k(softmax_fwd_kernel, ceil_div(rows * 32, 256), 256, 0, (cudaStream_t)stream, s, mask, probs, pd, rows, L,
                                                                                  rows_per_b, p, seed_ptr, salt);
    return check_launch("softmax_fwd");
}
int dv3_softmax_bwd(const float* probs, const float* dpd, const float* dprobs_ext, float* ds, int rows, int L,
                    float p, const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    launch_k(softmax_bwd_kernel, ceil_div(rows * 32, 256), 256, 0, (cudaStream_t)stream, probs, dpd, dprobs_ext, ds,
                                                                                  rows, L, p, seed_ptr, salt);
    return check_launch("softmax_bwd");
}

int dv3_interleave2(const float* in, float* out, int B, int C, int T, int inverse, void* stream) {
    launch_k(interleave2_kernel, ew_blocks((long long)B * C * 2 * T, 256), 256, 0, (cudaStream_t)stream, in, out, B, C,
                                                                                                  T, inverse);
    return check_launch("interleave2");
}

int dv3_mask_time(const float* x, float* y, const long long* lengths, int mult, int B, int C, int T, void* stream) {
    DV3_REQUIRE(B >= 1 && C >= 1 && T >= 1 && mult >= 1, "mask_time: bad shape");
    const long long total = (long long)B * C * T;
    launch_k(mask_time_kernel, ew_blocks(total, 256), 256, 0, (cudaStream_t)stream, x, y, lengths, 1, mult, C, T, total);
    return check_launch("mask_time");
}

int dv3_mask_frames(const float* x, float* y, const long long* extent, int mult, int B, int C, int T, void* stream) {
    DV3_REQUIRE(B >= 1 && C >= 1 && T >= 1 && mult >= 1 && extent != nullptr, "mask_frames: bad arguments");
    const long long total = (long long)B * C * T;
    launch_k(mask_time_kernel, ew_blocks(total, 256), 256, 0, (cudaStream_t)stream, x, y, extent, 0, mult, C, T, total);
    return check_launch("mask_frames");
}

}  // extern "C"
