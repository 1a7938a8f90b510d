// Autoregressive (incremental) decoding, one time step per launch sequence -- reference conv.py:17-46
// (Conv1d.incremental_forward: ring buffer of the last (k-1)*dilation+1 inputs x linearised weight),
// modules.py:145-167 / 200-226 (gate epilogues on a (B,1,C) slice), deepvoice3.py:132-176 (attention with the
// monotonic window) and the decoder loops deepvoice3.py:367-485 / nyanko.py:250-338.
//
// Design: a decoder step is ~40 dependent matrix-VECTOR products (B is 1..16, M = 1), i.e. pure weight
// streaming out of L2 (the 10-25 MB of decoder weights stay resident in the 50 MB L2) and launch latency.  So the
// step is a fixed sequence of small kernels with ALL loop state in device memory -- the step counter t, the ring
// buffers, the monotonic-attention cursor, the output arrays indexed by t -- which makes the sequence identical
// from step to step: the host captures it once in a CUDA graph and replays it, checking the done flags only every
// few steps.  Every pointer of a step record can advance by a per-step stride (x + b*ld + t*t_stride), so frames /
// decoder states / alignments are written in place and teacher-forced inputs are read in place.
// Arithmetic is exact fp32 (fmaf accumulation, one warp per output channel).
#include "common.cuh"
#include "../../include/dv3b200.h"

namespace dv3 {

constexpr float kSqrtHalf = 0.70710678118654752f;
constexpr int kAttnScratch = 9;    // floats of reduction scratch ahead of q and the scores in the attention step

// step index of row b: one shared counter t_ptr[0], or (SLOTS) one counter per row t_ptr[b]
template <bool SLOTS>
__device__ __forceinline__ long long step_of(const int* t_ptr, int b) {
    return t_ptr ? (long long)t_ptr[SLOTS ? b : 0] : 0;
}

// ring slot of the input of time t - back (the ring is zero-initialised, so times before the start read zeros)
__device__ __forceinline__ int ring_slot(long long t, long long back, int L) {
    const long long tj = t - back;
    return (int)(((tj % L) + L) % L);
}

// one warp per output channel c (GLU / highway: rows c and C + c); BT batch rows per pass.
// SLOTS: every row has its own step counter t_ptr[b] (continuous batching), so the ring slot of each tap, the filing
// slot and every per-step stride are per row; the fmaf chain of each output is the same as with the shared counter.
template <int BT, bool SLOTS>
__global__ void __launch_bounds__(256) inc_conv_step_kernel(const __grid_constant__ Dv3IncStep p) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int gated = p.mode != 0;
    const int C = gated ? p.Cout / 2 : p.Cout;
    const long long t0 = step_of<false>(p.t_ptr, 0);      // the shared counter (unused with SLOTS)
    const int k = p.k, Cin = p.Cin, L = (k - 1) * p.dilation + 1;
    if (warp < C) {
        const int c = warp;
        const float* __restrict__ wa = p.w + (size_t)c * k * Cin;
        const float* __restrict__ wb = p.w + (size_t)(C + c) * k * Cin;
        for (int b0 = 0; b0 < p.B; b0 += BT) {
            float acc_a[BT], acc_b[BT];
            long long tr[BT];                                // step of each row of this pass
#pragma unroll
            for (int i = 0; i < BT; ++i) {
                acc_a[i] = 0.f; acc_b[i] = 0.f;
                tr[i] = SLOTS ? (b0 + i < p.B ? step_of<true>(p.t_ptr, b0 + i) : 0) : t0;
            }
            for (int j = 0; j < k; ++j) {
                const bool cur = (j == k - 1);
                // tap j sees the input of time t - (k-1-j)*dilation; older than the sequence start = zero (ring is
                // zero-initialised), the current input comes straight from x (+ add)
                const long long back = (long long)(k - 1 - j) * p.dilation;
                const int slot0 = cur || SLOTS ? 0 : ring_slot(t0, back, L);
                int slots[BT];
#pragma unroll
                for (int i = 0; i < BT; ++i) slots[i] = cur || !SLOTS ? slot0 : ring_slot(tr[i], back, L);
                const float* wja = wa + (size_t)j * Cin;
                const float* wjb = wb + (size_t)j * Cin;
                if (p.vec4) {
                    for (int ci = lane * 4; ci < Cin; ci += 128) {
                        const float4 a4 = *reinterpret_cast<const float4*>(wja + ci);
                        float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (gated) b4 = *reinterpret_cast<const float4*>(wjb + ci);
#pragma unroll
                        for (int i = 0; i < BT; ++i) {
                            const int b = b0 + i;
                            if (b >= p.B) break;
                            const long long t = tr[i];
                            float4 x4;
                            if (cur) {
                                x4 = *reinterpret_cast<const float4*>(p.x + b * p.x_ld + t * p.x_t + ci);
                                if (p.add) {
                                    const float4 e4 = *reinterpret_cast<const float4*>(p.add + b * p.add_ld + t * p.add_t + ci);
                                    x4.x += e4.x; x4.y += e4.y; x4.z += e4.z; x4.w += e4.w;
                                }
                            } else {
                                x4 = *reinterpret_cast<const float4*>(p.ring + ((size_t)b * L + slots[i]) * Cin + ci);
                            }
                            acc_a[i] = fmaf(a4.x, x4.x, acc_a[i]); acc_a[i] = fmaf(a4.y, x4.y, acc_a[i]);
                            acc_a[i] = fmaf(a4.z, x4.z, acc_a[i]); acc_a[i] = fmaf(a4.w, x4.w, acc_a[i]);
                            if (gated) {
                                acc_b[i] = fmaf(b4.x, x4.x, acc_b[i]); acc_b[i] = fmaf(b4.y, x4.y, acc_b[i]);
                                acc_b[i] = fmaf(b4.z, x4.z, acc_b[i]); acc_b[i] = fmaf(b4.w, x4.w, acc_b[i]);
                            }
                        }
                    }
                } else {
                    for (int ci = lane; ci < Cin; ci += 32) {
                        const float a1 = wja[ci];
                        const float b1 = gated ? wjb[ci] : 0.f;
#pragma unroll
                        for (int i = 0; i < BT; ++i) {
                            const int b = b0 + i;
                            if (b >= p.B) break;
                            const long long t = tr[i];
                            float xv;
                            if (cur) {
                                xv = p.x[b * p.x_ld + t * p.x_t + ci];
                                if (p.add) xv += p.add[b * p.add_ld + t * p.add_t + ci];
                            } else {
                                xv = p.ring[((size_t)b * L + slots[i]) * Cin + ci];
                            }
                            acc_a[i] = fmaf(a1, xv, acc_a[i]);
                            if (gated) acc_b[i] = fmaf(b1, xv, acc_b[i]);
                        }
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < BT; ++i) {
                const int b = b0 + i;
                if (b >= p.B) break;                       // uniform across the warp
                const long long t = tr[i];
                float a = warp_sum(acc_a[i]);
                float g = gated ? warp_sum(acc_b[i]) : 0.f;
                if (lane != 0) continue;
                a += p.bias[c];
                float y;
                if (p.mode == 0) {
                    y = a;
                    if (p.act == 1) y = fmaxf(y, 0.f);
                    else if (p.act == 2) y = sigmoidf_(y);
                } else {
                    g += p.bias[C + c];
                    const float s = sigmoidf_(g);
                    const float xin = p.x[b * p.x_ld + t * p.x_t + c];      // gated blocks: Cin == C
                    if (p.mode == 1) {
                        if (p.spk) a += p.spk[b * p.spk_ld + c];
                        y = a * s;
                    } else {
                        y = s * a + (1.f - s) * xin;
                    }
                }
                if (p.res1) y = (y + p.res1[b * p.res1_ld + t * p.res1_t + c]) * kSqrtHalf;
                if (p.res2) y = (y + p.res2[b * p.res2_ld + t * p.res2_t + c]) * kSqrtHalf;
                p.y[b * p.y_ld + t * p.y_t + c] = y;
                if (p.y2) {
                    float y2 = y;
                    if (p.y2_mode == 1) y2 = sigmoidf_(y);
                    else if (p.y2_mode == 2) y2 = y + p.yadd[b * p.yadd_ld + t * p.yadd_t + c];
                    p.y2[b * p.y2_ld + t * p.y2_t + c] = y2;
                }
            }
        }
    }
    // the last CTA also files the current input into the ring (slot t mod L is not read by anybody this step)
    if (p.ring && blockIdx.x == gridDim.x - 1) {
        for (int i = threadIdx.x; i < p.B * Cin; i += blockDim.x) {
            const int b = i / Cin, ci = i - b * Cin;
            const long long t = SLOTS ? step_of<true>(p.t_ptr, b) : t0;
            const int slot_now = (int)(t % L);
            float xv = p.x[b * p.x_ld + t * p.x_t + ci];
            if (p.add) xv += p.add[b * p.add_ld + t * p.add_t + ci];
            p.ring[((size_t)b * L + slot_now) * Cin + ci] = xv;
        }
    }
}

// one CTA per batch row: scores = q . keys, monotonic window, softmax, context = probs . values * float(Ts*sqrt(1/Ts)).
// ROWS (ragged batch): row b sees only its own Ts = text_len[b] keys (the key pitch stays p.Ts) and keeps its own
// cursor; with Ts substituted, the arithmetic is that of the single-row launch, so each row matches it bit for bit.
// SLOTS (with ROWS): row b runs at its own step t_ptr[b] -- alignment row and cursor parity follow it.
// PATH (with ROWS): guided attention -- the window's centre is the prescribed token path[b*path_ld + t] instead of the
// previous step's argmax, and no cursor is written; everything else is the ROWS arithmetic.
template <bool ROWS, bool SLOTS, bool PATH>
__global__ void __launch_bounds__(256) inc_attn_step_kernel(const __grid_constant__ Dv3IncAttn p, const int* text_len,
                                                            const int* path, long long path_ld) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    extern __shared__ float sm[];  // all of it dynamic, so the host's size check is the whole budget
    float* red = sm;               // [kAttnScratch]: 8 per-warp partials + the broadcast slot red[8]
    float* q = sm + kAttnScratch;  // [E]
    float* sc = q + p.E;           // [Ts]
    float& bcast = red[8];
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long t = step_of<SLOTS>(p.t_ptr, b);
    const int Ts = ROWS ? text_len[b] : p.Ts;
    // cursor slots: [2] (row 0 leads every row, reference deepvoice3.py:443) or [2][B] (one per row)
    const int cur_rd = ROWS ? (int)(t & 1) * p.B + b : (int)(t & 1);
    const int cur_wr = ROWS ? (int)((t + 1) & 1) * p.B + b : (int)((t + 1) & 1);
    for (int e = tid; e < p.E; e += 256) q[e] = p.q[b * p.q_ld + e];
    __syncthreads();
    int lo = 0, hi = Ts;                                    // unmasked key range
    if (PATH || p.last_attended) {
        const int la = PATH ? path[b * path_ld + t] : p.last_attended[cur_rd];
        const int backward = la - p.window_backward;
        if (backward > 0) lo = backward;
        const int ahead = la + p.window_ahead;
        if (ahead < Ts) hi = ahead;
    }
    const float* __restrict__ K = p.keys + (size_t)b * p.E * p.Ts;
    float mx = -INFINITY;
    for (int s = tid; s < Ts; s += 256) {
        float acc = 0.f;
        for (int e = 0; e < p.E; ++e) acc = fmaf(q[e], K[(size_t)e * p.Ts + s], acc);
        if (s < lo || s >= hi) acc = -INFINITY;
        sc[s] = acc;
        mx = fmaxf(mx, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    __syncthreads();
    if (tid == 0) { float m = red[0]; for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]); bcast = m; }
    __syncthreads();
    mx = bcast;
    float sum = 0.f;
    for (int s = tid; s < Ts; s += 256) { const float e = expf(sc[s] - mx); sc[s] = e; sum += e; }
    sum = warp_sum(sum);
    __syncthreads();                                        // everybody has read bcast
    if ((tid & 31) == 0) red[tid >> 5] = sum;
    __syncthreads();
    if (tid == 0) { float s = 0.f; for (int i = 0; i < 8; ++i) s += red[i]; bcast = s; }
    __syncthreads();
    const float inv = 1.f / bcast;
    for (int s = tid; s < Ts; s += 256) {
        const float pr = sc[s] * inv;
        sc[s] = pr;
        if (p.align) p.align[b * p.align_ld + t * p.align_t + s] = pr * p.align_scale;
    }
    if (ROWS && p.align)
        for (int s = Ts + tid; s < p.Ts; s += 256) p.align[b * p.align_ld + t * p.align_t + s] = 0.f;
    __syncthreads();
    if (!PATH && p.last_attended && (ROWS || b == 0) && tid == 0) {  // reference: alignment.max(-1)[1] of batch row 0
        int best = 0; float bv = sc[0];
        for (int s = 1; s < Ts; ++s) if (sc[s] > bv) { bv = sc[s]; best = s; }
        p.last_attended[cur_wr] = best;
    }
    const float* __restrict__ V = p.values + (size_t)b * p.Ts * p.E;
    const float scale = context_scale(Ts);                  // float(Ts*sqrt(1/Ts)) rounded once, as the reference
    for (int e = tid; e < p.E; e += 256) {
        float acc = 0.f;
        for (int s = 0; s < Ts; ++s) acc = fmaf(sc[s], V[(size_t)s * p.E + e], acc);
        p.ctx[b * p.ctx_ld + e] = acc * scale;
    }
}

__global__ void inc_advance_kernel(int* t) {
    pdl_trigger(); pdl_wait(); *t += 1; }

// per-row counters: a row that has stopped (stop[b] != 0) keeps its step, so it recomputes that same step -- the
// same inputs give the same bits, and no row ever writes past frame max_decoder_steps + 1
__global__ void inc_advance_rows_kernel(int* t, const int* stop, int B) {
    pdl_trigger(); pdl_wait();
    for (int b = threadIdx.x; b < B; b += blockDim.x)
        if (!stop || stop[b] == 0) t[b] += 1;
}

// the reference stop rule (incremental._stop_step) on each row alone, after step t[b] wrote done[b*done_ld + t[b]]:
// n = t[b] + 1 steps ran; stop after them if done > 0.5 and n > min_steps, or if n > max_steps.  Written once.
__global__ void inc_stop_rows_kernel(const float* done, long long done_ld, const int* t, int* stop, int B,
                                     int min_steps, int max_steps) {
    pdl_trigger(); pdl_wait();
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        if (stop[b] != 0) continue;
        const int n = t[b] + 1;
        if ((done[b * done_ld + t[b]] > 0.5f && n > min_steps) || n > max_steps) stop[b] = n;
    }
}

// guided decoding: row b stops once t[b] + 1 reaches its prescribed step count total[b]; the done flag plays no part.
// Rows that are idle (stop[b] = -1) or stopped keep their value.  Written once.
__global__ void inc_stop_rows_total_kernel(const int* t, int* stop, const int* total, int B) {
    pdl_trigger(); pdl_wait();
    for (int b = threadIdx.x; b < B; b += blockDim.x)
        if (stop[b] == 0 && t[b] + 1 >= total[b]) stop[b] = t[b] + 1;
}

// entry e, slot list index i: row slots[i] of e.dst <- row i of e.src (zeros when e.src is NULL), in 4-byte words
__global__ void __launch_bounds__(256) inc_refill_kernel(const Dv3IncRefill* table, const int* slots) {
    pdl_trigger(); pdl_wait();
    const Dv3IncRefill e = table[blockIdx.y];
    const int i = blockIdx.z, b = slots[i];
    int* dst = reinterpret_cast<int*>(reinterpret_cast<char*>(e.dst) + (size_t)b * e.dst_row_stride);
    const int* src = e.src ? reinterpret_cast<const int*>(reinterpret_cast<const char*>(e.src) +
                                                          (size_t)i * e.src_row_stride) : nullptr;
    const long long n = e.row_bytes / 4;
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < n; w += (long long)gridDim.x * blockDim.x)
        dst[w] = src ? src[w] : 0;
}

}  // namespace dv3

using namespace dv3;

// dynamic shared memory of the attention step: the reduction scratch, q and the scores (the kernel has no static part)
static size_t attn_smem(const Dv3IncAttn* p) { return (size_t)(kAttnScratch + p->E + p->Ts) * sizeof(float); }
static constexpr int kAttnMaxKeys = 48 * 1024 / (int)sizeof(float) - kAttnScratch;    // largest E + Ts

extern "C" {

int dv3_inc_conv_step(const Dv3IncStep* p, void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->Cin > 0 && p->Cout > 0 && p->k >= 1 && p->dilation >= 1,
                "inc_conv_step: bad shape");
    DV3_REQUIRE(p->mode == 0 || (p->Cout == 2 * p->Cin), "inc_conv_step: gated blocks need Cout == 2*Cin");
    DV3_REQUIRE(p->k == 1 || p->ring != nullptr, "inc_conv_step: k > 1 needs a ring buffer");
    const int C = p->mode != 0 ? p->Cout / 2 : p->Cout;
    const int blocks = (C * 32 + 255) / 256;
    cudaStream_t st = (cudaStream_t)stream;
    if (p->B == 1) launch_k(inc_conv_step_kernel<1, false>, blocks, 256, 0, st, *p);
    else if (p->B == 2) launch_k(inc_conv_step_kernel<2, false>, blocks, 256, 0, st, *p);
    else launch_k(inc_conv_step_kernel<4, false>, blocks, 256, 0, st, *p);
    return check_launch("inc_conv_step");
}

int dv3_inc_conv_step_slots(const Dv3IncStep* p, void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->Cin > 0 && p->Cout > 0 && p->k >= 1 && p->dilation >= 1,
                "inc_conv_step_slots: bad shape");
    DV3_REQUIRE(p->mode == 0 || (p->Cout == 2 * p->Cin), "inc_conv_step_slots: gated blocks need Cout == 2*Cin");
    DV3_REQUIRE(p->k == 1 || p->ring != nullptr, "inc_conv_step_slots: k > 1 needs a ring buffer");
    DV3_REQUIRE(p->t_ptr != nullptr, "inc_conv_step_slots: needs the per-row step counters t_ptr[B]");
    const int C = p->mode != 0 ? p->Cout / 2 : p->Cout;
    const int blocks = (C * 32 + 255) / 256;
    cudaStream_t st = (cudaStream_t)stream;
    if (p->B == 1) launch_k(inc_conv_step_kernel<1, true>, blocks, 256, 0, st, *p);
    else if (p->B == 2) launch_k(inc_conv_step_kernel<2, true>, blocks, 256, 0, st, *p);
    else launch_k(inc_conv_step_kernel<4, true>, blocks, 256, 0, st, *p);
    return check_launch("inc_conv_step_slots");
}

int dv3_inc_attn_step(const Dv3IncAttn* p, void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->E > 0 && p->Ts > 0, "inc_attn_step: bad shape");
    const size_t smem = attn_smem(p);
    DV3_REQUIRE(smem <= 48 * 1024, "inc_attn_step: E + Ts = %d floats exceed the %d that fit in 48 KB of shared memory",
                p->E + p->Ts, kAttnMaxKeys);
    launch_k(inc_attn_step_kernel<false, false, false>, p->B, 256, smem, (cudaStream_t)stream, *p, (const int*)nullptr,
             (const int*)nullptr, 0LL);
    return check_launch("inc_attn_step");
}

int dv3_inc_attn_step_rows(const Dv3IncAttn* p, const int* text_len, void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->E > 0 && p->Ts > 0 && text_len, "inc_attn_step_rows: bad shape");
    const size_t smem = attn_smem(p);
    DV3_REQUIRE(smem <= 48 * 1024, "inc_attn_step_rows: E + Ts = %d floats exceed the %d that fit in 48 KB of shared memory",
                p->E + p->Ts, kAttnMaxKeys);
    launch_k(inc_attn_step_kernel<true, false, false>, p->B, 256, smem, (cudaStream_t)stream, *p, text_len,
             (const int*)nullptr, 0LL);
    return check_launch("inc_attn_step_rows");
}

int dv3_inc_attn_step_slots(const Dv3IncAttn* p, const int* text_len, void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->E > 0 && p->Ts > 0 && text_len && p->t_ptr, "inc_attn_step_slots: bad shape");
    const size_t smem = attn_smem(p);
    DV3_REQUIRE(smem <= 48 * 1024, "inc_attn_step_slots: E + Ts = %d floats exceed the %d that fit in 48 KB of shared memory",
                p->E + p->Ts, kAttnMaxKeys);
    launch_k(inc_attn_step_kernel<true, true, false>, p->B, 256, smem, (cudaStream_t)stream, *p, text_len,
             (const int*)nullptr, 0LL);
    return check_launch("inc_attn_step_slots");
}

int dv3_inc_attn_step_path(const Dv3IncAttn* p, const int* text_len, const int* path, long long path_ld,
                           void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->E > 0 && p->Ts > 0 && text_len && path && path_ld >= 1,
                "inc_attn_step_path: bad shape");
    const size_t smem = attn_smem(p);
    DV3_REQUIRE(smem <= 48 * 1024, "inc_attn_step_path: E + Ts = %d floats exceed the %d that fit in 48 KB of shared memory",
                p->E + p->Ts, kAttnMaxKeys);
    launch_k(inc_attn_step_kernel<true, false, true>, p->B, 256, smem, (cudaStream_t)stream, *p, text_len, path,
             path_ld);
    return check_launch("inc_attn_step_path");
}

int dv3_inc_attn_step_slots_path(const Dv3IncAttn* p, const int* text_len, const int* path, long long path_ld,
                                 void* stream) {
    DV3_REQUIRE(p && p->B > 0 && p->E > 0 && p->Ts > 0 && text_len && p->t_ptr && path && path_ld >= 1,
                "inc_attn_step_slots_path: bad shape");
    const size_t smem = attn_smem(p);
    DV3_REQUIRE(smem <= 48 * 1024,
                "inc_attn_step_slots_path: E + Ts = %d floats exceed the %d that fit in 48 KB of shared memory",
                p->E + p->Ts, kAttnMaxKeys);
    launch_k(inc_attn_step_kernel<true, true, true>, p->B, 256, smem, (cudaStream_t)stream, *p, text_len, path,
             path_ld);
    return check_launch("inc_attn_step_slots_path");
}

int dv3_inc_advance(int* t_ptr, void* stream) {
    launch_k(inc_advance_kernel, 1, 1, 0, (cudaStream_t)stream, t_ptr);
    return check_launch("inc_advance");
}

int dv3_inc_advance_rows(int* t, const int* stop, int B, void* stream) {
    DV3_REQUIRE(t && B > 0 && B <= 1024, "inc_advance_rows: bad shape (B = %d)", B);
    launch_k(inc_advance_rows_kernel, 1, B, 0, (cudaStream_t)stream, t, stop, B);
    return check_launch("inc_advance_rows");
}

int dv3_inc_stop_rows(const float* done, long long done_ld, const int* t, int* stop, int B, int min_steps,
                      int max_steps, void* stream) {
    DV3_REQUIRE(done && t && stop && B > 0 && B <= 1024 && done_ld > max_steps, "inc_stop_rows: bad shape");
    launch_k(inc_stop_rows_kernel, 1, B, 0, (cudaStream_t)stream, done, done_ld, t, stop, B, min_steps, max_steps);
    return check_launch("inc_stop_rows");
}

int dv3_inc_stop_rows_total(const int* t, int* stop, const int* total, int B, void* stream) {
    DV3_REQUIRE(t && stop && total && B > 0 && B <= 1024, "inc_stop_rows_total: bad shape (B = %d)", B);
    launch_k(inc_stop_rows_total_kernel, 1, B, 0, (cudaStream_t)stream, t, stop, total, B);
    return check_launch("inc_stop_rows_total");
}

int dv3_inc_refill(const Dv3IncRefill* table, int n_entries, const int* slots, int n_slots, void* stream) {
    DV3_REQUIRE(table && slots && n_entries > 0 && n_entries <= 65535 && n_slots >= 0 && n_slots <= 65535,
                "inc_refill: bad table (%d entries, %d slots)", n_entries, n_slots);
    if (n_slots == 0) return 0;
    launch_k(inc_refill_kernel, dim3(16, n_entries, n_slots), 256, 0, (cudaStream_t)stream, table, slots);
    return check_launch("inc_refill");
}

}  // extern "C"
