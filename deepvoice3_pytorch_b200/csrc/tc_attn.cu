// Fused dot-product attention of the teacher-forced decoder on wgmma tensor cores -- reference
// deepvoice3.py:132-176 (AttentionLayer.forward between the projections):
//     S = Q.K^T (no 1/sqrt(d)) -> mask padded keys with -inf -> softmax over keys -> [return P] -> dropout
//       -> O = scale * Pd.V                                                     (scale = Ts * sqrt(1/Ts))
// and its backward.  Layouts are the channel-major ones the decoder already holds: q (B,E,Td), k, v (B,E,Ts),
// out (B,E,Td), probabilities (B,Td,Ts) (materialised: the guided-attention loss reads them, train.py:734-738).
//
// Arithmetic: fp32-equivalent split-bf16 (hi*hi in one register accumulator, hi*lo + lo*hi in a second one, summed
// in fp32 by the epilogue -- same scheme as tc_gemm.cu).  The fp32 operands are split INSIDE the kernel while they are
// staged into shared memory in the wgmma canonical layouts (there is no pre-pass and nothing but q/k/v/probs ever
// touches HBM):
//   * operands whose contraction index is the ROW of the global tensor (q, k, dO, v in the score GEMMs; P, dS in the
//     key/value-gradient GEMMs) are written MN-major: [contraction row][64 elements = 128 B], 16-byte chunk c of row
//     r at chunk position c ^ (r & 7) (SWIZZLE_128B), 64-element column groups 8 KB apart;
//   * operands whose contraction index is contiguous in memory (v, k in the context GEMMs; dO, q in the gradient
//     GEMMs; the softmax output, produced by the epilogue threads themselves) are written K-major: [row][64
//     contraction elements = 128 B], 8-row atoms of 1024 B, same XOR swizzle.
//
// Kernels (256 threads = two warpgroups; every output tile is 64 rows, one warpgroup's M, so that the grid has enough
// CTAs to spread over the SMs -- the problem is small and each CTA is a latency chain, not a throughput one):
//   attn_rows_kernel<BWD=0>  one CTA per (64 query rows, utterance): S GEMM (warpgroup w: keys [64 w, 64 w + 64)) ->
//                            softmax epilogue on all 8 warps (writes P, stages dropout(P) as the A operand of the
//                            second GEMM) -> O GEMM (warpgroup w: channels [128 w, 128 w + 128)) -> store.
//   attn_rows_kernel<BWD=1>  same skeleton for the backward: dPd = dO^T.V -> softmax backward epilogue (reads P and
//                            dprobs once, writes dS) -> dQ = dS.K^T.
//   attn_cols_kernel         one CTA per (64 channels, utterance, dV or dK): dV = scale * dO.Pd or dK = Q.dS; the
//                            contraction over the query axis stays inside the CTA (no reduction, no atomics), through
//                            a two-stage staging ring so that the loads of one query chunk run under the MMAs of the
//                            previous one.
#include "tc_common.cuh"

namespace dv3 {

using namespace tc;

constexpr int AT_THREADS = 256;
constexpr int AT_NS = 128;                 // key tile: Ts <= 128 (longer memories use the SIMT path)
constexpr int AT_RT = 64;                  // output rows per CTA

struct AttnParams {
    const float* a1;        // rows kernel: q (fwd) / dO (bwd), (B,E,Td)
    const float* b1;        // rows kernel: k (fwd) / v (bwd), (B,E,Ts)
    const float* b2;        // rows kernel: v (fwd) / k (bwd), (B,E,Ts)
    const unsigned char* mask;   // (B,Ts) 1 = padding, or null (fwd)
    float* probs;           // (B,Td,Ts): written by fwd, read by bwd
    const float* dprobs;    // bwd: gradient arriving at the returned probabilities, or null
    float* ds;              // bwd: dS (B,Td,Ts) out (consumed by attn_cols_kernel)
    float* out;             // (B,E,Td): context (fwd) / dq (bwd)
    int B, E, Td, Ts;
    float scale, p_drop;
    const unsigned long long* seed_ptr;
    uint32_t salt;
    const long long* ts_log;   // logical key count in device memory, or null: scale = ts_log * sqrt(1/ts_log) then
};

// 8 fp32 -> 8 bf16 hi (16 bytes) + 8 bf16 lo
__device__ __forceinline__ void split8(const float* x, uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(x[2 * i]), h1 = __float2bfloat16_rn(x[2 * i + 1]);
        const __nv_bfloat16 l0 = __float2bfloat16_rn(x[2 * i] - __bfloat162float(h0));
        const __nv_bfloat16 l1 = __float2bfloat16_rn(x[2 * i + 1] - __bfloat162float(h1));
        h[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        l[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// split 8 floats and store hi at dst, lo at dst + plane_bytes
__device__ __forceinline__ void store_split8(uint8_t* dst, uint32_t plane_bytes, const float* x) {
    uint4 hi, lo;
    split8(x, hi, lo);
    *reinterpret_cast<uint4*>(dst) = hi;
    *reinterpret_cast<uint4*>(dst + plane_bytes) = lo;
}

// 8 consecutive floats row[c0 .. c0+8) with bounds (cols >= ncols read as 0); vectorised when aligned
__device__ __forceinline__ void load8(const float* __restrict__ row, int c0, int ncols, bool row_ok, bool vec_ok,
                                      float* x) {
    if (row_ok && vec_ok && c0 + 8 <= ncols) {
        const float4 u = __ldg(reinterpret_cast<const float4*>(row + c0));
        const float4 w = __ldg(reinterpret_cast<const float4*>(row + c0 + 4));
        x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w; x[4] = w.x; x[5] = w.y; x[6] = w.z; x[7] = w.w;
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = (row_ok && c0 + i < ncols) ? __ldg(row + c0 + i) : 0.f;
    }
}

// Swizzled byte offsets of the 16-byte chunk holding elements [8c, 8c + 8) of row r: MN-major (64-element column
// groups 8 KB apart, c counts over all groups) and K-major (8-row atoms of 1024 B).
__device__ __forceinline__ uint32_t off_mn(int r, int c) {
    return (uint32_t)(c >> 3) * 8192u + (uint32_t)r * 128u + (uint32_t)(((c & 7) ^ (r & 7)) << 4);
}
__device__ __forceinline__ uint32_t off_k(int r, int c) {
    return (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u + (uint32_t)((c ^ (r & 7)) << 4);
}

// One staging round: every thread issues the global loads of its N 8-float groups (load(u, x)) before the first
// split and shared store (store(u, x)), so that N x 32 bytes per thread are in flight at once.
template <int N, typename Load, typename Store>
__device__ __forceinline__ void stage_round(Load load, Store store) {
    float x[N][8];
#pragma unroll
    for (int u = 0; u < N; ++u) load(u, x[u]);
#pragma unroll
    for (int u = 0; u < N; ++u) store(u, x[u]);
}

// Stage a K-major operand: nrows_tile rows (global rows r0.., row stride ld) x 64 contraction columns starting at c_base.
constexpr int ST_UNR = 8;
__device__ __forceinline__ void stage_k(uint8_t* dst, uint32_t plane_bytes, const float* __restrict__ src, long long ld,
                                        int r0, int nrows_valid, int nrows_tile, int c_base, int ncols, bool vec_ok,
                                        int tid) {
    const int total = nrows_tile * 8;
    for (int g0 = tid; g0 < total; g0 += AT_THREADS * ST_UNR) {
        stage_round<ST_UNR>(
            [&](int u, float* x) {
                const int g = g0 + u * AT_THREADS, r = g >> 3, c = g & 7;
                load8(src + (long long)(r0 + r) * ld, c_base + c * 8, ncols, g < total && r0 + r < nrows_valid, vec_ok, x);
            },
            [&](int u, float* x) {
                const int g = g0 + u * AT_THREADS;
                if (g < total) store_split8(dst + off_k(g >> 3, g & 7), plane_bytes, x);
            });
    }
}

__device__ __forceinline__ uint64_t desc_kmajor(uint32_t saddr) {            // [row][64 k] 128-byte rows, SWIZZLE_128B
    return make_wgmma_desc(saddr, 16, 1024, WG_SW128);
}
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t saddr, uint32_t lbo) {   // [k row][64 mn], chunk stride lbo
    return make_wgmma_desc(saddr, lbo, 1024, WG_SW128);
}

// 64 x N tile of one warpgroup: main (acc[0, N/2)) (+)= Ahi*Bhi ; cross (acc[N/2, N)) (+)= Ahi*Blo + Alo*Bhi
template <int N, int TA, int TB>
__device__ __forceinline__ void mma3(float* acc, uint64_t ahi, uint64_t alo, uint64_t bhi, uint64_t blo) {
    wgmma_mma<N, TA, TB>(true, acc, ahi, bhi, 1);
    wgmma_mma<N, TA, TB>(true, acc + N / 2, ahi, blo, 1);
    wgmma_mma<N, TA, TB>(true, acc + N / 2, alo, bhi, 1);
}

// The 64 x 128 GEMM with a query- or channel-axis contraction that both kernels start with: nk chunks of 64
// contraction elements, each staged by stage(kc, st) into one of two 48 KB stages
//     A hi 8 KB | A lo 8 KB | B hi 16 KB | B lo 16 KB      (A: 64 rows, MN-major if TA else K-major; B: MN-major,
//                                                           128 columns = two 64-column groups)
// while the MMAs of the previous chunk run.  Warpgroup wg accumulates columns [64 wg, 64 wg + 64) in acc[64].
constexpr int STAGE_BYTES = 49152;
constexpr int GEMM_GROUPS = 6;             // 8-float groups per thread and stage: (64 x 8 + 64 x 16) / 256
template <int TA, typename Stage>
__device__ __forceinline__ void gemm_64x128(float* acc, uint8_t* smem, int nk, int wg, Stage stage) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kc = 0; kc < nk; ++kc) {
        if (kc >= 2) __syncthreads();                       // both warpgroups retired the MMAs that read this stage
        uint8_t* st = smem + (kc & 1) * STAGE_BYTES;
        stage(kc, st);
        fence_proxy_async();
        __syncthreads();
        const uint32_t sa = smem_u32(st), sb = sa + 16384 + wg * 8192;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint32_t a = sa + (TA ? kk * 2048 : kk * 32), b = sb + kk * 2048;
            const uint64_t ahi = TA ? desc_mnmajor(a, 8192) : desc_kmajor(a);
            const uint64_t alo = TA ? desc_mnmajor(a + 8192, 8192) : desc_kmajor(a + 8192);
            mma3<64, TA, 1>(acc, ahi, alo, desc_mnmajor(b, 8192), desc_mnmajor(b + 16384, 8192));
        }
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
}

// Shared-memory map of attn_rows_kernel (bytes, after 1024-byte alignment):
//   [0, 128 KB)     GEMM 1 stages (2 x 48 KB), then B2: per key slab [hi E*128 | lo E*128]  (<= 2 x 64 KB)
//   RS_SC           scores ([64][SC_PITCH] fp32, summed accumulators), then the per-warp transposing tiles
//   RS_A2           A2 = the second GEMM's A operand: hi 16 KB | lo 16 KB (2 key slabs x 64 rows x 128 B)
//   RS_RED          row partials of the softmax reductions: [2][4 key quarters][64 rows] fp32
// The epilogue warps exchange 32 x 32 tiles with global memory through a per-warp transposing buffer: the thread of
// lane l owns ROW l of its warp's 32 x 32 block of the score tile, and a row of the (B,Td,Ts) probability tensors is
// contiguous along the keys -- a direct per-thread access touches 32 different 128-byte lines per warp instruction.
// Through the buffer every global access is one full 128-byte line per instruction.
constexpr int TILE_PITCH = 33;
constexpr int TILE_FLOATS = 32 * TILE_PITCH;
constexpr int SC_PITCH = AT_NS + 1;
constexpr int RS_SC = 131072;
constexpr int RS_A2 = RS_SC + 8 * TILE_FLOATS * 4;         // 8 tiles (33 KB) >= the scores (64 x 129 x 4 B)
constexpr int RS_RED = RS_A2 + 32768;
constexpr int ROWS_SMEM = RS_RED + 2 * 4 * AT_RT * 4 + 1024;
static_assert(AT_RT * SC_PITCH <= 8 * TILE_FLOATS, "scores and tiles share a region");
static_assert(RS_A2 % 1024 == 0, "A2 is a swizzled wgmma operand");

// global rows [0, rows_valid) x columns [c0, c0+32) of a row-major matrix (row stride ld) starting at src -> tile
__device__ __forceinline__ void tile_load(float* tile, const float* __restrict__ src, int ld, int rows_valid, int c0,
                                          int ncols, int lane) {
    __syncwarp();
    const bool cok = c0 + lane < ncols;
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr)
        tile[rr * TILE_PITCH + lane] = (cok && rr < rows_valid) ? __ldg(src + (size_t)rr * ld + c0 + lane) : 0.f;
    __syncwarp();
}
// tile -> global rows [0, rows_valid) x columns [c0, c0+32)
__device__ __forceinline__ void tile_store(const float* tile, float* __restrict__ dst, int ld, int rows_valid, int c0,
                                           int ncols, int lane) {
    __syncwarp();
    const bool cok = c0 + lane < ncols;
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr)
        if (cok && rr < rows_valid) dst[(size_t)rr * ld + c0 + lane] = tile[rr * TILE_PITCH + lane];
    __syncwarp();
}

// A row sum of the softmax epilogues, taken in key order as one sequential pass over the row: the warps of key
// quarter j continue, with step(value), from the value quarter j - 1 left in *slot.  Every thread of the CTA calls it
// (four barriers); it returns the whole row's value.  Keeping the one-pass order keeps each probability and dS the
// value a single thread per row computes -- the row sums near 1 that the softmax backward subtracts cancel to a few
// ulps, and a different order moves those ulps.
template <typename Step>
__device__ __forceinline__ float row_chain(float* slot, int kq, Step step) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (kq == j) *slot = step(j == 0 ? 0.f : *slot);
        __syncthreads();
    }
    return *slot;
}

template <int BWD>
__global__ void __launch_bounds__(AT_THREADS, 1) attn_rows_kernel(const __grid_constant__ AttnParams p) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3;
    const int b = blockIdx.y, t0 = blockIdx.x * AT_RT;
    const int E = p.E, Td = p.Td, Ts = p.Ts;
    const float* A1 = p.a1 + (size_t)b * E * Td;
    const float* B1 = p.b1 + (size_t)b * E * Ts;
    const float* B2 = p.b2 + (size_t)b * E * Ts;
    const bool vec_td = (Td & 3) == 0, vec_ts = (Ts & 3) == 0;
    float* sc = reinterpret_cast<float*>(smem + RS_SC);
    float* red = reinterpret_cast<float*>(smem + RS_RED);
    pdl_wait();                 // global memory from here on
    const float scale = p.ts_log ? context_scale(*p.ts_log) : p.scale;

    // ---------------- GEMM 1: D1[t][s] = sum_e A1[e][t0+t] * B1[e][s] -----------------------------------
    float acc1[64];
    gemm_64x128<1>(acc1, smem, (E + 63) / 64, wg, [&](int kc, uint8_t* st) {
        stage_round<GEMM_GROUPS>(
            [&](int u, float* x) {
                if (u < 2) {                                // A1: 64 channels x 64 query columns
                    const int g = tid + u * AT_THREADS, r = g >> 3, e = kc * 64 + r;
                    load8(A1 + (long long)e * Td, t0 + (g & 7) * 8, Td, e < E, vec_td, x);
                } else {                                    // B1: 64 channels x 128 keys
                    const int g = tid + (u - 2) * AT_THREADS, r = g >> 4, e = kc * 64 + r;
                    load8(B1 + (long long)e * Ts, (g & 15) * 8, Ts, e < E, vec_ts, x);
                }
            },
            [&](int u, float* x) {
                if (u < 2) {
                    const int g = tid + u * AT_THREADS;
                    store_split8(st + off_mn(g >> 3, g & 7), 8192, x);
                } else {
                    const int g = tid + (u - 2) * AT_THREADS;
                    store_split8(st + 16384 + off_mn(g >> 4, g & 15), 16384, x);
                }
            });
    });
#pragma unroll
    for (int i = 0; i < 32; ++i)
        sc[frag_row(i, wq, lane) * SC_PITCH + 64 * wg + frag_col(i, lane)] = acc1[i] + acc1[32 + i];
    __syncthreads();                                        // scores complete; every MMA retired: the stages are free

    // ---------------- B2 staging (into the GEMM 1 stages) ---------------------------------------------------------
    const int nslab = (Ts + 63) / 64;                       // 64-key slabs of the second contraction
    const uint32_t b2_plane = (uint32_t)E * 128u;           // one plane of one slab: E rows x 128 B
    for (int sl = 0; sl < nslab; ++sl)
        stage_k(smem + sl * 2 * b2_plane, b2_plane, B2, Ts, 0, E, E, sl * 64, Ts, vec_ts, tid);

    // ---------------- epilogue (all warps; warp = 32 rows x 32 keys, thread = one row of it) ------------------------
    {
        const int rh = warp & 1, kq = warp >> 1, c0 = 32 * kq;
        const int row = 32 * rh + lane, t = t0 + row;
        const bool tv = t < Td, live = c0 < Ts;             // live: uniform per warp
        const DropCfg drop = make_drop(p.p_drop, p.seed_ptr, p.salt);
        const size_t rbase = ((size_t)b * Td + (tv ? t : 0)) * Ts;
        float sv[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) sv[i] = sc[row * SC_PITCH + c0 + i];
        // key c0 + i is excluded (padding or beyond Ts) <=> bit i of mb
        const unsigned char* mrow = p.mask ? p.mask + (size_t)b * Ts : nullptr;
        const int sl_ = c0 + lane;
        const uint32_t mb = __ballot_sync(0xffffffffu, sl_ >= Ts || (mrow && mrow[sl_ < Ts ? sl_ : 0]));
        __syncthreads();                                    // scores in registers: the region becomes the tiles
        float* tile = reinterpret_cast<float*>(smem + RS_SC) + warp * TILE_FLOATS;
        const int tw0 = t0 + 32 * rh, rows_valid = min(max(Td - tw0, 0), 32);
        const size_t wbase = ((size_t)b * Td + min(tw0, Td - 1)) * Ts;
        float o[32];                                        // fwd: the probability; bwd: dS
        if (BWD == 0) {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < 32; ++i) mx = fmaxf(mx, ((mb >> i) & 1u) ? -INFINITY : sv[i]);
            red[kq * AT_RT + row] = mx;
            __syncthreads();
            mx = fmaxf(fmaxf(red[row], red[AT_RT + row]), fmaxf(red[2 * AT_RT + row], red[3 * AT_RT + row]));
            float ex[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) ex[i] = ((mb >> i) & 1u) ? 0.f : expf(sv[i] - mx);
            const float inv = 1.f / row_chain(red + 4 * AT_RT + row, kq, [&](float sum) {
#pragma unroll
                for (int i = 0; i < 32; ++i) sum += ex[i];
                return sum;
            });
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = (tv && c0 + i < Ts) ? ex[i] * inv : 0.f;
        } else {
            float pv[32], g[32];
            if (live) {
                tile_load(tile, p.probs + wbase, Ts, rows_valid, c0, Ts, lane);
#pragma unroll
                for (int i = 0; i < 32; ++i) pv[i] = tile[lane * TILE_PITCH + i];
                if (p.dprobs) tile_load(tile, p.dprobs + wbase, Ts, rows_valid, c0, Ts, lane);
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                g[i] = 0.f;
                if (live && tv && c0 + i < Ts) {
                    g[i] = scale * sv[i] * drop_scale(drop, (uint32_t)(rbase + c0 + i));
                    if (p.dprobs) g[i] += tile[lane * TILE_PITCH + i];
                }
            }
            const float dot = row_chain(red + row, kq, [&](float d) {
#pragma unroll
                for (int i = 0; i < 32; ++i)
                    if (live && tv && c0 + i < Ts) d = fmaf(g[i], pv[i], d);
                return d;
            });
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = (live && tv && c0 + i < Ts) ? pv[i] * (g[i] - dot) : 0.f;
        }
        if (live) {
            __syncwarp();
#pragma unroll
            for (int i = 0; i < 32; ++i) tile[lane * TILE_PITCH + i] = o[i];
            tile_store(tile, (BWD == 0 ? p.probs : p.ds) + wbase, Ts, rows_valid, c0, Ts, lane);
        }
        // the A operand of the second GEMM: dropout(P) (fwd) or dS (bwd), K-major, key slabs 8 KB apart
        if (c0 < nslab * 64) {
            if (BWD == 0) {
#pragma unroll
                for (int i = 0; i < 32; ++i) o[i] *= drop_scale(drop, (uint32_t)(rbase + c0 + i));
            }
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                const int s = c0 + c8 * 8;
                store_split8(smem + RS_A2 + (s >> 6) * 8192 + off_k(row, (s & 63) >> 3), 16384, o + c8 * 8);
            }
        }
    }
    fence_proxy_async();
    __syncthreads();

    // ---------------- GEMM 2: D2[t][e] = sum_s A2[t][s] * B2[e][s], warpgroup w: channels [128 w, 128 w + 128) ------
    const float scl = BWD == 0 ? scale : 1.f;
    float* __restrict__ out = p.out + (size_t)b * E * Td;
    const uint32_t sa = smem_u32(smem + RS_A2), sb = smem_u32(smem);
    float acc[128];
    for (int e0 = 128 * wg; e0 < E; e0 += 256) {           // rows of B2 past E are never stored
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        wgmma_fence();
        for (int sl = 0; sl < nslab; ++sl) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a_hi = sa + sl * 8192 + kk * 32, b_hi = sb + sl * 2 * b2_plane + e0 * 128 + kk * 32;
                mma3<AT_NS, 0, 0>(acc, desc_kmajor(a_hi), desc_kmajor(a_hi + 16384), desc_kmajor(b_hi),
                                  desc_kmajor(b_hi + b2_plane));
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            const int t = t0 + frag_row(i, wq, lane), e = e0 + frag_col(i, lane);
            if (t < Td && e < E) out[(size_t)e * Td + t] = scl * (acc[i] + acc[64 + i]);
        }
    }
}

// dV[e][s] = scale * sum_t dO[e][t] * Pd[t][s] (blockIdx.z = 0) or dK[e][s] = sum_t Q[e][t] * dS[t][s] (blockIdx.z = 1)
// for 64 channels e; staging per 64-query chunk: A (dO or q, K-major) | B (Pd or dS, MN-major) as in gemm_64x128
constexpr int COLS_SMEM = 2 * STAGE_BYTES + 1024;

struct AttnColsParams {
    const float* dout; const float* q; const float* probs; const float* ds;
    float* dv; float* dk;
    int B, E, Td, Ts;
    float scale, p_drop;
    const unsigned long long* seed_ptr;
    uint32_t salt;
    const long long* ts_log;   // as AttnParams::ts_log
};

__global__ void __launch_bounds__(AT_THREADS, 1) attn_cols_kernel(const __grid_constant__ AttnColsParams p) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3;
    const int b = blockIdx.y, e0 = blockIdx.x * 64, pass = blockIdx.z;   // pass 0: dV (A = dO, B = Pd), 1: dK (q, dS)
    const int E = p.E, Td = p.Td, Ts = p.Ts;
    const bool vec_td = (Td & 3) == 0, vec_ts = (Ts & 3) == 0;
    const DropCfg drop = make_drop(p.p_drop, p.seed_ptr, p.salt);
    const bool drop_b = pass == 0 && drop.on;
    pdl_wait();                 // global memory from here on
    const float scale = p.ts_log ? context_scale(*p.ts_log) : p.scale;

    const float* A = (pass == 0 ? p.dout : p.q) + (size_t)b * E * Td;
    const float* Bm = (pass == 0 ? p.probs : p.ds) + (size_t)b * Td * Ts;
    float acc[64];
    gemm_64x128<0>(acc, smem, (Td + 63) / 64, wg, [&](int kc, uint8_t* st) {
        stage_round<GEMM_GROUPS>(
            [&](int u, float* x) {
                if (u < 2) {                                // A: rows e0.. of (E,Td), 64 query columns
                    const int g = tid + u * AT_THREADS, r = g >> 3;
                    load8(A + (long long)(e0 + r) * Td, kc * 64 + (g & 7) * 8, Td, e0 + r < E, vec_td, x);
                } else {                                    // B: 64 query rows of (Td,Ts)
                    const int g = tid + (u - 2) * AT_THREADS, t = kc * 64 + (g >> 4);
                    load8(Bm + (long long)t * Ts, (g & 15) * 8, Ts, t < Td, vec_ts, x);
                }
            },
            [&](int u, float* x) {
                if (u < 2) {
                    const int g = tid + u * AT_THREADS;
                    store_split8(st + off_k(g >> 3, g & 7), 8192, x);
                } else {
                    const int g = tid + (u - 2) * AT_THREADS, r = g >> 4, cg = g & 15;
                    if (drop_b) {                           // Pd = P * the dropout mask, regenerated from the index
                        const size_t idx0 = ((size_t)b * Td + kc * 64 + r) * Ts + cg * 8;
#pragma unroll
                        for (int i = 0; i < 8; ++i) x[i] *= drop_scale(drop, (uint32_t)(idx0 + i));
                    }
                    store_split8(st + 16384 + off_mn(r, cg), 16384, x);
                }
            });
    });
    // rows e of dV / dK are contiguous along the keys
    float* __restrict__ dst = (pass == 0 ? p.dv : p.dk) + (size_t)b * E * Ts;
    const float scl = pass == 0 ? scale : 1.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        const int e = e0 + frag_row(i, wq, lane), s = 64 * wg + frag_col(i, lane);
        if (e < E && s < Ts) dst[(size_t)e * Ts + s] = scl * (acc[i] + acc[32 + i]);
    }
}

template <typename K>
static int set_smem(K kern, int bytes, const char* what) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) { set_error("%s: cannot set %d B dynamic smem: %s", what, bytes, cudaGetErrorString(e)); return 1; }
    return 0;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

// 1 if the tensor-core attention kernels cover this shape (else the caller uses dv3_bgemm + dv3_softmax_*)
int dv3_tc_attn_supported(int B, int E, int Td, int Ts) {
    return B >= 1 && B <= 65535 && E >= 16 && E <= 256 && (E % 16) == 0 && Ts >= 1 && Ts <= AT_NS && Td >= 1;
}

static int tc_attn_fwd(const float* q, const float* k, const float* v, const unsigned char* mask, float* probs,
                       float* out, int B, int E, int Td, int Ts, float scale, const long long* ts_log, float p_drop,
                       const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    DV3_REQUIRE(dv3_tc_attn_supported(B, E, Td, Ts), "tc_attn_fwd: unsupported shape B=%d E=%d Td=%d Ts=%d", B, E, Td, Ts);
    static bool configured = false;
    if (!configured) { if (set_smem(attn_rows_kernel<0>, ROWS_SMEM, "tc_attn_fwd")) return 1; configured = true; }
    AttnParams p = {};
    p.a1 = q; p.b1 = k; p.b2 = v; p.mask = mask; p.probs = probs; p.out = out;
    p.B = B; p.E = E; p.Td = Td; p.Ts = Ts; p.scale = scale; p.p_drop = p_drop; p.seed_ptr = seed_ptr; p.salt = salt;
    p.ts_log = ts_log;
    launch_k(attn_rows_kernel<0>, dim3((Td + AT_RT - 1) / AT_RT, B), AT_THREADS, ROWS_SMEM, (cudaStream_t)stream, p);
    return check_launch("tc_attn_fwd");
}

int dv3_tc_attn_fwd(const float* q, const float* k, const float* v, const unsigned char* mask, float* probs,
                    float* out, int B, int E, int Td, int Ts, float scale, float p_drop,
                    const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    return tc_attn_fwd(q, k, v, mask, probs, out, B, E, Td, Ts, scale, nullptr, p_drop, seed_ptr, salt, stream);
}

// the context scale Ts*sqrt(1/Ts) taken from a logical key count in device memory (a batch padded to a bucket)
int dv3_tc_attn_fwd_ext(const float* q, const float* k, const float* v, const unsigned char* mask, float* probs,
                        float* out, int B, int E, int Td, int Ts, const long long* ts_log, float p_drop,
                        const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    DV3_REQUIRE(ts_log != nullptr, "tc_attn_fwd_ext: ts_log is NULL");
    return tc_attn_fwd(q, k, v, mask, probs, out, B, E, Td, Ts, 0.f, ts_log, p_drop, seed_ptr, salt, stream);
}

// ds: scratch (B,Td,Ts) fp32 written by the first launch and read by the second; dprobs may be null
static int tc_attn_bwd(const float* dout, const float* q, const float* k, const float* v, const float* probs,
                       const float* dprobs, float* ds, float* dq, float* dk, float* dv, int B, int E, int Td, int Ts,
                       float scale, const long long* ts_log, float p_drop, const unsigned long long* seed_ptr,
                       unsigned salt, void* stream) {
    DV3_REQUIRE(dv3_tc_attn_supported(B, E, Td, Ts), "tc_attn_bwd: unsupported shape B=%d E=%d Td=%d Ts=%d", B, E, Td, Ts);
    static bool configured = false;
    if (!configured) {
        if (set_smem(attn_rows_kernel<1>, ROWS_SMEM, "tc_attn_bwd")) return 1;
        if (set_smem(attn_cols_kernel, COLS_SMEM, "tc_attn_bwd")) return 1;
        configured = true;
    }
    AttnParams p = {};
    p.a1 = dout; p.b1 = v; p.b2 = k; p.probs = const_cast<float*>(probs); p.dprobs = dprobs; p.ds = ds; p.out = dq;
    p.B = B; p.E = E; p.Td = Td; p.Ts = Ts; p.scale = scale; p.p_drop = p_drop; p.seed_ptr = seed_ptr; p.salt = salt;
    p.ts_log = ts_log;
    launch_k(attn_rows_kernel<1>, dim3((Td + AT_RT - 1) / AT_RT, B), AT_THREADS, ROWS_SMEM, (cudaStream_t)stream, p);
    if (check_launch("tc_attn_bwd(rows)")) return 1;
    AttnColsParams c = {};
    c.dout = dout; c.q = q; c.probs = probs; c.ds = ds; c.dv = dv; c.dk = dk;
    c.B = B; c.E = E; c.Td = Td; c.Ts = Ts; c.scale = scale; c.p_drop = p_drop; c.seed_ptr = seed_ptr; c.salt = salt;
    c.ts_log = ts_log;
    launch_k(attn_cols_kernel, dim3((E + 63) / 64, B, 2), AT_THREADS, COLS_SMEM, (cudaStream_t)stream, c);
    return check_launch("tc_attn_bwd(cols)");
}

int dv3_tc_attn_bwd(const float* dout, const float* q, const float* k, const float* v, const float* probs,
                    const float* dprobs, float* ds, float* dq, float* dk, float* dv, int B, int E, int Td, int Ts,
                    float scale, float p_drop, const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    return tc_attn_bwd(dout, q, k, v, probs, dprobs, ds, dq, dk, dv, B, E, Td, Ts, scale, nullptr, p_drop, seed_ptr,
                       salt, stream);
}

int dv3_tc_attn_bwd_ext(const float* dout, const float* q, const float* k, const float* v, const float* probs,
                        const float* dprobs, float* ds, float* dq, float* dk, float* dv, int B, int E, int Td, int Ts,
                        const long long* ts_log, float p_drop, const unsigned long long* seed_ptr, unsigned salt,
                        void* stream) {
    DV3_REQUIRE(ts_log != nullptr, "tc_attn_bwd_ext: ts_log is NULL");
    return tc_attn_bwd(dout, q, k, v, probs, dprobs, ds, dq, dk, dv, B, E, Td, Ts, 0.f, ts_log, p_drop, seed_ptr, salt,
                       stream);
}

}  // extern "C"
