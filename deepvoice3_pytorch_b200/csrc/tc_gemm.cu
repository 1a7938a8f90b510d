// wgmma tensor-core path of the ConvBlock and of the plain (1x1 / k-tap) weight-normed convolutions: forward,
// data-gradient and weight-gradient as implicit GEMMs with fp32-class accuracy from split 16-bit operands.
// Every fp32 operand travels as a pair of planes p0 = rn16(x), p1 = rn16((x - p0) * 2^11) (common.cuh): fp16 pairs in
// the forward GEMMs, bf16 pairs in the gradient GEMMs.  Each K-step issues p0*p0 + p0*p1 + p1*p0 (single-pass TF32
// would miss the rtol=1e-3/atol=1e-4 parity bar after ~30 blocks).  The tensor core adds each MMA into the fp32
// accumulator with truncation (bias ~N_mma x 2^-25), so the main term p0*p0 and the cross terms (2^-11 smaller in
// effect with fp16 pairs, 2^-8 with bf16 pairs) accumulate in two separate register accumulators that the epilogue
// adds in fp32 as main + cross * 2^-11 (tools/precision_report.py).
//
//   GATED : D[t, (a|b) c] = sum_{j,ci} Xd[b, t+off_j, ci] * W[j, (a|b) c, ci]    M = 128 time steps, N = 64 a | 64 b
//   CONV  : D[t, n]       = sum_{j,kc} A[b, t+off_j, kc]  * W[j, n, kc]           M = 128 time steps, N = 64 or 128
//           (plain conv forward with bias/ReLU, and every data gradient: A = dY or dAB, W = transposed weight)
//   WGRAD : D[m, n] (j)   = sum_{b,t}  dY[b, t, m] * Xd[b, t+off_j, n]            MN-major operands, M = 128, N <= 256
//
// Each K = 16 step issues three MMAs: p0(A) x p0(W) into the main accumulator, then p0(A) x p1(W) and p1(A) x p0(W)
// into the cross accumulator.  Main and cross are two disjoint register tuples: when an in-flight MMA's accumulator
// partially overlaps the next one's, ptxas serialises the whole wgmma chain (C7511), whatever the register budget.
//
// Single-pass mode (NPL = 1, ops.conv_math = "tc1", DESIGN.md section 2.7): each operand travels as its plane p0 alone
// (fp16 forward, bf16 gradients) and each K = 16 step issues the one MMA p0(A) x p0(W) into the main accumulator: the
// producer loads one plane per operand, there is no cross accumulator, and the hand-off writes main * gmain.  One
// kernel body serves both plane counts.
//
// Both kernels run one PERSISTENT, warp-specialised pipeline (tc_pipeline): min(work units, SMs) CTAs, CTA c walks
// units c, c + grid, ... of a static list, and the TMA ring streams across unit boundaries.  512 threads, one
// setmaxnreg budget per warpgroup:
//   * warpgroup 2 = producer (24 registers): one thread issues the TMA loads of each K-iteration into the next stage of
//     a STAGES-deep ring (full[s]: one arrival plus the stage's transaction bytes; empty[s]: one arrival per consumer
//     warpgroup).  Each configuration names its measured depth in tc_ring.cuh: 4 stages of 32 KB for the gated
//     forward and the 128-column conv, 4 of 48 KB for the 64-column conv at BK = 64, 5 of 32 KB for the two-plane
//     weight gradient, 6 for the smaller stages;
//   * warpgroups 0 and 1 = consumers (168 registers): each accumulates 64 of the 128 tile rows in registers (wgmma),
//     keeping one stage of MMAs in flight (wait_group 1, then release the previous stage), then writes
//     main * gmain + cross * 2^-11 into a full-tile fp32 shared-memory hand-off tile (acc_tile, layout in
//     tc_ring.cuh) and goes straight on to the next unit's MMAs;
//   * warpgroup 3 = epilogue (152 registers): reads acc_tile and stores the unit's output.
// Two mbarriers pass acc_tile back and forth: acc_full (all 256 consumer threads have written it) and acc_empty (128
// arrivals: the epilogue is done with it).  So the epilogue of unit n runs while the consumers issue the MMAs of unit
// n+1.  A CTA's last unit has nothing to overlap with: the consumers, which have no next unit, join its epilogue and
// the three warpgroups split it (a one-wave launch is all last units).  While the MMAs run, the epilogue warpgroup
// prefetches the unit's global epilogue inputs into L2.  A kernel supplies only its unit list, the TMA loads of one K-iteration, the MMAs of one stage, its gmain, its
// epilogue and the loads of its epilogue's staged inputs.
//
// tc_conv_kernel (GATED, CONV): a unit is one 128-step x NCOLS output tile of one utterance.  Operands are 16-bit
// (B,T,C) planes fetched by TMA as K-major tiles of 128 rows x BK (BK = 64: 128-byte rows, SWIZZLE_128B; BK = 32:
// 64-byte rows, SWIZZLE_64B; the host launchers pick BK per configuration); the conv's zero padding, the causal shift,
// ragged T / channel tails are TMA out-of-bounds zero fill.  Its hand-off tile is the dense image of the output's
// TMA boxes: epilogue thread r owns time step r and fuses the launch's own math only (gate, bias, speaker bias,
// residual, dropout mask, addend, ReLU) in place in the tile, and the fp32 (B,C,T) outputs leave as TMA bulk tensor
// stores clipped at T and C; the gated forward's residual tile arrives by TMA into a staging buffer (see the epilogues).
// The operand planes of the next GEMM come from the split kernels of tc_split.cu, which run at full occupancy rather
// than on one warpgroup per SM.
//
// tc_wgrad_mn_kernel (WGRAD): MN-major operands and batch-range work units, see the comment at the kernel.
#include "tc_common.cuh"
#include "tc_ring.cuh"
#include "../../include/dv3b200.h"

namespace dv3 {

using namespace tc;

constexpr int TC_CONV_THREADS = 512;        // tc_conv_kernel, tc_wgrad_mn_kernel: consumers 0-1, producer 2,
                                            // epilogue 3 (warpgroups)
constexpr int TC_PRODUCER_REGS = 24;        // setmaxnreg budgets: 128 x 24 + 256 x 168 + 128 x 152 = 65 536 registers
constexpr int TC_CONSUMER_REGS = 168;
constexpr int TC_EPILOGUE_REGS = 152;       // > 65 536 / 512: claimed with setmaxnreg.inc (.dec may not raise it)
static_assert(TC_PRODUCER_REGS <= 65536 / TC_CONV_THREADS && TC_CONSUMER_REGS >= 65536 / TC_CONV_THREADS &&
              TC_EPILOGUE_REGS >= 65536 / TC_CONV_THREADS, "setmaxnreg direction of each warpgroup");
static_assert(128 * TC_PRODUCER_REGS + 256 * TC_CONSUMER_REGS + 128 * TC_EPILOGUE_REGS <= 65536, "register file");
constexpr int TC_EPILOGUE_LEAD = 3 * 128;   // thread 0 of the epilogue warpgroup: issues its bulk stores
constexpr int TC_LAST_PARTS = 3;            // warpgroups sharing a CTA's last epilogue: consumers 0, 1 and epilogue 3
constexpr int MAX_TAPS_TC = 8;
enum { TC_GATED = 0, TC_CONV = 1 };

struct TcMaps { CUtensorMap a[2]; CUtensorMap b[2]; };

struct TcParams {
    int T;
    int Nc;                    // output channels (GATED: C per half)
    int rows_per_tap;          // rows of the weight matrix per tap (GATED: 2C, CONV: Nc)
    int k, kb_n;               // taps; K blocks per tap
    int tap_off[MAX_TAPS_TC];
    // gated epilogue
    const float* bias; const float* spk; const float* res;
    float* y; float* save_a; float* save_s;
    int gate_mode, residual;
    // conv epilogue: out = acc*dropmask + bias + addend ; relu
    float* out; const float* e1; const float* e2; float alpha; int addmode, relu;
    float p_drop; const unsigned long long* seed_ptr; uint32_t salt;
    // Compensation of the tensor core's truncating accumulation: every MMA adds its K = 16 partial product into the
    // fp32 accumulator rounding TOWARD ZERO, a small expected relative loss per event on the running sum; over the
    // n_mma events of one output that is a systematic shrink of ~gcoef * n_mma (tools/trunc_bias.py measures gcoef).
    // The epilogue multiplies the main accumulator by gmain = 1 + gcoef * n_mma (the cross terms are 2^-8 or more
    // smaller in effect: their loss is below fp32 resolution).
    float gmain;
    int operand_bf16;          // operand format of the MMAs: 0 = fp16 planes (forward), 1 = bf16 planes (gradients)
    int tma_out;               // 1: outputs (and the gated residual) through the TcOutMaps; 0: per-thread accesses
};

template <int BK> struct SwizzleOf;
template <> struct SwizzleOf<64> { static constexpr uint32_t layout = WG_SW128, sbo = 1024; };
template <> struct SwizzleOf<32> { static constexpr uint32_t layout = WG_SW64, sbo = 512; };

template <int BK>
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return make_wgmma_desc(saddr, 16, SwizzleOf<BK>::sbo, SwizzleOf<BK>::layout);
}

// ---- epilogues -----------------------------------------------------------------------------------------------
// Both conv epilogues compute in place in the dense hand-off tile (tc_ring.cuh): epilogue thread r owns time step r of
// the unit and reads / writes its column entries (a warp covers one 128-byte row of a box: conflict-free), then the
// tile goes out as TMA bulk tensor stores, four 32-step boxes per output, issued by one elected thread after a
// proxy fence and a named barrier of the epilogue warpgroup.  The tensor maps carry the logical (B, Nc, T) extent, so
// TMA clipping drops the time steps past T and the channels past Nc; the thread that issued the stores waits until
// they have read shared memory (not until they have landed) and then releases the tile for all 128 threads.  Global
// fp32 rows must be 16-byte aligned for a TMA map (T % 4 == 0, aligned pointers); otherwise (p.tma_out == 0) every
// thread stores its own time step from the tile, coalesced along T, as the per-thread epilogue always did.  The math
// per element is that of the per-thread epilogue, in the same order.
// Addend / speaker-bias reads go through __ldg (ld.global.nc) in batches of 32 independent loads BEFORE the dependent
// math of the chunk: with plain loads the compiler must order every load after the previous iteration's stores.

// float offset of channel c, time step (threadIdx.x % 128) in a dense tile of NC channels
template <int NC>
__device__ __forceinline__ int dense_at(int c) {
    const int r = threadIdx.x & 127;
    return (r >> 5) * NC * 32 + c * 32 + ((((r >> 2) & 7) ^ (c & 7)) << 2) + (r & 3);
}

struct TcOutMaps { CUtensorMap out[3]; CUtensorMap res; };   // y | a | s (GATED) or out (CONV); the residual input

// Where an epilogue finds its shared memory: the hand-off tile, the staging buffer, the barriers.
struct Handoff { float* tile; float* staging; uint64_t* acc_empty; uint64_t* in_full; };

// Release the hand-off tile after the bulk stores of this unit, or, with per-thread stores, after this thread's.  Only
// the epilogue warpgroup releases it: the consumers that join a CTA's last epilogue have no next unit to hand off.
// The wait is for the stores to have READ the tile, also after the last unit: the global writes of bulk stores still
// in flight when the CTA exits complete before the grid does.
__device__ __forceinline__ void release_tile(const Handoff& h, bool tma) {
    if (threadIdx.x < TC_EPILOGUE_LEAD) return;
    if (!tma) mbar_arrive(h.acc_empty);
    else if (threadIdx.x == TC_EPILOGUE_LEAD) {
        bulk_commit();
        bulk_wait_read();
        mbar_arrive_cnt(h.acc_empty, 128);
    }
}

// L2 prefetch of the part of a (B, C, T) fp32 epilogue input that unit (t0, b, channels [c0, c0 + nc)) reads, issued
// by the epilogue warpgroup while the unit's MMAs run: warp q covers time steps [t0 + 32 q, t0 + 32 q + 32), lane l
// channels l, l + 32, ..., both ends of each 128-byte row segment (which may straddle two lines).
__device__ __forceinline__ void prefetch_bct(const float* x, int T, int C, int b, int c0, int nc, int t0) {
    const int ta = t0 + 32 * ((threadIdx.x >> 5) & 3), lane = threadIdx.x & 31;
    if (ta >= T) return;
    const int tb = min(ta + 31, T - 1);
    for (int c = lane; c < nc && c0 + c < C; c += 32) {
        const float* row = x + ((size_t)b * C + c0 + c) * T;
        prefetch_l2(row + ta);
        prefetch_l2(row + tb);
    }
}

// The gated forward's residual tile (128 steps x BR channels) into the staging buffer by TMA: issued for the next
// unit as soon as the current unit's y stores have read the buffer, so it lands under the next unit's MMAs.
template <int BR>
__device__ __forceinline__ void stage_residual(const TcParams& p, const TcOutMaps& om, const Handoff& h, int a_row0,
                                               int a_z, int b_row0) {
    if (!p.tma_out || !((p.gate_mode != 0) || p.residual) || (threadIdx.x & 127) != 0) return;
    mbar_arrive_expect_tx(h.in_full, 128 * BR * 4);
#pragma unroll
    for (int q = 0; q < 4; ++q) tma_load_3d(h.staging + q * BR * 32, &om.res, h.in_full, a_row0 + 32 * q, b_row0, a_z);
}

// Gated: a = acc_a (+ speaker) + bias_a, s = sigmoid(acc_b + bias_b), y from a, s and the residual.  y replaces the
// residual in the staging buffer, a and s replace the two accumulator halves; the speaker bias (multi-speaker presets
// only) stays on __ldg.
template <int BR, int CW>
__device__ __forceinline__ void epilogue_gated(const TcParams& p, const TcOutMaps& om, const Handoff& h, int n,
                                               int a_row0, int a_z, int b_row0, int part, int nparts) {
    constexpr int NC = 2 * BR;                             // a | b halves of the tile
    static_assert(BR % CW == 0, "whole channel chunks");
    const int t = a_row0 + (threadIdx.x & 127), b = a_z, C = p.Nc;
    const bool tv = t < p.T, tma = p.tma_out != 0;
    const float* __restrict__ bias = p.bias;
    const float* __restrict__ res = p.res;
    const float* __restrict__ spk = p.spk;
    float* __restrict__ yo = p.y;
    float* __restrict__ ao = p.save_a;
    float* __restrict__ so = p.save_s;
    float* tile = h.tile;
    float* st = h.staging;
    const bool need_res = (p.gate_mode != 0) || p.residual;
    const size_t base = ((size_t)b * C + b_row0) * p.T + (tv ? t : 0);
    if (need_res && tma) mbar_wait(h.in_full, n & 1);
#pragma unroll 1
    for (int c32 = part * CW; c32 < BR; c32 += nparts * CW) {   // this warpgroup's chunks of CW channels
        float sp[CW], ba[CW], bb[CW];                      // speaker bias; bias of the a and b halves
        const size_t cb = base + (size_t)c32 * p.T;
        if (need_res && !tma) {
#pragma unroll 8
            for (int i = 0; i < CW; ++i) st[dense_at<BR>(c32 + i)] = tv ? __ldg(&res[cb + (size_t)i * p.T]) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < CW; ++i) {
            ba[i] = __ldg(&bias[b_row0 + c32 + i]);
            bb[i] = __ldg(&bias[C + b_row0 + c32 + i]);
            if (spk) sp[i] = tv ? __ldg(&spk[cb + (size_t)i * p.T]) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < CW; ++i) {
            const int cl = c32 + i;
            float va = tile[dense_at<NC>(cl)];
            if (spk) va += sp[i];
            const float a = va + ba[i];
            const float s = sigmoidf_(tile[dense_at<NC>(BR + cl)] + bb[i]);
            const float rr = need_res ? st[dense_at<BR>(cl)] : 0.f;
            float y;
            if (p.gate_mode == 0) {
                y = a * s;
                if (p.residual) y = (y + rr) * 0.70710678118654752f;
            } else {
                y = s * a + (1.f - s) * rr;
            }
            st[dense_at<BR>(cl)] = y;
            tile[dense_at<NC>(cl)] = a;
            tile[dense_at<NC>(BR + cl)] = s;
        }
    }
    if (tma) {
        fence_proxy_async();
        named_bar_sync(1, 128 * nparts);
        if (threadIdx.x == TC_EPILOGUE_LEAD) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int t0 = a_row0 + 32 * q;
                if (t0 >= p.T) break;
                tma_store_3d(&om.out[0], st + q * BR * 32, t0, b_row0, b);
                if (ao) tma_store_3d(&om.out[1], tile + q * NC * 32, t0, b_row0, b);
                if (so) tma_store_3d(&om.out[2], tile + q * NC * 32 + BR * 32, t0, b_row0, b);
            }
        }
    } else if (tv) {
#pragma unroll 1
        for (int c32 = part * CW; c32 < BR; c32 += nparts * CW) {
#pragma unroll 8
            for (int c = c32; c < c32 + CW; ++c) {
                const size_t idx = base + (size_t)c * p.T;
                yo[idx] = st[dense_at<BR>(c)];
                if (ao) ao[idx] = tile[dense_at<NC>(c)];
                if (so) so[idx] = tile[dense_at<NC>(BR + c)];
            }
        }
    }
    release_tile(h, tma);
}

// Conv: out = acc * dropmask + bias + addend, then ReLU.
template <int NCOLS, int CW>
__device__ __forceinline__ void epilogue_conv(const TcParams& p, const TcOutMaps& om, const Handoff& h, int a_row0,
                                              int a_z, int b_row0, int part, int nparts) {
    static_assert(NCOLS % CW == 0, "whole channel chunks");
    const int t = a_row0 + (threadIdx.x & 127), b = a_z;
    const bool tv = t < p.T, tma = p.tma_out != 0;
    const DropCfg drop = make_drop(p.p_drop, p.seed_ptr, p.salt);
    const float* __restrict__ bias = p.bias;
    const float* __restrict__ e1 = p.e1;
    const float* __restrict__ e2 = p.e2;
    float* __restrict__ out = p.out;
    float* tile = h.tile;
    const size_t base = ((size_t)b * p.Nc + b_row0) * p.T + (tv ? t : 0);
#pragma unroll 1
    for (int c32 = part * CW; c32 < NCOLS; c32 += nparts * CW) {   // not unrolled: interleaving the chunks spilled
        float bz[CW], v[CW], x2[CW];                        // bias; addends e1, e2
        const int n0 = b_row0 + c32;
        const size_t cb = base + (size_t)c32 * p.T;
#pragma unroll
        for (int i = 0; i < CW; ++i) {
            const bool ok = tv && n0 + i < p.Nc;
            bz[i] = (bias && n0 + i < p.Nc) ? __ldg(&bias[n0 + i]) : 0.f;
            v[i] = (p.addmode != 0 && ok) ? __ldg(&e1[cb + (size_t)i * p.T]) : 0.f;
            x2[i] = (p.addmode == 2 && ok) ? __ldg(&e2[cb + (size_t)i * p.T]) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < CW; ++i) {
            float& d = tile[dense_at<NCOLS>(c32 + i)];
            float g = d * drop_scale(drop, (uint32_t)(cb + (size_t)i * p.T));
            if (bias) g += bz[i];
            if (p.addmode == 1) g += p.alpha * v[i];
            else if (p.addmode == 2) g += v[i] * (1.f - x2[i]);
            if (p.relu) g = fmaxf(g, 0.f);
            d = g;
        }
    }
    if (tma) {
        fence_proxy_async();
        named_bar_sync(1, 128 * nparts);
        if (threadIdx.x == TC_EPILOGUE_LEAD) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int t0 = a_row0 + 32 * q;
                if (t0 >= p.T) break;
                tma_store_3d(&om.out[0], tile + q * NCOLS * 32, t0, b_row0, b);
            }
        }
    } else if (tv) {
#pragma unroll 1
        for (int c32 = part * CW; c32 < NCOLS; c32 += nparts * CW) {
#pragma unroll 8
            for (int c = c32; c < c32 + CW; ++c)
                if (b_row0 + c < p.Nc) out[base + (size_t)c * p.T] = tile[dense_at<NCOLS>(c)];
        }
    }
    release_tile(h, tma);
}

// ------------------------------------------------------------------------------------------------
// The persistent warp-specialised pipeline of both GEMM kernels (see file header), with the shared-memory layout of
// Cfg (a RingCfg) and NPL operand planes.  The kernel supplies the parts specific to its GEMM as force-inlined lambdas:
//   decode(u) -> w                work unit u; w.n_iters is its number of K-iterations (ring stages)
//   load(w, kit, stage, bar)      the TMA loads of K-iteration kit of w into `stage`, completing on bar (the producer
//                                 has already armed bar with the stage's Cfg::STAGE bytes)
//   mma(stage, wg, acc, xacc)     consumer warpgroup wg's MMAs of one stage: p0 x p0 into acc and, with two planes,
//                                 p0 x p1 + p1 x p0 into xacc (64 rows x NCOLS columns, NCOLS / 2 registers each)
//   gmain(w)                      the factor of w's main accumulator (TcParams::gmain)
//   epilogue(w, n, h, part, nparts)  stores w, this CTA's n-th unit, from the hand-off tile h.tile (layout:
//                                 Cfg::DENSE, tc_ring.cuh).  nparts = 1: the epilogue warpgroup alone (part 0).
//                                 nparts = TC_LAST_PARTS, for the CTA's last unit only: consumer warpgroups 0 and 1
//                                 (parts 0, 1) have no next unit and share it with the epilogue warpgroup (part 2),
//                                 each taking its own slices of the tile; every output element keeps the expression
//                                 (and the thread's time step or column) it has with one part.  Contract: the epilogue
//                                 warpgroup arrives on h.acc_empty 128 times per unit, once its last access of the
//                                 tile is done (by a thread or by the bulk stores it issued), so the consumers can
//                                 overwrite the tile while the epilogue's last global stores are still under way.
//   stage(w, h)                   issues the loads of unit w's epilogue inputs into h.staging, completing on
//                                 h.in_full (phase n for the n-th unit), and L2 prefetches of those it reads from
//                                 global memory: called by every epilogue thread for the first unit up front and for
//                                 each next unit right after the current epilogue, so both run under w's MMAs.
// ------------------------------------------------------------------------------------------------
template <class Cfg, int NPL, class Decode, class Load, class Mma, class Gmain, class Epilogue, class Stage>
__device__ __forceinline__ void tc_pipeline(const TcMaps& maps, int num_units, Decode decode, Load load, Mma mma,
                                            Gmain gmain, Epilogue epilogue, Stage stage) {
    static_assert(NPL == 1 || NPL == 2, "one or two operand planes");
    static_assert(Cfg::NCOLS <= 128, "main + cross accumulators must fit in the registers of a consumer thread");
    static_assert(Cfg::STAGES >= 2, "pipeline needs at least two stages");
    constexpr int STAGE = Cfg::STAGE, STAGES = Cfg::STAGES;
    constexpr int NR = Cfg::NCOLS / 2;                       // registers per accumulator per thread
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    // 1 KB aligned by pointer arithmetic on the __shared__ array (not through an integer), so that the compiler keeps
    // knowing the address space: shared loads / stores (LDS / STS) instead of generic ones, which it may not reorder
    // with the epilogue's global loads.
    uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
    float* acc_tile = reinterpret_cast<float*>(smem + STAGES * STAGE);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE + Cfg::ACC_TILE + Cfg::STAGING);
    uint64_t* empty = full + STAGES;
    uint64_t* acc_full = empty + STAGES;                     // the consumers have written acc_tile (256 arrivals)
    uint64_t* acc_empty = acc_full + 1;                      // the epilogue is done with acc_tile (128 arrivals)
    uint64_t* in_full = acc_empty + 1;                       // the staged epilogue inputs have landed
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) prefetch_tmap(&maps.a[pl]);
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) prefetch_tmap(&maps.b[pl]);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        mbar_init(acc_full, 256);
        mbar_init(acc_empty, 128);
        mbar_init(in_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                    // everything above overlapped the previous kernel's tail; global memory from here

    if (warp >= 12) {
        setmaxnreg_inc<TC_EPILOGUE_REGS>();                  // up from the launch's 65 536 / 512 = 128 per thread
        const Handoff h = {acc_tile, acc_tile + Cfg::ACC_TILE / 4, acc_empty, in_full};
        if (blockIdx.x < num_units) stage(decode(blockIdx.x), h);
        int n = 0;
        for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++n) {
            const auto w = decode(u);
            const bool last = u + gridDim.x >= num_units;
            mbar_wait(acc_full, n & 1);
            if (last) epilogue(w, n, h, TC_LAST_PARTS - 1, TC_LAST_PARTS);
            else {
                epilogue(w, n, h, 0, 1);
                stage(decode(u + gridDim.x), h);
            }
        }
    } else if (warp >= 8) {
        setmaxnreg_dec<TC_PRODUCER_REGS>();
        if (warp == 8 && lane == 0) {
            int it = 0;
            for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
                const auto w = decode(u);
                for (int kit = 0; kit < w.n_iters; ++kit, ++it) {
                    const int s = it % STAGES, ph = (it / STAGES) & 1;
                    mbar_wait(&empty[s], ph ^ 1);
                    mbar_arrive_expect_tx(&full[s], STAGE);
                    load(w, kit, smem + s * STAGE, &full[s]);
                }
            }
        }
    } else {
        setmaxnreg_inc<TC_CONSUMER_REGS>();
        const int wg = warp >> 2, wq = warp & 3;
        // Two disjoint register tuples: an MMA in flight may not share accumulator registers with the next one, or
        // ptxas serialises every wgmma of the chain.
        float acc[NR], xacc[NPL == 2 ? NR : 1];              // main (p0 x p0), cross (p0 x p1 + p1 x p0)
        int it = 0, n = 0;
        for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++n) {
            const auto w = decode(u);
#pragma unroll
            for (int i = 0; i < NR; ++i) {
                acc[i] = 0.f;
                if constexpr (NPL == 2) xacc[i] = 0.f;
            }
            for (int kit = 0; kit < w.n_iters; ++kit, ++it) {
                const int s = it % STAGES, ph = (it / STAGES) & 1;
                mbar_wait(&full[s], ph);
                wgmma_fence();
                mma(smem + s * STAGE, wg, acc, xacc);
                wgmma_commit();
                wgmma_wait<1>();                                  // the previous stage's MMAs have retired
                if (kit > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
            }
            wgmma_wait<0>();
            if (w.n_iters > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
            const float gm = gmain(w);
            mbar_wait(acc_empty, (n & 1) ^ 1);                        // the epilogue is done with the previous unit
            // Dense tile: register i sits at time step 64 wg + 16 wq + lane / 4 + 8 ((i >> 1) & 1), i.e. in box
            // 2 wg + wq / 2, chunk 4 (wq & 1) + lane / 16 + 2 ((i >> 1) & 1), and at channel 8 (i >> 2) + 2 (lane & 3)
            // + (i & 1), so its swizzled chunk is sw ^ (i & 3) with a per-thread sw: four per-thread bases, each
            // plus an immediate offset per register.
            const int sw = (((wq & 1) << 2) | (lane >> 4)) ^ ((lane & 3) << 1);
            float* const frag0 = Cfg::DENSE ? acc_tile + (2 * wg + (wq >> 1)) * Cfg::NCOLS * 32 + (lane & 3) * 64 +
                                                  ((lane >> 2) & 3)
                                            : acc_tile;
#pragma unroll
            for (int i = 0; i < NR; ++i) {                            // lo planes carry 2^11
                float* dst = Cfg::DENSE
                    ? frag0 + (i >> 2) * 256 + (i & 1) * 32 + ((sw ^ (i & 3)) << 2)
                    : &acc_tile[(64 * wg + frag_row(i, wq, lane)) * Cfg::ACC_PITCH + frag_col(i, lane)];
                if constexpr (NPL == 2) *dst = fmaf(xacc[i], LO_INV, acc[i] * gm);
                else *dst = acc[i] * gm;
            }
            mbar_arrive(acc_full);
            if (u + gridDim.x >= num_units) {                       // no next unit: join the last epilogue
                const Handoff h = {acc_tile, acc_tile + Cfg::ACC_TILE / 4, acc_empty, in_full};
                mbar_wait(acc_full, n & 1);
                epilogue(w, n, h, wg, TC_LAST_PARTS);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// GATED / CONV kernel.  A unit is one output tile; tile ids run channel tiles fastest, then time tiles, then the
// batch, so that concurrently running CTAs share the activation tile in L2.  N per tile is limited to 128 columns.
// ------------------------------------------------------------------------------------------------
template <int MODE, int NBOX, int BR, int BK, bool BF16, int NPL>
__global__ void __launch_bounds__(TC_CONV_THREADS, 1)
tc_conv_kernel(const __grid_constant__ TcMaps maps, const __grid_constant__ TcOutMaps om,
               const __grid_constant__ TcParams p, int tiles_x, int tiles_y, int num_tiles) {
    using Cfg = TcCfg<NBOX, BK, BR, NPL>;
    constexpr int NCOLS = Cfg::NCOLS;
    constexpr int TILE = 128 * BK * 2, TILE_B = BR * BK * 2;   // one plane of the A tile (128 rows), one B box
    constexpr int B_OFF = NPL * TILE;
    constexpr int A_HALF = 64 * BK * 2;                      // rows [64 wg, 64 wg + 64) of the A tile
    const int n_iters = p.k * p.kb_n;

    struct Tile { int a_row0, a_z, b_row0, b_row1, n_iters; };
    auto decode = [&](int tile) {
        Tile w;
        const int ty = tile % tiles_y, r = tile / tiles_y;
        w.a_z = r / tiles_x;
        w.a_row0 = (r % tiles_x) * 128;
        if (MODE == TC_GATED) { w.b_row0 = ty * BR; w.b_row1 = p.Nc + ty * BR; }
        else { w.b_row0 = ty * BR * NBOX; w.b_row1 = w.b_row0 + BR; }
        w.n_iters = n_iters;
        return w;
    };
    auto load = [&](const Tile& w, int kit, uint8_t* st, uint64_t* bar) {
        const int j = kit / p.kb_n, kb = kit - j * p.kb_n;
        const int ax = kb * BK, ay = w.a_row0 + p.tap_off[j];
        const int by0 = j * p.rows_per_tap + w.b_row0, by1 = j * p.rows_per_tap + w.b_row1;
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) {
            tma_load_3d(st + pl * TILE, &maps.a[pl], bar, ax, ay, w.a_z);
            uint8_t* bdst = st + B_OFF + pl * NBOX * TILE_B;
            tma_load_3d(bdst, &maps.b[pl], bar, ax, by0, 0);
            if (NBOX == 2) tma_load_3d(bdst + TILE_B, &maps.b[pl], bar, ax, by1, 0);
        }
    };
    auto mma = [&](const uint8_t* st, int wg, float* acc, float* xacc) {
        const uint32_t sa = smem_u32(st) + wg * A_HALF, sb = smem_u32(st + B_OFF);
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
            const uint32_t ko = kk * 32;
            const uint64_t a0 = make_desc<BK>(sa + ko), b0 = make_desc<BK>(sb + ko);
            wgmma_mma<NCOLS, 0, 0>(BF16, acc, a0, b0, 1);
            if constexpr (NPL == 2) {
                const uint64_t a1 = make_desc<BK>(sa + TILE + ko), b1 = make_desc<BK>(sb + NBOX * TILE_B + ko);
                wgmma_mma<NCOLS, 0, 0>(BF16, xacc, a0, b1, 1);
                wgmma_mma<NCOLS, 0, 0>(BF16, xacc, a1, b0, 1);
            }
        }
    };
    auto gmain = [&](const Tile&) { return p.gmain; };
    // 32-channel chunks for the epilogue warpgroup alone; eight chunks of the tile's channels when three warpgroups
    // share the last unit (3 + 3 + 2, the epilogue warpgroup, which also issues the stores, taking 2)
    auto epilogue = [&](const Tile& w, int n, const Handoff& h, int part, int nparts) {
        if (MODE == TC_GATED) {
            if (nparts == 1) epilogue_gated<BR, 32>(p, om, h, n, w.a_row0, w.a_z, w.b_row0, 0, 1);
            else epilogue_gated<BR, BR / 8>(p, om, h, n, w.a_row0, w.a_z, w.b_row0, part, nparts);
        } else {
            if (nparts == 1) epilogue_conv<NCOLS, 32>(p, om, h, w.a_row0, w.a_z, w.b_row0, 0, 1);
            else epilogue_conv<NCOLS, NCOLS / 8>(p, om, h, w.a_row0, w.a_z, w.b_row0, part, nparts);
        }
    };
    auto stage = [&](const Tile& w, const Handoff& h) {
        if (MODE == TC_GATED) {
            stage_residual<BR>(p, om, h, w.a_row0, w.a_z, w.b_row0);
            if (p.spk) prefetch_bct(p.spk, p.T, p.Nc, w.a_z, w.b_row0, BR, w.a_row0);
        } else {
            if (p.addmode != 0) prefetch_bct(p.e1, p.T, p.Nc, w.a_z, w.b_row0, NCOLS, w.a_row0);
            if (p.addmode == 2) prefetch_bct(p.e2, p.T, p.Nc, w.a_z, w.b_row0, NCOLS, w.a_row0);
        }
    };
    tc_pipeline<Cfg, NPL>(maps, num_tiles, decode, load, mma, gmain, epilogue, stage);
}

// ------------------------------------------------------------------------------------------------
// Weight gradient straight from the (B,T,C) planes the forward / data-gradient GEMMs already use:
//     D[m, n] (tap j) = sum_{b,t} dY[b, t, m] * Xd[b, t + off_j, n]
// Both operands are "MN-major" here (channels contiguous, the contraction index t is the row): 64-channel x 32-row
// TMA boxes (128-byte rows, SWIZZLE_128B), wgmma descriptors with the MN-major canonical layout
// ((64 channels contiguous, chunk stride LBO), (8 rows x 128 B, group stride SBO)) and both operands transposed in the
// instruction.  The tap shift is a ROW coordinate of the TMA box (any alignment, out-of-bounds rows are zero = the
// conv padding), so no time-shifted copies of the input are needed.
//
// A work unit is one 128 (m) x 128 (n) tile of one tap j and one split s: the sum over the utterances
// [s * bps, min(B, (s + 1) * bps)) of the split, all their 32-row time chunks, written to slot s.  In the unit list the
// split index varies slowest, so every split but the last (the only one that can be short) comes first: units run
// longest first.  The schedule, and with it every value, is a function of the shape and the SM count.
// ------------------------------------------------------------------------------------------------
struct TcMnParams {
    int T, B, Mw, Nw, k;
    int tap_off[MAX_TAPS_TC];
    int nsplit, batches_per_split, kb_n;      // kb_n = 32-row time chunks per utterance
    int tiles_n, tiles_m, num_units;          // units: n-tile fastest, then m-tile, tap, split
    float* dw; long long split_stride;
    int msplit; long long s_m, s_mh, s_n, s_j;
    float gcoef;                              // see TcParams::gmain (n_mma = 2 per 32-row time chunk)
};

template <int NPL>
__global__ void __launch_bounds__(TC_CONV_THREADS, 1)
tc_wgrad_mn_kernel(const __grid_constant__ TcMaps maps, const __grid_constant__ TcMnParams p) {
    using Cfg = WgCfg<NPL>;
    constexpr int A_PL = 2 * WG_BOX, B_PL = 2 * WG_BOX;
    constexpr uint32_t LBO = 4096, SBO = 1024;           // 64-channel chunks one TMA box apart; 8-row groups 1 KB apart

    // unit -> (m0, n0, tap, split, first utterance, K-iterations)
    struct Unit { int m0, n0, j, s, b_beg, n_iters; };
    auto decode = [&](int u) {
        Unit w;
        w.n0 = (u % p.tiles_n) * 128;
        int r = u / p.tiles_n;
        w.m0 = (r % p.tiles_m) * 128;
        r /= p.tiles_m;
        w.j = r % p.k;
        w.s = r / p.k;
        w.b_beg = w.s * p.batches_per_split;
        const int b_end = min(p.B, w.b_beg + p.batches_per_split);
        w.n_iters = (b_end > w.b_beg ? b_end - w.b_beg : 0) * p.kb_n;
        return w;
    };
    auto load = [&](const Unit& w, int kit, uint8_t* st, uint64_t* bar) {
        const int bi = kit / p.kb_n, tc_ = kit - bi * p.kb_n;
        const int b = w.b_beg + bi, t0 = tc_ * 32;
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
                tma_load_3d(st + pl * A_PL + h * WG_BOX, &maps.a[pl], bar, w.m0 + h * 64, t0, b);
#pragma unroll
            for (int q = 0; q < 2; ++q)
                tma_load_3d(st + NPL * A_PL + pl * B_PL + q * WG_BOX, &maps.b[pl], bar, w.n0 + q * 64,
                            t0 + p.tap_off[w.j], b);
        }
    };
    // A = gradient planes, B = the bf16 copy of the forward operand planes; both MN-major
    auto mma = [&](const uint8_t* st, int wg, float* acc, float* xacc) {
        const uint32_t sa = smem_u32(st);
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {                        // 2 x K = 16 rows of 128 B
            const uint32_t ko = kk * 16 * 128;
            const uint64_t a0 = make_wgmma_desc(sa + wg * WG_BOX + ko, LBO, SBO, WG_SW128);
            const uint64_t b0 = make_wgmma_desc(sa + NPL * A_PL + ko, LBO, SBO, WG_SW128);
            wgmma_mma<128, 1, 1>(true, acc, a0, b0, 1);
            if constexpr (NPL == 2) {
                const uint64_t a1 = make_wgmma_desc(sa + A_PL + wg * WG_BOX + ko, LBO, SBO, WG_SW128);
                const uint64_t b1 = make_wgmma_desc(sa + 2 * A_PL + B_PL + ko, LBO, SBO, WG_SW128);
                wgmma_mma<128, 1, 1>(true, xacc, a0, b1, 1);
                wgmma_mma<128, 1, 1>(true, xacc, a1, b0, 1);
            }
        }
    };
    auto gmain = [&](const Unit& w) { return 1.f + p.gcoef * (float)(2 * w.n_iters); };
    // Tap-major layout (s_n == 1): thread r owns column n0 + r and walks the rows, a warp storing 32 consecutive floats
    // of one row.  Otherwise (ConvTranspose layout, consecutive m two floats apart): thread r owns row m0 + r and walks
    // the columns.  The warpgroups sharing a last unit walk interleaved 16-row (16-column) slices of the tile.
    auto epilogue = [&](const Unit& w, int, const Handoff& h, int part, int nparts) {
        const float* acc_tile = h.tile;
        const int r = threadIdx.x & 127;
        const int cw = nparts == 1 ? 128 : 16;
        float* __restrict__ out = p.dw + (size_t)w.s * p.split_stride + (size_t)w.j * p.s_j;
        const int rows = min(128, p.Mw - w.m0), cols = min(128, p.Nw - w.n0);
        if (p.s_n == 1) {
            if (r < cols) {
                float* __restrict__ o = out + w.n0 + r;
#pragma unroll 1
                for (int i0 = part * cw; i0 < rows; i0 += nparts * cw) {
                    const int i1 = min(i0 + cw, rows);
                    // row m = m0 + i at (m % msplit) * s_m + (m / msplit) * s_mh: one division per slice, then the
                    // remainder and quotient stepped along the rows
                    int mr = (w.m0 + i0) % p.msplit, mq = (w.m0 + i0) / p.msplit;
#pragma unroll 4
                    for (int i = i0; i < i1; ++i) {
                        o[(size_t)mr * p.s_m + (size_t)mq * p.s_mh] = acc_tile[i * Cfg::ACC_PITCH + r];
                        if (++mr == p.msplit) { mr = 0; ++mq; }
                    }
                }
            }
        } else if (r < rows) {
            const int m = w.m0 + r;
            float* __restrict__ o = out + (size_t)(m % p.msplit) * p.s_m + (size_t)(m / p.msplit) * p.s_mh +
                                    (size_t)w.n0 * p.s_n;
            const float* arow = acc_tile + r * Cfg::ACC_PITCH;
#pragma unroll 1
            for (int c0 = part * cw; c0 < cols; c0 += nparts * cw) {
                const int c1 = min(c0 + cw, cols);
#pragma unroll 4
                for (int c = c0; c < c1; ++c) o[(size_t)c * p.s_n] = arow[c];
            }
        }
        if (threadIdx.x >= TC_EPILOGUE_LEAD) mbar_arrive(h.acc_empty);
    };
    tc_pipeline<Cfg, NPL>(maps, p.num_units, decode, load, mma, gmain, epilogue, [](const Unit&, const Handoff&) {});
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static const EncodeTiledFn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres);
        return (e == cudaSuccess) ? (EncodeTiledFn)f : (EncodeTiledFn) nullptr;
    }();
    return fn;
}

// bf16 3-D tensor map; box = (box0, box1, 1); swizzle chosen from the box width (64 or 128 bytes)
int encode_tmap_bf16_3d(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                        uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1) {
    const EncodeTiledFn enc = encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
    cuuint32_t box[3] = {box0, box1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUtensorMapSwizzle sw = box0 * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): dims=(%llu,%llu,%llu) strides=(%llu,%llu) box=(%u,%u)", (int)r,
                  (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
                  (unsigned long long)stride1_bytes, (unsigned long long)stride2_bytes, box0, box1);
        return 1;
    }
    return 0;
}

// fp32 (B, Nc, T) tensor as TMA boxes of 32 time steps x box_c channels, SWIZZLE_128B: the boxes of the dense
// hand-off tile (tc_ring.cuh).  The extent is the logical one, so TMA clips every box at T and at Nc.
static int encode_tmap_f32_bct(CUtensorMap* map, const float* base, int B, int Nc, int T, int box_c) {
    const EncodeTiledFn enc = encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
    cuuint64_t dims[3] = {(cuuint64_t)T, (cuuint64_t)Nc, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)T * 4, (cuuint64_t)Nc * T * 4};
    cuuint32_t box[3] = {32, (cuuint32_t)box_c, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): fp32 (B,C,T) = (%d,%d,%d) box=(32,%d)", (int)r, B, Nc, T, box_c);
        return 1;
    }
    return 0;
}

// A TMA map needs 16-byte aligned rows: T % 4 == 0 and a 16-byte aligned base (or no tensor at all).
static bool tma_rows(const float* base, int T) { return T % 4 == 0 && ((uintptr_t)base & 15) == 0; }

template <typename K>
static int ensure_smem(K kern, int bytes, const char* what) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) { set_error("%s: cannot set %d B dynamic smem: %s", what, bytes, cudaGetErrorString(e)); return 1; }
    return 0;
}

// Persistent launch of a tc_pipeline kernel with the shared-memory layout Cfg: min(units, SMs) CTAs.
template <class Cfg, auto kern, typename... Args>
static int launch_persistent(int units, cudaStream_t st, const char* what, const Args&... args) {
    static const int configured = ensure_smem(kern, Cfg::SMEM, what);       // once per instantiation, thread-safe
    if (configured) return 1;
    const int sms = config().sms, grid = units < sms ? units : sms;
    cudaError_t e = launch_k(kern, dim3(grid), dim3(TC_CONV_THREADS), (size_t)Cfg::SMEM, st, args...);
    if (e != cudaSuccess) { set_error("%s: launch failed: %s", what, cudaGetErrorString(e)); return 1; }
    return check_launch(what);
}

template <int MODE, int NBOX, int BR, int BK, bool BF16, int NPL>
static int launch_conv_fmt(const TcMaps& maps, const TcOutMaps& om, const TcParams& p, int tiles_x, int tiles_y,
                           int batch, cudaStream_t st, const char* what) {
    const int num_tiles = tiles_x * tiles_y * batch;
    return launch_persistent<TcCfg<NBOX, BK, BR, NPL>, tc_conv_kernel<MODE, NBOX, BR, BK, BF16, NPL>>(
        num_tiles, st, what, maps, om, p, tiles_x, tiles_y, num_tiles);
}

template <int MODE, int NBOX, int BR, int BK, int NPL = 2>
static int launch_conv(const TcMaps& maps, const TcOutMaps& om, const TcParams& p, int tiles_x, int tiles_y, int batch,
                       cudaStream_t st, const char* what) {
    if (p.operand_bf16)
        return launch_conv_fmt<MODE, NBOX, BR, BK, true, NPL>(maps, om, p, tiles_x, tiles_y, batch, st, what);
    return launch_conv_fmt<MODE, NBOX, BR, BK, false, NPL>(maps, om, p, tiles_x, tiles_y, batch, st, what);
}

static void fill_taps_tc(int* tap_off, int k, int dilation, int causal, bool transpose) {
    const int padl = causal ? (k - 1) * dilation : (k - 1) / 2 * dilation;
    for (int j = 0; j < MAX_TAPS_TC; ++j)
        tap_off[j] = j < k ? (transpose ? (padl - j * dilation) : (j * dilation - padl)) : 0;
}

// plane p of a [nplanes][...] bf16 buffer
static inline const void* plane(const void* base, int pl, long long plane_elems) {
    return (const char*)base + (size_t)pl * plane_elems * 2;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

// 1 if the tensor-core ConvBlock path supports this block shape (else the caller uses the exact-fp32 kernels)
int dv3_tc_supported(int B, int C, int T, int k) {
    return (C % 128 == 0) && T >= 1 && k >= 1 && k <= MAX_TAPS_TC && B >= 1 && B <= 65535;
}
// plain convs: any channel counts (planes are padded to a multiple of 8 channels); k-tap convs need
// Cout % 128 == 0 so a weight box never straddles two taps
int dv3_tc_conv_supported(int B, int Cin, int Cout, int T, int k) {
    return T >= 1 && k >= 1 && k <= MAX_TAPS_TC && B >= 1 && B <= 65535 && (k == 1 || Cout % 128 == 0) && Cin >= 8 &&
           Cout >= 1;
}

// Gated forward.  xd: [npl][B][T][C] fp16 planes of the (dropped-out) input; w: [npl][k][2C][C] fp16 planes of the
// normalised weight; the rest as dv3_convblock_fwd.  64-channel tiles (64 a | 64 b columns).  Two planes: BK = 32,
// a BK = 64 stage (64 KB) leaves room for only two ring stages, BK = 32 for four (with five, H100: 1.45x faster at
// C=512, T=800).  One plane: BK = 64 (C % 128 == 0), four 32 KB stages.
int dv3_tc_convblock_fwd(const void* xd, const void* w, int npl, const float* bias, const float* spk,
                         const float* res, float* y, float* save_a, float* save_s, int B, int C, int T, int k,
                         int dilation, int causal, int mode, int residual, const void* fuse, void* stream) {
    DV3_REQUIRE(dv3_tc_supported(B, C, T, k), "tc_convblock_fwd: unsupported shape B=%d C=%d T=%d k=%d", B, C, T, k);
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_convblock_fwd: npl must be 1 or 2");
    DV3_REQUIRE(fuse == nullptr, "tc_convblock_fwd: fuse must be NULL");
    TcMaps maps;
    const int t_tiles = (T + 127) / 128;
    const int BK = npl == 2 ? 32 : 64;
    for (int pl = 0; pl < npl; ++pl) {
        if (encode_tmap_bf16_3d(&maps.a[pl], plane(xd, pl, (long long)B * T * C), C, T, B, (uint64_t)C * 2,
                                (uint64_t)T * C * 2, BK, 128)) return 1;
        if (encode_tmap_bf16_3d(&maps.b[pl], plane(w, pl, (long long)k * 2 * C * C), C, (uint64_t)k * 2 * C, 1,
                                (uint64_t)C * 2, (uint64_t)k * 2 * C * C * 2, BK, 64)) return 1;
    }
    TcParams p = {};
    p.T = T; p.Nc = C; p.rows_per_tap = 2 * C; p.k = k; p.kb_n = C / BK;
    fill_taps_tc(p.tap_off, k, dilation, causal, false);
    p.bias = bias; p.spk = spk; p.res = res; p.y = y; p.save_a = save_a; p.save_s = save_s;
    p.gate_mode = mode; p.residual = residual;
    p.gmain = 1.f + config().tc_gamma * (float)(p.k * p.kb_n * (BK / 16));
    const bool need_res = mode != 0 || residual;
    TcOutMaps om = {};
    p.tma_out = tma_rows(y, T) && (!save_a || tma_rows(save_a, T)) && (!save_s || tma_rows(save_s, T)) &&
                (!need_res || tma_rows(res, T));
    if (p.tma_out) {
        const float* outs[3] = {y, save_a, save_s};
        for (int i = 0; i < 3; ++i)
            if (outs[i] && encode_tmap_f32_bct(&om.out[i], outs[i], B, C, T, 64)) return 1;
        if (need_res && encode_tmap_f32_bct(&om.res, res, B, C, T, 64)) return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    // forward operands: fp16 planes (BF16 = false)
    if (npl == 1)
        return launch_conv_fmt<TC_GATED, 2, 64, 64, false, 1>(maps, om, p, t_tiles, C / 64, B, st, "tc_convblock_fwd");
    return launch_conv_fmt<TC_GATED, 2, 64, 32, false, 2>(maps, om, p, t_tiles, C / 64, B, st, "tc_convblock_fwd");
}

// Generic conv / data-gradient:  out (B, Nc, T) fp32 = sum_j A[b, t+off_j, :] . W[j, n, :]  (+ epilogue)
//   a: [npl][B][T][Kp] planes, Kp = Kc rounded up to 8;  w: [npl][k][Nc][Kp] planes (fp16 for a forward conv, bf16
//   for a data gradient).  transpose_taps = 1 for a data gradient (offsets padl - j*d), 0 for a forward conv.
// Tile width: 128 output channels, or 64 when 128-wide tiles would leave most of the SMs idle.  BK with two planes:
// 32 for 128-wide tiles (a 64 KB BK = 64 stage would leave two ring stages, BK = 32 gives four); 64 for 64-wide tiles
// when Kc % 64 == 0 (else 32: the 80-channel mel input, the 513-wide linear output, the 16-wide speaker embedding).
// One plane: 64 whenever Kc % 64 == 0, at both tile widths (stages of half the bytes), else 32.
int dv3_tc_conv(const void* a, const void* w, int npl, float* out, int B, int Kc, int Nc, int T, int k, int dilation,
                int causal, int transpose_taps, const float* bias, int relu, float p_drop,
                const unsigned long long* seed_ptr, unsigned salt, int addmode, const float* e1, const float* e2,
                float alpha, const void* fuse, void* stream) {
    DV3_REQUIRE(k >= 1 && k <= MAX_TAPS_TC && (k == 1 || Nc % 128 == 0) && B <= 65535,
                "tc_conv: unsupported shape B=%d Kc=%d Nc=%d T=%d k=%d", B, Kc, Nc, T, k);
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_conv: npl must be 1 or 2");
    DV3_REQUIRE(fuse == nullptr, "tc_conv: fuse must be NULL");
    const int Kp = (Kc + 7) / 8 * 8;
    const int t_tiles = (T + 127) / 128;
    cudaStream_t st = (cudaStream_t)stream;
    const long long tiles128 = (long long)t_tiles * ((Nc + 127) / 128) * B;
    const bool narrow = Nc > 64 && (k == 1 || Nc % 64 == 0) && tiles128 < 100;
    const bool k64 = Kc % 64 == 0;
    const int bk = ((narrow || npl == 1) && k64) ? 64 : 32, br = narrow ? 64 : 128;
    TcMaps maps;
    for (int pl = 0; pl < npl; ++pl) {
        if (encode_tmap_bf16_3d(&maps.a[pl], plane(a, pl, (long long)B * T * Kp), Kc, T, B, (uint64_t)Kp * 2,
                                (uint64_t)T * Kp * 2, bk, 128)) return 1;
        if (encode_tmap_bf16_3d(&maps.b[pl], plane(w, pl, (long long)k * Nc * Kp), Kc, (uint64_t)k * Nc, 1,
                                (uint64_t)Kp * 2, (uint64_t)k * Nc * Kp * 2, bk, br)) return 1;
    }
    TcParams p = {};
    p.T = T; p.Nc = Nc; p.rows_per_tap = Nc; p.k = k; p.kb_n = (Kc + bk - 1) / bk;
    fill_taps_tc(p.tap_off, k, dilation, causal, transpose_taps != 0);
    p.out = out; p.bias = bias; p.relu = relu; p.e1 = e1; p.e2 = e2; p.alpha = alpha; p.addmode = addmode;
    p.p_drop = p_drop; p.seed_ptr = seed_ptr; p.salt = salt;
    p.gmain = 1.f + config().tc_gamma * (float)(p.k * p.kb_n * (bk / 16));
    // forward conv: fp16 activation x fp16 weight planes; data gradient: bf16 gradient x bf16 weight planes
    p.operand_bf16 = transpose_taps ? 1 : 0;
    TcOutMaps om = {};
    p.tma_out = tma_rows(out, T);
    if (p.tma_out && encode_tmap_f32_bct(&om.out[0], out, B, Nc, T, br)) return 1;
    const int tiles_y = (Nc + br - 1) / br;
    if (npl == 1) {
        if (narrow) {
            if (k64) return launch_conv<TC_CONV, 1, 64, 64, 1>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(64)");
            return launch_conv<TC_CONV, 1, 64, 32, 1>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(64,bk32)");
        }
        if (k64) return launch_conv<TC_CONV, 1, 128, 64, 1>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(128,bk64)");
        return launch_conv<TC_CONV, 1, 128, 32, 1>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(128)");
    }
    if (narrow) {
        if (k64) return launch_conv<TC_CONV, 1, 64, 64>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(64)");
        return launch_conv<TC_CONV, 1, 64, 32>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(64,bk32)");
    }
    return launch_conv<TC_CONV, 1, 128, 32>(maps, om, p, t_tiles, tiles_y, B, st, "tc_conv(128)");
}

// Split count of the weight gradient, chosen for the persistent grid.  A candidate is a batch range of
// bps = ceil(B / nsplit) utterances per split; it is costed in 32-row K-iterations with the schedule the kernel runs:
//   tk = m-tiles * n-tiles * k units per split, U = tk * nsplit units, G = min(U, sms) CTAs; a unit of a full split
//   runs L = bps * kb_n iterations, one of the last split L_last <= L.  Dealt round-robin longest first, CTA 0 carries
//   the most: ceil(U_full / G) long units (U_full = tk * (nsplit - 1)) and ceil(U / G) units in all, so
//     makespan = ceil(U_full / G) * (L - L_last) + ceil(U / G) * (L_last + WG_UNIT_ITERS)
//   plus the partial slabs, nsplit * Mw * Nw * k * 8 bytes (written here, read by the weight-norm backward), at
//   WG_SLAB_BYTES_PER_ITER bytes per iteration for the whole GPU.
// The smallest nsplit within 3 % of the cheapest wins.  The result depends on the shape and the SM count only.
// Both constants from tools/wgrad_time.py --fit on an H100 SXM (700 W): t = 6.6 us + 0.47 us per K-iteration of CTA 0
// + 11.6 us per unit of CTA 0, i.e. about 25 iterations per unit; 0.47 us at 3.35 TB/s (data sheet) is 1.5 MB.
constexpr double WG_UNIT_ITERS = 25.0;             // per-unit cost in K-iterations
constexpr double WG_SLAB_BYTES_PER_ITER = 1.5e6;   // HBM bytes per K-iteration of time, whole GPU
int dv3_tc_wgrad_nsplit(int B, int Mw, int Nw, int T, int k) {
    const long long tk = (long long)((Mw + 127) / 128) * ((Nw + 127) / 128) * k;
    const long long kb_n = (T + 31) / 32, sms = config().sms;
    const double slab = (double)Mw * Nw * k * 8.0 / WG_SLAB_BYTES_PER_ITER;
    auto cost = [&](int ns) {
        const long long bps = (B + ns - 1) / ns, U = tk * ns, U_full = tk * (ns - 1), G = U < sms ? U : sms;
        const long long L = bps * kb_n, L_last = (B - (ns - 1) * bps) * kb_n;
        return (double)((U_full + G - 1) / G) * (double)(L - L_last) +
               (double)((U + G - 1) / G) * ((double)L_last + WG_UNIT_ITERS) + ns * slab;
    };
    // the distinct batch-range splits, ascending: ns = ceil(B / bps) for bps = B, B - 1, ..., 1
    double best = 0.0;
    for (int bps = B, prev = 0; bps >= 1; --bps) {
        const int ns = (B + bps - 1) / bps;
        if (ns != prev && (prev == 0 || cost(ns) < best)) best = cost(ns);
        prev = ns;
    }
    for (int bps = B, prev = 0; bps >= 1; --bps) {
        const int ns = (B + bps - 1) / bps;
        if (ns != prev && cost(ns) <= 1.03 * best) return ns;
        prev = ns;
    }
    return 1;
}

// Weight gradient from (B,T,C) planes.  dy: [npl][B][T][pad8(Mw)], xd: [npl][B][T][pad8(Nw)]; partial element
// (m, n, j) at (m%msplit)*s_m + (m/msplit)*s_mh + n*s_n + j*s_j of split `s` at dw_partials + s*split_stride.
int dv3_tc_wgrad_mn_npl(const void* dy, const void* xd, int npl, float* dw_partials, long long split_stride, int B,
                        int Mw, int Nw, int T, int k, int dilation, int causal, int msplit, long long s_m,
                        long long s_mh, long long s_n, long long s_j, void* stream) {
    DV3_REQUIRE(k >= 1 && k <= MAX_TAPS_TC && B <= 65535, "tc_wgrad_mn: unsupported shape k=%d", k);
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_wgrad_mn: npl must be 1 or 2");
    const int Mp = (Mw + 7) / 8 * 8, Np = (Nw + 7) / 8 * 8;
    TcMaps maps;
    for (int pl = 0; pl < npl; ++pl) {
        if (encode_tmap_bf16_3d(&maps.a[pl], plane(dy, pl, (long long)B * T * Mp), Mw, T, B, (uint64_t)Mp * 2,
                                (uint64_t)T * Mp * 2, 64, 32)) return 1;
        if (encode_tmap_bf16_3d(&maps.b[pl], plane(xd, pl, (long long)B * T * Np), Nw, T, B, (uint64_t)Np * 2,
                                (uint64_t)T * Np * 2, 64, 32)) return 1;
    }
    TcMnParams p = {};
    p.T = T; p.B = B; p.Mw = Mw; p.Nw = Nw; p.k = k; p.kb_n = (T + 31) / 32;
    fill_taps_tc(p.tap_off, k, dilation, causal, false);
    p.nsplit = dv3_tc_wgrad_nsplit(B, Mw, Nw, T, k);
    p.batches_per_split = (B + p.nsplit - 1) / p.nsplit;
    p.tiles_n = (Nw + 127) / 128; p.tiles_m = (Mw + 127) / 128;
    const long long units = (long long)p.tiles_n * p.tiles_m * k * p.nsplit;
    DV3_REQUIRE(units < (1ll << 31), "tc_wgrad_mn: %lld work units", units);
    p.num_units = (int)units;
    p.dw = dw_partials; p.split_stride = split_stride;
    p.msplit = msplit; p.s_m = s_m; p.s_mh = s_mh; p.s_n = s_n; p.s_j = s_j;
    p.gcoef = config().tc_gamma;
    cudaStream_t st = (cudaStream_t)stream;
    if (npl == 1)
        return launch_persistent<WgCfg<1>, tc_wgrad_mn_kernel<1>>(p.num_units, st, "tc_wgrad_mn", maps, p);
    return launch_persistent<WgCfg<2>, tc_wgrad_mn_kernel<2>>(p.num_units, st, "tc_wgrad_mn", maps, p);
}

int dv3_tc_wgrad_mn(const void* dy, const void* xd, float* dw_partials, long long split_stride, int B, int Mw,
                    int Nw, int T, int k, int dilation, int causal, int msplit, long long s_m, long long s_mh,
                    long long s_n, long long s_j, void* stream) {
    return dv3_tc_wgrad_mn_npl(dy, xd, 2, dw_partials, split_stride, B, Mw, Nw, T, k, dilation, causal, msplit, s_m,
                               s_mh, s_n, s_j, stream);
}

}  // extern "C"
