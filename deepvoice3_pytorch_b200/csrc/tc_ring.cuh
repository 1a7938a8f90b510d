// Shared-memory layout of the tensor-core GEMM pipeline (tc_pipeline in tc_gemm.cu): the ring depth and the bytes of
// every kernel configuration.  Plain constexpr C++ with no CUDA dependency, so that a host compiler can print the
// table (tests/test_tc_ring_host.py).
#pragma once

namespace dv3 {

constexpr int SMEM_LIMIT = 232448;          // 227 KB opt-in dynamic shared memory per CTA
constexpr int RING_SLACK = 1024 + 512;      // 1 KB alignment slack of the dynamic base + the barriers

// STAGES ring stages of STAGE bytes, the consumer -> epilogue hand-off tile (the whole fp32 output tile), STAGING bytes
// of epilogue input staging, then the barriers full[STAGES], empty[STAGES], acc_full, acc_empty, in_full.  The depth is
// chosen per configuration (measured, DESIGN.md section 2.4); MAX_STAGES is the deepest ring that would fit.
// Two hand-off layouts:
//   * DENSE (the conv kernel): the shared-memory image of four TMA boxes over a (B, C, T) fp32 tensor, so that the
//     epilogue stores it with bulk tensor copies.  Box q holds time steps [32 q, 32 q + 32) of all NCOLS channels:
//     channel c is one 128-byte row (time contiguous) at q * NCOLS * 128 + c * 128, and SWIZZLE_128B places time
//     step tt of that row in 16-byte chunk (tt / 4) ^ (c % 8).  The consumers' fragment-order writes and the
//     epilogue's reads (a warp reads one channel of 32 consecutive time steps) are both conflict-free; the swizzle of
//     a consumer write is a per-thread constant XOR the fragment index (tc_pipeline).
//   * padded [128 rows][NCOLS + 1] (the weight gradient): the odd pitch keeps the epilogue's column reads
//     conflict-free; the consumers' fragment-order writes are 4-way conflicted.
template <int STAGE_BYTES, int TILE_COLS, int DEPTH, bool DENSE_TILE = false, int STAGING_BYTES = 0>
struct RingCfg {
    static constexpr int STAGE = STAGE_BYTES;
    static constexpr int NCOLS = TILE_COLS;              // columns of the output tile and of each accumulator
    static constexpr bool DENSE = DENSE_TILE;
    static constexpr int ACC_PITCH = DENSE ? NCOLS : NCOLS + 1;
    static constexpr int ACC_TILE = 128 * ACC_PITCH * 4;
    static constexpr int STAGING = STAGING_BYTES;
    static constexpr int STAGES = DEPTH;
    static constexpr int SMEM = STAGES * STAGE + ACC_TILE + STAGING + RING_SLACK;
    static constexpr int MAX_STAGES = (SMEM_LIMIT - ACC_TILE - STAGING - RING_SLACK) / STAGE;
    static_assert(STAGE % 1024 == 0, "ring stages keep the 1 KB alignment of the swizzled TMA tiles");
    static_assert(ACC_TILE % 1024 == 0 || !DENSE, "the dense tile and the staging buffer are swizzled TMA boxes");
    static_assert(STAGES >= 2, "pipeline needs at least two stages");
    static_assert(SMEM <= SMEM_LIMIT, "ring + hand-off tile + staging + barriers exceed the 227 KB of a CTA");
};

// Conv ring: a stage holds NPL planes of one 128-row A tile and NBOX B boxes of BR rows, each BK 16-bit channels wide.
// BR = rows of one B-operand box (128, or 64 for problems too small to fill the machine with 128-wide tiles); NPL =
// operand planes per stage (2: hi / lo pairs, 1: single pass).  Every configuration the launchers use names its depth,
// measured per configuration over every GEMM shape of the deepvoice3_ljspeech step (tools/ring_ab.py, DESIGN.md
// section 2.4).  A fifth 32 KB stage (with the padded 66 KB hand-off tile of the time) made the multi-wave gated
// forwards and 128-column convs 1-5 % slower and the one-wave ones at most 1 % faster, so those stay at 4; a fourth
// 48 KB stage made the 64-column BK = 64 GEMMs 4-17 % faster.  The gated forward's 4 x 32 KB ring, 64 KB tile and
// 32 KB residual staging take 230 912 of the 232 448 bytes.
template <int NBOX, int BK, int BR, int NPL> struct ConvRing;
// two planes
template <> struct ConvRing<2, 32, 64, 2> { static constexpr int STAGES = 4; };    // gated forward, 32 KB stages
template <> struct ConvRing<1, 32, 128, 2> { static constexpr int STAGES = 4; };   // 128-column conv, 32 KB stages
template <> struct ConvRing<1, 64, 64, 2> { static constexpr int STAGES = 4; };    // 64-column conv at BK = 64, 48 KB
template <> struct ConvRing<1, 32, 64, 2> { static constexpr int STAGES = 6; };    // 64-column conv at BK = 32, 24 KB
// single pass: BK = 64 wherever the contraction is a multiple of 64 channels, so a one-plane stage carries 32 KB or
// 24 KB and feeds the MMA 4 K-steps per barrier round trip (a one-plane BK = 32 stage would carry 12-16 KB for 2).
// Chosen from the bytes per stage, not from an A/B of the two BK values (DESIGN.md section 2.7).
template <> struct ConvRing<2, 64, 64, 1> { static constexpr int STAGES = 4; };    // gated forward, 32 KB stages
template <> struct ConvRing<1, 64, 128, 1> { static constexpr int STAGES = 4; };   // 128-column conv at BK = 64, 32 KB
template <> struct ConvRing<1, 32, 128, 1> { static constexpr int STAGES = 6; };   // 128-column conv at BK = 32, 16 KB
template <> struct ConvRing<1, 64, 64, 1> { static constexpr int STAGES = 6; };    // 64-column conv at BK = 64, 24 KB
template <> struct ConvRing<1, 32, 64, 1> { static constexpr int STAGES = 6; };    // 64-column conv at BK = 32, 12 KB

// Dense hand-off tile; the gated forward (NBOX = 2) also stages the unit's 128-step x BR-channel fp32 residual tile
// (32 KB), which its epilogue overwrites with y before storing it.
template <int NBOX, int BK, int BR, int NPL = 2>
using TcCfg = RingCfg<NPL * (128 + NBOX * BR) * BK * 2, BR * NBOX, ConvRing<NBOX, BK, BR, NPL>::STAGES, true,
                      NBOX == 2 ? 128 * BR * 4 : 0>;

// Weight-gradient ring: per plane 128 channels of m and 128 channels of n, each as two 64-channel x 32-row boxes.
// The [128][129] hand-off tile (66 KB) leaves room for five 32 KB two-plane stages.
constexpr int WG_BOX = 64 * 32 * 2;                      // 64 channels x 32 time steps of bf16 = 4 KB
template <int NPL>
using WgCfg = RingCfg<NPL * 4 * WG_BOX, 128, NPL == 2 ? 5 : 6>;

}  // namespace dv3
