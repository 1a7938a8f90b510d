// Weight norm for ALL weight-normed convolutions of the model in one launch per phase.
// The per-layer kernels (weightnorm.cu: wn_norm_kernel + wn_pack_split_kernel in the forward, wn_bwd_kernel in the
// backward) are tiny: 127 launches per training step that together move ~0.5 GB but cost ~1.1 ms of GPU time because
// each one is latency bound (6-14 us for a few hundred KB).  The weights do not depend on activations, so the training step
// prepares every layer's packed bf16 operand planes up front (norm, then pack: 2 launches) and folds every layer's
// split-K reduction + g/v gradient into one launch after the backward pass.  A device-resident table of Dv3WnEntry
// records (built once on the host) maps a block index to (layer, block-within-layer).
#include "wn_device.cuh"
#include "../../include/dv3b200.h"

namespace dv3 {

// entry whose [blk0, next blk0) range contains block b; blk0 of field F is ascending over the table
template <int FIELD>
__device__ __forceinline__ int blk0_of(const Dv3WnEntry& e) {
    return FIELD == 0 ? e.blk_norm : FIELD == 1 ? e.blk_pack : e.blk_bwd;
}
template <int FIELD>
__device__ __forceinline__ int find_entry(const Dv3WnEntry* __restrict__ tab, int n, int b) {
    int lo = 0, hi = n - 1;                 // last entry with blk0 <= b
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (blk0_of<FIELD>(tab[mid]) <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) wn_norm_batched_kernel(const Dv3WnEntry* __restrict__ tab, int n) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int ei = find_entry<0>(tab, n, blockIdx.x);
    const Dv3WnEntry e = tab[ei];
    const int lb = blockIdx.x - e.blk_norm;
    wn_norm_row(e.v, e.g, e.inv_norm, e.scale, e.Cout, e.Cin * e.k, (lb * 256 + threadIdx.x) >> 5, threadIdx.x & 31);
}

// same layouts as dv3_tc_weightnorm_fwd: wfwd [NPL][k][Cout][Cinp], wbwd [NPL][k][Cin][Coutp]
template <int NPL>
__global__ void __launch_bounds__(256) wn_pack_batched_kernel(const Dv3WnEntry* __restrict__ tab, int n) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float tile[32][33];
    const int ei = find_entry<1>(tab, n, blockIdx.x);
    const Dv3WnEntry e = tab[ei];
    const int lb = blockIdx.x - e.blk_pack;
    const int by = lb / e.pack_gx, bx = lb - by * e.pack_gx;
    const long long Cinp = (e.Cin + 7) / 8 * 8, Coutp = (e.Cout + 7) / 8 * 8;
    wn_pack_split_tile<FMT_F16, FMT_BF16, NPL>(e.v, e.scale, e.wfwd, Cinp, 1, (long long)e.Cout * Cinp,
                             (long long)e.k * e.Cout * Cinp, e.wbwd, 1, Coutp, (long long)e.Cin * Coutp,
                             (long long)e.k * e.Cin * Coutp, e.Cout, e.Cin, e.k, bx, by, tile);
}

// tap-major partials [split][j][Cout][Cin] (what dv3_tc_wgrad_mn writes) -> dv, dg
__global__ void __launch_bounds__(256) wn_bwd_batched_kernel(const Dv3WnEntry* __restrict__ tab, int n,
                                                             int accumulate) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int ei = find_entry<2>(tab, n, blockIdx.x);
    const Dv3WnEntry e = tab[ei];
    const int r = blockIdx.x - e.blk_bwd;
    if (r >= e.Cout) return;
    wn_bwd_row(e.partials, e.split_stride, e.nsplit, e.Cin, e.v, e.g, e.inv_norm, e.dv, e.dg, e.Cout, e.Cin * e.k,
               accumulate, r);
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_tc_weightnorm_fwd_batched_npl(const Dv3WnEntry* table_dev, int n, int norm_blocks, int pack_blocks, int npl,
                                      void* stream) {
    DV3_REQUIRE(n > 0 && norm_blocks > 0 && pack_blocks > 0, "tc_weightnorm_fwd_batched: empty table");
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_weightnorm_fwd_batched: npl must be 1 or 2");
    cudaStream_t st = (cudaStream_t)stream;
    launch_k(wn_norm_batched_kernel, norm_blocks, 256, 0, st, table_dev, n);
    if (int e = check_launch("tc_weightnorm_fwd_batched(norm)")) return e;
    if (npl == 1) launch_k(wn_pack_batched_kernel<1>, pack_blocks, dim3(32, 8), 0, st, table_dev, n);
    else launch_k(wn_pack_batched_kernel<2>, pack_blocks, dim3(32, 8), 0, st, table_dev, n);
    return check_launch("tc_weightnorm_fwd_batched(pack)");
}

int dv3_tc_weightnorm_fwd_batched(const Dv3WnEntry* table_dev, int n, int norm_blocks, int pack_blocks,
                                  void* stream) {
    return dv3_tc_weightnorm_fwd_batched_npl(table_dev, n, norm_blocks, pack_blocks, 2, stream);
}

int dv3_weightnorm_bwd_batched(const Dv3WnEntry* table_dev, int n, int bwd_blocks, int accumulate, void* stream) {
    DV3_REQUIRE(n > 0 && bwd_blocks > 0, "weightnorm_bwd_batched: empty table");
    launch_k(wn_bwd_batched_kernel, bwd_blocks, 256, 0, (cudaStream_t)stream, table_dev, n, accumulate);
    return check_launch("weightnorm_bwd_batched");
}

}  // extern "C"
