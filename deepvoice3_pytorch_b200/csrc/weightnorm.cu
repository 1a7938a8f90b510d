// Per-layer weight normalisation  w = g * v / ||v||  (reference modules.py:85,100,109 -- old-style
// torch.nn.utils.weight_norm, dim=0, re-evaluated by a forward-pre-hook on every call).
// The forward writes w directly in the two packed layouts the conv kernels consume (forward operand and
// data-gradient operand): fp32 for the exact-fp32 kernels (dv3_weightnorm_fwd), 16-bit operand planes for the
// tensor-core kernels (dv3_tc_weightnorm_fwd, dv3_tc_weightnorm_convt_fwd), so no separate transpose/pack pass exists;
// the backward folds the split-K reduction of the weight-gradient partials into the g/v gradient.  The kernel bodies
// (wn_device.cuh) are shared with the all-layers-in-one-launch form of wn_batched.cu.
#include "common.cuh"
#include "wn_device.cuh"

namespace dv3 {

// one warp per row r: inv_norm[r] = 1/||v[r,:]||, scale[r] = g[r]*inv_norm[r]
__global__ void wn_norm_kernel(const float* __restrict__ v, const float* __restrict__ g,
                               float* __restrict__ inv_norm, float* __restrict__ scale, int R, int L) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    wn_norm_row(v, g, inv_norm, scale, R, L, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, threadIdx.x & 31);
}

// pack of one 32 x 32 tile per CTA (block 32x8), see wn_pack_split_tile
template <int FMTA, int FMTB, int NPL>
__global__ void wn_pack_split_kernel(const float* __restrict__ v, const float* __restrict__ scale,
                                     void* __restrict__ outA, long long a_r, long long a_x, long long a_j,
                                     long long a_plane, void* __restrict__ outB, long long b_r, long long b_x,
                                     long long b_j, long long b_plane, int R, int X, int k) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float tile[32][33];
    wn_pack_split_tile<FMTA, FMTB, NPL>(v, scale, outA, a_r, a_x, a_j, a_plane, outB, b_r, b_x, b_j, b_plane, R, X, k,
                                   blockIdx.x, blockIdx.y, tile);
}

// backward, one CTA (256 threads) per row (body in wn_device.cuh)
__global__ void __launch_bounds__(256) wn_bwd_kernel(float* __restrict__ dw_partials, long long split_stride,
                                                     int nsplit, int jmajor_X, const float* __restrict__ v,
                                                     const float* __restrict__ g,
                                                     const float* __restrict__ inv_norm, float* __restrict__ dv,
                                                     float* __restrict__ dg, int R, int L, int accumulate) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    wn_bwd_row(dw_partials, split_stride, nsplit, jmajor_X, v, g, inv_norm, dv, dg, R, L, accumulate, blockIdx.x);
}

// norm of R rows of length X*k, then the pack of both layouts: outA with lanes along (x,j), outB with lanes along r
template <int FMTA, int FMTB, int NPL = 2>
static int weightnorm_launch(const float* v, const float* g, float* inv_norm, float* scale, void* outA, long long a_r,
                             long long a_x, long long a_j, long long a_plane, void* outB, long long b_r, long long b_x,
                             long long b_j, long long b_plane, int R, int X, int k, cudaStream_t st, const char* what) {
    const int L = X * k;
    launch_k(wn_norm_kernel, ceil_div(R * 32, 256), 256, 0, st, v, g, inv_norm, scale, R, L);
    if (int e = check_launch(what)) return e;
    launch_k(wn_pack_split_kernel<FMTA, FMTB, NPL>, dim3(ceil_div(L, 32), ceil_div(R, 32)), dim3(32, 8), 0, st, v, scale,
             outA, a_r, a_x, a_j, a_plane, outB, b_r, b_x, b_j, b_plane, R, X, k);
    return check_launch(what);
}

}  // namespace dv3

using namespace dv3;

extern "C" {

// v: [R][X][k] (k fastest).  out1[r*s1r + x*s1x + j*s1j], out2[...]; inv_norm/scale: [R] workspaces.
int dv3_weightnorm_fwd(const float* v, const float* g, float* inv_norm, float* scale, float* out1,
                       float* out2, int R, int X, int k, long long s1r, long long s1x, long long s1j,
                       long long s2r, long long s2x, long long s2j, void* stream) {
    DV3_REQUIRE(R > 0 && X > 0 && k > 0, "weightnorm_fwd: empty weight");
    // out2 is written with lanes along (x,j), out1 with lanes along r
    return weightnorm_launch<FMT_F32, FMT_F32>(v, g, inv_norm, scale, out2, s2r, s2x, s2j, 0, out1, s1r, s1x, s1j, 0,
                                               R, X, k, (cudaStream_t)stream, "weightnorm_fwd");
}

// dw_partials: [nsplit][R*X*k] (slot 0 is overwritten with the reduced dW); tap_major = 0: v's own layout
// (r, x, j); 1: [j][r][x].  accumulate = 1 adds into dv / dg instead of overwriting them.
int dv3_weightnorm_bwd(float* dw_partials, long long split_stride, int nsplit, int tap_major, const float* v,
                       const float* g, const float* inv_norm, float* dv, float* dg, int R, int X, int k,
                       int accumulate, void* stream) {
    launch_k(wn_bwd_kernel, R, 256, 0, (cudaStream_t)stream,
        dw_partials, split_stride, nsplit, tap_major ? X : 0, v, g, inv_norm, dv, dg, R, X * k, accumulate);
    return check_launch("weightnorm_bwd");
}

// Weight norm + split for a conv weight v (Cout, Cin, k), g [Cout]:
//   wfwd: [npl][k][Cout][Cinp] fp16 planes (forward operand: rows co, K = ci)
//   wbwd: [npl][k][Cin][Coutp] bf16 planes (data-gradient operand, multiplied with bf16 gradient planes)
int dv3_tc_weightnorm_fwd(const float* v, const float* g, float* inv_norm, float* scale, void* wfwd, int npl,
                          void* wbwd, int Cout, int Cin, int k, void* stream) {
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_weightnorm_fwd: npl must be 1 or 2");
    const long long Cinp = (Cin + 7) / 8 * 8, Coutp = (Cout + 7) / 8 * 8;
    auto launch = npl == 1 ? weightnorm_launch<FMT_F16, FMT_BF16, 1> : weightnorm_launch<FMT_F16, FMT_BF16, 2>;
    return launch(v, g, inv_norm, scale, wfwd, Cinp, 1, (long long)Cout * Cinp, (long long)k * Cout * Cinp, wbwd, 1,
                  Coutp, (long long)Cin * Coutp, (long long)k * Cin * Coutp, Cout, Cin, k, (cudaStream_t)stream,
                  "tc_weightnorm_fwd");
}

// ConvTranspose1d(k=2,s=2) weight v (Cin, Cout, 2), g [Cin] (norm over dim 0 = Cin), run as a 1x1 conv with
// 2*Cout output rows ordered (j, co):
//   wfwd: [npl][2*Cout][Cinp] fp16, rows (j,co), K = ci        wbwd: [npl][Cin][K2p] bf16, rows ci, K = (j,co)
int dv3_tc_weightnorm_convt_fwd(const float* v, const float* g, float* inv_norm, float* scale, void* wfwd, int npl,
                                void* wbwd, int Cin, int Cout, void* stream) {
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_weightnorm_convt_fwd: npl must be 1 or 2");
    const long long Cinp = (Cin + 7) / 8 * 8, K2p = (2 * Cout + 7) / 8 * 8;
    // r = ci, x = co, j: outA (lanes along (x,j)) = wbwd [ci][j*Cout+co] ; outB (lanes along r) = wfwd [(j*Cout+co)][ci]
    auto launch = npl == 1 ? weightnorm_launch<FMT_BF16, FMT_F16, 1> : weightnorm_launch<FMT_BF16, FMT_F16, 2>;
    return launch(v, g, inv_norm, scale, wbwd, K2p, 1, (long long)Cout, (long long)Cin * K2p, wfwd, 1, Cinp,
                  (long long)Cout * Cinp, (long long)2 * Cout * Cinp, Cin, Cout, 2, (cudaStream_t)stream,
                  "tc_weightnorm_convt_fwd");
}

// ConvTranspose1d(k=s, stride=s) weight v (Cin, Cout, s), g [Cin], s in [2, 8], as a 1x1 conv with s*Cout rows ordered
// (j, co): the layouts of dv3_tc_weightnorm_convt_fwd with s taps.
int dv3_tc_weightnorm_convt_s_fwd(const float* v, const float* g, float* inv_norm, float* scale, void* wfwd, int npl,
                                  void* wbwd, int Cin, int Cout, int stride, void* stream) {
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_weightnorm_convt_s_fwd: npl must be 1 or 2");
    DV3_REQUIRE(stride >= 2 && stride <= 8, "tc_weightnorm_convt_s_fwd: stride %d outside [2, 8]", stride);
    const long long Cinp = (Cin + 7) / 8 * 8, Ksp = ((long long)stride * Cout + 7) / 8 * 8;
    auto launch = npl == 1 ? weightnorm_launch<FMT_BF16, FMT_F16, 1> : weightnorm_launch<FMT_BF16, FMT_F16, 2>;
    return launch(v, g, inv_norm, scale, wbwd, Ksp, 1, (long long)Cout, (long long)Cin * Ksp, wfwd, 1, Cinp,
                  (long long)Cout * Cinp, (long long)stride * Cout * Cinp, Cin, Cout, stride, (cudaStream_t)stream,
                  "tc_weightnorm_convt_s_fwd");
}

}  // extern "C"
