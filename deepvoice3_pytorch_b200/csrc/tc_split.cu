// Activation and gradient operand preparation for the tensor-core path (tc_gemm.cu): every fp32 operand x becomes a
// 16-bit (hi, lo * 2^11) pair (common.cuh: fp16 pairs for forward operands, bf16 pairs for gradients), written in the
// (B,T,C) layout each implicit GEMM consumes (K-major for the forward / data gradient, MN-major for the weight
// gradient).  The weight operands come from the weight norm (weightnorm.cu per layer, wn_batched.cu for all layers at
// once).  These passes are pure HBM streaming and absorb work the fp32 path does inside its loaders: the conv-input
// dropout mask, the ReLU mask of the incoming gradient, the bias-gradient reduction and the (B,C,T) <-> (B,T,C)
// layout change.  Channel pitches are padded to a multiple of 8 (16 bytes, the TMA stride granularity); pad columns
// are never read (the tensor maps carry the true extent).  With one plane (single-pass mode, npl = 1) only the hi
// plane is computed and written: the same bits as plane 0 of the pair.
#include <cuda_bf16.h>
#include "common.cuh"

namespace dv3 {

// ---- activation-side operand preparation: ONE kernel template, three uses ------------------------------------
//   SPLIT_INPUT  x (B,C,T) -> conv-input dropout -> fp16 planes (B,T,Cp) [forward operand] and, when wg != NULL, the same
//                values as a bf16 pair [operand of the weight gradient, which multiplies them with bf16 gradient
//                planes: a wgmma cannot mix fp16 and bf16 operands]
//   SPLIT_GATE   gate backward (conv.cu gate_bwd_kernel) of dy with the saved a, s (, x) -> dAB = [da | db] as bf16
//                planes (B,T,2C); dbias[2C] += sums over (b,t)                           [data-/weight-gradient operand]
//   SPLIT_GRAD   g = dy * (relu ? y > 0 : 1) -> bf16 planes (B,T,Cp); dbias[C] += sums
// A CTA (256 threads) owns 64 channels x 64 time steps of one utterance: float4 loads along T (16 threads per channel
// row, 3-4 tensors in flight per thread), bias-gradient sums reduced across those 16 lanes (one atomic per row and
// tile), transpose through shared memory, and 16-byte stores of 8 channels per thread -- 8 threads cover the 128
// contiguous bytes of one (b,t) row of a plane.  (The round-1 kernels used 32x32 tiles with 2-byte stores, 64 B per
// warp-store row: 25 % of the HBM roof over a training step.)
enum { SPLIT_INPUT = 0, SPLIT_GATE = 1, SPLIT_GRAD = 2 };

struct SplitParams {
    const float* in0;          // x | dy | dy
    const float* in1;          // - | a  | y (relu) or null
    const float* in2;          // - | s  | -
    const float* in3;          // - | x (highway) | -
    bf16* planes;              // [npl][B][T][pitch]
    bf16* wg;                  // SPLIT_INPUT: bf16 copy [npl][B][T][pitch] or null
    float* dbias;              // null | [2C] | [C]
    int B, C, T, pitch;
    int mode, residual, relu;  // gate mode (0 GLU, 1 highway), GLU residual flag; ReLU flag
    float p; const unsigned long long* seed_ptr; unsigned salt;     // SPLIT_INPUT dropout
    const long long* tlen; int tmult;   // or null: frames t >= tmult * tlen[0] are written as 0 (and leave dbias)
};

// two consecutive channels -> their 16-bit hi words (and, with two planes, lo words) packed as one 32-bit word each
template <int FMT, int NPL>
__device__ __forceinline__ void pack_planes(float x0, float x1, uint32_t& h, uint32_t& l) {
    if constexpr (NPL == 1) {
        h = (uint32_t)split_hi<FMT>(x0) | ((uint32_t)split_hi<FMT>(x1) << 16);
    } else {
        uint16_t h0, l0, h1, l1;
        split_pair<FMT>(x0, h0, l0);
        split_pair<FMT>(x1, h1, l1);
        h = (uint32_t)h0 | ((uint32_t)h1 << 16);
        l = (uint32_t)l0 | ((uint32_t)l1 << 16);
    }
}

// 6 CTAs per SM: holds the gate split (33 KB of shared memory: 6 fit) at 40 registers with the extent mask, no spills.
// DET (deterministic mode, its own instantiations): p.dbias is a scratch [B * gridDim.x][2C | C] instead; every
// (utterance, 64-frame tile) stores its per-channel sums in its own row -- frames past the extent are already zero in
// them -- and bias_reduce_kernel (conv.cu) adds the rows to the bias gradient in a fixed order.
template <int KIND, int NPL, bool DET = false>
__global__ void __launch_bounds__(256, 6) plane_split_kernel(const __grid_constant__ SplitParams p) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    __shared__ float sa[64][65];
    __shared__ float sb[KIND == SPLIT_GATE ? 64 : 1][65];
    const int tid = threadIdx.x;
    const int b = blockIdx.z, c0 = blockIdx.y * 64, t0 = blockIdx.x * 64;
    const int C = p.C, T = p.T;
    // the logical extent of a batch padded to a bucket (device memory): the frames past it read as zeros
    const int TL = p.tlen ? (int)min((long long)T, (long long)p.tmult * *p.tlen) : T;
    const bool vec = (T & 3) == 0;
    const DropCfg drop = make_drop(KIND == SPLIT_INPUT ? p.p : 0.f, p.seed_ptr, p.salt);
    const float gs = (KIND == SPLIT_GATE && p.mode == 0 && p.residual) ? 0.70710678118654752f : 1.f;
    const int q = tid & 15;                                  // float4 slot along T
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int r = (tid >> 4) + 16 * j, c = c0 + r, t = t0 + 4 * q;
        float v0[4] = {0.f, 0.f, 0.f, 0.f}, v1[4] = {0.f, 0.f, 0.f, 0.f};
        if (c < C && t < T) {
            const size_t row = ((size_t)b * C + c) * T + t;
            float x0[4], x1[4], x2[4], x3[4];
            const bool full = vec && t + 3 < T;
            auto ld = [&](const float* src, float* dst) {
                if (full) {
                    const float4 u = __ldg(reinterpret_cast<const float4*>(src + row));
                    dst[0] = u.x; dst[1] = u.y; dst[2] = u.z; dst[3] = u.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) dst[e] = (t + e < T) ? __ldg(src + row + e) : 0.f;
                }
            };
            ld(p.in0, x0);
            if (KIND == SPLIT_GATE) { ld(p.in1, x1); ld(p.in2, x2); if (p.mode != 0) ld(p.in3, x3); }
            if (KIND == SPLIT_GRAD && p.relu) ld(p.in1, x1);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (KIND == SPLIT_INPUT) {
                    v0[e] = x0[e] * drop_scale(drop, (uint32_t)(row + e));
                } else if (KIND == SPLIT_GATE) {
                    const float g = x0[e] * gs, av = x1[e], sv = x2[e];
                    v0[e] = g * sv;
                    v1[e] = g * (p.mode == 0 ? av : (av - x3[e])) * sv * (1.f - sv);
                } else {
                    v0[e] = (p.relu && !(x1[e] > 0.f)) ? 0.f : x0[e];
                }
                if (t + e >= TL) { v0[e] = 0.f; v1[e] = 0.f; }
            }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            sa[r][4 * q + e] = v0[e];
            if (KIND == SPLIT_GATE) sb[r][4 * q + e] = v1[e];
        }
        if (KIND != SPLIT_INPUT && p.dbias) {                // all 32 lanes take part: 16 lanes share a channel row
            float s0 = v0[0] + v0[1] + v0[2] + v0[3], s1 = v1[0] + v1[1] + v1[2] + v1[3];
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) {
                s0 += __shfl_xor_sync(0xffffffffu, s0, o);
                if (KIND == SPLIT_GATE) s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            }
            if (DET) {
                if (q == 0 && c < C) {
                    float* row = p.dbias + ((size_t)b * gridDim.x + blockIdx.x) * (KIND == SPLIT_GATE ? 2 * C : C);
                    row[c] = s0;
                    if (KIND == SPLIT_GATE) row[C + c] = s1;
                }
            } else if (q == 0 && c < C) {
                atomicAdd(&p.dbias[c], s0);
                if (KIND == SPLIT_GATE) atomicAdd(&p.dbias[C + c], s1);
            }
        }
    }
    __syncthreads();
    constexpr int FMT = KIND == SPLIT_INPUT ? FMT_F16 : FMT_BF16;
    const size_t plane = (size_t)p.B * T * p.pitch;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int slot = tid + 256 * j, tt = slot >> 3, cg = slot & 7, t = t0 + tt, c = c0 + cg * 8;
        if (t >= T || c >= (KIND == SPLIT_GATE ? C : p.pitch)) continue;
        const size_t off = ((size_t)b * T + t) * p.pitch + c;
#pragma unroll
        for (int half = 0; half < (KIND == SPLIT_GATE ? 2 : 1); ++half) {
            float e[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) e[i] = half ? sb[(cg * 8 + i) % 64][tt] : sa[cg * 8 + i][tt];
            uint32_t h[4], l[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) pack_planes<FMT, NPL>(e[2 * i], e[2 * i + 1], h[i], l[i]);
            uint16_t* d = reinterpret_cast<uint16_t*>(p.planes) + off + (half ? C : 0);
            *reinterpret_cast<uint4*>(d) = make_uint4(h[0], h[1], h[2], h[3]);
            if constexpr (NPL == 2) *reinterpret_cast<uint4*>(d + plane) = make_uint4(l[0], l[1], l[2], l[3]);
            if (KIND == SPLIT_INPUT && p.wg) {
#pragma unroll
                for (int i = 0; i < 4; ++i) pack_planes<FMT_BF16, NPL>(e[2 * i], e[2 * i + 1], h[i], l[i]);
                uint16_t* w = reinterpret_cast<uint16_t*>(p.wg) + off;
                *reinterpret_cast<uint4*>(w) = make_uint4(h[0], h[1], h[2], h[3]);
                if constexpr (NPL == 2) *reinterpret_cast<uint4*>(w + plane) = make_uint4(l[0], l[1], l[2], l[3]);
            }
        }
    }
}

static dim3 split_grid(int B, int C, int T) { return dim3((T + 63) / 64, (C + 63) / 64, B); }

template <int KIND>
static int launch_split(const SplitParams& p, int npl, void* stream, const char* what) {
    if (npl == 1) launch_k(plane_split_kernel<KIND, 1>, split_grid(p.B, p.C, p.T), dim3(256), 0, (cudaStream_t)stream, p);
    else launch_k(plane_split_kernel<KIND, 2>, split_grid(p.B, p.C, p.T), dim3(256), 0, (cudaStream_t)stream, p);
    return check_launch(what);
}

// deterministic bias gradient: partial rows from the split itself (p.dbias = scratch), then the fixed-order reduction
template <int KIND>
static int launch_split_det(SplitParams p, int npl, float* dbias, float* scratch, long long scratch_floats,
                            void* stream, const char* what) {
    const int nch = KIND == SPLIT_GATE ? 2 * p.C : p.C;
    const dim3 grid = split_grid(p.B, p.C, p.T);
    const long long nparts = (long long)p.B * grid.x;
    if (!dbias || !scratch || scratch_floats < nparts * nch) {
        set_error("%s: dbias and a scratch of >= %lld floats required", what, nparts * nch);
        return 1;
    }
    p.dbias = scratch;
    if (npl == 1) launch_k(plane_split_kernel<KIND, 1, true>, grid, dim3(256), 0, (cudaStream_t)stream, p);
    else launch_k(plane_split_kernel<KIND, 2, true>, grid, dim3(256), 0, (cudaStream_t)stream, p);
    if (int e = check_launch(what)) return e;
    return bias_reduce(scratch, (int)nparts, nch, dbias, (cudaStream_t)stream);
}

}  // namespace dv3

using namespace dv3;

extern "C" {

static int split_input(const float* x, void* btc, int npl, void* bct, int B, int C, int T, float p_drop,
                       const unsigned long long* seed_ptr, unsigned salt, const long long* tlen, int tmult,
                       void* stream) {
    DV3_REQUIRE(B <= 65535 && (C + 63) / 64 <= 65535, "tc_split_input: grid too large");
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_split_input: npl must be 1 or 2");
    DV3_REQUIRE(!tlen || tmult >= 1, "tc_split_input: tmult must be >= 1");
    SplitParams p = {};
    p.in0 = x; p.planes = (bf16*)btc; p.wg = (bf16*)bct; p.B = B; p.C = C; p.T = T; p.pitch = (C + 7) / 8 * 8;
    p.p = p_drop; p.seed_ptr = seed_ptr; p.salt = salt; p.tlen = tlen; p.tmult = tmult;
    return launch_split<SPLIT_INPUT>(p, npl, stream, "tc_split_input");
}

static int gate_bwd_split(const float* dy, const float* a, const float* s, const float* x, void* btc, int npl,
                          void* bct, float* dbias, int B, int C, int T, int mode, int residual, const long long* tlen,
                          int tmult, void* stream, bool det = false, float* scratch = nullptr,
                          long long scratch_floats = 0) {
    DV3_REQUIRE(bct == nullptr, "tc_gate_bwd_split: bct must be NULL");
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_gate_bwd_split: npl must be 1 or 2");
    DV3_REQUIRE(C % 8 == 0 && (mode == 0 || x != nullptr), "tc_gate_bwd_split: C %% 8 != 0 or highway without x");
    DV3_REQUIRE(!tlen || tmult >= 1, "tc_gate_bwd_split: tmult must be >= 1");
    SplitParams p = {};
    p.in0 = dy; p.in1 = a; p.in2 = s; p.in3 = x; p.planes = (bf16*)btc; p.dbias = dbias;
    p.B = B; p.C = C; p.T = T; p.pitch = 2 * C; p.mode = mode; p.residual = residual; p.tlen = tlen; p.tmult = tmult;
    if (det) return launch_split_det<SPLIT_GATE>(p, npl, dbias, scratch, scratch_floats, stream, "tc_gate_bwd_split_det");
    return launch_split<SPLIT_GATE>(p, npl, stream, "tc_gate_bwd_split");
}

static int grad_split(const float* dy, const float* y, void* btc, int npl, void* bct, float* dbias, int B, int C,
                      int T, int relu, const long long* tlen, int tmult, void* stream, bool det = false,
                      float* scratch = nullptr, long long scratch_floats = 0) {
    DV3_REQUIRE(bct == nullptr, "tc_grad_split: bct must be NULL");
    DV3_REQUIRE(npl == 1 || npl == 2, "tc_grad_split: npl must be 1 or 2");
    DV3_REQUIRE(!relu || y != nullptr, "tc_grad_split: ReLU backward needs the forward output");
    DV3_REQUIRE(!tlen || tmult >= 1, "tc_grad_split: tmult must be >= 1");
    SplitParams p = {};
    p.in0 = dy; p.in1 = y; p.planes = (bf16*)btc; p.dbias = dbias;
    p.B = B; p.C = C; p.T = T; p.pitch = (C + 7) / 8 * 8; p.relu = relu; p.tlen = tlen; p.tmult = tmult;
    if (det) return launch_split_det<SPLIT_GRAD>(p, npl, dbias, scratch, scratch_floats, stream, "tc_grad_split_det");
    return launch_split<SPLIT_GRAD>(p, npl, stream, "tc_grad_split");
}

int dv3_tc_split_input(const float* x, void* btc, int npl, void* bct, int B, int C, int T, int k, int dilation,
                       int causal, float p_drop, const unsigned long long* seed_ptr, unsigned salt, void* stream) {
    (void)k; (void)dilation; (void)causal;
    return split_input(x, btc, npl, bct, B, C, T, p_drop, seed_ptr, salt, nullptr, 1, stream);
}

int dv3_tc_gate_bwd_split(const float* dy, const float* a, const float* s, const float* x, void* btc, void* bct,
                          float* dbias, int B, int C, int T, int mode, int residual, void* stream) {
    return gate_bwd_split(dy, a, s, x, btc, 2, bct, dbias, B, C, T, mode, residual, nullptr, 1, stream);
}

int dv3_tc_grad_split(const float* dy, const float* y, void* btc, void* bct, float* dbias, int B, int C, int T,
                      int relu, void* stream) {
    return grad_split(dy, y, btc, 2, bct, dbias, B, C, T, relu, nullptr, 1, stream);
}

// The same with an optional logical time extent in device memory (a batch padded to a bucket): tlen null behaves as
// above; otherwise frames t >= tmult * tlen[0] of the input (forward operand) or of the incoming gradient are taken
// as 0 -- the time mask of the padded frames and its gradient, folded into the passes that read those tensors anyway.
int dv3_tc_split_input_ext(const float* x, void* btc, int npl, void* bct, int B, int C, int T, float p_drop,
                           const unsigned long long* seed_ptr, unsigned salt, const long long* tlen, int tmult,
                           void* stream) {
    return split_input(x, btc, npl, bct, B, C, T, p_drop, seed_ptr, salt, tlen, tmult, stream);
}

int dv3_tc_gate_bwd_split_ext(const float* dy, const float* a, const float* s, const float* x, void* btc, void* bct,
                              float* dbias, int B, int C, int T, int mode, int residual, const long long* tlen,
                              int tmult, void* stream) {
    return gate_bwd_split(dy, a, s, x, btc, 2, bct, dbias, B, C, T, mode, residual, tlen, tmult, stream);
}

int dv3_tc_grad_split_ext(const float* dy, const float* y, void* btc, void* bct, float* dbias, int B, int C, int T,
                          int relu, const long long* tlen, int tmult, void* stream) {
    return grad_split(dy, y, btc, 2, bct, dbias, B, C, T, relu, tlen, tmult, stream);
}

// Both gradient splits with the plane count (1 or 2) and the nullable extent: one entry point each for every form.
int dv3_tc_gate_bwd_split_npl(const float* dy, const float* a, const float* s, const float* x, void* btc, int npl,
                              void* bct, float* dbias, int B, int C, int T, int mode, int residual,
                              const long long* tlen, int tmult, void* stream) {
    return gate_bwd_split(dy, a, s, x, btc, npl, bct, dbias, B, C, T, mode, residual, tlen, tmult, stream);
}

int dv3_tc_grad_split_npl(const float* dy, const float* y, void* btc, int npl, void* bct, float* dbias, int B, int C,
                          int T, int relu, const long long* tlen, int tmult, void* stream) {
    return grad_split(dy, y, btc, npl, bct, dbias, B, C, T, relu, tlen, tmult, stream);
}

// Deterministic forms of the two calls above (same planes, bit for bit): the per-(utterance, 64-frame tile) channel
// sums go to scratch (>= dv3_bias_det_scratch_floats(B, 2C | C, T, 1) floats) and are added to dbias in a fixed order by
// a second launch.  dbias is required.
int dv3_tc_gate_bwd_split_det(const float* dy, const float* a, const float* s, const float* x, void* btc, int npl,
                              float* dbias, float* scratch, long long scratch_floats, int B, int C, int T, int mode,
                              int residual, const long long* tlen, int tmult, void* stream) {
    return gate_bwd_split(dy, a, s, x, btc, npl, nullptr, dbias, B, C, T, mode, residual, tlen, tmult, stream, true,
                          scratch, scratch_floats);
}

int dv3_tc_grad_split_det(const float* dy, const float* y, void* btc, int npl, float* dbias, float* scratch,
                          long long scratch_floats, int B, int C, int T, int relu, const long long* tlen, int tmult,
                          void* stream) {
    return grad_split(dy, y, btc, npl, nullptr, dbias, B, C, T, relu, tlen, tmult, stream, true, scratch,
                      scratch_floats);
}

}  // extern "C"
