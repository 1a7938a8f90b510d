// Shared device/host helpers for the dv3b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

namespace dv3 {

// ---- error plumbing (no exceptions across the C ABI) -------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);     // counts the launch; cudaGetLastError() -> 0 / error code + message
unsigned long long launch_count();

#define DV3_REQUIRE(cond, ...)                                    \
    do {                                                          \
        if (!(cond)) { ::dv3::set_error(__VA_ARGS__); return 1; } \
    } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---- process-wide settings: read ONCE (thread-safe static initialisation) from the environment, immutable after ----
struct Config {
    int pdl;            // DV3_PDL=0 disables programmatic dependent launch (default on)
    int sms;            // multiprocessor count of the current device at first use
    float tc_gamma;     // per-MMA truncation compensation of the tensor-core accumulators (tc_gemm.cu TcParams::gmain)
};
const Config& config();

// ---- programmatic dependent launch -------------------------------------------------------------------------
// Every kernel of this library begins with pdl_trigger() -- the next kernel on the stream may be scheduled onto SMs as
// they free up and run its own set-up (barrier init, descriptor prefetch) under this kernel's tail --
// and calls pdl_wait() before its first access to global memory, which blocks until the preceding kernel has completed
// and its writes are visible.  Launches go through launch_k(), which sets the programmatic-serialisation attribute
// (a plain full dependency when the predecessor is not a kernel of ours, or when DV3_PDL=0).  A captured CUDA graph
// keeps these edges as programmatic dependencies.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                   Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = config().pdl;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ---- attention context scale Ts * sqrt(1/Ts) (reference deepvoice3.py:170-171) of a key count read from device memory:
// a batch padded to a larger bucket scales by its logical text length, not by the padded one -------------------------
__device__ __forceinline__ float context_scale(long long ts) {
    const double t = (double)(ts < 1 ? 1 : ts);
    return (float)(t * sqrt(1.0 / t));
}

// ---- counter-based dropout mask ----------------------------------------------------------------
// keep(idx) is a pure function of (step seed in device memory, call-site salt, element index), so the
// backward pass and the weight-gradient pass regenerate exactly the mask the forward used, and a
// replayed CUDA graph gets a fresh mask by bumping the 8-byte seed in device memory.
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
struct DropCfg {
    uint32_t s0, s1;      // derived per launch from *seed_ptr and salt
    uint32_t thresh;      // drop iff hash < thresh ; thresh = p * 2^32
    float scale;          // 1/(1-p)
    int on;
};
__device__ __forceinline__ DropCfg make_drop(float p, const unsigned long long* seed_ptr, uint32_t salt) {
    DropCfg d;
    d.on = (p > 0.f) && (seed_ptr != nullptr);
    if (d.on) {
        unsigned long long s = *seed_ptr;
        d.s0 = mix32((uint32_t)s ^ (salt * 0x9E3779B1U));
        d.s1 = mix32((uint32_t)(s >> 32) + salt + 0x85ebca6bU);
        double t = (double)p * 4294967296.0;
        d.thresh = t >= 4294967295.0 ? 0xFFFFFFFFU : (uint32_t)t;
        d.scale = 1.f / (1.f - p);
    } else { d.s0 = d.s1 = d.thresh = 0; d.scale = 1.f; }
    return d;
}
__device__ __forceinline__ float drop_scale(const DropCfg& d, uint32_t idx) {
    // returns 0 (dropped) or 1/(1-p) (kept); 1 when dropout is off
    if (!d.on) return 1.f;
    uint32_t h = mix32(mix32(idx ^ d.s0) + d.s1);
    return h < d.thresh ? 0.f : d.scale;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---- 16-bit operand planes of the tensor-core path -----------------------------------------------------------
// Every fp32 operand x travels as two 16-bit planes: hi = rn16(x), lo = rn16((x - hi) * 2^11).  The products
// hi*hi (main accumulator) and hi*lo + lo*hi (cross accumulator, carrying the 2^11) are summed as
// main + cross * 2^-11 by the epilogue.  Two formats:
//   FMT_F16   forward operands (activations O(1), normalised weights): fp16 hi carries 11 significant bits, the scaled
//             fp16 lo another 11 -> 22-bit operands, products exact to ~2^-23: fp32-class results.  Values are clamped
//             to the fp16 range (+-65504); the scale keeps lo out of the fp16 subnormals.
//   FMT_BF16  gradients (magnitudes down to 1e-10: need the fp32 exponent range): 8 + 8 bits, products to ~2^-17.
constexpr float LO_SCALE = 2048.f, LO_INV = 1.f / 2048.f;
enum { FMT_BF16 = 2, FMT_F16 = 16 };
typedef __nv_bfloat16 bf16;
template <int FMT>
__device__ __forceinline__ void split_pair(float v, uint16_t& hi, uint16_t& lo) {
    if (FMT == FMT_F16) {
        v = fminf(fmaxf(v, -65504.f), 65504.f);
        const __half h = __float2half_rn(v);
        hi = __half_as_ushort(h);
        lo = __half_as_ushort(__float2half_rn((v - __half2float(h)) * LO_SCALE));
    } else {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi = __bfloat16_as_ushort(h);
        lo = __bfloat16_as_ushort(__float2bfloat16_rn((v - __bfloat162float(h)) * LO_SCALE));
    }
}

// The single-pass operand (ops.conv_math = "tc1"): plane hi of split_pair alone, the same bits.
template <int FMT>
__device__ __forceinline__ uint16_t split_hi(float v) {
    if (FMT == FMT_F16) return __half_as_ushort(__float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f)));
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- deterministic mode: dbias[c] += sum_i scratch[i][c], i < nparts, in a fixed order (conv.cu bias_reduce_kernel) ----
int bias_reduce(const float* scratch, int nparts, int nch, float* dbias, cudaStream_t st);

}  // namespace dv3
