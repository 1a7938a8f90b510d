// Flat-arena optimizer step for the data-parallel training loop: gradient-norm clipping
// (reference train.py:756-758, torch.nn.utils.clip_grad_norm_) + Adam (train.py:975-979, :759) over ONE
// contiguous fp32 parameter arena in two launches, with no host synchronisation: the clip coefficient is read
// from device memory, and lr / bias corrections come from a 4-float device block so a captured CUDA graph can
// be replayed with a new learning rate.
#include "common.cuh"

namespace dv3 {

// out[0] = sum(x^2), DETERMINISTIC: every block writes its partial to scratch[blockIdx.x]; the block that takes the
// last ticket sums the partials in index order, so the result does not depend on the order blocks finish in -- all
// data-parallel replicas (which hold bit-identical all-reduced gradients) get the same clip coefficient.
// scratch: >= DV3_SUMSQ_SCRATCH floats; scratch[DV3_SUMSQ_SCRATCH-1] is the ticket counter (zero before first use;
// the kernel leaves it zero).
constexpr int SUMSQ_MAX_BLOCKS = 132 * 8;
constexpr int SUMSQ_SCRATCH = 2048;
__global__ void sumsq_kernel(const float* __restrict__ x, long long n, float* __restrict__ out,
                             float* __restrict__ scratch) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    float s = 0.f;
    const long long n4 = n >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x) {
        const float4 v = x4[i];
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
    }
    for (long long i = (n4 << 2) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        s = fmaf(x[i], x[i], s);
    __shared__ float red[32];
    __shared__ bool last;
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        s = warp_sum(s);
        if (threadIdx.x == 0) {
            scratch[blockIdx.x] = s;
            __threadfence();
            unsigned* ticket = reinterpret_cast<unsigned*>(scratch + SUMSQ_SCRATCH - 1);
            last = atomicAdd(ticket, 1u) == gridDim.x - 1;
        }
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // fixed-order tree over the per-block partials: thread t sums partials t, t+256, ... then a block reduction
    float t = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += __ldcg(&scratch[i]);
    t = warp_sum(t);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x < 32) {
        t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        t = warp_sum(t);
        if (threadIdx.x == 0) {
            out[0] = t;
            *reinterpret_cast<unsigned*>(scratch + SUMSQ_SCRATCH - 1) = 0u;
        }
    }
}

// hyper = {lr, bias_correction1, bias_correction2, grad_scale}; sumsq[0] = ||g*grad_scale||^2 before clipping.
// WD: torch.optim.Adam's L2 weight decay, g' = clipped g + wd*p before the moments.  AMS: AMSGrad, the denominator
// takes vmax = max(vmax, v).  <false, false> is the plain clip + Adam step.
template <bool WD, bool AMS>
__global__ void adam_clip_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                 float* __restrict__ v, float* __restrict__ vmax, long long n,
                                 const float* __restrict__ hyper, const float* __restrict__ sumsq, float beta1,
                                 float beta2, float eps, float max_norm, float wd) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const float lr = hyper[0], bc1 = hyper[1], bc2 = hyper[2], gscale = hyper[3];
    float coef = gscale;
    if (max_norm > 0.f) {
        const float total = sqrtf(sumsq[0]) * gscale;
        const float c = max_norm / (total + 1e-6f);
        coef *= (c < 1.f ? c : 1.f);
    }
    const float step = lr / bc1, rs2 = rsqrtf(bc2);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        float gi = g[i] * coef;
        if (WD) gi += wd * p[i];
        const float mi = beta1 * m[i] + (1.f - beta1) * gi;
        const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
        m[i] = mi; v[i] = vi;
        float vd = vi;
        if (AMS) { vd = fmaxf(vmax[i], vi); vmax[i] = vd; }
        p[i] -= step * mi / (sqrtf(vd) * rs2 + eps);
    }
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_sumsq_scratch_floats(void) { return SUMSQ_SCRATCH; }

int dv3_sumsq(const float* x, long long n, float* out, float* scratch, void* stream) {
    DV3_REQUIRE(((uintptr_t)x & 15) == 0, "sumsq: pointer must be 16-byte aligned");
    DV3_REQUIRE(scratch != nullptr, "sumsq: scratch buffer required");
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > SUMSQ_MAX_BLOCKS) blocks = SUMSQ_MAX_BLOCKS;
    if (blocks < 1) blocks = 1;
    launch_k(sumsq_kernel, (int)blocks, 256, 0, (cudaStream_t)stream, x, n, out, scratch);
    return check_launch("sumsq");
}

static long long adam_blocks(long long n) {
    long long blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    return blocks;
}

int dv3_adam_clip(float* p, const float* g, float* m, float* v, long long n, const float* hyper,
                  const float* sumsq, float beta1, float beta2, float eps, float max_norm, void* stream) {
    launch_k(adam_clip_kernel<false, false>, (int)adam_blocks(n), 256, 0, (cudaStream_t)stream, p, g, m, v,
             (float*)nullptr, n, hyper, sumsq, beta1, beta2, eps, max_norm, 0.f);
    return check_launch("adam_clip");
}

int dv3_adam_clip_opts(float* p, const float* g, float* m, float* v, float* vmax, long long n, const float* hyper,
                       const float* sumsq, float beta1, float beta2, float eps, float max_norm, float weight_decay,
                       void* stream) {
    DV3_REQUIRE(weight_decay >= 0.f, "adam_clip_opts: weight_decay=%g < 0", weight_decay);
    const int blocks = (int)adam_blocks(n);
    const bool wd = weight_decay != 0.f, ams = vmax != nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    if (wd && ams)
        launch_k(adam_clip_kernel<true, true>, blocks, 256, 0, st, p, g, m, v, vmax, n, hyper, sumsq, beta1, beta2,
                 eps, max_norm, weight_decay);
    else if (wd)
        launch_k(adam_clip_kernel<true, false>, blocks, 256, 0, st, p, g, m, v, vmax, n, hyper, sumsq, beta1, beta2,
                 eps, max_norm, weight_decay);
    else if (ams)
        launch_k(adam_clip_kernel<false, true>, blocks, 256, 0, st, p, g, m, v, vmax, n, hyper, sumsq, beta1, beta2,
                 eps, max_norm, weight_decay);
    else
        launch_k(adam_clip_kernel<false, false>, blocks, 256, 0, st, p, g, m, v, vmax, n, hyper, sumsq, beta1, beta2,
                 eps, max_norm, weight_decay);
    return check_launch("adam_clip_opts");
}

}  // extern "C"
