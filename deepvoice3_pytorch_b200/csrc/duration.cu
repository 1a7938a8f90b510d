// Duration-predictor loss (DESIGN.md section 2.22): the mean over rows of the per-row mean over the row's n_b tokens of
// (y - log d)^2, with y the predicted log-duration and d >= 1 the target duration in decoder steps.
//
// Every sum has one fixed order and no atomics, so the loss is bit-reproducible and a row's bits do not depend on the
// rest of the batch: one CTA per row squares its tokens' errors in fp64 into shared memory and thread 0 adds them in
// token order; a one-thread kernel then adds the rows' means in row order.  The gradient
// dy[b, j] = d_loss * 2 (y - log d) / (n_b B) is formed in fp64 and rounded once; it is 0 past n_b.
// A row whose length is outside [1, L] or that holds a duration below 1 sets *err_flag and adds 0 to the loss and to
// the gradient.
#include "common.cuh"
#include "../../include/dv3b200.h"

namespace dv3 {

constexpr int DUR_MAX_TOKENS = 1024;
constexpr int kDurThreads = 256;

// row b's validity: 1 <= n <= L and every duration of its first n tokens >= 1 (a CTA-wide vote)
__device__ __forceinline__ bool dur_row_ok(const int* __restrict__ d, int n, int L) {
    if (n < 1 || n > L) return false;
    int bad = 0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) bad |= d[j] < 1;
    return !__syncthreads_or(bad);
}

__global__ void __launch_bounds__(kDurThreads) dur_loss_rows_kernel(const float* __restrict__ y, long long y_ld,
                                                                    const int* __restrict__ dur, long long d_ld,
                                                                    const int* __restrict__ lengths, int L,
                                                                    double* __restrict__ row_loss,
                                                                    int* __restrict__ err_flag) {
    pdl_trigger(); pdl_wait();
    __shared__ double sq[DUR_MAX_TOKENS];
    const int b = blockIdx.x;
    const int n = lengths[b];
    const float* yr = y + b * y_ld;
    const int* dr = dur + b * d_ld;
    if (!dur_row_ok(dr, n, L)) {
        if (threadIdx.x == 0) { *err_flag = 1; row_loss[b] = 0.0; }
        return;
    }
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const double e = (double)yr[j] - log((double)dr[j]);
        sq[j] = e * e;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int j = 0; j < n; ++j) s += sq[j];
        row_loss[b] = s / n;
    }
}

__global__ void dur_loss_reduce_kernel(const double* __restrict__ row_loss, int B, float* __restrict__ loss) {
    pdl_trigger(); pdl_wait();
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += row_loss[b];
    *loss = (float)(s / B);
}

__global__ void __launch_bounds__(kDurThreads) dur_loss_grad_kernel(const float* __restrict__ y, long long y_ld,
                                                                    const int* __restrict__ dur, long long d_ld,
                                                                    const int* __restrict__ lengths, int B, int L,
                                                                    const float* __restrict__ d_loss,
                                                                    float* __restrict__ dy) {
    pdl_trigger(); pdl_wait();
    const int b = blockIdx.x;
    const int n = lengths[b];
    const float* yr = y + b * y_ld;
    const int* dr = dur + b * d_ld;
    float* g = dy + (size_t)b * L;
    const bool ok = dur_row_ok(dr, n, L);
    const double scale = ok ? 2.0 * (double)d_loss[0] / ((double)n * (double)B) : 0.0;
    for (int j = threadIdx.x; j < L; j += blockDim.x)
        g[j] = ok && j < n ? (float)(scale * ((double)yr[j] - log((double)dr[j]))) : 0.f;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_duration_max_tokens(void) { return DUR_MAX_TOKENS; }

int dv3_duration_loss_fwd(const float* y, long long y_ld, const int* durations, long long d_ld, const int* lengths,
                          int B, int L, double* row_loss, float* loss, int* err_flag, void* stream) {
    DV3_REQUIRE(y && durations && lengths && row_loss && loss && err_flag, "duration_loss_fwd: null operand");
    DV3_REQUIRE(B >= 1 && B <= 65535 && L >= 1 && L <= DUR_MAX_TOKENS, "duration_loss_fwd: B=%d, L=%d", B, L);
    DV3_REQUIRE(y_ld >= L && d_ld >= L, "duration_loss_fwd: strides (%lld, %lld) below L=%d", y_ld, d_ld, L);
    cudaStream_t st = (cudaStream_t)stream;
    launch_k(dur_loss_rows_kernel, B, kDurThreads, 0, st, y, y_ld, durations, d_ld, lengths, L, row_loss, err_flag);
    launch_k(dur_loss_reduce_kernel, 1, 1, 0, st, (const double*)row_loss, B, loss);
    return check_launch("duration_loss_fwd");
}

int dv3_duration_loss_bwd(const float* y, long long y_ld, const int* durations, long long d_ld, const int* lengths,
                          int B, int L, const float* d_loss, float* dy, void* stream) {
    DV3_REQUIRE(y && durations && lengths && d_loss && dy, "duration_loss_bwd: null operand");
    DV3_REQUIRE(B >= 1 && B <= 65535 && L >= 1 && L <= DUR_MAX_TOKENS, "duration_loss_bwd: B=%d, L=%d", B, L);
    DV3_REQUIRE(y_ld >= L && d_ld >= L, "duration_loss_bwd: strides (%lld, %lld) below L=%d", y_ld, d_ld, L);
    launch_k(dur_loss_grad_kernel, B, kDurThreads, 0, (cudaStream_t)stream, y, y_ld, durations, d_ld, lengths, B, L,
             d_loss, dy);
    return check_launch("duration_loss_bwd");
}

}  // extern "C"
