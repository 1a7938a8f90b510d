// Monotonic alignment search (MAS, the Viterbi recursion of Glow-TTS) over attention alignments, and the per-step
// statistics of attention-error counting, in one pass over the alignment (alignment.py, DESIGN.md section 2.19).
//
// Row b is the alignment A_b(t, j) = A[b * stride_b + t * stride_t + j], t < N_b decoder steps, j < L_b tokens, and
// lp(t, j) = logf(fmaxf(A_b(t, j), 1e-8f)) (fmaxf also takes a NaN cell to the floor).  A cell is on some path from
// (0, 0) to (N_b - 1, L_b - 1) iff j <= t and L_b - 1 - j <= N_b - 1 - t; every other cell has Q = -inf.
//   Q(0, 0) = lp(0, 0),   Q(t, j) = lp(t, j) + max(Q(t-1, j), Q(t-1, j-1)),
// ties to (t-1, j): the path stays on the token unless the previous token scores strictly higher.  One predecessor bit a
// cell (1: from (t-1, j-1)), 32 columns a word, one word per warp per step by __ballot_sync.
//
// Forward: one CTA per row, thread j owns column j (L <= 1024), walking t = 0 .. N_b - 1 with one named barrier per step
// over the row's own ceil(L_b / 32) warps (the others exit at once).  Q(t-1, j-1) comes from lane j-1 by __shfl_up_sync,
// or for lane 0 from lane 31 of the warp before through a double-buffered shared slot.  Each thread streams its own
// column of A by cp.async through a MAS_RING-deep shared-memory ring (only the thread that copies a value reads it, so
// the ring needs no barrier).  The same pass keeps the per-step argmax p_t (ties to the lowest j) and maximum m_t -- a
// warp shuffle reduction, then warp 0 combines the warps' partials of step t after the barrier that already ends the
// step -- and the per-token coverage c_j = sum_t A_b(t, j) in increasing t.  NaN cells count as -inf in p_t and m_t.
// Backtrace: one warp per row; lane k fetches the direction word of step t0 - k in the current 32-token column, and the
// whole warp walks those 32 steps in registers, so a row costs about (N_b + L_b) / 32 dependent loads.
// No atomics: a row's bits depend on its own cells and lengths alone.
#include "common.cuh"
#include "dtw.cuh"

namespace dv3 {

constexpr int MAS_MAX_TOKENS = 1024;     // one column per thread: the largest max_positions of the presets
constexpr int MAS_RING = 8;              // steps of A in flight per thread
constexpr int MAS_BT_WARPS = 4;          // rows per backtrace CTA

static inline long long mas_dir_words(int steps, int tokens) { return (long long)steps * ((tokens + 31) / 32); }

__global__ void __launch_bounds__(MAS_MAX_TOKENS)
mas_forward_kernel(const float* __restrict__ A, long long stride_b, long long stride_t, const int* __restrict__ steps,
                   const int* __restrict__ tokens, int N_max, int L_max, const long long* __restrict__ dir_off,
                   unsigned* __restrict__ dirs, int* __restrict__ argmax, float* __restrict__ maxv,
                   float* __restrict__ coverage, float* __restrict__ score) {
    pdl_trigger(); pdl_wait();
    const int b = blockIdx.x;
    const int N = steps[b], L = tokens[b];
    const int nw = (L + 31) >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = threadIdx.x;
    if (warp >= nw) return;
    const int nthr = nw * 32;
    extern __shared__ float smem[];
    float* ring = smem;                                              // MAS_RING x blockDim.x
    float* edge = ring + MAS_RING * blockDim.x;                      // 2 x 32: Q of each warp's lane 31
    float* part_m = edge + 64;                                       // 2 x 32: each warp's max
    int* part_p = reinterpret_cast<int*>(part_m + 64);               // 2 x 32: and its argmax
    const bool col = j < L;
    const float* a_col = A + b * stride_b + j;
    unsigned* dir = dirs + dir_off[b];
    const float NEG = __int_as_float(0xff800000);
    auto issue = [&](int t) {
        if (col && t < N) cp_async4(ring + (t % MAS_RING) * blockDim.x + j, a_col + t * stride_t);
        cp_async_commit();
    };
#pragma unroll
    for (int s = 0; s < MAS_RING - 1; ++s) issue(s);
    float q = NEG, cov = 0.f;
    for (int t = 0; t < N; ++t) {
        issue(t + MAS_RING - 1);
        cp_async_wait<MAS_RING - 1>();
        const float a = col ? ring[(t % MAS_RING) * blockDim.x + j] : 0.f;
        const int buf = t & 1;
        float ql = __shfl_up_sync(0xffffffffu, q, 1);                // Q(t-1, j-1)
        if (lane == 0) ql = warp > 0 ? edge[(buf ^ 1) * 32 + warp - 1] : NEG;
        const bool on = col && j <= t && L - 1 - j <= N - 1 - t;
        const bool diag = ql > q;
        const float lp = logf(fmaxf(a, 1e-8f));
        q = on ? lp + (t == 0 ? 0.f : (diag ? ql : q)) : NEG;
        const unsigned bits = __ballot_sync(0xffffffffu, on && diag);
        if (lane == 0) dir[(long long)t * nw + warp] = bits;
        if (lane == 31) edge[buf * 32 + warp] = q;
        if (col) cov += a;
        if (col && t == N - 1 && j == L - 1) score[b] = q;
        float m = col && a == a ? a : NEG;
        int p = col ? j : 0x7fffffff;                                // ties prefer real columns, then the lowest j
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, m, o);
            const int op = __shfl_xor_sync(0xffffffffu, p, o);
            if (om > m || (om == m && op < p)) { m = om; p = op; }
        }
        if (lane == 0) { part_m[buf * 32 + warp] = m; part_p[buf * 32 + warp] = p; }
        asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
        if (warp == 0) {
            m = lane < nw ? part_m[buf * 32 + lane] : NEG;
            p = lane < nw ? part_p[buf * 32 + lane] : 0x7fffffff;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float om = __shfl_xor_sync(0xffffffffu, m, o);
                const int op = __shfl_xor_sync(0xffffffffu, p, o);
                if (om > m || (om == m && op < p)) { m = om; p = op; }
            }
            if (lane == 0) { argmax[(long long)b * N_max + t] = p; maxv[(long long)b * N_max + t] = m; }
        }
    }
    cp_async_wait_0();
    if (col) coverage[(long long)b * L_max + j] = cov;
}

// One warp per row: durations[b, j] = the steps the path spends on token j (0 for j >= L_b, all 0 when N_b < L_b).  The
// walk moves to j - 1 where the bit says so, and also where staying would leave the grid (j >= t) and never below j = 0,
// so it ends at (0, 0) whatever the bits hold: every duration is >= 1 and they sum to N_b.
__global__ void __launch_bounds__(MAS_BT_WARPS * 32)
mas_backtrace_kernel(const int* __restrict__ steps, const int* __restrict__ tokens, int B, int L_max,
                     const long long* __restrict__ dir_off, const unsigned* __restrict__ dirs,
                     int* __restrict__ durations) {
    pdl_trigger(); pdl_wait();
    const int b = blockIdx.x * MAS_BT_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    const int N = steps[b], L = tokens[b], nw = (L + 31) >> 5;
    int* dur = durations + (long long)b * L_max;
    const bool path = N >= L;
    for (int j = path ? L + lane : lane; j < L_max; j += 32) dur[j] = 0;
    if (!path) return;
    const unsigned* dir = dirs + dir_off[b];
    int t = N - 1, j = L - 1, run = 0;
    for (;;) {
        const int wc = j >> 5, t0 = t;
        const unsigned mine = t0 - lane >= 1 ? dir[(long long)(t0 - lane) * nw + wc] : 0u;
        bool done = false;
        for (int k = 0; k < 32; ++k) {                       // cell (t, j), t = t0 - k
            ++run;
            if (t == 0) { done = true; break; }
            const unsigned w = __shfl_sync(0xffffffffu, mine, k);
            const bool back = j >= t || (j > 0 && ((w >> (j & 31)) & 1u));
            --t;
            if (back) {
                if (lane == 0) dur[j] = run;
                run = 0;
                --j;
                if ((j >> 5) != wc) break;
            }
        }
        if (done) break;
    }
    if (lane == 0) dur[0] = run;
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_mas_max_tokens(void) { return MAS_MAX_TOKENS; }

long long dv3_mas_dir_words(int steps, int tokens) {
    return steps >= 1 && tokens >= 1 && tokens <= MAS_MAX_TOKENS ? mas_dir_words(steps, tokens) : 0;
}

int dv3_mas_forward(const float* A, long long stride_b, long long stride_t, const int* steps, const int* tokens, int B,
                    int N_max, int L_max, const long long* dir_off, unsigned* dirs, int* argmax, float* maxv,
                    float* coverage, float* score, void* stream) {
    DV3_REQUIRE(A && steps && tokens && dir_off && dirs && argmax && maxv && coverage && score, "mas_forward: null operand");
    DV3_REQUIRE(B >= 1 && N_max >= 1 && L_max >= 1 && L_max <= MAS_MAX_TOKENS,
                "mas_forward: B=%d, N_max=%d, L_max=%d (L_max must lie in [1, %d])", B, N_max, L_max, MAS_MAX_TOKENS);
    DV3_REQUIRE(stride_t >= L_max && stride_b >= 0, "mas_forward: strides (%lld, %lld) for L_max=%d", stride_b,
                stride_t, L_max);
    const long long extent = (long long)(B - 1) * stride_b + (long long)(N_max - 1) * stride_t + L_max;
    DV3_REQUIRE(extent < (1LL << 31) && (long long)B * N_max < (1LL << 31) && (long long)B * L_max < (1LL << 31),
                "mas_forward: %lld alignment elements (B=%d, N_max=%d) too large for 32-bit indexing", extent, B, N_max);
    const int threads = (L_max + 31) / 32 * 32;
    const size_t smem = ((size_t)MAS_RING * threads + 192) * sizeof(float);       // <= 33 KB: no opt-in needed
    launch_k(mas_forward_kernel, (unsigned)B, threads, smem, (cudaStream_t)stream, A, stride_b, stride_t, steps, tokens,
             N_max, L_max, dir_off, dirs, argmax, maxv, coverage, score);
    return check_launch("mas_forward");
}

int dv3_mas_backtrace(const int* steps, const int* tokens, int B, int L_max, const long long* dir_off,
                      const unsigned* dirs, int* durations, void* stream) {
    DV3_REQUIRE(steps && tokens && dir_off && dirs && durations, "mas_backtrace: null operand");
    DV3_REQUIRE(B >= 1 && L_max >= 1 && L_max <= MAS_MAX_TOKENS && (long long)B * L_max < (1LL << 31),
                "mas_backtrace: B=%d, L_max=%d", B, L_max);
    launch_k(mas_backtrace_kernel, (unsigned)ceil_div(B, MAS_BT_WARPS), MAS_BT_WARPS * 32, 0, (cudaStream_t)stream,
             steps, tokens, B, L_max, dir_off, dirs, durations);
    return check_launch("mas_backtrace");
}

}  // extern "C"
