// Fused audio front-end: preemphasis -> sqrt-Hann STFT (1024 / hop 256, 768-sample zero padding on both sides)
// -> |.| -> { linear: dB, normalise } and { mel filterbank -> dB, normalise } in ONE pass over the waveform.
// Replaces reference audio.py:31-34 (spectrogram) and :46-51 (melspectrogram), which run TWO independent lws
// STFTs per clip on the CPU (ljspeech.py:63-67).  HBM-bound by construction (about 32 FLOP/B): every sample is read
// once, and only the (513 + n_mels) floats the trainer stores per frame are written back.
//
// Work decomposition: one CTA (8 warps) walks 64 consecutive frames of one clip, 8 at a time -- ONE WARP PER FRAME.
//   * the 11*256 raw samples the 8 frames overlap on are staged once in shared memory by 16-byte cp.async (zero-filled
//     outside the clip), the copy for the next 8 frames in flight while the mel rows of the current ones are formed;
//   * each warp runs the register-resident radix-8 transform of stft_core.cuh: two butterflies per lane held as
//     register PAIRS, all arithmetic pair-wise (stft_core.cuh), pre-emphasis and window
//     applied as the points are read, two exchanges through its private work area (__syncwarp only), then the split
//     into the 513-bin half spectrum four bins at a time; the normalised dB row goes straight to global memory
//     (coalesced) and the magnitudes stay in shared memory;
//   * the mel rows are sparse (mel_start / mel_len): once per CTA the non-zero weights are packed per QUAD of filters
//     (rows aligned to 4 bins, zero-padded to the quad's longest row); lane = (frame, filter of the quad) then runs
//     pure 128-bit loads + FMAs over all 8 frames at once (conflict-free because consecutive frames' planes are an odd
//     number of 16-byte words apart).  Filterbanks that do not fit the packed form take a plain (slow) loop;
//   * window, twiddles and split factors come from one table built once per device in double precision (init kernel),
//     copied into shared memory per CTA; dB through lg2.approx.
// Frames beyond a clip's own count (ragged batches) are zero-filled by the kernel, so callers pass uninitialised
// output buffers.
#include "tc_common.cuh"
#include "stft_core.cuh"

namespace dv3 {

using namespace stftc;

constexpr int FFT_N = 1024, HOP = 256, NH = 512, NBINS = 513, PAD = FFT_N - HOP;
constexpr int STFT_WARPS = 8, STFT_GROUPS = 8, STFT_FRAMES = STFT_WARPS * STFT_GROUPS;     // frames per CTA
constexpr int STAGE_N = (STFT_WARPS + 3) * HOP;                                            // samples 8 frames span
constexpr int MAX_MELS = 128, MAX_QUADS = MAX_MELS / 4;
constexpr int MEL_NNZ = 2048;           // packed (zero-padded) mel weights kept in shared memory (1.1 k for the presets)
constexpr int MEL_REACH = 568;          // a packed row may read magnitude-plane words below this index (all written)

struct StftParams {
    const float* wav;          // (nclips, max_len)
    const int* lengths;        // (nclips) valid samples per clip
    const float* mel_basis;    // (n_mels, 513) dense
    const int* mel_start;      // (n_mels) first non-zero bin
    const int* mel_len;        // (n_mels) number of non-zero bins
    float* linear;             // (nclips, max_frames, 513) or null
    float* mel;                // (nclips, max_frames, n_mels) or null
    int max_len, max_frames, n_mels;
    float preemph;
    // normalised dB: clip((20*log10(max(min_level, v)) - ref - min_db) / -min_db, 0, 1)   (audio.py:79-81, :88-89)
    //   = sat(c2 * log2(max(min_level, v)) + c0);  on p4 = |2X|^2 (log2(v) = log2(p4)/2 - 1): sat(c2h * log2(max(min_p4, p4)) + c0l)
    float c2, c0, min_level, c2h, c0l, min_p4;
    int aligned16;             // every clip starts on a 16-byte boundary: 16-byte staging copies
};

__device__ f4 g_stft_tab[TAB_N];        // window / twiddle tables, see stft_core.cuh

__global__ void stft_tables_kernel() {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < TAB_N) g_stft_tab[i] = table_entry(i);
}

struct StftSmem {
    alignas(16) float raw[STAGE_N + 8];   // raw[4 + i] = x[s0 + i] (16-byte aligned frames), raw[3] = x[s0 - 1]
    f4 tab[TAB_N];
    alignas(16) float wt[MEL_NNZ];        // packed mel weights: quad Q at qoff[Q], row q at + q*L4, zero padded
    int4 frow[MAX_MELS];                  // per filter: (start4 / 4, zero weights in front = start - start4, len, start)
    int2 qinfo[MAX_QUADS];                // per quad: (offset in wt[] / 4, padded row length / 4)
    int badw[4];                          // per warp of the set-up: a row of its filters reaches past MEL_REACH
    int packed;                           // 1: every quad fits the packed form
    alignas(8) uint64_t mbar;             // completion of the bulk (TMA) staging copies
    alignas(16) float work[STFT_WARPS][2][WORK];      // per-warp re / im planes; the magnitudes end up in plane 0
};
static_assert((2 * WORK) % 4 == 0 && ((2 * WORK) / 4) % 2 == 1, "frame planes must sit an odd number of 16-byte words apart");
static_assert((WORK * 4) % 8 == 0, "the im plane must be 8-byte aligned");

__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sqrt_approx(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// raw samples x[s0-4 .. s0+STAGE_N) of the clip -> sm.raw[0 ..], zero outside [0, len).  Three ways:
//   BULK   the whole span lies inside the clip and is 16-byte aligned: ONE cp.async.bulk (TMA) issued by thread 0,
//          completion on sm.mbar -- no LSU instructions or shared-memory wavefronts spent on staging;
//   A16    16-byte cp.async pieces with zero fill (a clip's first / last groups);
//   else   4-byte cp.async pieces (rows that do not start on 16-byte boundaries).
constexpr int STAGE_BYTES = (STAGE_N + 4) * 4;
static_assert(STAGE_BYTES % 16 == 0, "bulk copies move multiples of 16 bytes");
__device__ __forceinline__ bool stage_is_bulk(bool a16, int s0, int len) { return a16 && s0 >= 4 && s0 + STAGE_N <= len; }
__device__ __forceinline__ void stage_async(float* raw, uint64_t* mbar, const float* x, int s0, int len, int tid,
                                            bool a16) {
    if (stage_is_bulk(a16, s0, len)) {                         // uniform over the CTA
        if (tid == 0) {
            tc::fence_proxy_async();                             // earlier generic-proxy reads of raw[] are ordered by the barrier
            tc::mbar_arrive_expect_tx(mbar, STAGE_BYTES);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(raw)), "l"(x + s0 - 4), "r"(STAGE_BYTES), "r"(tc::smem_u32(mbar)) : "memory");
        }
        return;
    }
    if (a16) {
        for (int i = tid; i < (STAGE_N + 4) / 4; i += STFT_WARPS * 32) {
            const int s = s0 - 4 + 4 * i;                        // multiple of 4: a piece never straddles sample 0
            const int nb = s < 0 ? 0 : min(max(len - s, 0), 4) * 4;
            const unsigned dst = (unsigned)__cvta_generic_to_shared(raw + 4 * i);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(x + (nb ? s : 0)), "r"(nb)
                         : "memory");
        }
    } else {
        for (int i = tid; i < STAGE_N + 1; i += STFT_WARPS * 32) {
            const int s = s0 - 1 + i;
            const bool ok = s >= 0 && s < len;
            const unsigned dst = (unsigned)__cvta_generic_to_shared(raw + 3 + i);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(x + (ok ? s : 0)), "r"(ok ? 4 : 0)
                         : "memory");
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

__global__ void __launch_bounds__(STFT_WARPS * 32, 3) stft_mel_kernel(const __grid_constant__ StftParams p) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    extern __shared__ __align__(16) unsigned char smem_raw[];
    StftSmem& sm = *reinterpret_cast<StftSmem*>(smem_raw);
    const int clip = blockIdx.y, f_begin = blockIdx.x * STFT_FRAMES, tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int len = p.lengths[clip];
    const int nframes = min((len + 2 * PAD - FFT_N + HOP - 1) / HOP + 1, p.max_frames);   // ceil((len+2*768-1024)/256)+1
    const int f_end = min(f_begin + STFT_FRAMES, p.max_frames);

    // frames of this chunk past the clip's own end: zero-fill (contiguous rows)
    {
        const int z0 = max(f_begin, nframes);
        if (z0 < f_end) {
            const size_t row0 = (size_t)clip * p.max_frames + z0;
            if (p.linear) {
                float* o = p.linear + row0 * NBINS;
                for (int i = tid; i < (f_end - z0) * NBINS; i += blockDim.x) o[i] = 0.f;
            }
            if (p.mel) {
                float* o = p.mel + row0 * p.n_mels;
                for (int i = tid; i < (f_end - z0) * p.n_mels; i += blockDim.x) o[i] = 0.f;
            }
        }
    }
    if (f_begin >= nframes) return;

    const float* x = p.wav + (size_t)clip * p.max_len;
    const bool a16 = p.aligned16 != 0;
    if (tid == 0) { tc::mbar_init(&sm.mbar, 1); tc::fence_barrier_init(); }   // thread 0 is also the only issuer
    stage_async(sm.raw, &sm.mbar, x, f_begin * HOP - PAD, len, tid, a16);     // in flight while the tables are set up
    uint32_t bulk_parity = 0;

    // ---- tables, once per CTA ----
    for (int i = tid; i < TAB_N; i += blockDim.x) sm.tab[i] = g_stft_tab[i];
    const int nquads = (p.n_mels + 3) >> 2;
    int myL4 = 0;
    if (p.mel && tid < MAX_MELS) {                 // warps 0-3: one thread per filter, a quad = 4 consecutive lanes
        const int m = tid;
        const int s = m < p.n_mels ? p.mel_start[m] : 0, l = m < p.n_mels ? p.mel_len[m] : 0;
        const int s4 = s & ~3, ext = l > 0 ? (s - s4) + l : 0;
        int mx = max(ext, __shfl_xor_sync(0xffffffffu, ext, 1));
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        myL4 = (mx + 3) & ~3;
        sm.frow[m] = make_int4(s4 >> 2, s - s4, l, s);
        if ((m & 3) == 0) sm.qinfo[m >> 2].y = myL4 >> 2;
        const bool bad = (l > 0 && s4 + myL4 > MEL_REACH) || myL4 > 64;       // the packing below covers 64 columns
        const bool anybad = __any_sync(0xffffffffu, bad);
        if (lane == 0) sm.badw[warp] = anybad;
    }
    __syncthreads();
    if (p.mel && warp == 0) {                      // exclusive scan of the quads' packed sizes (in 16-byte words)
        const int sz = lane < nquads ? 4 * sm.qinfo[lane].y : 0;
        int inc = sz;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        sm.qinfo[lane].x = inc - sz;
        const int total = __shfl_sync(0xffffffffu, inc, 31);
        if (lane == 0) sm.packed = (!(sm.badw[0] | sm.badw[1] | sm.badw[2] | sm.badw[3]) && 4 * total <= MEL_NNZ) ? 1 : 0;
    }
    __syncthreads();
    const bool packed = p.mel && sm.packed == 1;
    if (packed) {
        // warp w packs rows w, w+8, ...: columns lane and lane+32 of each; four rows' loads are issued before the
        // first store so that the (L2-latency) loads overlap
        const int nrows = 4 * nquads;
        for (int m0 = warp; m0 < nrows; m0 += 4 * STFT_WARPS) {
            float v[4][2];
            int dst[4], L4s[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int m = m0 + r * STFT_WARPS;
                v[r][0] = v[r][1] = 0.f; dst[r] = 0; L4s[r] = 0;
                if (m < nrows) {
                    const int4 fr = sm.frow[m];
                    const int2 qi = sm.qinfo[m >> 2];
                    L4s[r] = 4 * qi.y; dst[r] = 4 * qi.x + (m & 3) * L4s[r];
                    const float* row = p.mel_basis + (size_t)m * NBINS + fr.w - fr.y;
                    const int j0 = lane - fr.y, j1 = lane + 32 - fr.y;
                    if (j0 >= 0 && j0 < fr.z) v[r][0] = __ldg(row + lane);
                    if (j1 >= 0 && j1 < fr.z) v[r][1] = __ldg(row + lane + 32);
                }
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                if (lane < L4s[r]) sm.wt[dst[r] + lane] = v[r][0];
                if (lane + 32 < L4s[r]) sm.wt[dst[r] + lane + 32] = v[r][1];
            }
        }
    }
    const float c2 = p.c2, c0 = p.c0, min_level = p.min_level, c2h = p.c2h, c0l = p.c0l, min_p4 = p.min_p4;

    float* re = sm.work[warp][0];
    float* im = sm.work[warp][1];
    const f4 *win = sm.tab + TAB_WIN, *tw1 = sm.tab + TAB_TW1, *tw2 = sm.tab + TAB_TW2, *wsp = sm.tab + TAB_WSP;

    for (int g = 0; g < STFT_GROUPS; ++g) {
        const int f0 = f_begin + g * STFT_WARPS;
        if (f0 >= nframes) break;                                   // uniform over the CTA
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        if (stage_is_bulk(a16, f0 * HOP - PAD, len)) { tc::mbar_wait(&sm.mbar, bulk_parity); bulk_parity ^= 1; }
        __syncthreads();                                            // raw[] landed; the previous group's mel stage is done
        const int frame = f0 + warp;
        const size_t fidx = (size_t)clip * p.max_frames + frame;
        if (frame < nframes) {                                      // warp-uniform
            pr vr[8], vi[8];
            const int lim = len - (frame * HOP - PAD);              // samples of the frame before the clip's end
            const float* xs = sm.raw + 4 + warp * HOP;
            if (lim < FFT_N) pass1<true>(lane, xs, p.preemph, lim, win, tw1, vr, vi);     // warp-uniform
            else pass1<false>(lane, xs, p.preemph, lim, win, tw1, vr, vi);
            store1(lane, vr, vi, re, im);
            __syncwarp();
            pass2(lane, re, im, tw2, vr, vi);
            __syncwarp();
            store2(lane, vr, vi, re, im);
            __syncwarp();
            pass3(lane, re, im, vr, vi);
            __syncwarp();
            store3(lane, vr, vi, re, im);
            __syncwarp();

            // split into the half spectrum, bins (k, k+32, 512-k, 480-k), k = lane + 64*j; dB row out, magnitudes back
            // into re[] (every index is read and written by exactly one lane in one step, so in place is safe)
            float* lin = p.linear ? p.linear + fidx * NBINS : nullptr;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int ka = lane + 64 * j;
                pr lo, hi;
                split4(ka, re, im, rot16(wsp[lane], j), lo, hi);
                if (lin) {
                    lin[ka] = __saturatef(fmaf(c2h, lg2_approx(fmaxf(lo.x, min_p4)), c0l));
                    lin[ka + 32] = __saturatef(fmaf(c2h, lg2_approx(fmaxf(lo.y, min_p4)), c0l));
                    lin[NH - ka] = __saturatef(fmaf(c2h, lg2_approx(fmaxf(hi.x, min_p4)), c0l));
                    lin[NH - 32 - ka] = __saturatef(fmaf(c2h, lg2_approx(fmaxf(hi.y, min_p4)), c0l));
                }
                re[ka] = 0.5f * sqrt_approx(lo.x);
                re[ka + 32] = 0.5f * sqrt_approx(lo.y);
                re[NH - ka] = 0.5f * sqrt_approx(hi.x);
                re[NH - 32 - ka] = 0.5f * sqrt_approx(hi.y);
            }
            if (lane == 0) {
                const float pn = split_nyquist(re, im);
                if (lin) lin[NH / 2] = __saturatef(fmaf(c2h, lg2_approx(fmaxf(pn, min_p4)), c0l));
                re[NH / 2] = 0.5f * sqrt_approx(pn);
            }
        }
        __syncthreads();                                            // all 8 frames' magnitudes are in place; raw[] is free
        if (g + 1 < STFT_GROUPS && f0 + STFT_WARPS < nframes)
            stage_async(sm.raw, &sm.mbar, x, (f0 + STFT_WARPS) * HOP - PAD, len, tid, a16);

        if (p.mel) {
            // lane = (frame fl, filter q of the quad): all 8 frames of the group in one go.  Quads are dealt to the
            // warps longest first in snake order (rows grow with the filter index), so the warps finish together.
            const int fl = lane & 7, q = lane >> 3;
            const float* magf = sm.work[fl][0];
            const bool fvalid = f0 + fl < nframes;
            float* out = p.mel + ((size_t)clip * p.max_frames + f0 + fl) * p.n_mels;
            for (int k = 0; 8 * k < nquads; ++k) {
                const int i = 8 * k + ((k & 1) ? STFT_WARPS - 1 - warp : warp);
                if (i >= nquads) continue;
                const int Q = nquads - 1 - i, m = 4 * Q + q;
                float acc = 0.f;
                if (packed) {
                    const int2 qi = sm.qinfo[Q];
                    const f4* w4 = reinterpret_cast<const f4*>(sm.wt) + qi.x + q * qi.y;
                    const f4* m4 = reinterpret_cast<const f4*>(magf) + sm.frow[m].x;
                    float acc1 = 0.f;
                    int jj = 0;
#pragma unroll 1
                    for (; jj + 1 < qi.y; jj += 2) {
                        const f4 a0 = m4[jj], b0 = w4[jj], a1 = m4[jj + 1], b1 = w4[jj + 1];
                        acc = fmaf(a0.x, b0.x, acc); acc1 = fmaf(a1.x, b1.x, acc1);
                        acc = fmaf(a0.y, b0.y, acc); acc1 = fmaf(a1.y, b1.y, acc1);
                        acc = fmaf(a0.z, b0.z, acc); acc1 = fmaf(a1.z, b1.z, acc1);
                        acc = fmaf(a0.w, b0.w, acc); acc1 = fmaf(a1.w, b1.w, acc1);
                    }
                    if (jj < qi.y) {
                        const f4 a0 = m4[jj], b0 = w4[jj];
                        acc = fmaf(a0.x, b0.x, acc); acc1 = fmaf(a0.y, b0.y, acc1);
                        acc = fmaf(a0.z, b0.z, acc); acc1 = fmaf(a0.w, b0.w, acc1);
                    }
                    acc += acc1;
                } else if (m < p.n_mels) {                           // general filterbank: weights from global memory
                    const int4 fr = sm.frow[m];
                    const float* w = p.mel_basis + (size_t)m * NBINS + fr.w;
#pragma unroll 1
                    for (int jj = 0; jj < fr.z; ++jj) acc = fmaf(w[jj], magf[fr.w + jj], acc);
                }
                if (fvalid && m < p.n_mels) out[m] = __saturatef(fmaf(c2, lg2_approx(fmaxf(acc, min_level)), c0));
            }
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

}  // namespace dv3

using namespace dv3;

extern "C" {

// frames produced for a clip of n samples: ceil((n + 2*768 - 1024)/256) + 1   (lws "perfectrec" padding)
int dv3_stft_num_frames(int n_samples) { return (n_samples + 2 * PAD - FFT_N + HOP - 1) / HOP + 1; }

// The table kernel runs once per device (synchronously, so that other streams may use the table afterwards); inside a
// stream capture it is simply recorded in front of every STFT launch (it is idempotent).
static int stft_tables(cudaStream_t st) {
    static bool done[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 1;
    if (done[dev]) return 0;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    stft_tables_kernel<<<(TAB_N + 127) / 128, 128, 0, st>>>();
    if (cudaGetLastError() != cudaSuccess) return 1;
    if (cap == cudaStreamCaptureStatusNone) {
        if (cudaStreamSynchronize(st) != cudaSuccess) return 1;
        done[dev] = true;
    }
    return 0;
}

int dv3_stft_mel(const float* wav, const int* lengths, const float* mel_basis, const int* mel_start,
                 const int* mel_len, float* linear, float* mel, int nclips, int max_len, int max_frames,
                 int n_mels, float preemph, float min_level_db, float ref_level_db, void* stream) {
    DV3_REQUIRE(nclips >= 1 && nclips <= 65535, "stft_mel: nclips %d out of range", nclips);
    DV3_REQUIRE(max_frames >= 1, "stft_mel: bad max_frames %d", max_frames);
    DV3_REQUIRE(n_mels >= 0 && n_mels <= MAX_MELS, "stft_mel: n_mels %d > %d", n_mels, MAX_MELS);
    DV3_REQUIRE(stft_tables((cudaStream_t)stream) == 0, "stft_mel: cannot build the transform tables");
    const int aligned16 = (reinterpret_cast<uintptr_t>(wav) % 16 == 0) && (max_len % 4 == 0);
    DV3_REQUIRE(min_level_db < 0.f, "stft_mel: min_level_db must be negative (got %g)", (double)min_level_db);
    const double inv = 1.0 / -(double)min_level_db, c2 = 20.0 * 0.30102999566398120 * inv;      // 20*log10(2) / -min_db
    const double c0 = 1.0 - (double)ref_level_db * inv, min_level = pow(10.0, (double)min_level_db / 20.0);
    StftParams p = {wav, lengths, mel_basis, mel_start, mel_len, linear, mel, max_len, max_frames, n_mels, preemph,
                    (float)c2, (float)c0, (float)min_level, (float)(0.5 * c2), (float)(c0 - c2),
                    (float)(4.0 * min_level * min_level), aligned16};
    static const cudaError_t attr = cudaFuncSetAttribute(stft_mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         (int)sizeof(StftSmem));
    DV3_REQUIRE(attr == cudaSuccess, "stft_mel: cannot reserve %zu bytes of shared memory", sizeof(StftSmem));
    launch_k(stft_mel_kernel, dim3((max_frames + STFT_FRAMES - 1) / STFT_FRAMES, nclips), STFT_WARPS * 32,
             sizeof(StftSmem), (cudaStream_t)stream, p);
    return check_launch("stft_mel");
}

}  // extern "C"
