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
//
// Output descriptor (StftParams::lead / ds / lin_rows / mel_rows): frame f of a clip goes to linear row lead + f, and
// to mel row (lead + f) / ds when (lead + f) % ds == 0; every other row of both outputs is written as zero.  With
// lead = 0, ds = 1 this is the preprocessing layout (dv3_stft_mel); with lead = r and ds = downsample_step it is the
// padded, decimated layout of the training batch (data.collate), so a batch's targets come straight from its
// waveforms (dv3_stft_mel_targets).  The mel stage then runs only on kept frames: for ds in {2, 4, 8} the 8/ds kept
// frames of a group take all lanes, ds quads of filters per warp pass instead of one.  The waveform is fp32 or int16
// PCM (template), the int16 staged as is (half the shared-memory bytes) and converted x / 32768 where pass 1 reads it;
// the optional per-clip rescale x / peak * gain is applied there too, with correctly rounded division and product.
#include <type_traits>

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
    const void* wav;           // (nclips, max_len) fp32 or int16 (kernel template)
    const int* lengths;        // (nclips) valid samples per clip
    const float* mel_basis;    // (n_mels, 513) dense
    const int* mel_start;      // (n_mels) first non-zero bin
    const int* mel_len;        // (n_mels) number of non-zero bins
    float* linear;             // (nclips, lin_rows, 513) or null
    float* mel;                // (nclips, mel_rows, n_mels) or null
    int max_len, max_frames, n_mels;     // max_frames: frames computed per clip (lead + max_frames <= lin_rows)
    int lead, ds, qsh;         // output descriptor (top of file); qsh = log2(ds) for ds in {2, 4, 8}, else 0
    int lin_rows, mel_rows;
    const float* peak;         // (nclips) max |x| of each clip: x -> x / peak * gain (kernel template SCALE), or null
    float gain;
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

// raw samples x[s0-VEC .. s0+STAGE_N) of the clip -> raw[0 ..], zero outside [0, len); VEC = samples per 16 bytes
// (4 fp32 / 8 int16), so that raw[VEC] (sample s0) is 16-byte aligned and raw[VEC-1] holds x[s0-1].  Three ways:
//   BULK   the whole span lies inside the clip and is 16-byte aligned: ONE cp.async.bulk (TMA) issued by thread 0,
//          completion on sm.mbar -- no LSU instructions or shared-memory wavefronts spent on staging;
//   A16    16-byte cp.async pieces with zero fill (a clip's first / last groups);
//   else   4-byte cp.async pieces (fp32 rows that do not start on 16-byte boundaries), or plain loads and stores
//          (int16 rows likewise: cp.async has no 2-byte form).
template <typename In> struct Stage {
    static constexpr int VEC = 16 / (int)sizeof(In), BYTES = (STAGE_N + VEC) * (int)sizeof(In);
    static_assert(BYTES % 16 == 0, "bulk copies move multiples of 16 bytes");
    static_assert(BYTES <= (int)sizeof(float) * (STAGE_N + 8), "the staged span must fit StftSmem::raw");
};
template <typename In>
__device__ __forceinline__ bool stage_is_bulk(bool a16, int s0, int len) {
    return a16 && s0 >= Stage<In>::VEC && s0 + STAGE_N <= len;
}
template <typename In>
__device__ __forceinline__ void stage_async(In* raw, uint64_t* mbar, const In* x, int s0, int len, int tid, bool a16) {
    constexpr int VEC = Stage<In>::VEC;
    if (stage_is_bulk<In>(a16, s0, len)) {                     // uniform over the CTA
        if (tid == 0) {
            tc::fence_proxy_async();                             // earlier generic-proxy reads of raw[] are ordered by the barrier
            tc::mbar_arrive_expect_tx(mbar, Stage<In>::BYTES);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(tc::smem_u32(raw)), "l"(x + s0 - VEC), "r"(Stage<In>::BYTES), "r"(tc::smem_u32(mbar))
                         : "memory");
        }
        return;
    }
    if (a16) {
        for (int i = tid; i < (STAGE_N + VEC) / VEC; i += STFT_WARPS * 32) {
            const int s = s0 - VEC + VEC * i;                    // multiple of VEC: a piece never straddles sample 0
            const int nb = s < 0 ? 0 : min(max(len - s, 0), VEC) * (int)sizeof(In);
            const unsigned dst = (unsigned)__cvta_generic_to_shared(raw + VEC * i);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(x + (nb ? s : 0)), "r"(nb)
                         : "memory");
        }
    } else if constexpr (sizeof(In) == 4) {
        for (int i = tid; i < STAGE_N + 1; i += STFT_WARPS * 32) {
            const int s = s0 - 1 + i;
            const bool ok = s >= 0 && s < len;
            const unsigned dst = (unsigned)__cvta_generic_to_shared(raw + VEC - 1 + i);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(x + (ok ? s : 0)), "r"(ok ? 4 : 0)
                         : "memory");
        }
    } else {
        for (int i = tid; i < STAGE_N + 1; i += STFT_WARPS * 32) {
            const int s = s0 - 1 + i;
            raw[VEC - 1 + i] = (s >= 0 && s < len) ? x[s] : In(0);
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

// pass-1 sample sources over the staged span (stft_core.cuh RawF32 is the plain fp32 one): int16 -> x / 32768 (exact),
// then, with SCALE, x / peak * gain with a correctly rounded division and product (numpy's float32 arithmetic)
template <bool SCALE> __device__ __forceinline__ float rescale(float v, float peak, float gain) {
    return SCALE ? __fmul_rn(__fdiv_rn(v, peak), gain) : v;
}
template <bool SCALE> struct StagedF32 {
    const float* x; float peak, gain;
    __device__ __forceinline__ f4 load4(int i) const {
        const f4 s = *reinterpret_cast<const f4*>(x + i);
        return f4{rescale<SCALE>(s.x, peak, gain), rescale<SCALE>(s.y, peak, gain), rescale<SCALE>(s.z, peak, gain),
                  rescale<SCALE>(s.w, peak, gain)};
    }
    __device__ __forceinline__ float load1(int i) const { return rescale<SCALE>(x[i], peak, gain); }
};
template <bool SCALE> struct StagedS16 {
    const short* x; float peak, gain;
    __device__ __forceinline__ float cvt(short v) const {
        return rescale<SCALE>(__fmul_rn((float)v, 3.0517578125e-05f), peak, gain);         // 1 / 32768
    }
    __device__ __forceinline__ f4 load4(int i) const {
        const short4 s = *reinterpret_cast<const short4*>(x + i);
        return f4{cvt(s.x), cvt(s.y), cvt(s.z), cvt(s.w)};
    }
    __device__ __forceinline__ float load1(int i) const { return cvt(x[i]); }
};
template <typename In, bool SCALE> struct SourceOf { typedef StagedF32<SCALE> type; };
template <bool SCALE> struct SourceOf<short, SCALE> { typedef StagedS16<SCALE> type; };

template <bool TAIL, typename In, bool SCALE>
__device__ __forceinline__ void pass1_staged(int lane, const In* xs, float peak, float gain, float c, int lim,
                                             const f4* win, const f4* tw1, pr (&vr)[8], pr (&vi)[8]) {
    if constexpr (std::is_same<In, float>::value && !SCALE) pass1<TAIL>(lane, xs, c, lim, win, tw1, vr, vi);
    else pass1_src<TAIL>(lane, typename SourceOf<In, SCALE>::type{xs, peak, gain}, c, lim, win, tw1, vr, vi);
}

template <typename In, bool SCALE>
__global__ void __launch_bounds__(STFT_WARPS * 32, 3) stft_mel_kernel(const __grid_constant__ StftParams p) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    extern __shared__ __align__(16) unsigned char smem_raw[];
    StftSmem& sm = *reinterpret_cast<StftSmem*>(smem_raw);
    const int clip = blockIdx.y, f_begin = blockIdx.x * STFT_FRAMES, tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int len = p.lengths[clip];
    const int nframes = min((len + 2 * PAD - FFT_N + HOP - 1) / HOP + 1, p.max_frames);   // ceil((len+2*768-1024)/256)+1
    const int f_end = min(f_begin + STFT_FRAMES, p.max_frames);
    const int lead = p.lead, ds = p.ds;

    // zero rows (contiguous runs): the rows of this chunk's frames past the clip's own end, and in the first chunk the
    // lead rows in front of frame 0; a mel row j belongs to frame j*ds - lead
    {
        const int z0 = max(f_begin, nframes);
        const int zr[2][2] = {{lead + z0, lead + f_end}, {0, blockIdx.x == 0 ? lead : 0}};
#pragma unroll
        for (int z = 0; z < 2; ++z) {
            const int r0 = zr[z][0], r1 = zr[z][1];
            if (r0 >= r1) continue;
            if (p.linear) {
                float* o = p.linear + ((size_t)clip * p.lin_rows + r0) * NBINS;
                for (int i = tid; i < (r1 - r0) * NBINS; i += blockDim.x) o[i] = 0.f;
            }
            if (p.mel) {
                const int m0 = (r0 + ds - 1) / ds, m1 = (r1 + ds - 1) / ds;
                float* o = p.mel + ((size_t)clip * p.mel_rows + m0) * p.n_mels;
                for (int i = tid; i < (m1 - m0) * p.n_mels; i += blockDim.x) o[i] = 0.f;
            }
        }
    }
    if (f_begin >= nframes) return;

    const In* x = reinterpret_cast<const In*>(p.wav) + (size_t)clip * p.max_len;
    In* raw = reinterpret_cast<In*>(sm.raw);
    const float peak = SCALE ? p.peak[clip] : 1.f, gain = p.gain;
    const bool a16 = p.aligned16 != 0;
    if (tid == 0) { tc::mbar_init(&sm.mbar, 1); tc::fence_barrier_init(); }   // thread 0 is also the only issuer
    stage_async(raw, &sm.mbar, x, f_begin * HOP - PAD, len, tid, a16);     // in flight while the tables are set up
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
        if (stage_is_bulk<In>(a16, f0 * HOP - PAD, len)) { tc::mbar_wait(&sm.mbar, bulk_parity); bulk_parity ^= 1; }
        __syncthreads();                                            // raw[] landed; the previous group's mel stage is done
        const int frame = f0 + warp;
        const size_t fidx = (size_t)clip * p.lin_rows + lead + frame;
        if (frame < nframes) {                                      // warp-uniform
            pr vr[8], vi[8];
            const int lim = len - (frame * HOP - PAD);              // samples of the frame before the clip's end
            const In* xs = raw + Stage<In>::VEC + warp * HOP;
            if (lim < FFT_N)                                        // warp-uniform
                pass1_staged<true, In, SCALE>(lane, xs, peak, gain, p.preemph, lim, win, tw1, vr, vi);
            else pass1_staged<false, In, SCALE>(lane, xs, peak, gain, p.preemph, lim, win, tw1, vr, vi);
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
            stage_async(raw, &sm.mbar, x, (f0 + STFT_WARPS) * HOP - PAD, len, tid, a16);

        if (p.mel) {
            // lane = (frame fl, filter q of the quad): all 8 frames of the group in one go.  Quads are dealt to the
            // warps longest first in snake order (rows grow with the filter index), so the warps finish together.
            // Decimated output (ds = 2^qsh): lane = (quad sub of the pass, kept frame kf, q) -- the 8/ds kept frames
            // times ds quads per pass; any other ds keeps lane = (fl, q) and drops the rows that are not kept.
            const int qsh = p.qsh, slot = lane & 7, q = lane >> 3;
            const int sub = slot >> (3 - qsh), kf = slot & ((8 >> qsh) - 1);
            const int fl = (qsh ? (-(lead + f0)) & (ds - 1) : 0) + (kf << qsh);     // < 8
            const int t = lead + f0 + fl;                                            // padded frame index
            const bool keep = qsh != 0 || ds == 1 || t % ds == 0;
            const float* magf = sm.work[fl][0];
            const bool fvalid = f0 + fl < nframes && keep;
            float* out = p.mel + ((size_t)clip * p.mel_rows + (qsh ? t >> qsh : (ds == 1 ? t : t / ds))) * p.n_mels;
            for (int k = 0; (8 * k << qsh) < nquads; ++k) {
                const int i = ((8 * k + ((k & 1) ? STFT_WARPS - 1 - warp : warp)) << qsh) + sub;
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

// peak[c] = max |x| over clip c's own samples (int16 as x / 32768): the rescaling divisor of preprocess._load.  One CTA
// per clip; a max is exact in any order.
constexpr int PEAK_THREADS = 1024;
template <typename In>
__global__ void __launch_bounds__(PEAK_THREADS) peak_abs_kernel(const In* wav, const int* lengths, int max_len,
                                                                float* peak) {
    pdl_trigger(); pdl_wait();
    __shared__ float part[PEAK_THREADS / 32];
    const int clip = blockIdx.x, len = lengths[clip];
    const In* x = wav + (size_t)clip * max_len;
    float m = 0.f;
    for (int i = threadIdx.x; i < len; i += PEAK_THREADS) {
        const float v = std::is_same<In, float>::value ? (float)x[i] : __fmul_rn((float)x[i], 3.0517578125e-05f);
        m = fmaxf(m, fabsf(v));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = part[threadIdx.x];
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (threadIdx.x == 0) peak[clip] = m;
    }
}

template <typename In, bool SCALE>
static int launch_stft(const StftParams& p, int nclips, cudaStream_t st, const char* what) {
    static const cudaError_t attr = cudaFuncSetAttribute(stft_mel_kernel<In, SCALE>,
                                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         (int)sizeof(StftSmem));
    DV3_REQUIRE(attr == cudaSuccess, "%s: cannot reserve %zu bytes of shared memory", what, sizeof(StftSmem));
    launch_k(stft_mel_kernel<In, SCALE>, dim3((p.max_frames + STFT_FRAMES - 1) / STFT_FRAMES, nclips),
             STFT_WARPS * 32, sizeof(StftSmem), st, p);
    return check_launch(what);
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

// the parameters shared by both entry points, in the identity layout (lead 0, ds 1, one row per frame)
static int stft_params(StftParams& p, const char* what, const void* wav, const int* lengths, const float* mel_basis,
                       const int* mel_start, const int* mel_len, float* linear, float* mel, int nclips, int max_len,
                       int max_frames, int n_mels, float preemph, float min_level_db, float ref_level_db,
                       int aligned16, void* stream) {
    DV3_REQUIRE(nclips >= 1 && nclips <= 65535, "%s: nclips %d out of range", what, nclips);
    DV3_REQUIRE(max_frames >= 1, "%s: bad max_frames %d", what, max_frames);
    DV3_REQUIRE(n_mels >= 0 && n_mels <= MAX_MELS, "%s: n_mels %d > %d", what, n_mels, MAX_MELS);
    DV3_REQUIRE(stft_tables((cudaStream_t)stream) == 0, "%s: cannot build the transform tables", what);
    DV3_REQUIRE(min_level_db < 0.f, "%s: min_level_db must be negative (got %g)", what, (double)min_level_db);
    const double inv = 1.0 / -(double)min_level_db, c2 = 20.0 * 0.30102999566398120 * inv;      // 20*log10(2) / -min_db
    const double c0 = 1.0 - (double)ref_level_db * inv, min_level = pow(10.0, (double)min_level_db / 20.0);
    p = StftParams{wav, lengths, mel_basis, mel_start, mel_len, linear, mel, max_len, max_frames, n_mels,
                   /*lead*/ 0, /*ds*/ 1, /*qsh*/ 0, /*lin_rows*/ max_frames, /*mel_rows*/ max_frames,
                   /*peak*/ nullptr, /*gain*/ 1.f, preemph, (float)c2, (float)c0, (float)min_level, (float)(0.5 * c2),
                   (float)(c0 - c2), (float)(4.0 * min_level * min_level), aligned16};
    return 0;
}

int dv3_stft_mel(const float* wav, const int* lengths, const float* mel_basis, const int* mel_start,
                 const int* mel_len, float* linear, float* mel, int nclips, int max_len, int max_frames,
                 int n_mels, float preemph, float min_level_db, float ref_level_db, void* stream) {
    StftParams p;
    const int aligned16 = (reinterpret_cast<uintptr_t>(wav) % 16 == 0) && (max_len % 4 == 0);
    if (stft_params(p, "stft_mel", wav, lengths, mel_basis, mel_start, mel_len, linear, mel, nclips, max_len,
                    max_frames, n_mels, preemph, min_level_db, ref_level_db, aligned16, stream))
        return 1;
    return launch_stft<float, false>(p, nclips, (cudaStream_t)stream, "stft_mel");
}

int dv3_stft_mel_targets(const void* wav, int wav_int16, const int* lengths, const float* peak, float rescaling_max,
                         const float* mel_basis, const int* mel_start, const int* mel_len, float* linear, float* mel,
                         int nclips, int max_len, int T_lin, int lead, int downsample_step, int n_mels, float preemph,
                         float min_level_db, float ref_level_db, void* stream) {
    const char* what = "stft_mel_targets";
    DV3_REQUIRE(lead >= 0 && lead < T_lin, "%s: lead %d must lie in [0, T_lin = %d)", what, lead, T_lin);
    DV3_REQUIRE(downsample_step >= 1, "%s: bad downsample_step %d", what, downsample_step);
    StftParams p;
    const int vec = wav_int16 ? 8 : 4;                            // samples per 16 bytes
    const int aligned16 = (reinterpret_cast<uintptr_t>(wav) % 16 == 0) && (max_len % vec == 0);
    if (stft_params(p, what, wav, lengths, mel_basis, mel_start, mel_len, linear, mel, nclips, max_len, T_lin - lead,
                    n_mels, preemph, min_level_db, ref_level_db, aligned16, stream))
        return 1;
    const int ds = downsample_step;
    p.lead = lead; p.ds = ds;
    p.qsh = ds == 2 ? 1 : ds == 4 ? 2 : ds == 8 ? 3 : 0;
    p.lin_rows = T_lin; p.mel_rows = (T_lin + ds - 1) / ds;
    p.peak = peak; p.gain = rescaling_max;
    const cudaStream_t st = (cudaStream_t)stream;
    if (wav_int16) return peak ? launch_stft<short, true>(p, nclips, st, what) : launch_stft<short, false>(p, nclips, st, what);
    return peak ? launch_stft<float, true>(p, nclips, st, what) : launch_stft<float, false>(p, nclips, st, what);
}

int dv3_peak_abs_batched(const void* wav, int wav_int16, const int* lengths, int max_len, int nclips, float* peak,
                         void* stream) {
    DV3_REQUIRE(nclips >= 1, "peak_abs: nclips %d out of range", nclips);
    if (wav_int16)
        launch_k(peak_abs_kernel<short>, dim3(nclips), PEAK_THREADS, 0, (cudaStream_t)stream,
                 reinterpret_cast<const short*>(wav), lengths, max_len, peak);
    else
        launch_k(peak_abs_kernel<float>, dim3(nclips), PEAK_THREADS, 0, (cudaStream_t)stream,
                 reinterpret_cast<const float*>(wav), lengths, max_len, peak);
    return check_launch("peak_abs");
}

}  // extern "C"
