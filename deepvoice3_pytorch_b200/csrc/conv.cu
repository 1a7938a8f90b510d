// Fused ConvBlock kernels (exact-fp32 math mode) -- replaces, per block, the reference's
//   F.dropout -> weight-normed nn.Conv1d (cuDNN) -> causal trim -> split -> +softsign(speaker) ->
//   sigmoid -> mul -> add -> mul chain (reference deepvoice3_pytorch/modules.py:145-164 Conv1dGLU,
//   :200-226 HighwayConv1d) and the plain weight-normed Conv1d (+ReLU) of modules.py:94-100.
//
// Layout: activations (B, C, T) fp32, T contiguous (the reference's conv layout).  The conv is an
// implicit GEMM  Y[co, (b,t)] = sum_{j,ci} W[j][ci][co] * Xd[b, ci, t + off_j]  with the (b,t) axis
// flattened into N = B*T so no tile is wasted on short sequences; the loader gathers the shifted,
// zero-padded, dropout-masked input straight into shared memory (im2col never touches HBM).
//   forward  : A = packed weights W_f[j][ci][co],  B = gather(x),   epilogue = bias/speaker/GLU|highway/residual
//   dgrad    : A = packed weights W_b[j][co][ci],  B = gather(dAB), epilogue = dropout mask + residual-path grads
//   wgrad    : A = dAB (K-contiguous),             B = gather(x) (K-contiguous), epilogue = split-K partials
#include "gemm_simt.cuh"

namespace dv3 {

constexpr int MAX_TAPS = 8;

struct ConvParams {
    // operands
    const float* x;        // (B, Cin, T) input of the gather
    const float* w;        // [k][Cin][Mtot]
    const float* bias;     // [Mtot] or null
    const float* spk;      // (B, Cg, T) or null          (gated forward)
    const float* res;      // (B, Cg, T) residual input    (gated forward)  == x of the block
    float* y;              // (B, Mout, T)
    float* save_a;         // (B, Cg, T) or null
    float* save_s;         // (B, Cg, T) or null
    // dgrad epilogue extras
    const float* e1;       // addend tensor 1 (B, Mtot, T) or null
    const float* e2;       // addend tensor 2
    float alpha;           // mode 1: y += alpha*e1 ; mode 2: y += e1*(1-e2)
    int addmode;
    // sizes
    int B, Cin, T, N;      // N = B*T
    int Mtot;              // rows of the implicit GEMM (2*Cg when gated)
    int Cg;                // gated: channels per half
    int k, cpt;            // taps, chunks per tap = ceil(Cin/BK)
    int tap_off[MAX_TAPS];
    int mode;              // gated: 0 GLU, 1 highway ; plain: bit0 = relu
    int residual;
    // dropout on the gathered operand (forward, wgrad) or on the output (dgrad)
    float p_drop;
    const unsigned long long* seed_ptr;
    uint32_t salt;
    int drop_on_output;
};

template <bool GATED>
struct ConvPolicy {
    using Params = ConvParams;

    struct ALoad {
        using Map = DirectMap<GEMM_BM>;
        static constexpr int N = Map::N;
        Map map;
        const float* w;
        int co, Cin, Mtot, cpt;
        bool valid;
        __device__ ALoad(const Params& p, int m_tile, int, int tid) : map(tid) {
            const int r = map.row(0);
            if (GATED) {
                const int c = m_tile * 64 + (r & 63);
                valid = c < p.Cg;
                co = (r < 64) ? c : p.Cg + c;
            } else {
                co = m_tile * GEMM_BM + r;
                valid = co < p.Mtot;
            }
            w = p.w; Cin = p.Cin; Mtot = p.Mtot; cpt = p.cpt;
        }
        __device__ void fetch(int chunk, float* r) const {
            const int j = chunk / cpt, ci0 = (chunk - j * cpt) * GEMM_BK;
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const int ci = ci0 + map.kk(i);
                r[i] = (valid && ci < Cin) ? __ldg(&w[((size_t)j * Cin + ci) * Mtot + co]) : 0.f;
            }
        }
        __device__ void store(float* S, const float* r) const { tile_store<GEMM_BM>(S, map, r); }
    };

    template <int BN>
    struct BLoad {
        using Map = DirectMap<BN>;
        static constexpr int N = Map::N;
        Map map;
        const float* x;
        const int* tap_off;
        int b, t, T, Cin, cpt;
        bool validn;
        DropCfg drop;
        __device__ BLoad(const Params& p, int n_tile, int, int tid) : map(tid) {
            const int n = n_tile * BN + map.row(0);
            validn = n < p.N;
            b = validn ? n / p.T : 0;
            t = n - b * p.T;
            x = p.x; T = p.T; Cin = p.Cin; cpt = p.cpt; tap_off = p.tap_off;
            drop = make_drop(p.drop_on_output ? 0.f : p.p_drop, p.seed_ptr, p.salt);
        }
        __device__ void fetch(int chunk, float* r) const {
            const int j = chunk / cpt, ci0 = (chunk - j * cpt) * GEMM_BK;
            const int tt = t + tap_off[j];
            const bool ok = validn && tt >= 0 && tt < T;
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const int ci = ci0 + map.kk(i);
                float v = 0.f;
                if (ok && ci < Cin) {
                    const uint32_t idx = (uint32_t)((b * Cin + ci) * T + tt);
                    v = __ldg(&x[idx]) * drop_scale(drop, idx);
                }
                r[i] = v;
            }
        }
        __device__ void store(float* S, const float* r) const { tile_store<BN>(S, map, r); }
    };

    __device__ static int num_chunks(const Params& p, int) { return p.k * p.cpt; }

    template <int BN>
    __device__ static void epilogue(const Params& p, const Acc<BN>& acc, int m_tile, int n_tile, int,
                                    int tx, int ty) {
        constexpr int NG = BN / 64;                 // column groups of 4 per thread
        const bool vec = (p.T & 3) == 0;
        const DropCfg drop = make_drop(p.drop_on_output ? p.p_drop : 0.f, p.seed_ptr, p.salt);
#pragma unroll
        for (int g = 0; g < NG; ++g) {
            const int n = n_tile * BN + g * 64 + tx * 4;
            if (n >= p.N) continue;
            int bq[4], tq[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int nn = n + q;
                bq[q] = nn / p.T; tq[q] = nn - bq[q] * p.T;
            }
            if (GATED) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int c = m_tile * 64 + ty * 4 + i;
                    if (c >= p.Cg) continue;
                    const float ba = p.bias ? p.bias[c] : 0.f;
                    const float bb = p.bias ? p.bias[p.Cg + c] : 0.f;
                    float yo[4], ao[4], so[4];
                    size_t idx[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        if (n + q >= p.N) { idx[q] = 0; yo[q] = ao[q] = so[q] = 0.f; continue; }
                        idx[q] = ((size_t)bq[q] * p.Cg + c) * p.T + tq[q];
                        float a = acc.v[i][g * 4 + q] + ba;
                        if (p.spk) a += p.spk[idx[q]];
                        const float s = sigmoidf_(acc.v[4 + i][g * 4 + q] + bb);
                        float y;
                        if (p.mode == 0) {
                            y = a * s;
                            if (p.residual) y = (y + p.res[idx[q]]) * 0.70710678118654752f;
                        } else {
                            const float xr = p.res[idx[q]];
                            y = s * a + (1.f - s) * xr;
                        }
                        yo[q] = y; ao[q] = a; so[q] = s;
                    }
                    if (vec && n + 3 < p.N) {
                        *reinterpret_cast<float4*>(&p.y[idx[0]]) = make_float4(yo[0], yo[1], yo[2], yo[3]);
                        if (p.save_a) *reinterpret_cast<float4*>(&p.save_a[idx[0]]) = make_float4(ao[0], ao[1], ao[2], ao[3]);
                        if (p.save_s) *reinterpret_cast<float4*>(&p.save_s[idx[0]]) = make_float4(so[0], so[1], so[2], so[3]);
                    } else {
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            if (n + q >= p.N) continue;
                            p.y[idx[q]] = yo[q];
                            if (p.save_a) p.save_a[idx[q]] = ao[q];
                            if (p.save_s) p.save_s[idx[q]] = so[q];
                        }
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int m = m_tile * GEMM_BM + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
                    if (m >= p.Mtot) continue;
                    const float bm = p.bias ? p.bias[m] : 0.f;
                    float yo[4];
                    size_t idx[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        if (n + q >= p.N) { idx[q] = 0; yo[q] = 0.f; continue; }
                        idx[q] = ((size_t)bq[q] * p.Mtot + m) * p.T + tq[q];
                        float y = acc.v[i][g * 4 + q] + bm;
                        if (p.drop_on_output) y *= drop_scale(drop, (uint32_t)idx[q]);
                        if (p.addmode == 1) y += p.alpha * p.e1[idx[q]];
                        else if (p.addmode == 2) y += p.e1[idx[q]] * (1.f - p.e2[idx[q]]);
                        if (p.mode & 1) y = fmaxf(y, 0.f);
                        yo[q] = y;
                    }
                    if (vec && n + 3 < p.N) {
                        *reinterpret_cast<float4*>(&p.y[idx[0]]) = make_float4(yo[0], yo[1], yo[2], yo[3]);
                    } else {
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            if (n + q < p.N) p.y[idx[q]] = yo[q];
                    }
                }
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// weight gradient:  dW[m][ci][j] = sum_{b,t} dAB[b,m,t] * Xd[b,ci,t+off_j]     (split over (b,t))
// ------------------------------------------------------------------------------------------------
struct WgradParams {
    const float* dab;      // (B, M, T)
    const float* x;        // (B, Cin, T)
    float* dw;             // partials [nsplit][...], element address = m_addr(m) + ci*s_n + j*s_j
    size_t split_stride;
    int B, M, Cin, T, N;
    int k, nsplit, chunks_per_split;
    int tap_off[MAX_TAPS];
    int msplit, s_m, s_mh, s_n, s_j;
    float p_drop;
    const unsigned long long* seed_ptr;
    uint32_t salt;
};

struct WgradPolicy {
    using Params = WgradParams;

    struct ALoad {
        using Map = TransMap<GEMM_BM>;
        static constexpr int N = Map::N;
        Map map;
        const float* dab;
        int m0, M, T, Ntot, nbase;
        __device__ ALoad(const Params& p, int m_tile, int z, int tid) : map(tid) {
            dab = p.dab; m0 = m_tile * GEMM_BM; M = p.M; T = p.T; Ntot = p.N;
            nbase = (z / p.k) * p.chunks_per_split * GEMM_BK;
        }
        __device__ void fetch(int chunk, float* r) const {
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const int n = nbase + chunk * GEMM_BK + map.kk(i);
                const int m = m0 + map.row(i);
                float v = 0.f;
                if (n < Ntot && m < M) {
                    const int b = n / T, t = n - b * T;
                    v = __ldg(&dab[((size_t)b * M + m) * T + t]);
                }
                r[i] = v;
            }
        }
        __device__ void store(float* S, const float* r) const { tile_store<GEMM_BM>(S, map, r); }
    };

    template <int BN>
    struct BLoad {
        using Map = TransMap<BN>;
        static constexpr int N = Map::N;
        Map map;
        const float* x;
        int c0, Cin, T, Ntot, nbase, off;
        DropCfg drop;
        __device__ BLoad(const Params& p, int n_tile, int z, int tid) : map(tid) {
            x = p.x; c0 = n_tile * BN; Cin = p.Cin; T = p.T; Ntot = p.N;
            nbase = (z / p.k) * p.chunks_per_split * GEMM_BK;
            off = p.tap_off[z % p.k];
            drop = make_drop(p.p_drop, p.seed_ptr, p.salt);
        }
        __device__ void fetch(int chunk, float* r) const {
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const int n = nbase + chunk * GEMM_BK + map.kk(i);
                const int ci = c0 + map.row(i);
                float v = 0.f;
                if (n < Ntot && ci < Cin) {
                    const int b = n / T, tt = n - b * T + off;
                    if (tt >= 0 && tt < T) {
                        const uint32_t idx = (uint32_t)((b * Cin + ci) * T + tt);
                        v = __ldg(&x[idx]) * drop_scale(drop, idx);
                    }
                }
                r[i] = v;
            }
        }
        __device__ void store(float* S, const float* r) const { tile_store<BN>(S, map, r); }
    };

    __device__ static int num_chunks(const Params& p, int z) {
        const int total = (p.N + GEMM_BK - 1) / GEMM_BK;
        const int beg = (z / p.k) * p.chunks_per_split;
        int n = total - beg;
        return n < 0 ? 0 : (n > p.chunks_per_split ? p.chunks_per_split : n);
    }

    template <int BN>
    __device__ static void epilogue(const Params& p, const Acc<BN>& acc, int m_tile, int n_tile, int z,
                                    int tx, int ty) {
        const int j = z % p.k, split = z / p.k;
        float* out = p.dw + (size_t)split * p.split_stride + (size_t)j * p.s_j;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m_tile * GEMM_BM + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
            if (m >= p.M) continue;
            const size_t ma = (size_t)(m % p.msplit) * p.s_m + (size_t)(m / p.msplit) * p.s_mh;
#pragma unroll
            for (int q = 0; q < Acc<BN>::NC; ++q) {
                const int ci = n_tile * BN + (q >> 2) * 64 + tx * 4 + (q & 3);
                if (ci < p.Cin) out[ma + (size_t)ci * p.s_n] = acc.v[i][q];
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// gate backward (elementwise) + bias gradient
//   GLU     : y = a*s [ (.+x)*sqrt.5 ]      da = g*s ; db = g*a*s*(1-s)            g = dy*(res?sqrt.5:1)
//   highway : y = s*a + (1-s)*x             da = dy*s ; db = dy*(a-x)*s*(1-s)
// writes dAB (B, 2C, T) = [da ; db], dbias[2C] += row sums.  One warp per (b, c) row.
// ------------------------------------------------------------------------------------------------
__global__ void gate_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ a,
                                const float* __restrict__ s, const float* __restrict__ x,
                                float* __restrict__ dab, float* __restrict__ dbias, int B, int C, int T,
                                int mode, int residual) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * C) return;
    const int b = warp / C, c = warp - b * C;
    const size_t in = (size_t)warp * T;
    const size_t oa = ((size_t)b * 2 * C + c) * T, ob = oa + (size_t)C * T;
    const float gs = (mode == 0 && residual) ? 0.70710678118654752f : 1.f;
    float sa = 0.f, sb = 0.f;
    for (int t = lane; t < T; t += 32) {
        const float g = dy[in + t] * gs, av = a[in + t], sv = s[in + t];
        const float da = g * sv;
        const float core = (mode == 0) ? av : (av - x[in + t]);
        const float db = g * core * sv * (1.f - sv);
        dab[oa + t] = da; dab[ob + t] = db;
        sa += da; sb += db;
    }
    sa = warp_sum(sa); sb = warp_sum(sb);
    if (lane == 0 && dbias) { atomicAdd(&dbias[c], sa); atomicAdd(&dbias[C + c], sb); }
}

// plain conv: dyr = dy * (relu ? y>0 : 1) ; dbias[c] += sum_{b,t} dyr.  One warp per (b,c) row.
__global__ void bias_act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                    float* __restrict__ dyr, float* __restrict__ dbias, int B, int C,
                                    int T, int relu) {
    pdl_trigger(); pdl_wait();     // programmatic dependent launch: see common.cuh
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * C) return;
    const int c = warp % C;
    const size_t base = (size_t)warp * T;
    float sum = 0.f;
    for (int t = lane; t < T; t += 32) {
        float g = dy[base + t];
        if (relu) { g = y[base + t] > 0.f ? g : 0.f; dyr[base + t] = g; }
        sum += g;
    }
    sum = warp_sum(sum);
    if (lane == 0 && dbias) atomicAdd(&dbias[c], sum);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int g_num_sms = 0;
static int num_sms() {
    if (!g_num_sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) g_num_sms = 132;
    }
    return g_num_sms;
}

template <class P, int BN>
static int launch_gemm(const typename P::Params& p, dim3 grid, cudaStream_t st, const char* what) {
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(gemm_simt_kernel<P, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             gemm_smem_bytes<BN>());
        configured = true;
    }
    launch_k(gemm_simt_kernel<P, BN>, grid, GEMM_THREADS, gemm_smem_bytes<BN>(), st, p);
    return check_launch(what);
}

static void fill_taps(int* tap_off, int k, int dilation, int causal, bool transpose) {
    const int padl = causal ? (k - 1) * dilation : (k - 1) / 2 * dilation;
    for (int j = 0; j < k; ++j) tap_off[j] = transpose ? (padl - j * dilation) : (j * dilation - padl);
}

template <bool GATED>
static int run_conv(ConvParams& p, cudaStream_t st, const char* what) {
    const int m_tiles = GATED ? ceil_div(p.Cg, 64) : ceil_div(p.Mtot, GEMM_BM);
    const int bn = pick_bn(p.N, m_tiles, 1, num_sms());
    if (bn == 128) return launch_gemm<ConvPolicy<GATED>, 128>(p, dim3(ceil_div(p.N, 128), m_tiles, 1), st, what);
    return launch_gemm<ConvPolicy<GATED>, 64>(p, dim3(ceil_div(p.N, 64), m_tiles, 1), st, what);
}

}  // namespace dv3

using namespace dv3;

extern "C" {

int dv3_convblock_fwd(const float* x, const float* w_f, const float* bias, const float* spk, float* y,
                      float* save_a, float* save_s, int B, int C, int T, int k, int dilation, int causal,
                      int mode, int residual, float p_drop, const unsigned long long* seed_ptr,
                      unsigned salt, void* stream) {
    DV3_REQUIRE(k >= 1 && k <= MAX_TAPS, "convblock_fwd: kernel size %d not in [1,%d]", k, MAX_TAPS);
    DV3_REQUIRE((long long)B * C * T < (1LL << 31),
                "convblock_fwd: tensor of %lld elements too large for 32-bit indexing", (long long)B * C * T);
    DV3_REQUIRE(mode == 0 || mode == 1, "convblock_fwd: mode must be 0 (GLU) or 1 (highway)");
    ConvParams p = {};
    p.x = x; p.w = w_f; p.bias = bias; p.spk = spk; p.res = x; p.y = y; p.save_a = save_a; p.save_s = save_s;
    p.B = B; p.Cin = C; p.T = T; p.N = B * T; p.Mtot = 2 * C; p.Cg = C; p.k = k;
    p.cpt = ceil_div(C, GEMM_BK);
    fill_taps(p.tap_off, k, dilation, causal, false);
    p.mode = mode; p.residual = residual;
    p.p_drop = p_drop; p.seed_ptr = seed_ptr; p.salt = salt; p.drop_on_output = 0;
    return run_conv<true>(p, (cudaStream_t)stream, "convblock_fwd");
}

int dv3_conv1d_fwd(const float* x, const float* w_f, const float* bias, float* y, int B, int Cin, int Cout,
                   int T, int k, int dilation, int causal, int relu, void* stream) {
    DV3_REQUIRE(k >= 1 && k <= MAX_TAPS, "conv1d_fwd: kernel size %d not in [1,%d]", k, MAX_TAPS);
    DV3_REQUIRE((long long)B * (Cin > Cout ? Cin : Cout) * T < (1LL << 31),
                "conv1d_fwd: tensor of %lld elements too large for 32-bit indexing",
                (long long)B * (Cin > Cout ? Cin : Cout) * T);
    ConvParams p = {};
    p.x = x; p.w = w_f; p.bias = bias; p.y = y;
    p.B = B; p.Cin = Cin; p.T = T; p.N = B * T; p.Mtot = Cout; p.k = k; p.cpt = ceil_div(Cin, GEMM_BK);
    fill_taps(p.tap_off, k, dilation, causal, false);
    p.mode = relu ? 1 : 0;
    return run_conv<false>(p, (cudaStream_t)stream, "conv1d_fwd");
}

// dx = mask * conv_transpose(dab, w) + addend ; w_b is [k][M][Cin]
int dv3_conv1d_dgrad(const float* dab, const float* w_b, float* dx, int B, int M, int Cin, int T, int k,
                     int dilation, int causal, float p_drop, const unsigned long long* seed_ptr,
                     unsigned salt, int addmode, const float* e1, const float* e2, float alpha,
                     void* stream) {
    DV3_REQUIRE(k >= 1 && k <= MAX_TAPS, "conv1d_dgrad: kernel size %d not in [1,%d]", k, MAX_TAPS);
    DV3_REQUIRE(addmode >= 0 && addmode <= 2, "conv1d_dgrad: bad addmode");
    DV3_REQUIRE((long long)B * (M > Cin ? M : Cin) * T < (1LL << 31),
                "conv1d_dgrad: tensor of %lld elements too large for 32-bit indexing",
                (long long)B * (M > Cin ? M : Cin) * T);
    ConvParams p = {};
    p.x = dab; p.w = w_b; p.y = dx;
    p.B = B; p.Cin = M; p.T = T; p.N = B * T; p.Mtot = Cin; p.k = k; p.cpt = ceil_div(M, GEMM_BK);
    fill_taps(p.tap_off, k, dilation, causal, true);
    p.p_drop = p_drop; p.seed_ptr = seed_ptr; p.salt = salt; p.drop_on_output = 1;
    p.addmode = addmode; p.e1 = e1; p.e2 = e2; p.alpha = alpha;
    return run_conv<false>(p, (cudaStream_t)stream, "conv1d_dgrad");
}

// Number of split-K partials dv3_conv1d_wgrad will write for this problem (caller sizes the workspace).
int dv3_conv1d_wgrad_nsplit(int B, int M, int Cin, int T, int k) {
    const int tiles = ceil_div(M, GEMM_BM) * ceil_div(Cin, 64) * k;
    const int chunks = ceil_div(B * T, GEMM_BK);
    int want = ceil_div(4 * num_sms(), tiles);
    int maxs = chunks / 8 > 0 ? chunks / 8 : 1;           // at least 8 chunks (128 samples) per split
    if (want > maxs) want = maxs;
    if (want < 1) want = 1;
    const int cps = ceil_div(chunks, want);
    return ceil_div(chunks, cps);
}

// dw partials: [nsplit][numel(v)], element (m, ci, j) at (m%msplit)*s_m + (m/msplit)*s_mh + ci*s_n + j*s_j
int dv3_conv1d_wgrad(const float* dab, const float* x, float* dw_partials, long long split_stride, int B,
                     int M, int Cin, int T, int k, int dilation, int causal, float p_drop,
                     const unsigned long long* seed_ptr, unsigned salt, int msplit, int s_m, int s_mh,
                     int s_n, int s_j, void* stream) {
    DV3_REQUIRE(k >= 1 && k <= MAX_TAPS, "conv1d_wgrad: kernel size %d not in [1,%d]", k, MAX_TAPS);
    DV3_REQUIRE((long long)B * (M > Cin ? M : Cin) * T < (1LL << 31),
                "conv1d_wgrad: tensor of %lld elements too large for 32-bit indexing",
                (long long)B * (M > Cin ? M : Cin) * T);
    WgradParams p = {};
    p.dab = dab; p.x = x; p.dw = dw_partials; p.split_stride = (size_t)split_stride;
    p.B = B; p.M = M; p.Cin = Cin; p.T = T; p.N = B * T; p.k = k;
    p.nsplit = dv3_conv1d_wgrad_nsplit(B, M, Cin, T, k);
    p.chunks_per_split = ceil_div(ceil_div(p.N, GEMM_BK), p.nsplit);
    fill_taps(p.tap_off, k, dilation, causal, false);
    p.msplit = msplit; p.s_m = s_m; p.s_mh = s_mh; p.s_n = s_n; p.s_j = s_j;
    p.p_drop = p_drop; p.seed_ptr = seed_ptr; p.salt = salt;
    dim3 grid(ceil_div(Cin, 64), ceil_div(M, GEMM_BM), p.nsplit * k);
    return launch_gemm<WgradPolicy, 64>(p, grid, (cudaStream_t)stream, "conv1d_wgrad");
}

int dv3_convblock_gate_bwd(const float* dy, const float* a, const float* s, const float* x, float* dab,
                           float* dbias, int B, int C, int T, int mode, int residual, void* stream) {
    const int warps = B * C, threads = 256;
    launch_k(gate_bwd_kernel, ceil_div(warps * 32, threads), threads, 0, (cudaStream_t)stream, 
        dy, a, s, x, dab, dbias, B, C, T, mode, residual);
    return check_launch("convblock_gate_bwd");
}

int dv3_bias_act_bwd(const float* dy, const float* y, float* dyr, float* dbias, int B, int C, int T,
                     int relu, void* stream) {
    const int warps = B * C, threads = 256;
    launch_k(bias_act_bwd_kernel, ceil_div(warps * 32, threads), threads, 0, (cudaStream_t)stream, 
        dy, y, dyr, dbias, B, C, T, relu);
    return check_launch("bias_act_bwd");
}

}  // extern "C"
