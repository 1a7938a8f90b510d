// Batched fp32 GEMM on the shared CUDA-core mainloop -- the contractions of the attention layer
// (reference deepvoice3.py:143 bmm(q,k), :167 bmm(p,v) and their gradients) in exact-fp32 mode.
//   C[b][m][n] = alpha * sum_k A_b(m,k) * B_b(k,n)  (+ C if accumulate)
// Operand element addressing is fully strided so that no operand ever needs a transpose in HBM:
//   A_b(m,k) = A[b*sAb + m*sAm + k*sAk],  B_b(k,n) = B[b*sBb + k*sBk + n*sBn],  C row-major (ldc).
// An operand whose unit stride is along M (resp. N) uses the "direct" tile map, one whose unit stride
// is along K uses the "transposed" map (see gemm_simt.cuh); both are coalesced.
#include "gemm_simt.cuh"
#include <type_traits>

namespace dv3 {

struct BgemmParams {
    const float* A; const float* B; float* C;
    long long sAb, sAm, sAk, sBb, sBk, sBn, sCb;
    int M, N, K, ldc;
    float alpha;
    int accumulate;
    const long long* alpha_ts;   // non-null: alpha = context_scale(*alpha_ts), read from device memory
};

template <bool A_KMAJOR, bool B_KMAJOR>
struct BgemmPolicy {
    using Params = BgemmParams;

    template <int W, bool KMAJOR>
    struct Load {
        using Map = typename std::conditional<KMAJOR, TransMap<W>, DirectMap<W>>::type;
        static constexpr int N = Map::N;
        Map map;
        const float* base;
        long long s_row, s_k;
        int row0, rows, K;
        __device__ Load(const float* ptr, long long sb, long long sr, long long sk, int tile, int nrows, int K_,
                        int z, int tid)
            : map(tid), base(ptr + (size_t)z * sb), s_row(sr), s_k(sk), row0(tile * W), rows(nrows), K(K_) {}
        __device__ void fetch(int chunk, float* r) const {
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const int row = row0 + map.row(i), k = chunk * GEMM_BK + map.kk(i);
                r[i] = (row < rows && k < K) ? __ldg(&base[row * s_row + k * s_k]) : 0.f;
            }
        }
        __device__ void store(float* S, const float* r) const { tile_store<W>(S, map, r); }
    };

    struct ALoad : Load<GEMM_BM, A_KMAJOR> {
        __device__ ALoad(const Params& p, int m_tile, int z, int tid)
            : Load<GEMM_BM, A_KMAJOR>(p.A, p.sAb, p.sAm, p.sAk, m_tile, p.M, p.K, z, tid) {}
    };
    template <int BN>
    struct BLoad : Load<BN, B_KMAJOR> {
        __device__ BLoad(const Params& p, int n_tile, int z, int tid)
            : Load<BN, B_KMAJOR>(p.B, p.sBb, p.sBn, p.sBk, n_tile, p.N, p.K, z, tid) {}
    };

    __device__ static int num_chunks(const Params& p, int) { return (p.K + GEMM_BK - 1) / GEMM_BK; }

    template <int BN>
    __device__ static void epilogue(const Params& p, const Acc<BN>& acc, int m_tile, int n_tile, int z, int tx,
                                    int ty) {
        float* C = p.C + (size_t)z * p.sCb;
        const float alpha = p.alpha_ts ? context_scale(*p.alpha_ts) : p.alpha;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m_tile * GEMM_BM + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
            if (m >= p.M) continue;
#pragma unroll
            for (int q = 0; q < Acc<BN>::NC; ++q) {
                const int n = n_tile * BN + (q >> 2) * 64 + tx * 4 + (q & 3);
                if (n >= p.N) continue;
                float* dst = &C[(size_t)m * p.ldc + n];
                const float v = alpha * acc.v[i][q];
                *dst = p.accumulate ? (*dst + v) : v;
            }
        }
    }
};

template <bool AK, bool BK_>
static int launch_bgemm(const BgemmParams& p, int batch, cudaStream_t st) {
    using P = BgemmPolicy<AK, BK_>;
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(gemm_simt_kernel<P, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             gemm_smem_bytes<64>());
        configured = true;
    }
    dim3 grid(ceil_div(p.N, 64), ceil_div(p.M, GEMM_BM), batch);
    launch_k(gemm_simt_kernel<P, 64>, grid, GEMM_THREADS, gemm_smem_bytes<64>(), st, p);
    return check_launch("bgemm");
}

}  // namespace dv3

using namespace dv3;

static int bgemm(const float* A, long long sAb, long long sAm, long long sAk, const float* B, long long sBb,
                 long long sBk, long long sBn, float* C, long long sCb, int ldc, int batch, int M, int N, int K,
                 float alpha, const long long* alpha_ts, int accumulate, void* stream) {
    DV3_REQUIRE(batch >= 1 && batch <= 65535, "bgemm: batch %d out of range", batch);
    DV3_REQUIRE(sAm == 1 || sAk == 1, "bgemm: A needs unit stride along M or K");
    DV3_REQUIRE(sBn == 1 || sBk == 1, "bgemm: B needs unit stride along N or K");
    BgemmParams p = {A, B, C, sAb, sAm, sAk, sBb, sBk, sBn, sCb, M, N, K, ldc, alpha, accumulate, alpha_ts};
    cudaStream_t st = (cudaStream_t)stream;
    const bool ak = (sAm != 1), bk = (sBn != 1);
    if (ak && bk) return launch_bgemm<true, true>(p, batch, st);
    if (ak) return launch_bgemm<true, false>(p, batch, st);
    if (bk) return launch_bgemm<false, true>(p, batch, st);
    return launch_bgemm<false, false>(p, batch, st);
}

extern "C" int dv3_bgemm(const float* A, long long sAb, long long sAm, long long sAk, const float* B,
                         long long sBb, long long sBk, long long sBn, float* C, long long sCb, int ldc,
                         int batch, int M, int N, int K, float alpha, int accumulate, void* stream) {
    return bgemm(A, sAb, sAm, sAk, B, sBb, sBk, sBn, C, sCb, ldc, batch, M, N, K, alpha, nullptr, accumulate, stream);
}

// alpha = Ts*sqrt(1/Ts) (the attention context scale) of a key count read from device memory
extern "C" int dv3_bgemm_ctx_scale(const float* A, long long sAb, long long sAm, long long sAk, const float* B,
                                   long long sBb, long long sBk, long long sBn, float* C, long long sCb, int ldc,
                                   int batch, int M, int N, int K, const long long* ts_log, int accumulate,
                                   void* stream) {
    DV3_REQUIRE(ts_log != nullptr, "bgemm_ctx_scale: ts_log is NULL");
    return bgemm(A, sAb, sAm, sAk, B, sBb, sBk, sBn, C, sCb, ldc, batch, M, N, K, 0.f, ts_log, accumulate, stream);
}
