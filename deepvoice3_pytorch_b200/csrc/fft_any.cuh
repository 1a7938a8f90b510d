// Mixed-radix FFT core of the general-geometry audio kernels (stft_any.cu, for every frame audio.check_geometry
// accepts): a shared-memory Stockham transform of length M = N/2 (radix-2/3/4/5 passes) and the real-packing
// split / merge between the packed complex transform and the N/2+1-bin half spectrum.  Written so that g++ compiles it
// too: tests/test_stft_geometry_host.py runs the passes "thread" by thread on the CPU against numpy.fft.
//
// Stockham pass with radix p after passes whose radices multiply to Ns (Ns = 1 for the first pass), butterfly
// j in [0, M/p), k = j mod Ns:
//     v[r] = in[j + r*M/p] * W_M^(k*r*M/(Ns*p)),   v <- DFT_p(v),   out[(j/Ns)*Ns*p + k + r*Ns] = v[r]
// Every pass reads one buffer and writes the other, so the passes need no index permutation and the output is in
// natural order.  Twiddle indices k*r*M/(Ns*p) stay below M.
//
// Table (fp32, built on the host in fp64 and rounded once: audio._geometry_table), 3N + 2 floats:
//     win[N]            w(i) = sqrt(hann(i + 1/2) * 2R/N), the analysis = synthesis window
//     tw [M]  (float2)  W_M^j = exp(-2 pi i j / M)
//     sp [M+1](float2)  W_N^k = exp(-2 pi i k / N)
// Real packing: z[n] = x[2n] + i x[2n+1], Z = FFT_M(z);  X[k] = E + W_N^k O with 2E = Z[k] + conj Z[M-k],
// 2O = -i (Z[k] - conj Z[M-k]) (Z[M] = Z[0]).  The inverse forms Z[k] = E + i conj(W_N^k) O from X and transforms
// conj Z forward: z = conj(FFT_M(conj Z)) / M.
#pragma once
#if defined(__CUDACC__)
#define FFTA_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#define FFTA_HD inline
#endif

namespace dv3 {
namespace fftany {

constexpr int MIN_N = 256, MAX_N = 4096, MAX_M = MAX_N / 2;

struct c2 { float x, y; };

// The passes in order: n4 radix-4 passes, then n2 (0 or 1) radix-2, then n3 radix-3 and n5 radix-5 passes.  Counts
// rather than an array of radices, so that a kernel indexes nothing at run time (no local-memory copy of the plan).
struct Plan {
    int M, n4, n2, n3, n5, npass;
    FFTA_HD int radix(int s) const { return s < n4 ? 4 : s < n4 + n2 ? 2 : s < n4 + n2 + n3 ? 3 : 5; }
};

// npass = 0 when M has a prime factor above 5
FFTA_HD Plan make_plan(int M) {
    Plan p{M, 0, 0, 0, 0, 0};
    int m = M;
    while (m % 4 == 0) { ++p.n4; m /= 4; }
    if (m % 2 == 0) { p.n2 = 1; m /= 2; }
    while (m % 3 == 0) { ++p.n3; m /= 3; }
    while (m % 5 == 0) { ++p.n5; m /= 5; }
    p.npass = m == 1 && M > 1 ? p.n4 + p.n2 + p.n3 + p.n5 : 0;
    return p;
}

FFTA_HD int tab_win(int) { return 0; }
FFTA_HD int tab_tw(int N) { return N; }          // float offsets into the table
FFTA_HD int tab_sp(int N) { return 2 * N; }
FFTA_HD int tab_floats(int N) { return 3 * N + 2; }

FFTA_HD c2 cadd(c2 a, c2 b) { return {a.x + b.x, a.y + b.y}; }
FFTA_HD c2 csub(c2 a, c2 b) { return {a.x - b.x, a.y - b.y}; }
FFTA_HD c2 cmul(c2 a, c2 b) { return {fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x)}; }
FFTA_HD c2 cmuli_neg(c2 a) { return {a.y, -a.x}; }              // -i * a

// in-place forward DFT of length P in {2, 3, 4, 5}
template <int P> FFTA_HD void dft(c2* v) {
    if constexpr (P == 2) {
        const c2 a = v[0], b = v[1];
        v[0] = cadd(a, b); v[1] = csub(a, b);
    } else if constexpr (P == 4) {
        const c2 s0 = cadd(v[0], v[2]), d0 = csub(v[0], v[2]), s1 = cadd(v[1], v[3]), d1 = csub(v[1], v[3]);
        v[0] = cadd(s0, s1); v[2] = csub(s0, s1);
        const c2 t = cmuli_neg(d1);
        v[1] = cadd(d0, t); v[3] = csub(d0, t);
    } else if constexpr (P == 3) {
        const float C = -0.5f, S = -0.86602540378443865f;        // exp(-2 pi i / 3)
        const c2 s = cadd(v[1], v[2]), d = csub(v[1], v[2]);
        const c2 a = {fmaf(C, s.x, v[0].x), fmaf(C, s.y, v[0].y)};
        const c2 b = {-S * d.y, S * d.x};                        // i*S*d
        v[0] = cadd(v[0], s); v[1] = cadd(a, b); v[2] = csub(a, b);
    } else {                                                     // p == 5
        const float C1 = 0.30901699437494742f, C2 = -0.80901699437494742f;
        const float S1 = -0.95105651629515357f, S2 = -0.58778525229247313f;     // sin(-2 pi / 5), sin(-4 pi / 5)
        const c2 s1 = cadd(v[1], v[4]), d1 = csub(v[1], v[4]), s2 = cadd(v[2], v[3]), d2 = csub(v[2], v[3]);
        const c2 a1 = {fmaf(C1, s1.x, fmaf(C2, s2.x, v[0].x)), fmaf(C1, s1.y, fmaf(C2, s2.y, v[0].y))};
        const c2 a2 = {fmaf(C2, s1.x, fmaf(C1, s2.x, v[0].x)), fmaf(C2, s1.y, fmaf(C1, s2.y, v[0].y))};
        const c2 b1 = {-fmaf(S1, d1.y, S2 * d2.y), fmaf(S1, d1.x, S2 * d2.x)};      // i*(S1 d1 + S2 d2)
        const c2 b2 = {-fmaf(S2, d1.y, -S1 * d2.y), fmaf(S2, d1.x, -S1 * d2.x)};    // i*(S2 d1 - S1 d2)
        v[0] = cadd(v[0], cadd(s1, s2));
        v[1] = cadd(a1, b1); v[4] = csub(a1, b1);
        v[2] = cadd(a2, b2); v[3] = csub(a2, b2);
    }
}

// one butterfly j of a pass (radix P, Ns, length M); load(i) gives in[i], out is the other buffer
template <int P, typename Load>
FFTA_HD void butterfly_p(const Load& load, c2* out, const c2* tw, int M, int Ns, int j) {
    c2 v[P];
    const int k = j % Ns, step = M / P, ts = M / (Ns * P);
#pragma unroll
    for (int r = 0; r < P; ++r) {
        v[r] = load(j + r * step);
        if (r && k) v[r] = cmul(v[r], tw[k * r * ts]);
    }
    dft<P>(v);
    const int o = (j / Ns) * Ns * P + k;
#pragma unroll
    for (int r = 0; r < P; ++r) out[o + r * Ns] = v[r];
}

// butterflies j0, j0 + stride, ... of one pass with radix p
template <typename Load>
FFTA_HD void fft_pass(const Load& load, c2* out, const c2* tw, int M, int p, int Ns, int j0, int stride) {
    const int nb = M / p;
    switch (p) {
        case 4: for (int j = j0; j < nb; j += stride) butterfly_p<4>(load, out, tw, M, Ns, j); break;
        case 2: for (int j = j0; j < nb; j += stride) butterfly_p<2>(load, out, tw, M, Ns, j); break;
        case 3: for (int j = j0; j < nb; j += stride) butterfly_p<3>(load, out, tw, M, Ns, j); break;
        default: for (int j = j0; j < nb; j += stride) butterfly_p<5>(load, out, tw, M, Ns, j); break;
    }
}

struct SmemLoad {
    const c2* a;
    FFTA_HD c2 operator()(int i) const { return a[i]; }
};

// half-spectrum bin k in [0, M] from the packed transform Z (natural order)
FFTA_HD c2 split_bin(const c2* Z, int M, int k, c2 w) {
    const c2 a = Z[k == M ? 0 : k], b = Z[k == 0 ? 0 : M - k];
    const c2 e = {0.5f * (a.x + b.x), 0.5f * (a.y - b.y)};
    const c2 o = {0.5f * (a.y + b.y), -0.5f * (a.x - b.x)};     // -i (a - conj b) / 2
    return cadd(e, cmul(w, o));
}

// conj of the packed inverse input Z[k], k in [0, M), from the half spectrum X (M+1 bins); w = W_N^k
FFTA_HD c2 merge_bin_conj(c2 a, c2 b, c2 w) {                    // a = X[k], b = X[M-k]
    const c2 e = {0.5f * (a.x + b.x), 0.5f * (a.y - b.y)};
    const c2 d = {0.5f * (a.x - b.x), 0.5f * (a.y + b.y)};      // (X[k] - conj X[M-k]) / 2
    const c2 o = cmul(d, c2{w.x, -w.y});                         // * conj(W_N^k)
    return {e.x - o.y, -(e.y + o.x)};                            // conj(E + i O)
}

}  // namespace fftany
}  // namespace dv3
