// CPU harness for csrc/fft_any.cuh: runs the Stockham passes butterfly by butterfly (a pass for all butterflies before
// the next = the barriers of the kernels), the real-packing split, and the inverse (merge, passes, conj / M).
// stdin: int32 N, float32 table[3N + 2] (audio._geometry_table), float32 frame x[N].
// stdout: float32 X[N/2 + 1] as (re, im) pairs = rfft(x), then float32 y[N] = irfft(X).  Built by
// tests/test_stft_geometry_host.py.
#include <cstdio>
#include <cstdint>
#include <vector>
#include "fft_any.cuh"
using namespace dv3::fftany;

template <typename Load>
static const c2* run(const Plan& pl, const Load& first, std::vector<c2>& a, std::vector<c2>& b, const c2* tw) {
    const int M = pl.M;
    fft_pass(first, a.data(), tw, M, pl.radix(0), 1, 0, 1);
    int Ns = pl.radix(0);
    c2 *pa = a.data(), *pb = b.data();
    for (int s = 1; s < pl.npass; ++s) {
        const int p = pl.radix(s);
        fft_pass(SmemLoad{pa}, pb, tw, M, p, Ns, 0, 1);
        Ns *= p;
        c2* t = pa; pa = pb; pb = t;
    }
    return pa;
}

int main() {
    int32_t N;
    if (fread(&N, 4, 1, stdin) != 1) return 2;
    std::vector<float> tab(tab_floats(N)), x(N);
    if (fread(tab.data(), 4, tab.size(), stdin) != tab.size()) return 2;
    if (fread(x.data(), 4, N, stdin) != (size_t)N) return 2;
    const int M = N / 2, K = M + 1;
    const Plan pl = make_plan(M);
    if (pl.npass == 0) return 3;
    const c2* tw = reinterpret_cast<const c2*>(tab.data() + tab_tw(N));
    const c2* sp = reinterpret_cast<const c2*>(tab.data() + tab_sp(N));
    c2 nan = {NAN, NAN};
    std::vector<c2> a(M, nan), b(M, nan);                  // NaN-poisoned: a read of an unwritten word shows
    struct Packed {
        const float* x;
        c2 operator()(int i) const { return {x[2 * i], x[2 * i + 1]}; }
    };
    const c2* Z = run(pl, Packed{x.data()}, a, b, tw);
    std::vector<c2> X(K);
    for (int k = 0; k < K; ++k) X[k] = split_bin(Z, M, k, sp[k]);
    fwrite(X.data(), 8, K, stdout);

    struct Merge {
        const c2* X; const c2* sp; int M;
        c2 operator()(int i) const { return merge_bin_conj(X[i], X[M - i], sp[i]); }
    };
    std::vector<c2> a2(M, nan), b2(M, nan);
    const c2* z = run(pl, Merge{X.data(), sp, M}, a2, b2, tw);
    std::vector<float> y(N);
    for (int n = 0; n < M; ++n) { y[2 * n] = z[n].x / M; y[2 * n + 1] = -z[n].y / M; }
    fwrite(y.data(), 4, N, stdout);
    return 0;
}
