// Per-warp 1024-point real STFT frame: the index arithmetic of stft.cu, written so that g++ can compile it too
// (tests/test_stft_core.py runs the stages lane by lane on the CPU and compares with numpy's rfft).
//
// One warp transforms one frame.  1024 real samples are packed as 512 complex points z[n] = x[2n] + i*x[2n+1];
// the 512-point transform is three radix-8 passes (512 = 8*8*8).  Every lane runs TWO butterflies per pass ("virtual
// threads" a and b) and keeps their data as PAIRS pr = (value of a, value of b): all arithmetic is pair-wise (two independent
// scalar instructions per pair, which keeps the issue of a lane dense).  The
// pairing of every pass is chosen so that the loads deliver pairs in adjacent registers (64/128-bit shared-memory
// accesses) with no register shuffling.  With n = 64*n2 + 8*n1 + n0 and k = k0 + 8*k1 + 64*k2:
//   pass 1  lane l: a,b = points t = 2l, 2l+1   A[k0]  = W512^(t*k0) * sum_n2 z[64*n2 + t]      * W8^(n2*k0)
//   pass 2  lane l = 4*k0 + m: a,b = n0 = 2m, 2m+1
//                                                 B[k1]  = W64^(n0*k1) * sum_n1 A[k0][8*n1 + n0]  * W8^(n1*k1)
//   pass 3  lane l = 4*k1 + u: a,b = k0 = 2u, 2u+1
//                                                 Z[k]   =               sum_n0 B[k0][k1][n0]     * W8^(n0*k2)
// Exchanges through the warp's work area (re / im planes of WORK floats, viewed as pairs):
//   exchange 1  pair (A[k0][2l], A[k0][2l+1]) at pair index 36*k0 + l     64-bit stores, 64-bit loads at 36*k0 + 4*n1 + m
//   exchange 2  B[k0][k1][n0] at float index 68*n0 + 8*k1 + k0            32-bit stores, 64-bit loads at pair 34*n0 + l
//   natural     pair (Z[2l + 64*k2], Z[2l + 1 + 64*k2]) at pair index l + 32*k2
// (row pitches 36 / 34 pairs make every warp-wide access conflict-free.)  The half spectrum follows from Z by the usual
// even/odd split, here four bins per step: k_a = lane + 64*j, k_b = k_a + 32 and their mirrors 512 - k.
#pragma once
#if defined(__CUDACC__)
#define STFT_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#define STFT_HD inline
#endif

namespace dv3 {
namespace stftc {

struct f2 { float x, y; };
struct alignas(16) f4 { float x, y, z, w; };
typedef f2 pr;                   // (virtual thread a, virtual thread b)

constexpr int WORK = 578;        // floats per plane (re / im) of a warp's work area; 2*WORK/4 is odd, see stft.cu
constexpr int PITCH1 = 36;       // exchange 1: pairs per k0 row
constexpr int PITCH2 = 34;       // exchange 2: pairs per n0 row

// ---- pair arithmetic: one instruction per pair on the device ----------------------------------------------------
#if defined(__CUDA_ARCH__)
// sm_90 has no packed f32x2 arithmetic: two scalar instructions per pair.  The _rn intrinsics keep nvcc from fusing a
// separate multiply and add into one FMA, so the device rounds exactly like the host build of this header.
__device__ __forceinline__ pr padd(pr a, pr b) { return {__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ pr psub(pr a, pr b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)}; }
__device__ __forceinline__ pr pmul(pr a, pr b) { return {__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ pr pfma(pr a, pr b, pr c) { return {__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ pr pfnma(pr a, pr b, pr c) { return {__fmaf_rn(-a.x, b.x, c.x), __fmaf_rn(-a.y, b.y, c.y)}; }
#else
STFT_HD pr padd(pr a, pr b) { return {a.x + b.x, a.y + b.y}; }
STFT_HD pr psub(pr a, pr b) { return {a.x - b.x, a.y - b.y}; }
STFT_HD pr pmul(pr a, pr b) { return {a.x * b.x, a.y * b.y}; }
STFT_HD pr pfma(pr a, pr b, pr c) { return {fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
STFT_HD pr pfnma(pr a, pr b, pr c) { return {fmaf(-a.x, b.x, c.x), fmaf(-a.y, b.y, c.y)}; }
#endif

// (r, i) <- (r, i) * (wx + i*wy), pair-wise
STFT_HD void cmulp(pr& r, pr& i, pr wx, pr wy) {
    const pr nr = pfnma(i, wy, pmul(r, wx));
    const pr ni = pfma(i, wx, pmul(r, wy));
    r = nr; i = ni;
}

// in-place 8-point forward DFT of two butterflies at once: a[k] <- sum_n a[n] * exp(-2*pi*i*n*k/8)
STFT_HD void radix8p(pr* r, pr* i) {
    const pr hh = {0.70710678118654752f, 0.70710678118654752f};
    const pr b0r = padd(r[0], r[4]), b0i = padd(i[0], i[4]), b1r = psub(r[0], r[4]), b1i = psub(i[0], i[4]);
    const pr b2r = padd(r[2], r[6]), b2i = padd(i[2], i[6]), b3r = psub(r[2], r[6]), b3i = psub(i[2], i[6]);
    const pr b4r = padd(r[1], r[5]), b4i = padd(i[1], i[5]), b5r = psub(r[1], r[5]), b5i = psub(i[1], i[5]);
    const pr b6r = padd(r[3], r[7]), b6i = padd(i[3], i[7]), b7r = psub(r[3], r[7]), b7i = psub(i[3], i[7]);
    const pr e0r = padd(b0r, b2r), e0i = padd(b0i, b2i), e2r = psub(b0r, b2r), e2i = psub(b0i, b2i);
    const pr e1r = padd(b1r, b3i), e1i = psub(b1i, b3r), e3r = psub(b1r, b3i), e3i = padd(b1i, b3r);   // b1 -/+ i*b3
    const pr o0r = padd(b4r, b6r), o0i = padd(b4i, b6i), o2r = psub(b4r, b6r), o2i = psub(b4i, b6i);
    const pr o1r = padd(b5r, b7i), o1i = psub(b5i, b7r), o3r = psub(b5r, b7i), o3i = padd(b5i, b7r);
    const pr s1 = padd(o1r, o1i), d1 = psub(o1i, o1r);       // (1-i)/sqrt2 * o1 = h*(s1, d1)
    const pr s3 = padd(o3r, o3i), d3 = psub(o3i, o3r);       // (-1-i)/sqrt2 * o3 = h*(d3, -s3)
    r[0] = padd(e0r, o0r); i[0] = padd(e0i, o0i); r[4] = psub(e0r, o0r); i[4] = psub(e0i, o0i);
    r[1] = pfma(s1, hh, e1r); i[1] = pfma(d1, hh, e1i); r[5] = pfnma(s1, hh, e1r); i[5] = pfnma(d1, hh, e1i);
    r[2] = padd(e2r, o2i); i[2] = psub(e2i, o2r); r[6] = psub(e2r, o2i); i[6] = padd(e2i, o2r);       // -i * o2
    r[3] = pfma(d3, hh, e3r); i[3] = pfnma(s3, hh, e3i); r[7] = pfnma(d3, hh, e3r); i[7] = pfma(s3, hh, e3i);
}

// ---- tables (built once by stft.cu's init kernel, and by the CPU harness) ----------------------------------------
// Only what cannot be formed cheaply in registers is tabulated (the kernel is bound by shared-memory wavefronts, not by
// arithmetic): the rest follows by angle addition / products of the tabulated factors.
//   win [l], win[32 + l]  = S*sin(a_j), S*cos(a_j) as (j=0, j=2, j=1, j=3); a_j = pi*(2*(4l+j)+1)/2048, S = sqrt(1/2):
//                           the frame window is w[i] = S*sin(pi*(2i+1)/2048) (sqrt-Hann * sqrt(2*hop/N)), and sample
//                           i = 128*n2 + 4l + j sits n2*pi/8 further on: w = S*sin(a_j)*cos(n2*pi/8) + S*cos(a_j)*sin(n2*pi/8)
//   tw1 [g*32 + l]        = (cos a, cos b, sin a, sin b) of W512^(t*k0),  t = 2l, 2l+1, k0 = 1 (g=0), 4 (g=1);
//                           k0 = 2, 3, 5, 6, 7 are products of these two (depth <= 3)
//   tw2 [g*4 + m]         = (cos a, cos b, sin a, sin b) of W64^(n0*k1),  n0 = 2m, 2m+1, k1 = 1, 4; the rest likewise
//   wsp [l]               = (cos a, cos b, sin a, sin b) of W1024^k,      k = l, l + 32; k + 64j = one rotation by W16^j
constexpr int TAB_WIN = 0, TAB_TW1 = 64, TAB_TW2 = TAB_TW1 + 64, TAB_WSP = TAB_TW2 + 8, TAB_N = TAB_WSP + 32;

// cos / sin of -2*pi*num/den in double precision (the init kernel and the CPU harness share table_entry)
STFT_HD void cs_(int num, int den, float& c, float& s) {
#if defined(__CUDA_ARCH__)
    double sd, cd; sincospi(-2.0 * (double)num / (double)den, &sd, &cd);
#else
    const double a = -2.0 * 3.14159265358979323846 * (double)num / (double)den, sd = std::sin(a), cd = std::cos(a);
#endif
    c = (float)cd; s = (float)sd;
}
// S*sin / S*cos of pi*(2i+1)/2048, S = sqrt(1/2)
STFT_HD void wsc_(int i, float& s, float& c) {
#if defined(__CUDA_ARCH__)
    double sd, cd; sincospi((2.0 * i + 1.0) / 2048.0, &sd, &cd);
#else
    const double a = 3.14159265358979323846 * (2.0 * i + 1.0) / 2048.0, sd = std::sin(a), cd = std::cos(a);
#endif
    s = (float)(0.70710678118654752440 * sd); c = (float)(0.70710678118654752440 * cd);
}
STFT_HD f4 table_entry(int idx) {
    f4 r;
    if (idx < TAB_TW1) {
        const int l = idx & 31;
        float s[4], c[4];
        for (int j = 0; j < 4; ++j) wsc_(4 * l + j, s[j], c[j]);
        if (idx < 32) { r.x = s[0]; r.y = s[2]; r.z = s[1]; r.w = s[3]; }
        else { r.x = c[0]; r.y = c[2]; r.z = c[1]; r.w = c[3]; }
    } else if (idx < TAB_TW2) {
        const int j = idx - TAB_TW1, k0 = (j >> 5) ? 4 : 1, l = j & 31;
        cs_(2 * l * k0, 512, r.x, r.z); cs_((2 * l + 1) * k0, 512, r.y, r.w);
    } else if (idx < TAB_WSP) {
        const int j = idx - TAB_TW2, k1 = (j >> 2) ? 4 : 1, m = j & 3;
        cs_(2 * m * k1, 64, r.x, r.z); cs_((2 * m + 1) * k1, 64, r.y, r.w);
    } else {
        const int l = idx - TAB_WSP;
        cs_(l, 1024, r.x, r.z); cs_(l + 32, 1024, r.y, r.w);
    }
    return r;
}

// twiddle pairs: c = a * b (complex, pair-wise)
struct tw { pr x, y; };
STFT_HD tw twmul(tw a, tw b) { return {pfnma(a.y, b.y, pmul(a.x, b.x)), pfma(a.y, b.x, pmul(a.x, b.y))}; }
// v[1..7] *= w^k given w^1 and w^4 (products of depth <= 3 instead of five more table loads)
STFT_HD void twiddle7(pr* vr, pr* vi, f4 t1, f4 t4) {
    const tw w1 = {{t1.x, t1.y}, {t1.z, t1.w}}, w4 = {{t4.x, t4.y}, {t4.z, t4.w}};
    const tw w2 = twmul(w1, w1), w3 = twmul(w2, w1);
    cmulp(vr[1], vi[1], w1.x, w1.y);
    cmulp(vr[2], vi[2], w2.x, w2.y);
    cmulp(vr[3], vi[3], w3.x, w3.y);
    cmulp(vr[4], vi[4], w4.x, w4.y);
    const tw w5 = twmul(w4, w1), w6 = twmul(w4, w2), w7 = twmul(w4, w3);
    cmulp(vr[5], vi[5], w5.x, w5.y);
    cmulp(vr[6], vi[6], w6.x, w6.y);
    cmulp(vr[7], vi[7], w7.x, w7.y);
}
// W1024^(k + 64j) = W1024^k * W16^j, j = 1..3 (compile-time constant rotations of the tabulated j = 0 factors)
STFT_HD f4 rot16(f4 w, int j) {
    const float C1 = 0.92387953251128674f, S1 = 0.38268343236508977f, H = 0.70710678118654752f;
    const float cx = j == 1 ? C1 : (j == 2 ? H : S1), cy = j == 1 ? -S1 : (j == 2 ? -H : -C1);
    if (j == 0) return w;
    const tw r = twmul(tw{{w.x, w.y}, {w.z, w.w}}, tw{{cx, cx}, {cy, cy}});
    return f4{r.x.x, r.x.y, r.y.x, r.y.y};
}

// Sample source of pass 1: the staged fp32 waveform itself.  stft.cu adds sources that convert staged int16 PCM and
// rescale as the samples are read; a source has load4(i) = samples i..i+3 (i a multiple of 4) and load1(i) = sample i.
struct RawF32 {
    const float* x;
    STFT_HD f4 load4(int i) const { return *reinterpret_cast<const f4*>(x + i); }
    STFT_HD float load1(int i) const { return x[i]; }
};

// pass 1: x -> sample 0 of the frame window in the RAW waveform (16-byte aligned, x[-1] readable; samples outside the
// clip are 0); pre-emphasis e[i] = x[i] - c*x[i-1] (audio.py:21-23) is applied on the fly.  TAIL: e[i] = 0 for
// i >= lim (the zero padding after the clip's last sample starts inside this frame).
template <bool TAIL, typename Src>
STFT_HD void pass1_src(int lane, const Src& x, float c, int lim, const f4* win, const f4* tw1, pr (&vr)[8],
                       pr (&vi)[8]) {
    const f4 ws = win[lane], wc = win[32 + lane];
    const pr sA = {ws.x, ws.y}, sB = {ws.z, ws.w}, cA = {wc.x, wc.y}, cB = {wc.z, wc.w};
    const float C1 = 0.92387953251128674f, S1 = 0.38268343236508977f, H = 0.70710678118654752f;
    const float CB[8] = {1.f, C1, H, S1, 0.f, -S1, -H, -C1}, SB[8] = {0.f, S1, H, C1, 1.f, C1, H, S1};   // n2*pi/8
#pragma unroll
    for (int n2 = 0; n2 < 8; ++n2) {
        const int i0 = 128 * n2 + 4 * lane;                  // first of the 4 samples of points a, b
        const f4 s = x.load4(i0);
#if defined(__CUDA_ARCH__)
        // x[i0 - 1] is the previous lane's last sample: a shuffle instead of a 4-way conflicting load
        float xm = __shfl_up_sync(0xffffffffu, s.w, 1);
        if (lane == 0) xm = x.load1(i0 - 1);
#else
        const float xm = x.load1(i0 - 1);
#endif
        float e0 = fmaf(-c, xm, s.x), e1 = fmaf(-c, s.x, s.y), e2 = fmaf(-c, s.y, s.z), e3 = fmaf(-c, s.z, s.w);
        if (TAIL) {
            if (i0 >= lim) e0 = 0.f;
            if (i0 + 1 >= lim) e1 = 0.f;
            if (i0 + 2 >= lim) e2 = 0.f;
            if (i0 + 3 >= lim) e3 = 0.f;
        }
        pr wA, wB;                                           // window at samples (i0, i0+2) and (i0+1, i0+3)
        if (n2 == 0) { wA = sA; wB = sB; }
        else if (n2 == 4) { wA = cA; wB = cB; }
        else {
            const pr cb = {CB[n2], CB[n2]}, sb = {SB[n2], SB[n2]};
            wA = pfma(cA, sb, pmul(sA, cb));
            wB = pfma(cB, sb, pmul(sB, cb));
        }
        vr[n2] = pmul(pr{e0, e2}, wA);
        vi[n2] = pmul(pr{e1, e3}, wB);
    }
    radix8p(vr, vi);
    twiddle7(vr, vi, tw1[lane], tw1[32 + lane]);
}
template <bool TAIL>
STFT_HD void pass1(int lane, const float* x, float c, int lim, const f4* win, const f4* tw1, pr (&vr)[8], pr (&vi)[8]) {
    pass1_src<TAIL>(lane, RawF32{x}, c, lim, win, tw1, vr, vi);
}
STFT_HD void store1(int lane, const pr (&vr)[8], const pr (&vi)[8], float* re, float* im) {
    f2* re2 = reinterpret_cast<f2*>(re);
    f2* im2 = reinterpret_cast<f2*>(im);
#pragma unroll
    for (int k0 = 0; k0 < 8; ++k0) {
        re2[PITCH1 * k0 + lane] = vr[k0];
        im2[PITCH1 * k0 + lane] = vi[k0];
    }
}
STFT_HD void pass2(int lane, const float* re, const float* im, const f4* tw2, pr (&vr)[8], pr (&vi)[8]) {
    const f2* re2 = reinterpret_cast<const f2*>(re);
    const f2* im2 = reinterpret_cast<const f2*>(im);
    const int k0 = lane >> 2, m = lane & 3;
#pragma unroll
    for (int n1 = 0; n1 < 8; ++n1) {
        vr[n1] = re2[PITCH1 * k0 + 4 * n1 + m];
        vi[n1] = im2[PITCH1 * k0 + 4 * n1 + m];
    }
    radix8p(vr, vi);
    twiddle7(vr, vi, tw2[m], tw2[4 + m]);
}
STFT_HD void store2(int lane, const pr (&vr)[8], const pr (&vi)[8], float* re, float* im) {
    const int k0 = lane >> 2, m = lane & 3;
    const int base = 2 * PITCH2 * (2 * m) + k0;              // float index of (n0 = 2m, k1 = 0, k0)
#pragma unroll
    for (int k1 = 0; k1 < 8; ++k1) {
        re[base + 8 * k1] = vr[k1].x;
        im[base + 8 * k1] = vi[k1].x;
        re[base + 2 * PITCH2 + 8 * k1] = vr[k1].y;
        im[base + 2 * PITCH2 + 8 * k1] = vi[k1].y;
    }
}
STFT_HD void pass3(int lane, const float* re, const float* im, pr (&vr)[8], pr (&vi)[8]) {
    const f2* re2 = reinterpret_cast<const f2*>(re);
    const f2* im2 = reinterpret_cast<const f2*>(im);
#pragma unroll
    for (int n0 = 0; n0 < 8; ++n0) {
        vr[n0] = re2[PITCH2 * n0 + lane];                    // pair (k0 = 2u, 2u+1) of (k1 = lane>>2, u = lane&3)
        vi[n0] = im2[PITCH2 * n0 + lane];
    }
    radix8p(vr, vi);
}
STFT_HD void store3(int lane, const pr (&vr)[8], const pr (&vi)[8], float* re, float* im) {     // natural order Z[k]
    f2* re2 = reinterpret_cast<f2*>(re);
    f2* im2 = reinterpret_cast<f2*>(im);
#pragma unroll
    for (int k2 = 0; k2 < 8; ++k2) {
        re2[lane + 32 * k2] = vr[k2];
        im2[lane + 32 * k2] = vi[k2];
    }
}
// bins k_a = lane + 64j, k_b = k_a + 32 (0 <= k < 256) and their mirrors 512 - k from Z[k], Z[512-k]; w = W1024^k.
// Returns p_lo = (|2X[k_a]|^2, |2X[k_b]|^2) and p_hi = (|2X[512-k_a]|^2, |2X[512-k_b]|^2):
//   2E = Z[k] + conj(Z[512-k]),  2O = -i*(Z[k] - conj(Z[512-k])),  X[k] = E + w*O,  X[512-k] = conj(E - w*O)
// (k = 0 pairs Z[0] with itself and yields bins 0 and 512; bin 256 is split_nyquist's.)
STFT_HD void split4(int ka, const float* re, const float* im, f4 w, pr& p_lo, pr& p_hi) {
    const int kb = ka + 32, ma = (512 - ka) & 511, mb = 512 - kb;
    const pr ar = {re[ka], re[kb]}, ai = {im[ka], im[kb]}, br = {re[ma], re[mb]}, bn = {im[ma], im[mb]};
    const pr er = padd(ar, br), ei = psub(ai, bn), dr = psub(ar, br), di = padd(ai, bn);
    const pr wx = {w.x, w.y}, wy = {w.z, w.w};
    const pr p = pfma(wx, di, pmul(wy, dr));                 // Re(w * 2O),  2O = (di, -dr)
    const pr q = pfnma(wx, dr, pmul(wy, di));                // Im(w * 2O)
    const pr xr = padd(er, p), xi = padd(ei, q), yr = psub(er, p), yi = psub(ei, q);
    p_lo = pfma(xr, xr, pmul(xi, xi));
    p_hi = pfma(yr, yr, pmul(yi, yi));
}
// |2X[256]|^2 = 4*|Z[256]|^2   (E = Re Z, O = Im Z, w = -i)
STFT_HD float split_nyquist(const float* re, const float* im) { return 4.f * (re[256] * re[256] + im[256] * im[256]); }

}  // namespace stftc
}  // namespace dv3
