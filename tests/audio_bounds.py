"""TEST INFRASTRUCTURE ONLY.  Elementwise error bounds for the audio kernels (csrc/stft.cu + stft_core.cuh, the
1024 / 256 front end; csrc/stft_any.cu + fft_any.cuh, the front end at every other frame and the complex STFT and
inverse STFT at every frame; csrc/istft.cu, dB -> amplitude and de-emphasis) against the fp64 oracles of
oracle/audio_oracle.py and tests/stft_geometry_oracle.py.  The reference values come from those oracles; this module adds the bounds.

Error model.  u = 2^-24 (unit roundoff of fp32).  Every bound is first order in u; the sums are scaled by
(1 + 2^-10) for the second-order terms (below (c u)^2 relative for the c of this file).  Errors of complex values are
measured in modulus.  The rules, each a rounding of the kernel's own code:
  * a complex add / sub rounds each component once: |d| <= u |a +- b| <= u (|a| + |b|); -a, conj a, +-i a are exact;
  * a complex product with two roundings per component (cmul, cmulp, twmul, split4's p / q, with or without FMA
    contraction): |d| <= 2 sqrt2 u |a| |t|  (CMUL);
  * a twiddle or split factor t with |t_hat - t| <= tau u: fp32 table entries rounded once from fp64 (audio._geometry_table,
    stft_core.cuh table_entry) have tau = 1; a product of two factors has tau_a + tau_b + CMUL.
  * A pass of the FFT maps values whose moduli sum, over the inputs that reach one output, to S; its outputs carry an
    error <= c_pass u S, with c_pass = D_p + tau + CMUL: D_p for the radix-p DFT (below), tau + CMUL for the twiddle
    multiply on either side of it.  Every intermediate value of a decimation FFT is a unit-modulus combination of a
    disjoint subset of the inputs, and reaches each output through unit-modulus coefficients; so the pass errors add,
    and the packed transform Z of z[n] = x[2n] + i x[2n+1] has |Z_hat_k - Z_k| <= c_Z u sum|x|, c_Z = sum c_pass.
        D_2 = 1 (one add);  D_4 = 2 (two add levels);
        D_8 = 5 (radix8p: three add levels; the odd rotation by (1 -+ i)/sqrt2 = h (s, d) adds the rounding of s, d
              (sqrt2 u |o|, times h) and of the constant h (u));
        D_3 = 5 (s, d: u; a = fma(C, s, v0): u (|v0| + |s| / 2); b = S d with S rounded: 2 u |S| |d|; a +- b: u; the
              propagated errors of s, d times |C| + |S| = 1.37: 1.37 + 0.5 + 1.73 + 1.37 < 5 per unit of sum|v|);
        D_5 = 10 (s1, d1, s2, d2: u, propagated with |C1| + |S1| and |C2| + |S2| < 1.4; four rounded constants < 1.4;
              the nested fmas and products of a1, b1 < 2.8 + 1.4; the final add < 2.8: < 10 per unit of sum|v|).
  * The split X_k = E + W_N^k O (2E = Z_k + conj Z_{M-k}, 2O = -i (Z_k - conj Z_{M-k})) has coefficients of modulus
    <= 1 on Z_k and Z_{M-k}, so it doubles the transform error, and rounds E, O (u (|a| + |b|) / 2 each), the product
    ((tau + CMUL) u (|a| + |b|) / 2) and the sum (u (|a| + |b|)); with |a| + |b| <= 2 sum|x|:
        c_fft = 2 c_Z + c_split,  c_split = 4 + tau + CMUL.
    The inverse merges the half spectrum into Z the same way (merge_bin_conj, istft_any_kernel), then runs the forward
    passes on conj Z:  |z_hat_n - z_n| <= (2 c_Z + c_split) u sum_k |X_k|   (sum|Z| <= 2 sum|X|).
  Per kernel (passes from make_plan, or the fixed plan of the 1024-point front end):
    stft1024   stft_core.cuh: 3 radix-8 passes, the first two followed by twiddle7 (tau up to 12.5 for w^7 = w^4 w^2 w^1
               as products of the tabulated w^1, w^4), split4 with W1024^k rotated by a rounded W16^j (tau = 2 + CMUL);
    any        fft_any.cuh: make_plan's radix-4 / 2 / 3 / 5 passes, table twiddles (tau = 1).

Input stage.  The kernels' input is reproduced exactly: int16 PCM x 2^-15, and with rescaling rn(rn(x / peak) * gain)
(numpy float32 division and product are correctly rounded like __fdiv_rn / __fmul_rn), peak = max|x[:len]|.
Pre-emphasis is one fmaf with the fp32 coefficient: |e_hat_n - e_n| <= u (|x_n| + c |x_{n-1}|) + |c_f32 - c| |x_{n-1}|
against e_n = x_n - c x_{n-1} with c = 0.97 in fp64.  Window: w_hat = w (1 + u) for the fp32 tables of fft_any.cuh;
stft_core.cuh builds w = S sin(a + b) = rn(rn(sA cb) + cA sb) from the tabulated sA = rn(S sin a), cA = rn(S cos a)
and the rounded constants cb, sb = cos b, sin b: |dw| <= u (3 |S sin a cos b| + 2 |S cos a sin b| + |w|) (exact table
entries at n2 = 0, 4).  The product e w is rounded (u).  An
input error reaches every bin with a coefficient of modulus 1, so the frame bound is
    B_f = c_fft u sum_n |w_n e_n| + sum_n (w_n de_n + dw_n |e_n| + u w_n |e_n|).

Magnitude and dB.  |X_hat| lies in [|X| - B, |X| + B], widened by the magnitude's own rounding: p4 = |2X|^2 by one
fma and a product (|X| relative u), then 0.5 sqrt.approx (stft1024 mel magnitudes), or sqrtf (correctly rounded,
stft_any: 2u).  Both ends go through the monotone map clip((20 log10(max(min_level, v)) - ref_db - min_db) / -min_db,
0, 1) in fp64 and are widened by the evaluation error of sat(fmaf(c2, log2(.), c0)): the log2 error (lg2.approx.ftz.f32:
absolute error 2^-22 per the PTX ISA; log2f: 1 ulp), the rounding of the fp32 constants c2, c0 and of the fmaf.
PTX ISA bounds sqrt.approx.f32 at a relative error of 2^-23; the bounds take 2^-22 for it.  The linear row of stft1024
takes lg2 of p4 = 4 |X|^2 with the constants c2 / 2 and c0 - c2.
Mel: the reference is sum_k B_jk |X_k| with the spec's own fp32 basis; the kernel's fmaf chains over the n non-zero
weights add at most gamma_n = n u / (1 - n u) relative, so the mel value lies in
[sum_k B_jk mag_lo_k (1 - gamma_n), sum_k B_jk mag_hi_k (1 + gamma_n)], and the dB map follows as above.

Magnitude projection (Griffin-Lim step) got = mag X_hat / |X_hat| (rounded: sqrt of the rounded |X_hat|^2, 2u; the
quotient and product, 2u): where |X| > 2B, |got - mag X / |X|| <= mag (2B / (|X| - B) + 5u); elsewhere only
||got| - mag| <= 5u mag is required, and X_hat == 0 gives (mag, 0).

Inverse STFT.  The kernels fold the imaginary parts of bins 0 and N/2 into the waveform, where numpy's irfft drops
them: ``packed_irfft`` restates the kernels' inverse in fp64 (Z_k = E_k + i conj(W_N^k) O_k, z = ifft_M(Z), x[2n] =
Re z_n, x[2n+1] = Im z_n).  Per frame |x_hat_n - x_n| <= c_fft u sum_k |X_k| / M; the scaling by 1/M (exact for a
power of two, else u) and the window (u + dw) follow; the Q overlapping frames are summed in launch order into a zeroed
buffer: Q u sum |w x| more.

dB -> amplitude (spec_to_amp): db = fmaf(v, 100, -100) + 20 (two roundings), t = db * 0.05f (the rounded constant and
the product), powf(10, t) and powf(., power) within 4 ulp each (CUDA C++ Programming Guide): relative error
power (ln10 |dt| + 8u) + 8u + |power_f32 - power| |ln amp|.
De-emphasis y_n = fmaf(c_f32, y_{n-1}, x_n) against Y_n = x_n + c Y_{n-1} in fp64:
E_n <= c_f32 E_{n-1} + |c_f32 - c| A_{n-1} + u A_n, with A_n = |x_n| + c A_{n-1} (recurrences on absolute values).
"""
import numpy as np
from scipy.signal import lfilter

from oracle import audio_oracle as A

U = 2.0 ** -24
CMUL = 2.0 * np.sqrt(2.0)
SECOND_ORDER = 1.0 + 2.0 ** -10
LG2_APPROX_ABS = 2.0 ** -22          # PTX ISA, lg2.approx.f32: maximum absolute error
SQRT_APPROX_REL = 2.0 ** -22         # PTX ISA, sqrt.approx.f32: 2^-23 relative; taken at twice that
ULP = 2.0 * U                        # one ulp of an fp32 value, relative to the value (at most)
POWF_ULP, LOG2F_ULP = 4, 1
D = {2: 1.0, 3: 5.0, 4: 2.0, 5: 10.0, 8: 5.0}
TAU_TAB = 1.0
KERNELS = ("stft1024", "any")


def plan(M):
    """fft_any.cuh make_plan: the radices in pass order."""
    r, m = [], M
    while m % 4 == 0:
        r.append(4); m //= 4
    if m % 2 == 0:
        r.append(2); m //= 2
    for p in (3, 5):
        while m % p == 0:
            r.append(p); m //= p
    assert m == 1
    return r


def _tw_product(ta, tb):
    return ta + tb + CMUL


def c_fft(kernel, N=1024):
    """The constant of |X_hat_k - X_k| <= c_fft u sum|x| (and of the inverse per sum|X|), from the kernel's passes."""
    if kernel == "stft1024":
        t1 = t4 = TAU_TAB
        t2 = _tw_product(t1, t1); t3 = _tw_product(t2, t1)
        tau7 = max(t1, t2, t3, t4, _tw_product(t4, t1), _tw_product(t4, t2), _tw_product(t4, t3))
        c_z = 2 * (D[8] + tau7 + CMUL) + D[8]
        tau_split = TAU_TAB + TAU_TAB + CMUL          # tabulated W1024^k times a rounded W16^j (rot16)
    elif kernel == "any":
        c_z = sum(D[p] + TAU_TAB + CMUL for p in plan(N // 2))
        tau_split = TAU_TAB
    else:
        raise ValueError(kernel)
    return 2 * c_z + 4 + tau_split + CMUL


def window_error(kernel, N, R):
    """(w, dw): the fp64 window and the bound on |w_hat - w| per sample of the frame."""
    w = A.lws_window(N, R)
    i = np.arange(N)
    if kernel == "any":
        return w, U * w
    if kernel == "stft1024":
        assert (N, R) == (1024, 256)
        S = np.sqrt(0.5)
        n2, rest = i // 128, i % 128
        a = np.pi * (2 * rest + 1) / 2048.0
        b = n2 * np.pi / 8
        dw = U * (3 * np.abs(S * np.sin(a) * np.cos(b)) + 2 * np.abs(S * np.cos(a) * np.sin(b)) + w)
        exact = (n2 == 0) | (n2 == 4)
        return w, np.where(exact, U * w, dw)
    raise ValueError(kernel)


# ---- input -------------------------------------------------------------------------------------------------------
def kernel_samples(row, n, int16=False, gain=None):
    """The fp32 samples a kernel reads from one clip row of n samples: int16 -> x * 2^-15 (exact), then with a gain
    rn(rn(x / peak) * gain), peak = max |x[:n]|.  -> (float32 samples, float32 peak)."""
    x = np.asarray(row[:n])
    x = (x.astype(np.float32) * np.float32(2.0 ** -15)) if int16 else x.astype(np.float32)
    peak = np.float32(np.abs(x).max()) if n else np.float32(0)
    if gain is not None:
        x = (x / peak) * np.float32(gain)
    return x.astype(np.float32), peak


def _frames(v, N, R, T):
    """(T, N): frame f = v[f R - (N - R) + i], zero outside v (the kernels' padding)."""
    pad = N - R
    need = (T - 1) * R + N
    buf = np.zeros(need + 2 * pad)
    buf[pad:pad + len(v)] = v
    idx = np.arange(N)[None, :] + R * np.arange(T)[:, None]
    return buf[idx]


class Forward:
    """fp64 reference spectrum and per-frame bound of one clip through one kernel.
    X (T, K) complex = oracle lws_stft of the pre-emphasised exact input; B (T,) the bound of |X_hat - X|."""

    def __init__(self, x32, N, R, kernel, preemph=0.97, T=None):
        x = np.asarray(x32, dtype=np.float64)
        T = A.num_frames(len(x), N, R) if T is None else T
        self.N, self.R, self.kernel, self.T = N, R, kernel, T
        if preemph is not None:
            e, de = A.preemphasis(x, preemph), preemphasis_error(x, preemph)
        else:
            e, de = x, np.zeros_like(x)
        self.X = A.lws_stft(e, N, R)[:T] if len(x) else np.zeros((T, N // 2 + 1), complex)
        if self.X.shape[0] < T:
            self.X = np.concatenate([self.X, np.zeros((T - self.X.shape[0], self.X.shape[1]), complex)])
        self.B = frame_bound(np.abs(_frames(e, N, R, T)), _frames(de, N, R, T), kernel, N, R)


def frame_bound(ae, ade, kernel, N, R):
    """B_f for frames of |e| (T, N) with input errors ade (T, N)."""
    w, dw = window_error(kernel, N, R)
    swe = (w * ae).sum(-1)
    return SECOND_ORDER * (c_fft(kernel, N) * U * swe + (w * ade + dw * ae + U * w * ae).sum(-1))


def preemphasis_error(x, c=0.97):
    """|e_hat - e| bound of the kernels' fmaf pre-emphasis on fp32 samples x (fp64 array)."""
    cf = float(np.float32(c))
    xprev = np.concatenate([[0.0], np.abs(x[:-1])])
    return U * (np.abs(x) + cf * xprev) + abs(cf - c) * xprev


def complex_ratio(got, fw):
    """max over the frames of |got - X| / B (got: (T, K) complex)."""
    err = np.abs(np.asarray(got, np.complex128) - fw.X)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / fw.B[:, None])
    return float(np.nan_to_num(r, nan=np.inf).max())


# ---- dB ----------------------------------------------------------------------------------------------------------
def _pre(v, min_db=-100.0, ref_db=20.0):
    """The dB map before its clip (the bound's own restatement of audio_oracle._amp_to_db / _normalize)."""
    min_level = 10.0 ** (min_db / 20.0)
    return (20.0 * np.log10(np.maximum(min_level, v)) - ref_db - min_db) / -min_db


def _eval_err(lo, hi, log_err, halved, min_db=-100.0, ref_db=20.0):
    """Evaluation error of sat(fmaf(c2, log2(arg), c0)) at arguments between lo and hi."""
    min_level = 10.0 ** (min_db / 20.0)
    c2 = 20.0 * np.log10(2.0) / -min_db
    c0 = 1.0 - ref_db / -min_db
    if halved:                                   # lg2 of p4 = 4 v^2 with c2 / 2, c0 - c2
        c2, c0 = 0.5 * c2, c0 - c2
        arg = lambda v: 4.0 * np.maximum(v, min_level) ** 2
    else:
        arg = lambda v: np.maximum(v, min_level)
    L = np.maximum(np.abs(np.log2(arg(lo))), np.abs(np.log2(arg(hi))))
    e_log = LG2_APPROX_ABS if log_err == "lg2" else LOG2F_ULP * ULP * L
    return c2 * e_log + U * (2 * c2 * L + 2 * abs(c0)) + 2.0 ** -30


def db_interval(v, lo, hi, log_err, halved):
    """(ref, lower, upper) of a normalised dB output whose linear value v (fp64 reference) lies in [lo, hi].  The
    interval is the unsaturated one moved onto the saturated reference: saturation is monotone and 1-Lipschitz, so
    |sat(y) - sat(pre(v))| <= |y - pre(v)|, and a value clipped at 0 or 1 is not scored against a zero-width end."""
    eps = _eval_err(lo, hi, log_err, halved)
    ref = A._normalize(A._amp_to_db(v) - 20.0)
    pv = _pre(v)
    return ref, ref - (pv - _pre(lo) + eps), ref + (_pre(hi) - pv + eps)


def interval_ratio(got, ref, lower, upper):
    """Largest error-to-bound ratio of got against ref within [lower, upper]: 1 at either end; inf for NaN."""
    got = np.asarray(got, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(got >= ref, (got - ref) / (upper - ref), (ref - got) / (ref - lower))
    r = np.where(got == ref, 0.0, r)
    return float(np.nan_to_num(r, nan=np.inf, posinf=np.inf).max()) if r.size else 0.0


MAG_REL = {"stft1024_lin": U, "stft1024_mel": U + SQRT_APPROX_REL, "any": 2 * U}
MAG_ABS = {"stft1024_lin": 0.0, "stft1024_mel": 2.0 ** -64, "any": 0.0}


def mag_interval(fw, which):
    a = np.abs(fw.X)
    B = fw.B[:, None]
    r = MAG_REL[which]
    return np.maximum(0.0, (a - B) * (1 - r)), (a + B) * (1 + r) + MAG_ABS[which]


def linear_db(fw):
    """(ref, lower, upper) of the linear row, (T, K)."""
    which = "stft1024_lin" if fw.kernel == "stft1024" else "any"
    lo, hi = mag_interval(fw, which)
    return db_interval(np.abs(fw.X), lo, hi, "lg2" if fw.kernel == "stft1024" else "log2f",
                       halved=fw.kernel == "stft1024")


def mel_db(fw, basis, start=None, length=None):
    """(ref, lower, upper) of the mel row, (T, n_mels), for the fp32 filterbank ``basis`` (its non-zero runs
    start / length; the whole row when not given)."""
    which = "stft1024_mel" if fw.kernel == "stft1024" else "any"
    lo, hi = mag_interval(fw, which)
    Bm = np.asarray(basis, np.float64)
    n = np.full(Bm.shape[0], Bm.shape[1]) if length is None else np.asarray(length)
    gamma = (n + 2) * U / (1 - (n + 2) * U)
    v = np.abs(fw.X) @ Bm.T
    return db_interval(v, (lo @ Bm.T) * (1 - gamma), (hi @ Bm.T) * (1 + gamma),
                       "lg2" if fw.kernel == "stft1024" else "log2f", halved=False)


def front_end_ratios(lin, mel, x32, N, R, kernel, basis, start=None, length=None):
    """(linear, mel) largest error-to-bound ratios of one clip's (T, K) linear and (T, n_mels) mel rows."""
    fw = Forward(x32, N, R, kernel)
    assert lin.shape == fw.X.shape and mel.shape == (fw.T, np.asarray(basis).shape[0]), (lin.shape, mel.shape)
    return (interval_ratio(lin, *linear_db(fw)), interval_ratio(mel, *mel_db(fw, basis, start, length)))


# ---- Griffin-Lim projection and inverse STFT -----------------------------------------------------------------------
def projection_ratio(got, fw, mag):
    """got = the kernel's mag X_hat / |X_hat| (T, K) complex; -> largest error-to-bound ratio."""
    got = np.asarray(got, np.complex128)
    mag = np.asarray(mag, np.float64)
    a, B = np.abs(fw.X), fw.B[:, None] * np.ones_like(mag)
    strong = a > 2 * B
    with np.errstate(divide="ignore", invalid="ignore"):
        want = np.where(a > 0, mag * fw.X / np.where(a > 0, a, 1.0), mag + 0j)
        bound = mag * (2 * B / (a - B) + 5 * U) + 1e-38
        r_strong = np.abs(got - want) / bound
        r_weak = np.abs(np.abs(got) - mag) / (5 * U * mag + 1e-38)
    r = np.where(strong, r_strong, r_weak)
    return float(np.nan_to_num(r, nan=np.inf).max())


def packed_irfft(X, N):
    """The kernels' inverse real FFT of the half spectrum X (..., N/2 + 1) in fp64: the imaginary parts of bins 0
    and N/2 are folded into the waveform instead of dropped (irfft when they are zero)."""
    X = np.asarray(X, np.complex128)
    M = N // 2
    k = np.arange(M)
    a, b = X[..., :M], np.conj(X[..., M - k])
    Z = 0.5 * (a + b) + 1j * (0.5 * (a - b) * np.exp(2j * np.pi * k / N))
    z = np.fft.ifft(Z, axis=-1)
    out = np.empty(X.shape[:-1] + (N,))
    out[..., 0::2], out[..., 1::2] = z.real, z.imag
    return out


def istft(spec, N, R, n, kernel):
    """(ref (n,), bound (n,)) of the inverse STFT of spec (T, K) complex into a zeroed clip of n samples."""
    spec = np.asarray(spec, np.complex128)
    T, M, pad = spec.shape[0], N // 2, N - R
    w, dw = window_error(kernel, N, R)
    x = packed_irfft(spec, N)
    S = np.abs(spec).sum(1)
    inv_err = 0.0 if M & (M - 1) == 0 else U
    fr_err = (w[None] * c_fft(kernel, N) * U * S[:, None] / M + np.abs(x) * (w[None] * (inv_err + 2 * U) + dw[None]))
    fr = x * w[None]
    L = (T - 1) * R + N
    y, err, absum = np.zeros(L), np.zeros(L), np.zeros(L)
    for f in range(T):
        y[f * R:f * R + N] += fr[f]
        err[f * R:f * R + N] += fr_err[f]
        absum[f * R:f * R + N] += np.abs(fr[f])
    sl = slice(pad, pad + n)
    return y[sl], SECOND_ORDER * (err[sl] + (N // R) * U * absum[sl])


def abs_ratio(got, ref, bound):
    err = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nan_to_num(r, nan=np.inf).max()) if r.size else 0.0


# ---- dB -> amplitude and de-emphasis ------------------------------------------------------------------------------
def spec_to_amp(s, min_db=-100.0, ref_db=20.0, power=1.4):
    """(ref, bound) of dv3_spec_to_amp on fp32 normalised dB values s."""
    v = np.clip(np.asarray(s, np.float64), 0, 1)
    lin = v * -min_db + min_db
    db = lin + ref_db
    t = db * 0.05
    ddb = U * (np.abs(v * -min_db) + np.abs(lin) + np.abs(db))
    dt = 0.05 * ddb + abs(float(np.float32(0.05)) - 0.05) * np.abs(db) + U * np.abs(t)
    amp = np.power(10.0, t * power)
    pf = float(np.float32(power))
    rel = power * (np.log(10.0) * dt + POWF_ULP * ULP) + POWF_ULP * ULP + abs(pf - power) * np.abs(np.log(10.0) * t)
    return amp, SECOND_ORDER * rel * amp + 1e-45


def deemphasis(x, c=0.97):
    """(ref, bound) of dv3_deemphasis on one fp32 clip."""
    x = np.asarray(x, np.float64)
    ref = A.inv_preemphasis(x, c)
    cf = float(np.float32(c))
    Aabs = lfilter([1.0], [1.0, -c], np.abs(x))
    prev = np.concatenate([[0.0], Aabs[:-1]])
    src = abs(cf - c) * prev + U * Aabs
    return ref, SECOND_ORDER * lfilter([1.0], [1.0, -cf], src)
