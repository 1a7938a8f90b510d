"""CPU: the elementwise bounds of tests/audio_bounds.py have teeth.  Each defect below is applied to the fp64
reference; on the test inputs the perturbed reference must leave the bound of the true one by more than a factor of
two on at least one element, so a kernel within its bound cannot carry the defect.  Also the fp64 restatement of the
kernels' packed inverse, and the de-emphasis bound against an fp32 emulation of the kernel's fmaf recurrence."""
import numpy as np
import pytest

import audio_bounds as AB
from oracle import audio_oracle as A

GEOMS = [(22050, 1024, 256, "stft1024"), (22050, 1024, 256, "any"), (16000, 800, 200, "any"),
         (48000, 2400, 600, "any")]


def _clip(N, n=6000, seed=0):
    """noise + a tone on a bin centre + DC + Nyquist, then 0.9-amplitude garbage past the clip's end."""
    rng = np.random.RandomState(seed)
    t = np.arange(n)
    x = 0.2 * rng.randn(n) + 0.3 * np.cos(2 * np.pi * 37 * t / N) + 0.1 + 0.05 * (-1.0) ** t
    garbage = rng.uniform(-0.9, 0.9, 64)
    return x.astype(np.float32), garbage.astype(np.float32)


def _stft(e, N, R, w=None):
    w = A.lws_window(N, R) if w is None else w
    return np.fft.rfft(AB._frames(e, N, R, A.num_frames(len(e), N, R)) * w, axis=1)


@pytest.mark.parametrize("sr,N,R,kernel", GEOMS, ids=["%d-%d-%s" % (N, R, k) for _, N, R, k in GEOMS])
def test_bounds_catch_defects(sr, N, R, kernel):
    x, garbage = _clip(N)
    fw = AB.Forward(x, N, R, kernel)
    T, M = fw.T, N // 2
    e = A.preemphasis(x.astype(np.float64))
    assert np.allclose(_stft(e, N, R), fw.X, atol=1e-12)
    lin_ref, lin_lo, lin_hi = AB.linear_db(fw)
    from deepvoice3_pytorch_b200 import audio
    old = dict(vars(audio.hparams))
    try:
        audio.hparams.sample_rate, audio.hparams.fft_size, audio.hparams.hop_size = sr, N, R
        basis = audio._build_mel_basis()
    finally:
        for k, v in old.items():
            setattr(audio.hparams, k, v)
    mel_ref, mel_lo, mel_hi = AB.mel_db(fw, basis)

    i = np.arange(N)
    factors = {}
    # window without its half-sample offset
    w0 = np.sqrt(0.5 * (1 - np.cos(2 * np.pi * i / N)) * 2 * R / N)
    factors["window without the half-sample offset"] = AB.complex_ratio(_stft(e, N, R, w=w0), fw)
    # pre-emphasis coefficient rounded to fp16
    e16 = A.preemphasis(x.astype(np.float64), float(np.float16(0.97)))
    factors["pre-emphasis 0.97 rounded to fp16"] = AB.complex_ratio(_stft(e16, N, R), fw)
    # every frame starts one sample late
    late = np.fft.rfft(AB._frames(np.concatenate([e[1:], [0.0]]), N, R, T) * A.lws_window(N, R), axis=1)
    factors["frame one sample late"] = AB.complex_ratio(late, fw)
    # the first garbage sample past len leaks into the frames (pre-emphasised like a clip sample)
    xl = np.concatenate([x, garbage[:1]]).astype(np.float64)
    el = A.preemphasis(xl)
    leak = np.fft.rfft(AB._frames(el, N, R, T) * A.lws_window(N, R), axis=1)
    factors["one sample past len"] = AB.complex_ratio(leak, fw)
    # DC and Nyquist bins exchanged (= the signs of Im Z_0 swapped in the split: X_0, X_M = Re Z_0 -+ Im Z_0)
    sw = fw.X.copy()
    sw[:, [0, M]] = sw[:, [M, 0]]
    factors["DC and Nyquist swapped"] = AB.interval_ratio(A._normalize(A._amp_to_db(np.abs(sw)) - 20.0),
                                                          lin_ref, lin_lo, lin_hi)
    # a mel filter shifted by one bin
    shifted = np.roll(basis.astype(np.float64), 1, axis=1)
    mel_sh = A._normalize(A._amp_to_db(np.abs(fw.X) @ shifted.T) - 20.0)
    factors["mel filters shifted by one bin"] = AB.interval_ratio(mel_sh, mel_ref, mel_lo, mel_hi)
    # dB of |X|^2 without the halving
    factors["dB of |X|^2 not halved"] = AB.interval_ratio(A._normalize(A._amp_to_db(np.abs(fw.X) ** 2) - 20.0),
                                                          lin_ref, lin_lo, lin_hi)
    print("\n%d / %d %s: defect / bound" % (N, R, kernel))
    for k, v in factors.items():
        print("  %-40s %10.3g" % (k, v))
    for k, v in factors.items():
        assert v > 2.0, (k, v)


def test_packed_inverse_is_irfft_without_imaginary_edge_bins():
    rng = np.random.RandomState(1)
    for N in (256, 800, 1024, 2400):
        X = rng.randn(5, N // 2 + 1) + 1j * rng.randn(5, N // 2 + 1)
        X[:, [0, N // 2]] = X[:, [0, N // 2]].real
        assert np.abs(AB.packed_irfft(X, N) - np.fft.irfft(X, n=N, axis=1)).max() < 1e-13
        X[:, 0] += 0.5j
        fold = np.abs(AB.packed_irfft(X, N) - np.fft.irfft(X, n=N, axis=1))
        assert np.allclose(fold, 0.5 / N, rtol=1e-9)                                        # folded, not dropped


def test_deemphasis_bound_holds_for_an_fp32_fmaf_recurrence():
    rng = np.random.RandomState(2)
    x = (0.5 * rng.randn(4000)).astype(np.float32)
    c = np.float32(0.97)
    y = np.empty_like(x)
    prev = np.float32(0)
    for n in range(len(x)):            # fmaf: the product is exact in fp64, one rounding to fp32
        prev = np.float32(float(c) * float(prev) + float(x[n]))
        y[n] = prev
    ref, bound = AB.deemphasis(x)
    r = AB.abs_ratio(y, ref, bound)
    print("de-emphasis fp32 emulation: error / bound %.3g" % r)
    assert 1e-3 < r <= 1.0
