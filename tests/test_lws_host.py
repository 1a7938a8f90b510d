"""CPU: LWS phase recovery (csrc/lws.cu) -- the fp64 oracle's weights and conventions against STFT(iSTFT(.)), its
quality against Griffin-Lim, argument checks that fire before any CUDA call, and the C ABI of the new entry points."""
import ctypes

import numpy as np
import pytest
import torch

import lws_oracle as O
from oracle import audio_oracle as A


def test_weights_are_the_linear_part_of_stft_of_istft():
    """For an impulse delta at (m0, k0) of an interior frame, the complex-linear part of G = STFT(iSTFT(.)) --
    (G(delta) - i G(i delta)) / 2, which removes the real signal's mirror term -- is beta_q(d) (-i)^{k0 q} at
    (m0 - q, k0 + d).  This pins the index and sign conventions of the weights and the phase factor."""
    beta = O.lws_weights()
    T, m0 = 20, 10
    G = lambda X: A.lws_stft(A.lws_istft(X))[:T]
    for k0 in (6, 37, 250, 506):
        D = np.zeros((T, 513), dtype=np.complex128)
        D[m0, k0] = 1.0
        H = (G(D) - 1j * G(1j * D)) / 2
        for q in range(-3, 4):
            for d in range(-5, 6):
                want = beta[q + 3, d + 5] * (-1j) ** ((k0 * q) % 4)
                assert abs(H[m0 - q, k0 + d] - want) < 1e-12, (k0, q, d)


def test_product_weights_equal_the_oracle():
    from deepvoice3_pytorch_b200 import audio
    beta = O.lws_weights()
    np.testing.assert_allclose(audio._lws_weights_fp64(), beta, rtol=0, atol=1e-15)
    assert abs(beta[3, 5] - 0.25) < 1e-15                    # beta_0(0) = sum w^2 / N = 1/4 (hop = N/4)


def test_local_sum_mirror_bins_are_real_at_the_spectrum_ends():
    """Y at bins 0 and 512 is real in exact arithmetic when X is a real signal's spectrum (the mirrored terms pair up as
    complex conjugates): the oracle's conjugate mirror and unreduced phase factor keep that."""
    rng = np.random.RandomState(1)
    X = A.lws_stft(rng.randn(30 * 256))[:30]
    Y = O.lws_local_sum(X, O.lws_weights())
    assert np.abs(Y[:, [0, 512]].imag).max() < 1e-12 * np.abs(Y).max()


def test_quality_against_griffin_lim():
    """Spectral convergence ||A - |STFT(x)||| / ||A|| of the no-future initialisation + 30 batch iterations against
    60 Griffin-Lim iterations, on three 200-frame synthetic clips (fp64 oracle).  Measured: 0.068 / 0.096 / 0.130
    against 0.141 / 0.176 / 0.124, ratios 0.48 / 0.54 / 1.04.  Over seeds 0..7 the ratio spans 0.48 .. 1.04 (median
    0.72): on some of these chirp-plus-noise clips LWS only matches Griffin-Lim-60.  So the bound is on the mean ratio
    (0.69 measured), with every clip no worse than Griffin-Lim-60 by more than 10 %, rather than 0.7 on each clip."""
    ratios = []
    for seed in (0, 1, 2):
        x = A.synthetic_clip(seed, n=199 * 256 - 512)
        amp = np.abs(A.lws_stft(x))
        assert amp.shape == (200, 513)
        gl = O.spectral_convergence(amp, A.griffin_lim(amp, 60))
        lw = O.spectral_convergence(amp, O.lws(amp, 30))
        ratios.append(lw / gl)
    assert max(ratios) <= 1.1, ratios
    assert np.mean(ratios) <= 0.7, ratios


def test_bad_method_and_counts_raise_before_any_cuda_call(monkeypatch):
    from deepvoice3_pytorch_b200 import audio, synthesis

    def no_cuda(*a, **k):
        raise AssertionError("reached a CUDA call")
    monkeypatch.setattr(audio.lib, "call", no_cuda)
    monkeypatch.setattr(torch.Tensor, "cuda", no_cuda)
    monkeypatch.setattr(torch.Tensor, "to", no_cuda)
    spec = np.zeros((513, 12), dtype=np.float32)
    for kw in (dict(method="bogus"), dict(method="LWS"), dict(method=None), dict(method="lws", n_iter=-1),
               dict(method="lws", n_iter=2.5)):
        with pytest.raises(ValueError):
            audio.inv_spectrogram(spec, **kw)
        with pytest.raises(ValueError):
            audio.inv_spectrogram_batch([spec, spec], **kw)
    mag = torch.zeros(2, 12, 513)
    for kw in (dict(n_iter=-1), dict(init_iters=-1), dict(n_iter=1.5), dict(init_iters="1")):
        with pytest.raises(ValueError):
            audio.lws_batch(mag, [12, 10], **kw)
        with pytest.raises(ValueError):
            audio.lws(mag[0], **kw)
    with pytest.raises(ValueError, match="method"):
        synthesis.tts_batch(None, [np.arange(2, 9)], vocoder="wavenet")
    with pytest.raises(ValueError, match="method"):
        synthesis.tts_stream(None, [np.arange(2, 9)], vocoder="wavenet")


def test_hparams_default():
    from deepvoice3_pytorch_b200 import audio
    assert audio.hparams.lws_iters == 30 and audio.hparams.griffin_lim_iters == 60


def test_lws_entry_points_match_the_header():
    """The LWS entry points are declared in include/dv3b200.h with the argument types audio.py passes and are exported
    by the library."""
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import parse_header, LIB_PATH
    _build.build()
    decls = parse_header()
    P, I = ctypes.c_void_p, ctypes.c_int
    want = {
        "dv3_lws_nofuture": [P, P, P, I, I, P],
        "dv3_lws_iterate": [P, P, P, P, I, P],
        "dv3_lws_nofuture_batched": [P, P, P, P, I, I, I, P],
        "dv3_lws_iterate_batched": [P, P, P, P, P, I, I, P],
    }
    dll = ctypes.CDLL(LIB_PATH)
    for name, args in want.items():
        assert name in decls, name
        assert [t for t, _ in decls[name][1]] == args, name
        assert decls[name][0] is ctypes.c_int, name
        assert hasattr(dll, name), name
