"""GPU: LWS phase recovery (csrc/lws.cu, audio.lws_batch) against the fp64 oracle (tests/lws_oracle.py; parity with
the reference's lws.run_lws is UNPINNED, see its header), its ragged-batch contract, and the synthesis entry points."""
import ctypes

import numpy as np
import pytest
import torch

import lws_oracle as O
from oracle import audio_oracle as A

pytestmark = pytest.mark.gpu


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _clip_mag(seed, T):
    x = A.synthetic_clip(seed, n=(T - 1) * 256 - 512)
    amp = np.abs(A.lws_stft(x)).astype(np.float32)
    assert amp.shape == (T, 513)
    return amp


def _to_dev(X):
    return torch.from_numpy(np.stack([X.real, X.imag], -1).astype(np.float32)).cuda()


def _from_dev(t):
    a = t.cpu().numpy().astype(np.float64)
    return a[..., 0] + 1j * a[..., 1]


def _scale(X, beta):
    """sum over the stencil of |beta| |X|: the size of the terms that cancel into Y (fp32 round-off scales with it)."""
    T = X.shape[0]
    Xe = np.abs(O._extend(X))
    s = np.zeros((T, 513))
    for q in range(-3, 4):
        for d in range(-5, 6):
            s += abs(beta[q + 3, d + 5]) * Xe[3 + q:3 + q + T, 5 - d:5 - d + 513]
    return s


def test_one_jacobi_iteration_matches_oracle():
    """From the same random-phase input: every bin, the mirrored ones (0-5, 507-512) and the first and last 3 frames
    included, within 1e-5 of the local magnitude wherever |Y| is not a cancellation (|Y| >= 1e-2 of its terms' size,
    where fp32 round-off moves the phase by < 1e-5)."""
    from deepvoice3_pytorch_b200 import audio
    T = 43                                                            # 6 frame tiles, the last one partial
    amp = _clip_mag(5, T)
    rng = np.random.RandomState(0)
    X = amp * np.exp(2j * np.pi * rng.rand(T, 513))
    X[:, [0, 512]] = X[:, [0, 512]].real                              # a real signal's spectrum is real there
    X = _from_dev(_to_dev(X))                                         # the fp32 values the kernel sees
    beta = O.lws_weights()
    want = O.lws_iterate(X, amp, beta)
    Y = O.lws_local_sum(X, beta)
    xin, xout = _to_dev(X), torch.full((T, 513, 2), float("nan"), device="cuda")
    mag = torch.from_numpy(amp).cuda()
    w = audio._lws_weights(mag.device)
    from deepvoice3_pytorch_b200._lib import lib
    lib.call("dv3_lws_iterate", _vp(mag), _vp(xin), _vp(xout), _vp(w), T, _st())
    got = _from_dev(xout)
    err = np.abs(got - want)
    ok = np.abs(Y) >= 1e-2 * _scale(X, beta)
    ok[:, [0, 512]] = np.abs(Y[:, [0, 512]].real) >= 1e-2 * _scale(X, beta)[:, [0, 512]]
    assert ok.mean() > 0.98, ok.mean()
    assert np.isfinite(got).all() and np.allclose(np.abs(got), amp, rtol=1e-5, atol=1e-6 * amp.max())
    bad = err > 1e-5 * amp + 1e-7 * amp.max()
    assert not (bad & ok).any(), (np.argwhere(bad & ok)[:10], (err / np.maximum(amp, 1e-30))[ok].max())
    for sel in (np.s_[:, :6], np.s_[:, 507:], np.s_[:3], np.s_[-3:]):     # edges were really compared
        assert ok[sel].mean() > 0.9
    assert not got[:, [0, 512]].imag.any()


def test_nofuture_scan_teacher_forced():
    """Frame m from the oracle, given the GPU's frames m-3..m-1, equals the GPU's frame m: each frame is checked
    alone, so fp32 drift does not compound along the scan."""
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    T = 60
    amp = _clip_mag(6, T)
    beta = O.lws_weights()
    mag = torch.from_numpy(amp).cuda()
    for init_iters in (0, 1, 3):
        spec = torch.full((T, 513, 2), float("nan"), device="cuda")
        lib.call("dv3_lws_nofuture", _vp(mag), _vp(spec), _vp(audio._lws_weights(mag.device)), T, init_iters, _st())
        got = _from_dev(spec)
        assert np.isfinite(got).all()
        prev = np.zeros((T + 3, 513), dtype=np.complex128)
        prev[3:] = got
        errs = []
        for m in range(T):
            want = O.lws_nofuture_frame(amp[m], prev[m:m + 3], beta, init_iters)
            errs.append(np.abs(got[m] - want) / (amp[m] + 1e-6 * amp.max()))
        errs = np.array(errs)
        # bins whose phase sits on a cancellation can differ; they are few and isolated
        assert (errs > 1e-4).mean() < 0.01, (init_iters, (errs > 1e-4).mean())
        assert np.median(errs) < 1e-6, (init_iters, np.median(errs))


def _sc(amp, x):
    return O.spectral_convergence(amp, x)


def test_end_to_end_quality():
    """lws on the GPU (no-future init + 30 iterations): within 5 % of the oracle's spectral convergence, and against
    the GPU's Griffin-Lim-60 the bound of tests/test_lws_host.py (mean ratio <= 0.7, every clip <= 1.1)."""
    from deepvoice3_pytorch_b200 import audio
    ratios = []
    for seed in (0, 1, 2):
        amp = _clip_mag(seed, 200)
        mag = torch.from_numpy(amp).cuda()
        y_lws = audio.lws(mag, n_iter=30).cpu().numpy()
        y_gl = audio.griffin_lim(mag, n_iter=60).cpu().numpy()
        assert y_lws.shape == y_gl.shape == (audio.inv_num_samples(200),)
        sc_gpu, sc_oracle, sc_gl = _sc(amp, y_lws), _sc(amp, O.lws(amp, 30)), _sc(amp, y_gl)
        assert abs(sc_gpu - sc_oracle) <= 0.05 * sc_oracle, (seed, sc_gpu, sc_oracle)
        ratios.append(sc_gpu / sc_gl)
    assert max(ratios) <= 1.1 and np.mean(ratios) <= 0.7, ratios


def test_ragged_batch_bit_identical_to_each_clip_alone():
    from deepvoice3_pytorch_b200 import audio
    frames = [37, 4, 120, 9, 61]
    T_max = max(frames)
    mags = [_clip_mag(30 + i, t) for i, t in enumerate(frames)]
    batch = torch.full((len(frames), T_max, 513), 1e3, device="cuda")    # loud padding: must not leak in
    for c, a in enumerate(mags):
        batch[c, :a.shape[0]] = torch.from_numpy(a)
    for n_iter, init_iters in ((5, 1), (0, 2)):
        y = audio.lws_batch(batch, frames, n_iter=n_iter, init_iters=init_iters)
        again = audio.lws_batch(batch, frames, n_iter=n_iter, init_iters=init_iters)
        assert torch.equal(y, again)
        rev = audio.lws_batch(batch.flip(0).contiguous(), frames[::-1], n_iter=n_iter, init_iters=init_iters).flip(0)
        assert y.shape == (len(frames), audio.inv_num_samples(T_max))
        for c, a in enumerate(mags):
            n = audio.inv_num_samples(frames[c])
            alone = audio.lws(torch.from_numpy(a).cuda(), n_iter=n_iter, init_iters=init_iters)
            assert alone.shape == (n,)
            assert torch.equal(y[c, :n], alone), c
            assert not y[c, n:].any(), c
            assert torch.equal(rev[c, :n], alone), c


def test_inv_spectrogram_lws_and_synthesis():
    """inv_spectrogram(method="lws") returns as many samples as Griffin-Lim; tts_batch(vocoder="lws") row b equals
    inv_spectrogram(spec_b, method="lws") of the linear spectrogram it vocoded; in exact-fp32 mode tts_stream equals
    tts_batch with the same vocoder; the default vocoder is still Griffin-Lim."""
    from deepvoice3_pytorch_b200 import audio, synthesis
    from test_gpu_synthesis import _conv_math, _model, _sequences
    S = audio.spectrogram(A.synthetic_clip(8, n=40 * 256 - 512))
    y_l = audio.inv_spectrogram(S, method="lws")
    y_g = audio.inv_spectrogram(S)
    assert y_l.dtype == np.float32 and y_l.shape == y_g.shape == (audio.inv_num_samples(S.shape[1]),)
    assert not np.array_equal(y_l, y_g)

    model = _model("nyanko_ljspeech", max_steps=24)
    seqs = _sequences([37, 5, 61, 20], seed=4)
    seen = []
    real = audio.inv_spectrogram_batch

    def spy(specs, n_iter=None, method="griffin_lim"):
        seen.append(([np.array(s) for s in specs], method))
        return real(specs, n_iter, method)
    with _conv_math("fp32"):
        synthesis.audio.inv_spectrogram_batch = spy
        try:
            got = synthesis.tts_batch(model, seqs, vocoder="lws")
            default = synthesis.tts_batch(model, seqs)
        finally:
            synthesis.audio.inv_spectrogram_batch = real
        streamed = dict(synthesis.tts_stream(model, seqs, slots=2, post_batch=3, vocoder="lws"))
    assert [m for _, m in seen] == ["lws", "griffin_lim"]
    order = sorted(range(len(seqs)), key=lambda i: -seqs[i].size)       # tts_batch's row order
    for row, i in enumerate(order):
        spec = seen[0][0][row]
        assert np.array_equal(got[i][0], audio.inv_spectrogram(spec, method="lws")), i
        assert np.array_equal(default[i][0], audio.inv_spectrogram(spec)), i
        for a, b in zip(streamed[i], got[i]):
            assert np.array_equal(a, b), i
