"""GPU: fused STFT->linear/mel kernel against the numpy restatement of audio.py (oracle/audio_oracle.py;
parity UNPINNED, see its header).  Values are held to the elementwise fp64 bounds of tests/audio_bounds.py (kernel
"stft1024" for the fused front end, "any" for the complex STFT / iSTFT of csrc/stft_any.cu)."""
import numpy as np
import pytest
import torch

import audio_bounds as AB

pytestmark = pytest.mark.gpu


def _check(lin, mel, x, basis=None, start=None, length=None):
    """lin (T, 513), mel (T, n_mels) of the fp32 clip x within the bounds of the fused kernel."""
    from deepvoice3_pytorch_b200 import audio
    if basis is None:
        basis, start, length = (t.cpu().numpy() for t in audio._device_basis(torch.device("cuda")))
    r_lin, r_mel = AB.front_end_ratios(lin, mel, x, 1024, 256, "stft1024", basis, start, length)
    assert r_lin <= 1.0 and r_mel <= 1.0, (r_lin, r_mel)


def test_single_clip_matches_oracle():
    from deepvoice3_pytorch_b200 import audio
    from oracle import audio_oracle as A
    x = A.synthetic_clip(3)
    lin = audio.spectrogram(x)
    mel = audio.melspectrogram(x)
    assert lin.shape == (513, 865) and mel.shape == (80, 865)
    _check(lin.T, mel.T, x)


def test_ragged_batch_and_edge_lengths():
    from deepvoice3_pytorch_b200 import audio
    from oracle import audio_oracle as A
    lens = [1, 255, 256, 257, 1023, 1024, 1025, 5000, 22050]
    clips = [A.synthetic_clip(10 + i, n=max(n, 2))[:n] for i, n in enumerate(lens)]
    wav = np.zeros((len(lens), max(lens)), dtype=np.float32)
    for i, c in enumerate(clips):
        wav[i, :len(c)] = c
    lin, mel = audio.stft_mel_batch(torch.from_numpy(wav).cuda(), torch.tensor(lens, dtype=torch.int32).cuda())
    lin, mel = lin.cpu().numpy(), mel.cpu().numpy()
    for i, (c, n) in enumerate(zip(clips, lens)):
        nf = A.num_frames(n)
        assert nf == audio.num_frames(n)
        _check(lin[i, :nf], mel[i, :nf], c)
        assert not lin[i, nf:].any() and not mel[i, nf:].any()     # untouched beyond the clip


def test_mel_basis_matches_librosa_definition():
    from deepvoice3_pytorch_b200 import audio
    from oracle import audio_oracle as A
    np.testing.assert_allclose(audio._build_mel_basis(), A.mel_basis(), rtol=1e-6, atol=1e-9)


def test_linearity_and_silence():
    """Size-independent properties: silence -> exactly the floor (0); scaling the input by 10 raises every
    unclipped bin by 20 dB (= 0.2 normalised)."""
    from deepvoice3_pytorch_b200 import audio
    from oracle import audio_oracle as A
    z = np.zeros(22050, dtype=np.float32)
    assert not audio.spectrogram(z).any() and not audio.melspectrogram(z).any()
    x = 0.05 * A.synthetic_clip(5, n=44100)
    a, b = audio.spectrogram(x), audio.spectrogram(10 * x)
    ok = (a > 0.05) & (b < 0.95)
    assert np.abs((b - a)[ok] - 0.2).max() < 2e-3


def test_complex_stft_and_istft_against_oracle():
    """At 1024 / 256: dv3_stft_complex_geom == the oracle's lws_stft (complex values), dv3_istft_geom == lws_istft, and
    istft(stft(x)) == x (the sqrt-Hann frame with 768-sample padding reconstructs perfectly)."""
    import ctypes
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    from oracle import audio_oracle as A
    rng = np.random.RandomState(0)
    n = 40 * 256 - 512                                       # hop-aligned: 41 frames
    x = (0.3 * rng.randn(n)).astype(np.float32)
    T = audio.num_frames(n)
    assert audio.inv_num_samples(T) == n
    xd = torch.from_numpy(x).cuda()
    spec = torch.zeros(T, 513, 2, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    tab = audio._geometry_table(xd.device, 1024, 256)
    nd = torch.tensor([n], dtype=torch.int32, device="cuda")
    fd = torch.tensor([T], dtype=torch.int32, device="cuda")

    def stft(mag):
        lib.call("dv3_stft_complex_geom", vp(xd), vp(nd), n, mag, vp(spec), vp(fd), T, 1, vp(tab), 1024, 256, st)
    stft(None)
    fw = AB.Forward(x, 1024, 256, "any", preemph=None, T=T)
    got = spec[..., 0].cpu().numpy().astype(np.float64) + 1j * spec[..., 1].cpu().numpy()
    assert AB.complex_ratio(got, fw) <= 1.0
    y = torch.zeros(n, device="cuda")
    lib.call("dv3_istft_geom", vp(spec), vp(y), vp(nd), n, vp(fd), T, 1, vp(tab), 1024, 256, st)
    np.testing.assert_allclose(y.cpu().numpy(), x, rtol=1e-3, atol=2e-5)            # perfect reconstruction
    ref_y, bound = AB.istft(got, 1024, 256, n, "any")
    assert AB.abs_ratio(y.cpu().numpy(), ref_y, bound) <= 1.0
    # magnitude projection (one Griffin-Lim step)
    mag_np = np.abs(fw.X).astype(np.float32) * 0.5
    magd = torch.from_numpy(mag_np).cuda()
    stft(vp(magd))
    got = spec[..., 0].cpu().numpy().astype(np.float64) + 1j * spec[..., 1].cpu().numpy()
    assert AB.projection_ratio(got, fw, mag_np) <= 1.0


def test_inv_spectrogram_round_trip_and_oracle():
    """reference audio.py:37-43: spectrogram(x) -> inv_spectrogram recovers a waveform whose spectrogram matches the
    input (spectral convergence of Griffin-Lim), the de-emphasis filter is exact, and a short run equals the numpy
    restatement of the same algorithm (parity with the reference's lws phase recovery is UNPINNED: lws is absent)."""
    from deepvoice3_pytorch_b200 import audio
    from oracle import audio_oracle as A
    x = A.synthetic_clip(3, n=60 * 256 - 512)
    S = audio.spectrogram(x)                                 # (513, T) normalised dB
    old_power = audio.hparams.power
    try:
        audio.hparams.power = 1.0                            # so that the re-analysed spectrogram is comparable
        y = audio.inv_spectrogram(S, n_iter=60)
        assert y.dtype == np.float32 and y.shape == (audio.inv_num_samples(S.shape[1]),)
        S2 = audio.spectrogram(y)
        assert S2.shape == S.shape
        loud = S > 0.45                                      # bins above ~ -55 dB: where the magnitude is meaningful
        assert np.abs(S2 - S)[loud].mean() < 0.03, np.abs(S2 - S)[loud].mean()
        # 4 iterations: the CUDA path against the numpy restatement of the same iteration
        y4 = audio.inv_spectrogram(S, n_iter=4)
        r4 = A.inv_spectrogram(S, power=1.0, n_iter=4)
        np.testing.assert_allclose(y4, r4, rtol=2e-2, atol=2e-3 * np.abs(r4).max())
    finally:
        audio.hparams.power = old_power
    # de-emphasis alone: the fp32 fmaf recurrence within its bound of the fp64 IIR
    z = torch.randn(3, 5000, device="cuda")
    got = audio.inv_preemphasis(z).cpu().numpy()
    for i in range(3):
        ref, bound = AB.deemphasis(z[i].cpu().numpy())
        assert AB.abs_ratio(got[i], ref, bound) <= 1.0


def test_general_filterbank_and_staging_paths():
    """(a) A dense 24 x 513 filterbank does not fit the packed per-quad form of the kernel: the plain loop must give
    basis @ |STFT| like numpy.  (b) The same clips staged through the 16-byte path (row pitch a multiple of 4 samples)
    and the 4-byte path (odd pitch) give bit-identical outputs."""
    import ctypes
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    from oracle import audio_oracle as A
    rng = np.random.RandomState(7)
    n = 6000
    clips = np.stack([A.synthetic_clip(40 + i, n=n) for i in range(3)])
    T = audio.num_frames(n)

    def run(wav_t, basis, start, length):
        nm = basis.shape[0]
        lin = torch.empty(wav_t.shape[0], T, 513, device="cuda")
        mel = torch.empty(wav_t.shape[0], T, nm, device="cuda")
        lens = torch.full((wav_t.shape[0],), n, dtype=torch.int32, device="cuda")
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        lib.call("dv3_stft_mel", p(wav_t), p(lens), p(basis), p(start), p(length), p(lin), p(mel), wav_t.shape[0],
                 wav_t.shape[1], T, nm, 0.97, -100.0, 20.0, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return lin.cpu().numpy(), mel.cpu().numpy()

    # (a) dense filterbank
    dense = (rng.rand(24, 513).astype(np.float32) + 0.1) / 513.0
    wav_t = torch.from_numpy(clips).cuda()
    lin, mel = run(wav_t, torch.from_numpy(dense).cuda(), torch.zeros(24, dtype=torch.int32).cuda(),
                   torch.full((24,), 513, dtype=torch.int32).cuda())
    for i in range(3):
        _check(lin[i], mel[i], clips[i], dense, np.zeros(24, np.int32), np.full(24, 513, np.int32))
    # (b) staging paths
    basis, start, length = audio._device_basis(wav_t.device)
    lin_a, mel_a = run(wav_t, basis, start, length)                                      # pitch 6000: 16-byte copies
    wide = torch.zeros(3, n + 1, device="cuda")
    wide[:, :n] = wav_t
    lin_b, mel_b = run(wide, basis, start, length)                                       # pitch 6001: 4-byte copies
    assert np.array_equal(lin_a, lin_b) and np.array_equal(mel_a, mel_b)
    _check(lin_a[0], mel_a[0], clips[0])
