"""GPU: the audio path at STFT frames other than 1024 / 256 (csrc/stft_any.cu, csrc/lws_any.cu, selected by
audio.check_geometry) against the fp64 oracles of tests/stft_geometry_oracle.py: the STFT kernels within the
elementwise bounds of tests/audio_bounds.py (kernel "any"), LWS within the bound of tests/test_gpu_lws.py; the
ragged-batch and bit-identity contracts; the training targets against the preprocessed corpus; synthesis; and that the
1024 / 256 frame calls its own forward and LWS kernels and the general complex-STFT and inverse-STFT ones."""
import contextlib
import ctypes
import os

import numpy as np
import pytest
import torch

import audio_bounds as AB
import stft_geometry_oracle as G
from oracle import audio_oracle as A

pytestmark = pytest.mark.gpu

GEOMS = [(16000, 256, 64), (16000, 512, 128), (16000, 800, 200), (22050, 1024, 512), (22050, 2048, 256),
         (24000, 1200, 300), (44100, 2048, 512), (48000, 2400, 600), (48000, 4096, 1024)]
IDS = ["%dk-%d-%d" % (sr // 1000, N, R) for sr, N, R in GEOMS]


@contextlib.contextmanager
def frame(sr, N, R):
    from deepvoice3_pytorch_b200 import audio
    keep = dict(vars(audio.hparams))
    audio.hparams.sample_rate, audio.hparams.fft_size, audio.hparams.hop_size = sr, N, R
    try:
        yield G.hp(sr, N, R)
    finally:
        for k in list(vars(audio.hparams)):
            delattr(audio.hparams, k)
        for k, v in keep.items():
            setattr(audio.hparams, k, v)


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(lin, mel, x, N, R, kernel="any"):
    """lin (T, K), mel (T, n_mels) of the fp32 clip x within the bounds of ``kernel`` at the frame (N, R), with the
    filterbank of the current hparams."""
    from deepvoice3_pytorch_b200 import audio
    basis, start, length = (t.cpu().numpy() for t in audio._device_basis(torch.device("cuda")))
    r_lin, r_mel = AB.front_end_ratios(lin, mel, x, N, R, kernel, basis, start, length)
    assert r_lin <= 1.0 and r_mel <= 1.0, (N, R, kernel, r_lin, r_mel)


def _clip(seed, n, sr):
    return A.synthetic_clip(seed, n=max(n, 2), sr=sr)[:n]


@pytest.mark.parametrize("sr,N,R", GEOMS, ids=IDS)
def test_forward_against_oracle_ragged_and_bit_identical(sr, N, R):
    from deepvoice3_pytorch_b200 import audio
    with frame(sr, N, R):
        lens = [1, R - 1, R, R + 1, N - 1, N, N + 1, 3 * sr // 2]
        clips = [_clip(20 + i, n, sr) for i, n in enumerate(lens)]
        wav = np.zeros((len(lens), max(lens)), np.float32)
        for i, c in enumerate(clips):
            wav[i, :len(c)] = c
        wd, ld = torch.from_numpy(wav).cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
        lin, mel = audio.stft_mel_batch(wd, ld)
        lin2, mel2 = audio.stft_mel_batch(wd, ld)
        assert torch.equal(lin, lin2) and torch.equal(mel, mel2)                       # two runs
        lin, mel = lin.cpu().numpy(), mel.cpu().numpy()
        assert lin.shape[2] == N // 2 + 1
        for i, (c, n) in enumerate(zip(clips, lens)):
            nf = A.num_frames(n, N, R)
            assert nf == audio.num_frames(n)
            _check(lin[i, :nf], mel[i, :nf], c, N, R)
            assert not lin[i, nf:].any() and not mel[i, nf:].any()
            a_lin, a_mel = audio.stft_mel_batch(torch.from_numpy(np.ascontiguousarray(c)).view(1, -1).cuda())
            assert np.array_equal(a_lin[0].cpu().numpy(), lin[i, :nf]), i                # alone == in the batch
            assert np.array_equal(a_mel[0].cpu().numpy(), mel[i, :nf]), i


def test_general_kernel_at_1024_256_agrees_with_the_specialised_one():
    """dv3_stft_mel_geom called directly at the default frame (nothing selects it there) and dv3_stft_mel: each
    within its own bound of the fp64 reference, and the same zero rows."""
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    lens = [1, 700, 1024, 15617, 22050 * 3]
    wav = np.zeros((len(lens), max(lens)), np.float32)
    for i, n in enumerate(lens):
        wav[i, :n] = _clip(50 + i, n, 22050)
    wd, ld = torch.from_numpy(wav).cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
    lin, mel = audio.stft_mel_batch(wd, ld)
    T = lin.shape[1]
    basis, start, length = audio._device_basis(wd.device)
    glin, gmel = torch.full_like(lin, float("nan")), torch.full_like(mel, float("nan"))
    lib.call("dv3_stft_mel_geom", _vp(wd), 0, _vp(ld), None, 1.0, _vp(audio._geometry_table(wd.device, 1024, 256)),
             _vp(basis), _vp(start), _vp(length), _vp(glin), _vp(gmel), len(lens), wav.shape[1], T, 0, 1, 80, 1024,
             256, 0.97, -100.0, 20.0, _st())
    lin, mel, glin, gmel = (t.cpu().numpy() for t in (lin, mel, glin, gmel))
    for i, n in enumerate(lens):
        nf = audio.num_frames(n)
        _check(glin[i, :nf], gmel[i, :nf], wav[i, :n], 1024, 256, "any")
        _check(lin[i, :nf], mel[i, :nf], wav[i, :n], 1024, 256, "stft1024")
        assert not glin[i, nf:].any() and not gmel[i, nf:].any()
        assert not lin[i, nf:].any() and not mel[i, nf:].any()


def _write_corpus(root, sr, n_clips=7, seed=3):
    from scipy.io import wavfile
    rng = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, "wavs"), exist_ok=True)
    lines = []
    for i in range(n_clips):
        n = sr // 4 if i == 0 else int(rng.randint(sr // 4, 3 * sr))         # collate needs >= r * ds frames
        t = np.arange(n) / sr
        x = (0.3 * np.sin(2 * np.pi * (200 + 50 * i) * t) + 0.05 * rng.randn(n)) * (0.2 + 0.7 * rng.rand())
        wavfile.write(os.path.join(root, "wavs", "C%03d.wav" % i), sr, (x * 32767).astype(np.int16))
        txt = "utterance number %d of the geometry corpus" % i
        lines.append("C%03d|%s|%s\n" % (i, txt, txt))
    with open(os.path.join(root, "metadata.csv"), "w", encoding="utf-8") as f:
        f.writelines(lines)


@pytest.mark.parametrize("sr,N,R", [(16000, 800, 200), (44100, 2048, 512)], ids=["16k-800-200", "44k-2048-512"])
def test_targets_equal_collate_of_the_preprocessed_corpus(tmp_path, sr, N, R):
    """stft_mel_targets on the corpus' PCM (int16, and fp32 = x / 32768) gives bit for bit data.collate of the .npy
    features preprocess.build_from_path wrote at the same frame, rescaling off and on, at several (r, ds)."""
    from scipy.io import wavfile
    from deepvoice3_pytorch_b200 import audio, data, preprocess
    in_dir = str(tmp_path / "in")
    _write_corpus(in_dir, sr)
    with frame(sr, N, R):
        for rescaling in (False, True):
            audio.hparams.rescaling = rescaling
            out_dir = str(tmp_path / ("out%d" % rescaling))
            os.makedirs(out_dir)
            rows = preprocess.build_from_path(in_dir, out_dir, batch_clips=4)
            assert len(rows) == 7
            feats = [(np.load(os.path.join(out_dir, s)), np.load(os.path.join(out_dir, m))) for s, m, _, _ in rows]
            assert all(lin.shape[1] == N // 2 + 1 and lin.shape[0] == nf for (lin, _), (_, _, nf, _) in zip(feats, rows))
            pcm = [wavfile.read(os.path.join(in_dir, "wavs", "C%03d.wav" % i))[1] for i in range(7)]
            lens = [len(p) for p in pcm]
            wav16 = np.zeros((7, max(lens) + 5), np.int16)
            for i, p in enumerate(pcm):
                wav16[i, :len(p)] = p
            for r, ds in ((1, 4), (4, 1), (2, 2), (3, 3)):
                ref = data.collate([(np.arange(3), m, l) for l, m in feats], r=r, downsample_step=ds)
                T_lin = ref["y"].shape[1]
                for wav in (torch.from_numpy(wav16).cuda(), torch.from_numpy(wav16.astype(np.float32) / 32768).cuda()):
                    y, mel = audio.stft_mel_targets(wav, lens, T_lin, r, ds)
                    assert torch.equal(y.cpu(), ref["y"]), (rescaling, r, ds, wav.dtype)
                    assert torch.equal(mel.cpu(), ref["mel"]), (rescaling, r, ds, wav.dtype)


@pytest.mark.parametrize("sr,N,R", GEOMS, ids=IDS)
def test_complex_stft_istft_and_griffin_lim_against_oracle(sr, N, R):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    with frame(sr, N, R):
        rng = np.random.RandomState(0)
        T = 41
        n = audio.inv_num_samples(T)
        assert A.num_frames(n, N, R) == T
        x = (0.3 * rng.randn(n)).astype(np.float32)
        xd = torch.from_numpy(x).cuda().view(1, -1)
        K = N // 2 + 1
        spec = torch.full((1, T, K, 2), float("nan"), device="cuda")
        nd, fd = torch.tensor([n], dtype=torch.int32).cuda(), torch.tensor([T], dtype=torch.int32).cuda()
        tab = audio._geometry_table(xd.device, N, R)
        lib.call("dv3_stft_complex_geom", _vp(xd), _vp(nd), n, None, _vp(spec), _vp(fd), T, 1, _vp(tab), N, R, _st())
        fw = AB.Forward(x, N, R, "any", preemph=None, T=T)
        got = _from_dev(spec[0])
        assert AB.complex_ratio(got, fw) <= 1.0
        y = torch.zeros(1, n, device="cuda")
        lib.call("dv3_istft_geom", _vp(spec), _vp(y), _vp(nd), n, _vp(fd), T, 1, _vp(tab), N, R, _st())
        np.testing.assert_allclose(y[0].cpu().numpy(), x, rtol=1e-3, atol=2e-5)                # perfect rec.
        ref_y, bound = AB.istft(got, N, R, n, "any")
        assert AB.abs_ratio(y[0].cpu().numpy(), ref_y, bound) <= 1.0
        mag_np = np.abs(fw.X).astype(np.float32) * 0.5
        lib.call("dv3_stft_complex_geom", _vp(xd), _vp(nd), n, _vp(torch.from_numpy(mag_np).cuda()), _vp(spec),
                 _vp(fd), T, 1, _vp(tab), N, R, _st())
        assert AB.projection_ratio(_from_dev(spec[0]), fw, mag_np) <= 1.0
        # Griffin-Lim: 4 iterations against the oracle's, as test_gpu_audio.py does for 1024 / 256
        amp = np.abs(A.lws_stft(_clip(3, n, sr), N, R)).astype(np.float32)
        g4 = audio.griffin_lim(torch.from_numpy(amp).cuda(), n_iter=4).cpu().numpy()
        r4 = G.griffin_lim(amp, 4, N, R)
        np.testing.assert_allclose(g4, r4, rtol=2e-2, atol=2e-3 * np.abs(r4).max())


@pytest.mark.parametrize("sr,N,R", [(16000, 800, 200), (22050, 1024, 512), (48000, 2400, 600), (48000, 4096, 1024),
                                    (22050, 2048, 256)], ids=["800-200", "1024-512", "2400-600", "4096-1024",
                                                              "2048-256"])
def test_ragged_griffin_lim_and_lws_bit_identical_alone(sr, N, R):
    from deepvoice3_pytorch_b200 import audio
    with frame(sr, N, R):
        frames = [23, 9, 60, 12]                                      # >= Q frames: at least one sample each
        K = N // 2 + 1
        mags = [np.abs(A.lws_stft(_clip(30 + i, audio.inv_num_samples(t), sr), N, R)).astype(np.float32)
                for i, t in enumerate(frames)]
        batch = torch.full((len(frames), max(frames), K), 1e3, device="cuda")              # loud padding
        for c, a in enumerate(mags):
            assert a.shape == (frames[c], K)
            batch[c, :a.shape[0]] = torch.from_numpy(a)
        for fn, kw in ((audio.griffin_lim_batch, dict(n_iter=5)), (audio.lws_batch, dict(n_iter=5, init_iters=1)),
                       (audio.lws_batch, dict(n_iter=0, init_iters=2))):
            y = fn(batch, frames, **kw)
            assert torch.equal(y, fn(batch, frames, **kw))
            for c, a in enumerate(mags):
                n = audio.inv_num_samples(frames[c])
                alone = fn(torch.from_numpy(a).cuda()[None], [frames[c]], **kw)[0]
                assert alone.shape == (n,)
                assert torch.equal(y[c, :n], alone), (fn.__name__, kw, c)
                assert not y[c, n:].any()


def _to_dev(X):
    return torch.from_numpy(np.stack([X.real, X.imag], -1).astype(np.float32)).cuda()


def _from_dev(t):
    a = t.cpu().numpy().astype(np.float64)
    return a[..., 0] + 1j * a[..., 1]


def _scale(X, beta, Q):
    T, K = X.shape
    H = Q - 1
    Xe = np.abs(G._extend(X, H))
    s = np.zeros((T, K))
    for q in range(-H, H + 1):
        for d in range(-5, 6):
            s += abs(beta[q + H, d + 5]) * Xe[H + q:H + q + T, 5 - d:5 - d + K]
    return s


LWS_GEOMS = [(16000, 256, 64), (16000, 800, 200), (22050, 1024, 512), (22050, 2048, 256), (48000, 4096, 1024)]


@pytest.mark.parametrize("sr,N,R", LWS_GEOMS, ids=["%d-%d" % (N, R) for _, N, R in LWS_GEOMS])
def test_lws_iteration_and_nofuture_scan_against_oracle(sr, N, R):
    """One Jacobi iteration elementwise (the bound of test_gpu_lws.py) and the no-future scan teacher-forced."""
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    Q, K = N // R, N // 2 + 1
    with frame(sr, N, R):
        T = 21
        amp = np.abs(A.lws_stft(_clip(5, audio.inv_num_samples(T), sr), N, R)).astype(np.float32)
        rng = np.random.RandomState(0)
        X = amp * np.exp(2j * np.pi * rng.rand(T, K))
        X[:, [0, K - 1]] = X[:, [0, K - 1]].real
        X = _from_dev(_to_dev(X))
        beta = G.lws_weights(N, R)
        want = G.lws_iterate(X, amp, beta, Q)
        Y = G.lws_local_sum(X, beta, Q)
        mag = torch.from_numpy(amp).cuda()
        g = audio.check_geometry(mel=False)
        w = audio._lws_weights(mag.device, g)
        fd = torch.tensor([T], dtype=torch.int32).cuda()
        xin, xout = _to_dev(X), torch.full((T, K, 2), float("nan"), device="cuda")
        lib.call("dv3_lws_iterate_geom", _vp(mag), _vp(xin), _vp(xout), _vp(w), _vp(fd), T, 1, N, R, _st())
        got = _from_dev(xout)
        sc = _scale(X, beta, Q)
        ok = np.abs(Y) >= 1e-2 * sc
        ok[:, [0, K - 1]] = np.abs(Y[:, [0, K - 1]].real) >= 1e-2 * sc[:, [0, K - 1]]
        assert ok.mean() > 0.95, ok.mean()
        assert np.isfinite(got).all() and np.allclose(np.abs(got), amp, rtol=1e-5, atol=1e-6 * amp.max())
        bad = np.abs(got - want) > 1e-5 * amp + 1e-7 * amp.max()
        assert not (bad & ok).any(), np.argwhere(bad & ok)[:10]
        assert not got[:, [0, K - 1]].imag.any()
        for init_iters in (0, 1, 3):
            spec = torch.full((T, K, 2), float("nan"), device="cuda")
            lib.call("dv3_lws_nofuture_geom", _vp(mag), _vp(spec), _vp(w), _vp(fd), T, 1, init_iters, N, R, _st())
            got = _from_dev(spec)
            assert np.isfinite(got).all()
            prev = np.zeros((T + Q - 1, K), dtype=np.complex128)
            prev[Q - 1:] = got
            errs = np.array([np.abs(got[m] - G.lws_nofuture_frame(amp[m], prev[m:m + Q - 1], beta, Q, init_iters))
                             / (amp[m] + 1e-6 * amp.max()) for m in range(T)])
            assert (errs > 1e-4).mean() < 0.01, (init_iters, (errs > 1e-4).mean())
            assert np.median(errs) < 1e-6, (init_iters, np.median(errs))


@pytest.mark.parametrize("sr,N,R", [(16000, 800, 200), (22050, 2048, 256)], ids=["800-200", "2048-256"])
def test_lws_end_to_end_quality_against_oracle(sr, N, R):
    """LWS (no-future + 30 iterations) within 5 % of the oracle's spectral convergence."""
    from deepvoice3_pytorch_b200 import audio
    with frame(sr, N, R):
        for seed in (0, 1):
            T = 120
            amp = np.abs(A.lws_stft(_clip(seed, audio.inv_num_samples(T), sr), N, R)).astype(np.float32)
            y = audio.lws(torch.from_numpy(amp).cuda(), n_iter=30).cpu().numpy()
            sc_gpu = G.spectral_convergence(amp, y, N, R)
            sc_oracle = G.spectral_convergence(amp, G.lws(amp, N, R, 30), N, R)
            assert abs(sc_gpu - sc_oracle) <= 0.05 * sc_oracle, (seed, sc_gpu, sc_oracle)


@pytest.mark.parametrize("sr,N,R", [(22050, 2048, 512), (24000, 1200, 300)], ids=["2048-512", "1200-300"])
def test_synthesis_at_other_frames(sr, N, R):
    """A model with linear_dim = N/2 + 1: tts_batch and tts_stream with both vocoders return inv_num_samples samples;
    in exact-fp32 mode each row equals synthesizing it alone, and tts_stream equals tts_batch."""
    from deepvoice3_pytorch_b200 import builder, ops, synthesis, audio
    from test_gpu_synthesis import _sequences
    K = N // 2 + 1
    with frame(sr, N, R):
        torch.manual_seed(7)
        model = builder.nyanko(n_vocab=149, embed_dim=128, mel_dim=80, linear_dim=K, r=1, downsample_step=4,
                               encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=512,
                               dropout=0.0).cuda().eval()
        dec = model.seq2seq.decoder
        dec.max_decoder_steps, dec.min_decoder_steps = 12, 6
        seqs = _sequences([21, 5, 33], seed=4)
        old = ops.conv_math
        ops.conv_math = "fp32"
        try:
            for vocoder in ("griffin_lim", "lws"):
                got = synthesis.tts_batch(model, seqs, vocoder=vocoder)
                streamed = dict(synthesis.tts_stream(model, seqs, slots=2, post_batch=2, vocoder=vocoder))
                for i, s in enumerate(seqs):
                    wav, _, spec, _ = got[i]
                    assert spec.shape[1] == K
                    assert wav.shape == (audio.inv_num_samples(spec.shape[0]),)
                    alone = synthesis.tts_batch(model, [s], vocoder=vocoder)[0]
                    assert np.array_equal(alone[0], wav), (vocoder, i)
                    for a, b in zip(streamed[i], got[i]):
                        assert np.array_equal(a, b), (vocoder, i)
        finally:
            ops.conv_math = old


def test_default_frame_entry_points(tmp_path):
    """At 1024 / 256: preprocessing and targets call only the specialised forward kernels (dv3_stft_mel /
    dv3_stft_mel_targets, never dv3_stft_mel_geom) and LWS only its specialised kernels; Griffin-Lim, LWS and tts_batch
    run the complex STFT and the inverse STFT through dv3_stft_complex_geom / dv3_istft_geom."""
    from deepvoice3_pytorch_b200 import audio, preprocess, synthesis, builder
    from deepvoice3_pytorch_b200._lib import lib
    from test_gpu_synthesis import _sequences
    seen = []
    real = lib.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)
    in_dir, out_dir = str(tmp_path / "in"), str(tmp_path / "out")
    _write_corpus(in_dir, 22050, n_clips=3)
    os.makedirs(out_dir)
    torch.manual_seed(7)
    model = builder.nyanko(n_vocab=149, embed_dim=128, mel_dim=80, linear_dim=513, r=1, downsample_step=4,
                           encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=512,
                           dropout=0.0).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = 8
    lib.call = spy
    try:
        preprocess.build_from_path(in_dir, out_dir, batch_clips=2)
        wav = torch.zeros(2, 5000, dtype=torch.int16, device="cuda")
        audio.stft_mel_targets(wav, [5000, 3000], 40, 1, 4)
        mag = torch.rand(2, 20, 513, device="cuda")
        audio.griffin_lim_batch(mag, [20, 11], n_iter=2)
        audio.lws_batch(mag, [20, 11], n_iter=2)
        synthesis.tts_batch(model, _sequences([9, 4], seed=2))
        synthesis.tts_batch(model, _sequences([9, 4], seed=2), vocoder="lws")
    finally:
        lib.call = real
    want = {"dv3_stft_mel", "dv3_stft_mel_targets", "dv3_stft_complex_geom", "dv3_istft_geom",
            "dv3_lws_nofuture_batched", "dv3_lws_iterate_batched"}
    assert not [n for n in seen if ("stft" in n or "lws" in n) and n not in want], sorted(set(seen))
    for name in sorted(want):
        assert name in seen, name


@pytest.mark.parametrize("N,R,mels", [(1024, 200, 80), (1102, 551, 80), (8192, 2048, 80), (1023, 341, 80),
                                      (4096, 256, 80), (1024, 256, 129)])
def test_refused_geometry_raises_before_any_launch(monkeypatch, N, R, mels):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import Dv3Error

    def no_call(*a, **k):
        raise AssertionError("reached a CUDA library call")
    wav = torch.zeros(2, 4096, device="cuda")
    mag = torch.zeros(2, 12, N // 2 + 1, device="cuda")
    with frame(22050, N, R):
        audio.hparams.num_mels = mels
        monkeypatch.setattr(audio.lib, "call", no_call)
        with pytest.raises(Dv3Error):
            audio.stft_mel_batch(wav)
        with pytest.raises(Dv3Error):
            audio.stft_mel_targets(wav, [4096, 100], 64, 1, 4)
        if mels <= 128:
            with pytest.raises(Dv3Error):
                audio.griffin_lim_batch(mag, [12, 10])
            with pytest.raises(Dv3Error):
                audio.lws_batch(mag, [12, 10])
