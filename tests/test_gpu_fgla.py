"""GPU: fast Griffin-Lim (csrc/stft_any.cu stft_complex_momentum_any_kernel at every frame;
audio.griffin_lim_batch(momentum > 0)) against the fp64 oracle of
tests/fgla_oracle.py: one momentum step elementwise within the bounds of tests/audio_bounds.py, bit identity with the
plain projection at beta = 0, the ragged-batch contract, end-to-end quality, the entry points each path calls, and
inv_spectrogram / synthesis with method "fast_griffin_lim"."""
import ctypes
import types

import numpy as np
import pytest
import torch

import audio_bounds as AB
import fgla_oracle as F
from oracle import audio_oracle as A
from test_fgla_host import RATIO_BOUND, clip_mags
from test_gpu_stft_geometry import GEOMS, IDS, frame

pytestmark = pytest.mark.gpu

ALL = [(22050, 1024, 256)] + GEOMS
ALL_IDS = ["22k-1024-256"] + IDS
BETA = float(np.float32(F.beta_of(0.99)))            # the fp32 coefficient the kernels receive at momentum 0.99


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _complex(t):
    a = t.cpu().numpy().astype(np.float64)
    return a[..., 0] + 1j * a[..., 1]


def _pairs(X):
    return torch.from_numpy(np.stack([X.real, X.imag], -1).astype(np.float32)).cuda()


class _Step:
    """Three clips of a ragged batch at the frame (N, R) with their magnitudes and a prev spectrum; runs the plain and
    the momentum entry points at that frame.  Clip 0 has a silent stretch of 3 N samples: there X == 0, and prev is
    set to 0, so C == 0."""

    def __init__(self, N, R):
        from deepvoice3_pytorch_b200 import audio
        self.N, self.R, self.K = N, R, N // 2 + 1
        self.frames = [41, 9, 3 * (N // R)]
        self.ns = [audio.inv_num_samples(t) for t in self.frames]
        self.pitch = max(self.ns) + 29
        self.Tm = max(self.frames)
        rng = np.random.RandomState(N + R)
        wav = np.zeros((3, self.pitch), np.float32)
        for c, n in enumerate(self.ns):
            wav[c, :n] = 0.4 * rng.randn(n) + A.synthetic_clip(c, n=max(n, 2))[:n]
        wav[:, -1] = 5.0                                        # past every clip: must not be read
        s0 = self.ns[0] // 3
        wav[0, s0:s0 + 3 * N] = 0.0
        self.wav = wav
        self.wd = torch.from_numpy(wav).cuda()
        self.nd = torch.tensor(self.ns, dtype=torch.int32).cuda()
        self.fd = torch.tensor(self.frames, dtype=torch.int32).cuda()
        self.refs = [AB.Forward(wav[c, :self.ns[c]], N, R, "any", preemph=None,
                                T=self.frames[c]) for c in range(3)]
        self.silent = [f for f in range(self.frames[0]) if not self.refs[0].X[f].any()]
        assert len(self.silent) >= 2, self.silent
        mags = np.full((3, self.Tm, self.K), 1e3, np.float32)              # loud padding: must not leak in
        prev = np.full((3, self.Tm, self.K), 7.0 - 3.0j)
        for c in range(3):
            X = self.refs[c].X
            T = self.frames[c]
            mags[c, :T] = (np.abs(X) * rng.uniform(0.5, 1.5, X.shape)).astype(np.float32)
            # prev: a spectrum of the same size with its own phase, as the previous iteration's X would be
            prev[c, :T] = np.abs(X) * rng.uniform(0.3, 1.7, X.shape) * np.exp(2j * np.pi * rng.rand(*X.shape))
        prev[0, self.silent] = 0.0
        mags[0, self.silent[0], :5] = 0.0                        # mag 0 on C == 0 bins: (0, 0)
        self.mags, self.md = mags, torch.from_numpy(mags).cuda()
        self.prev = _complex(_pairs(prev))                        # the fp32 values the kernel reads
        self.tab = audio._geometry_table(self.wd.device, N, R)

    def plain(self, mag):
        from deepvoice3_pytorch_b200._lib import lib
        spec = torch.full((3, self.Tm, self.K, 2), float("nan"), device="cuda")
        lib.call("dv3_stft_complex_geom", _vp(self.wd), _vp(self.nd), self.pitch, _vp(mag), _vp(spec),
                 _vp(self.fd), self.Tm, 3, _vp(self.tab), self.N, self.R, _st())
        return spec

    def momentum(self, beta):
        """-> (prev after the call, spec) as device tensors; spec starts NaN."""
        from deepvoice3_pytorch_b200._lib import lib
        prev = _pairs(self.prev)
        spec = torch.full((3, self.Tm, self.K, 2), float("nan"), device="cuda")
        lib.call("dv3_stft_complex_momentum_geom", _vp(self.wd), _vp(self.nd), self.pitch, _vp(self.md),
                 _vp(prev), _vp(spec), _vp(self.fd), self.Tm, 3, beta, _vp(self.tab), self.N, self.R, _st())
        return prev, spec


def _c_forward(fw, prev, beta):
    """The reference of C = X - beta prev in projection_ratio's form: X = the fp64 C, B = per-frame bound of
    |C_hat - C|.  C_hat = rn(X_hat - beta prev) per component (one fmaf, beta and prev exact fp32 inputs), so
    |C_hat - C| <= |X_hat - X| + u (|C| + |X_hat - X|) <= B_X (1 + u) + u max_k |C|."""
    C = fw.X - beta * prev
    return types.SimpleNamespace(X=C, B=AB.SECOND_ORDER * (fw.B * (1 + AB.U) + AB.U * np.abs(C).max(-1)))


@pytest.mark.parametrize("sr,N,R", ALL, ids=ALL_IDS)
def test_zero_beta_is_the_plain_projection_bit_for_bit(sr, N, R):
    """beta = 0: spec equals the plain projected STFT and prev the plain unprojected STFT, bit for bit, whatever prev
    held before."""
    with frame(sr, N, R):
        s = _Step(N, R)
        prev, spec = s.momentum(0.0)
        want_spec, want_X = s.plain(s.md), s.plain(None)
        for c, T in enumerate(s.frames):
            assert torch.equal(spec[c, :T], want_spec[c, :T]), c
            assert torch.equal(prev[c, :T], want_X[c, :T]), c


@pytest.mark.parametrize("sr,N,R", ALL, ids=ALL_IDS)
def test_one_momentum_step_against_fp64(sr, N, R):
    """Given x and prev: prev out within complex_ratio of X, spec within projection_ratio of the projection of
    C = X - beta prev; frames with X == 0 and prev == 0 give exactly (mag, 0); frames past a clip's count untouched."""
    with frame(sr, N, R):
        s = _Step(N, R)
        prev_d, spec_d = s.momentum(BETA)
        prev_out, spec = _complex(prev_d), _complex(spec_d)
        for c, T in enumerate(s.frames):
            fw = s.refs[c]
            assert AB.complex_ratio(prev_out[c, :T], fw) <= 1.0, c
            assert AB.projection_ratio(spec[c, :T], _c_forward(fw, s.prev[c, :T], BETA), s.mags[c, :T]) <= 1.0, c
            # untouched past the clip's frames
            assert np.isnan(spec[c, T:]).all(), c
            assert np.array_equal(prev_out[c, T:], s.prev[c, T:]), c
        for f in s.silent:
            assert np.array_equal(spec[0, f], s.mags[0, f] + 0j), f
            assert not prev_out[0, f].any(), f
        # the momentum really enters: spec differs from the plain projection of X
        plain = _complex(s.plain(s.md))
        assert not np.array_equal(spec[0, :s.frames[0]], plain[0, :s.frames[0]])


RAGGED = [(22050, 1024, 256), (16000, 800, 200), (22050, 1024, 512), (48000, 2400, 600), (48000, 4096, 1024),
          (22050, 2048, 256)]


@pytest.mark.parametrize("sr,N,R", RAGGED, ids=["%d-%d" % (N, R) for _, N, R in RAGGED])
def test_ragged_batch_bit_identical_alone_and_reproducible(sr, N, R):
    from deepvoice3_pytorch_b200 import audio
    with frame(sr, N, R):
        frames = [23, 9, 60, 12]
        K = N // 2 + 1
        mags = [np.abs(A.lws_stft(A.synthetic_clip(40 + i, n=audio.inv_num_samples(t), sr=sr), N, R))
                .astype(np.float32) for i, t in enumerate(frames)]
        batch = torch.full((len(frames), max(frames), K), 1e3, device="cuda")
        for c, a in enumerate(mags):
            batch[c, :a.shape[0]] = torch.from_numpy(a)
        y = audio.griffin_lim_batch(batch, frames, n_iter=5, momentum=0.99)
        assert torch.equal(y, audio.griffin_lim_batch(batch, frames, n_iter=5, momentum=0.99))
        plain = audio.griffin_lim_batch(batch, frames, n_iter=5)
        assert not torch.equal(y, plain)
        for c, a in enumerate(mags):
            n = audio.inv_num_samples(frames[c])
            alone = audio.griffin_lim(torch.from_numpy(a).cuda(), n_iter=5, momentum=0.99)
            assert alone.shape == (n,)
            assert torch.equal(y[c, :n], alone), c
            assert not y[c, n:].any(), c


@pytest.mark.parametrize("sr,N,R,T", [(22050, 1024, 256, 200), (22050, 2048, 512, 120)], ids=["1024-256", "2048-512"])
def test_end_to_end_quality(sr, N, R, T):
    """FGLA-n on the GPU within 5 % of the oracle's spectral convergence at n = 10, 30, 60, and against the GPU's
    GL-n the bound of tests/test_fgla_host.py (mean ratio <= RATIO_BOUND[n], every clip below GL-n)."""
    from deepvoice3_pytorch_b200 import audio
    with frame(sr, N, R):
        mags = clip_mags(sr, N, R, T)
        ratios = {n: [] for n in RATIO_BOUND}
        for a in mags:
            a32 = a.astype(np.float32)
            oracle = F.sc_sweep(a32, RATIO_BOUND, N, R)
            mag = torch.from_numpy(a32).cuda()
            for n in RATIO_BOUND:
                y = audio.griffin_lim(mag, n_iter=n, momentum=0.99).cpu().numpy()
                gl = audio.griffin_lim(mag, n_iter=n).cpu().numpy()
                sc, sc_gl = F.spectral_convergence(a32, y, N, R), F.spectral_convergence(a32, gl, N, R)
                assert abs(sc - oracle[n]) <= 0.05 * oracle[n], (n, sc, oracle[n])
                assert sc < sc_gl, (n, sc, sc_gl)
                ratios[n].append(sc / sc_gl)
        for n, r in ratios.items():
            assert np.mean(r) <= RATIO_BOUND[n], (n, r)


def _recorded(fn):
    from deepvoice3_pytorch_b200._lib import lib
    seen = []
    real = lib.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)
    lib.call = spy
    try:
        fn()
    finally:
        lib.call = real
    return seen


AUDIO = ("stft", "istft", "lws", "spec_to_amp", "deemphasis")


def test_existing_paths_call_the_same_entry_points():
    """Griffin-Lim without momentum, the default inv_spectrogram, LWS and the default tts_batch call exactly the
    sequence of audio entry points they call without this feature; the momentum entry points appear only with
    momentum > 0."""
    from deepvoice3_pytorch_b200 import audio, synthesis
    from test_gpu_synthesis import _model, _sequences
    gl = ["dv3_istft_geom"] + ["dv3_stft_complex_geom", "dv3_istft_geom"] * 3
    mag = torch.rand(2, 20, 513, device="cuda")
    assert _recorded(lambda: audio.griffin_lim_batch(mag, [20, 11], n_iter=3)) == gl
    assert _recorded(lambda: audio.griffin_lim_batch(mag, [20, 11], n_iter=3, momentum=0)) == gl
    assert _recorded(lambda: audio.griffin_lim_batch(mag, [20, 11], n_iter=3, momentum=0.5)) == \
        ["dv3_istft_geom"] + ["dv3_stft_complex_momentum_geom", "dv3_istft_geom"] * 3
    assert _recorded(lambda: audio.lws_batch(mag, [20, 11], n_iter=2)) == \
        ["dv3_lws_nofuture_batched"] + ["dv3_lws_iterate_batched"] * 2 + ["dv3_istft_geom"]
    S = audio.spectrogram(A.synthetic_clip(8, n=40 * 256 - 512))
    default_inv = ["dv3_spec_to_amp", "dv3_istft_geom"] + ["dv3_stft_complex_geom", "dv3_istft_geom"] * 60 \
        + ["dv3_deemphasis"]
    assert _recorded(lambda: audio.inv_spectrogram(S)) == default_inv
    fast = _recorded(lambda: audio.inv_spectrogram(S, method="fast_griffin_lim"))
    assert fast == ["dv3_spec_to_amp", "dv3_istft_geom"] + \
        ["dv3_stft_complex_momentum_geom", "dv3_istft_geom"] * audio.hparams.fast_griffin_lim_iters + \
        ["dv3_deemphasis"]
    model = _model("nyanko_ljspeech", max_steps=16)
    seqs = _sequences([9, 4], seed=2)
    calls = _recorded(lambda: synthesis.tts_batch(model, seqs))
    assert not [n for n in calls if "momentum" in n]
    assert [n for n in calls if any(a in n for a in AUDIO)] == default_inv
    calls = _recorded(lambda: synthesis.tts_batch(model, seqs, vocoder="fast_griffin_lim"))
    assert "dv3_stft_complex_momentum_geom" in calls and "dv3_stft_complex_geom" not in calls


@pytest.mark.parametrize("preset", ["deepvoice3_ljspeech", "nyanko_ljspeech", "deepvoice3_vctk"])
def test_inv_spectrogram_and_synthesis_fast_griffin_lim(preset):
    """inv_spectrogram(method="fast_griffin_lim") is griffin_lim_batch with the two hparams; tts_batch and tts_stream
    with vocoder="fast_griffin_lim": every row bit-identical to its utterance synthesized alone (exact-fp32 mode)."""
    from deepvoice3_pytorch_b200 import audio, synthesis
    from test_gpu_synthesis import _conv_math, _model, _sequences
    S = audio.spectrogram(A.synthetic_clip(8, n=40 * 256 - 512))
    y = audio.inv_spectrogram(S, method="fast_griffin_lim")
    assert y.dtype == np.float32 and y.shape == (audio.inv_num_samples(S.shape[1]),)
    assert not np.array_equal(y, audio.inv_spectrogram(S))
    assert np.array_equal(audio.inv_spectrogram(S, n_iter=7, method="fast_griffin_lim"),
                          audio.inv_spectrogram_batch([S], 7, "fast_griffin_lim")[0])

    model = _model(preset, max_steps=24)
    seqs = _sequences([37, 5, 61, 20], seed=4)
    spk = [3, 17, 0, 54] if model.n_speakers > 1 else None
    with _conv_math("fp32"):
        got = synthesis.tts_batch(model, seqs, speaker_ids=spk, vocoder="fast_griffin_lim")
        streamed = dict(synthesis.tts_stream(model, seqs, speaker_ids=spk, slots=2, post_batch=3,
                                             vocoder="fast_griffin_lim"))
        for i, s in enumerate(seqs):
            alone = synthesis.tts_batch(model, [s], speaker_ids=None if spk is None else [spk[i]],
                                        vocoder="fast_griffin_lim")[0]
            for a, b in zip(alone, got[i]):
                assert np.array_equal(a, b), i
            for a, b in zip(streamed[i], got[i]):
                assert np.array_equal(a, b), i
            assert got[i][0].shape == (audio.inv_num_samples(got[i][2].shape[0]),)
