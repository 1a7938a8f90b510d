"""Host tests of the neural vocoder: the fp64 oracle of the multi-resolution STFT loss against torch autograd, the STFT
adjoint and its inverse-STFT form, the alignment rule, refusals before any library call, the C ABI and ptxas report of
csrc/vocoder.cu, and VocoderBatches."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import vocoder_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = ((512, 128), (1024, 256), (2048, 512))


def _pair(seed, n):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 0.3
    return x + 0.2 * rng.standard_normal(n), x


def test_oracle_gradient_matches_torch_fp64_autograd():
    ys, xs = zip(*[_pair(s, n) for s, n in ((0, 3000), (1, 2500))])
    res = ((512, 128), (1024, 256))
    yt = [torch.tensor(y, requires_grad=True) for y in ys]
    L = VO.torch_loss(yt, [torch.tensor(x) for x in xs], res)
    L.backward()
    assert abs(L.item() - VO.loss(ys, xs, res)) <= 1e-12 * L.item()
    for g, t in zip(VO.grad_wave(ys, xs, res), yt):
        np.testing.assert_allclose(g, t.grad.numpy(), rtol=1e-9, atol=1e-12 * np.abs(g).max())


@pytest.mark.parametrize("N,R", RES + ((768, 128), (1024, 512)))
def test_stft_adjoint_identity_fp64(N, R):
    rng = np.random.default_rng(N + R)
    n = 3 * N + 17
    x = rng.standard_normal(n)
    X = VO.stft(x, N, R)
    G = rng.standard_normal(X.shape) + 1j * rng.standard_normal(X.shape)
    lhs = np.sum(X.real * G.real + X.imag * G.imag)
    adj = VO.stft_adjoint(G, N, R, n)
    assert abs(lhs - np.dot(x, adj)) <= 1e-10 * np.abs(x).sum() * np.abs(adj).max()
    # the kernels' form: the inverse STFT of the rescaled spectrum (imaginary parts of DC / Nyquist dropped)
    np.testing.assert_allclose(VO.istft(VO.adjoint_spectrum(G, N), N, R, n), adj, rtol=0, atol=1e-10 * np.abs(adj).max())


@pytest.mark.parametrize("N,R", ((1024, 256), (512, 128), (2048, 256), (768, 192)))
def test_output_length_and_crop_offset(N, R):
    from deepvoice3_pytorch_b200 import audio, vocoder
    from oracle.audio_oracle import lws_window
    old = audio.hparams.fft_size, audio.hparams.hop_size
    audio.hparams.fft_size, audio.hparams.hop_size = N, R
    try:
        off = vocoder.alignment_offset()
        assert off == (N - R) // 2
        for T in (4, 9, 33):
            n = vocoder.output_length(T)
            assert n == (T - 1) * R - (N - 2 * R) == audio.inv_num_samples(T)
            assert audio.num_frames_host(n) == T
            assert off + n <= T * R                              # the crop lies inside the generated samples
        # frame f owns generator samples [fR, fR + R): their centre, as output sample, is frame f's window centre
        w = lws_window(N, R)
        centre_win = np.sum(np.arange(N) * w) / np.sum(w) - (N - R)     # relative to fR, in output samples
        assert abs((R - 1) / 2.0 - off - centre_win) <= 0.5
    finally:
        audio.hparams.fft_size, audio.hparams.hop_size = old


@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


def test_refusals_before_any_library_call(no_lib):
    from deepvoice3_pytorch_b200 import audio, vocoder
    from deepvoice3_pytorch_b200.data import VocoderBatches
    with pytest.raises(ValueError):
        vocoder.NeuralVocoder(upsample=(4, 4, 4, 2))
    with pytest.raises(ValueError):
        vocoder.NeuralVocoder(upsample=(16, 16))
    for bad in ([], [(1000, 256)], [(1024, 100)], [(1024, 1024)], [(8192, 2048)], [(1024,)], None):
        with pytest.raises(ValueError):
            vocoder.check_resolutions(bad)
        with pytest.raises(ValueError):
            vocoder.stft_loss(torch.zeros(1, 4096), torch.zeros(1, 4096), bad)
    with pytest.raises(ValueError):
        vocoder.vocoder_batch({"pcm": torch.zeros(1, 10000), "lengths": [10000], "starts": [0]}, 0)
    with pytest.raises(ValueError):
        VocoderBatches([np.zeros(10000, np.float32)] * 4, 2, seg_frames=0)
    voc = vocoder.NeuralVocoder.__new__(vocoder.NeuralVocoder)      # an instance: no parameters needed to refuse
    torch.nn.Module.__init__(voc)
    spec = np.zeros((513, 10), np.float32)
    with pytest.raises(ValueError):
        audio.inv_spectrogram(spec, n_iter=10, method=voc)
    with pytest.raises(ValueError):
        audio.inv_spectrogram_batch([spec], n_iter=0, method=voc)
    for bad in ("wavenet", None, 3):
        with pytest.raises(ValueError):
            audio.check_phase_method(bad)
        with pytest.raises(ValueError):
            audio.inv_spectrogram_batch([spec], method=bad)
    assert audio.check_phase_method(voc) is voc
    assert no_lib == []


def test_check_frame_is_check_geometry_rules():
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import Dv3Error
    for N, R in ((1024, 256), (512, 128), (2048, 512), (768, 96), (4096, 512)):
        assert audio.check_frame(N, R) == (N, R)
    for N, R in ((1022, 511), (254, 127), (4100, 1025), (1024, 1024), (1024, 100), (1024.5, 256), (14 * 64, 112)):
        with pytest.raises(Dv3Error):
            audio.check_frame(N, R)


def test_conv_transpose_accepts_kernel_equal_stride_only():
    from deepvoice3_pytorch_b200.conv import ConvTranspose1d
    for s in range(2, 9):
        m = ConvTranspose1d(8, 4, s, stride=s)
        assert tuple(m.weight_v.shape) == (8, 4, s) and m.stride == (s,)
    for k, s, p in ((3, 2, 0), (2, 2, 1), (9, 9, 0), (1, 1, 0), (4, 2, 0)):
        with pytest.raises(ValueError):
            ConvTranspose1d(8, 4, k, stride=s, padding=p)


def test_default_topology():
    from deepvoice3_pytorch_b200 import conv as C, modules as Mo, vocoder
    v = vocoder.NeuralVocoder()
    kinds = [type(m).__name__ for m in v.layers]
    assert kinds == (["Conv1d", "ReLU"] + ["Conv1dGLU"] * 2 + (["ConvTranspose1d"] + ["Conv1dGLU"] * 3) * 4
                     + ["Conv1d"])
    ups = [m for m in v.layers if isinstance(m, C.ConvTranspose1d)]
    assert [(m.in_channels, m.out_channels, m.stride[0]) for m in ups] == [(256, 128, 4)] + [(128, 128, 4)] * 3
    glus = [m for m in v.layers if isinstance(m, Mo.Conv1dGLU)]
    assert [m.conv.dilation[0] for m in glus] == [1, 3] + [1, 3, 9] * 4
    assert all(m.residual and not m.causal and m.dropout == 0 and m.speaker_proj is None for m in glus)
    assert v.layers[0].in_channels == 513 and v.layers[-1].out_channels == 1


NAMES = ("dv3_mrstft_ws_doubles", "dv3_mrstft_loss_fwd", "dv3_mrstft_loss_total", "dv3_mrstft_loss_bwd",
         "dv3_vocoder_gather", "dv3_interleave", "dv3_tc_weightnorm_convt_s_fwd")


def test_c_abi_declares_and_exports_the_vocoder_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    for n in NAMES:
        assert n in d, n
    assert [a for _, a in d["dv3_mrstft_loss_bwd"][1]] == ["spec_y", "spec_x", "stats", "B", "max_frames", "n_fft",
                                                           "hop", "M", "d_loss", "adjoint", "dspec", "stream"]
    assert d["dv3_mrstft_ws_doubles"][0] == ctypes.c_longlong
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in NAMES:
            assert re.search(r"\bT %s\b" % name, nm), name
        lib = ctypes.CDLL(so)
        lib.dv3_mrstft_ws_doubles.restype = ctypes.c_longlong
        assert lib.dv3_mrstft_ws_doubles(16, 70) == 16 * 9 * 3


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "vocoder.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    kernels = sorted(re.sub(r"^_ZN3dv3\d+(\w+?)E.*$", r"\1", n) for n, *_ in frames)
    assert kernels == ["interleave_s_kernel", "mrstft_bwd_kernel", "mrstft_clip_kernel", "mrstft_partials_kernel",
                       "mrstft_total_kernel", "voc_gather_kernel"], rep
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


def test_vocoder_batches_deterministic_in_seed_and_epoch(tmp_path):
    from deepvoice3_pytorch_b200.data import VocoderBatches
    from deepvoice3_pytorch_b200.audio import num_frames_host
    rng = np.random.default_rng(0)
    wavs = [rng.standard_normal(int(n)).astype(np.float32) for n in rng.integers(2000, 20000, 11)]
    wavs.append((rng.standard_normal(500) * 1000).astype(np.int16))           # too short for 8 frames
    vb = VocoderBatches(wavs, 3, seg_frames=8, seed=5)
    assert len(vb) == len(vb.eligible) // 3 and 11 not in vb.eligible

    def draw(v, epoch):
        v.set_epoch(epoch)
        return [{k: t.numpy().copy() for k, t in b.items()} for b in v]
    a, b = draw(vb, 0), draw(VocoderBatches(wavs, 3, seg_frames=8, seed=5), 0)
    c = draw(vb, 1)
    assert len(a) == len(vb)
    for p, q in zip(a, b):
        for k in p:
            np.testing.assert_array_equal(p[k], q[k])
    assert any(not np.array_equal(p["items"], q["items"]) or not np.array_equal(p["starts"], q["starts"])
               for p, q in zip(a, c))
    for batch in a:
        assert batch["pcm"].dtype == np.float32 and batch["pcm"].shape[0] == 3
        for row, (i, n, s) in enumerate(zip(batch["items"], batch["lengths"], batch["starts"])):
            assert n == wavs[i].size and 0 <= s <= num_frames_host(n) - 8
            np.testing.assert_array_equal(batch["pcm"][row, :n], wavs[i])
    with pytest.raises(ValueError):
        VocoderBatches(wavs, 12, seg_frames=8)
    with pytest.raises(ValueError):
        VocoderBatches(wavs, 2, seg_frames=10 ** 4)


def test_vocoder_batches_from_a_wav_dataset(tmp_path):
    """Rows of a WavDataset source are whole utterances at the training rate: the pcm length of each row gives the
    item's frame_lengths; a segmented (VCTK) dataset, whose items are raw spans at the file's rate, is refused."""
    from scipy.io import wavfile
    from deepvoice3_pytorch_b200.audio import num_frames_host, hparams
    from deepvoice3_pytorch_b200.data import VocoderBatches, WavDataset
    rng = np.random.default_rng(3)
    items = []
    for k, (sr, n) in enumerate(((hparams.sample_rate, 9000), (44100, 20000), (hparams.sample_rate, 15000),
                                 (16000, 7000))):
        path = str(tmp_path / ("u%d.wav" % k))
        wavfile.write(path, sr, (rng.standard_normal(n) * 3000).astype(np.int16))
        items.append((path, "text %d" % k))
    ds = WavDataset(items, lambda t: [1, 2, 3])
    vb = VocoderBatches(ds, 2, seg_frames=8, seed=1)
    seen = 0
    for batch in vb:
        for row, (i, n, s) in enumerate(zip(batch["items"].tolist(), batch["lengths"].tolist(),
                                            batch["starts"].tolist())):
            assert num_frames_host(n) == ds.frame_lengths[i]
            assert 0 <= s <= ds.frame_lengths[i] - 8
            pcm = np.asarray(ds[i][1])
            want = pcm.astype(np.float32) / np.float32(32768.0) if pcm.dtype == np.int16 else pcm
            np.testing.assert_array_equal(batch["pcm"][row, :n].numpy(), want)
            seen += 1
    assert seen == 4
    ds._segments = [(48000, 100, True, 0, 100, 0, 100)] * len(ds.items)      # what from_vctk builds
    with pytest.raises(ValueError):
        VocoderBatches(ds, 2, seg_frames=8)
