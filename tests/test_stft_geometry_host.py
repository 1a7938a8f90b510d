"""CPU: the STFT geometries beyond 1024 / 256 (audio.check_geometry, csrc/fft_any.cuh, csrc/stft_any.cu,
csrc/lws_any.cu) -- the geometry rule, the mixed-radix FFT core under g++ against numpy.fft for every supported length,
the fp64 tables, the general LWS weights and oracle against the 1024 / 256 ones, the C ABI of the new entry points and
the ptxas report of the new kernels."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import lws_oracle as O4
import stft_geometry_oracle as G
from oracle import audio_oracle as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc")


def _smooth(m):
    for p in (2, 3, 5):
        while m % p == 0:
            m //= p
    return m == 1


SUPPORTED_N = [n for n in range(256, 4097, 2) if _smooth(n // 2)]


@pytest.fixture
def hp():
    from deepvoice3_pytorch_b200 import audio
    keep = dict(vars(audio.hparams))
    yield audio.hparams
    for k in list(vars(audio.hparams)):
        delattr(audio.hparams, k)
    for k, v in keep.items():
        setattr(audio.hparams, k, v)


def test_supported_lengths():
    assert len(SUPPORTED_N) > 40
    for n in (256, 512, 800, 960, 1024, 1200, 2048, 2400, 4096):
        assert n in SUPPORTED_N
    for n in (1102, 1000 + 2 * 7, 8192, 254, 1023):
        assert n not in SUPPORTED_N


@pytest.mark.parametrize("N,R,mels", [(1024, 200, 80), (1102, 551, 80), (8192, 2048, 80), (1023, 341, 80),
                                      (4096, 256, 80), (1024, 256, 129), (1024, 1024, 80), (128, 64, 80)])
def test_refused_geometries_raise_before_any_launch(hp, monkeypatch, N, R, mels):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import Dv3Error

    def no_cuda(*a, **k):
        raise AssertionError("reached a CUDA call")
    monkeypatch.setattr(audio.lib, "call", no_cuda)
    monkeypatch.setattr(audio.lib, "raw", no_cuda)
    monkeypatch.setattr(torch.Tensor, "cuda", no_cuda)
    hp.fft_size, hp.hop_size, hp.num_mels = N, R, mels
    with pytest.raises(Dv3Error):
        audio.check_geometry()
    if mels <= 128:
        with pytest.raises(Dv3Error):
            audio.check_geometry(mel=False)
        with pytest.raises(Dv3Error):
            audio.num_frames(1000)
        with pytest.raises(Dv3Error):
            audio.inv_spectrogram_batch([np.zeros((N // 2 + 1, 12), np.float32)])
    else:
        assert audio.check_geometry(mel=False).default


@pytest.mark.parametrize("sr,N,R", [(16000, 256, 64), (16000, 512, 128), (16000, 800, 200), (22050, 1024, 512),
                                    (22050, 2048, 256), (24000, 1200, 300), (44100, 2048, 512), (48000, 2400, 600),
                                    (48000, 4096, 1024), (22050, 1024, 256)])
def test_accepted_geometries(hp, sr, N, R):
    from deepvoice3_pytorch_b200 import audio
    hp.sample_rate, hp.fft_size, hp.hop_size = sr, N, R
    g = audio.check_geometry()
    assert (g.n_fft, g.hop, g.bins, g.overlap, g.default) == (N, R, N // 2 + 1, N // R, (N, R) == (1024, 256))
    for n in (0, 1, R - 1, R, R + 1, N - 1, N, N + 1, 10 * sr):
        assert audio.num_frames_host(n) == A.num_frames(n, N, R)


def test_fmax_above_nyquist_is_refused(hp):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import Dv3Error
    hp.sample_rate = 8000
    with pytest.raises(Dv3Error, match="Nyquist"):
        audio.check_geometry()
    assert audio.check_geometry(mel=False).default


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fftany") / "fft_any_harness")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", CSRC, os.path.join(ROOT, "tests", "native",
                                                                                 "fft_any_harness.cpp"), "-o", exe])
    return exe


def test_fft_core_matches_numpy_for_every_supported_length(harness):
    """Forward rfft and the inverse (merge + passes) of the g++ build against numpy, for every N the geometry rule
    accepts (radix-2/3/4/5 passes in every combination), within the bounds of tests/audio_bounds.py (kernel "any"):
    |X_hat - X| <= c_fft u sum|x|, and the inverse against the fp64 packed inverse of the harness' own spectrum,
    c_fft u sum|X| / M plus the rounding of the division by M.  Noise, a tone with DC and Nyquist, and an impulse."""
    import audio_bounds as AB
    from deepvoice3_pytorch_b200 import audio
    rng = np.random.default_rng(0)
    worst = {}
    for N in SUPPORTED_N:
        n = np.arange(N)
        signals = {"noise": rng.standard_normal(N),
                   "tone": 0.5 * np.cos(2 * np.pi * (N // 7) * n / N) + 0.25 + 0.125 * (-1.0) ** n,
                   "impulse": (n == 3).astype(np.float64)}
        tab = audio._geometry_table_fp64(N, N // 4 if N % 4 == 0 else N // 2)
        flat = np.concatenate([tab[0], np.stack([tab[1].real, tab[1].imag], -1).ravel(),
                               np.stack([tab[2].real, tab[2].imag], -1).ravel()]).astype(np.float32)
        for name, sig in signals.items():
            x = sig.astype(np.float32)
            out = subprocess.run([harness], input=np.int32(N).tobytes() + flat.tobytes() + x.tobytes(),
                                 stdout=subprocess.PIPE, check=True).stdout
            got = np.frombuffer(out, dtype=np.float32)
            K, M = N // 2 + 1, N // 2
            X = got[:2 * K].astype(np.float64).view(np.complex128)
            y = got[2 * K:].astype(np.float64)
            assert np.isfinite(got).all(), N
            ref = np.fft.rfft(x.astype(np.float64))
            c = AB.c_fft("any", N)
            r_fwd = np.abs(X - ref).max() / (c * AB.U * np.abs(x).sum())
            yref = AB.packed_irfft(X, N)
            r_inv = (np.abs(y - yref) / (c * AB.U * np.abs(X).sum() / M + AB.U * np.abs(yref))).max()
            assert r_fwd <= 1.0 and r_inv <= 1.0, (N, name, r_fwd, r_inv)
            # normwise, and the round trip back to x: tighter than the elementwise bound on noise
            assert np.abs(X - ref).max() <= 1e-5 * np.abs(ref).max(), (N, name)
            assert np.abs(y - x).max() <= 1e-5 * np.abs(x).max(), (N, name)
            worst[name] = max(worst.get(name, (0, 0)), (r_fwd, r_inv))
            worst[name + " u*sum|x|"] = max(worst.get(name + " u*sum|x|", 0),
                                            np.abs(X - ref).max() / (AB.U * np.abs(x).sum()))
    print("fft_any harness, largest (forward, inverse) error / bound and forward error in u sum|x|:", worst)


def test_plan_covers_every_supported_length():
    """make_plan's radices multiply to N / 2 (restated: 4s, then one 2, then 3s and 5s)."""
    for N in SUPPORTED_N:
        m, radices = N // 2, []
        while m % 4 == 0:
            radices.append(4); m //= 4
        if m % 2 == 0:
            radices.append(2); m //= 2
        for p in (3, 5):
            while m % p == 0:
                radices.append(p); m //= p
        assert m == 1 and int(np.prod(radices)) == N // 2


@pytest.mark.parametrize("N,R", [(256, 64), (800, 200), (1024, 256), (1200, 300), (2400, 600), (4096, 1024),
                                 (1024, 512), (2048, 256)])
def test_tables_against_closed_forms(N, R):
    from deepvoice3_pytorch_b200 import audio
    win, tw, sp = audio._geometry_table_fp64(N, R)
    np.testing.assert_allclose(win, A.lws_window(N, R), rtol=0, atol=1e-15)
    np.testing.assert_allclose(np.sum(win.reshape(N // R, R) ** 2, axis=0), 1.0, rtol=0, atol=1e-14)   # perfect rec.
    j = np.arange(N // 2)
    np.testing.assert_allclose(tw, np.cos(2 * np.pi * j / (N // 2)) - 1j * np.sin(2 * np.pi * j / (N // 2)), atol=1e-15)
    k = np.arange(N // 2 + 1)
    np.testing.assert_allclose(sp, np.cos(np.pi * k * 2 / N) - 1j * np.sin(2 * np.pi * k / N), atol=1e-15)
    dev_tab = audio._geometry_table("cpu", N, R).numpy()
    assert dev_tab.shape == (3 * N + 2,) and dev_tab.dtype == np.float32
    want = np.concatenate([win, np.stack([tw.real, tw.imag], -1).ravel(), np.stack([sp.real, sp.imag], -1).ravel()])
    assert np.array_equal(dev_tab, want.astype(np.float32))                               # rounded once from fp64


def _lws_weights_1024_256():
    """audio._lws_weights_fp64 as it was written for the 1024 / 256 frame only."""
    N, R = 1024, 256
    n = np.arange(N)
    w = np.sqrt(0.5 * (1.0 - np.cos(2.0 * np.pi * (n + 0.5) / N)) * 2.0 * R / N)
    beta = np.zeros((7, 11), dtype=np.complex128)
    for q in range(-3, 4):
        j = n - q * R
        ok = (j >= 0) & (j < N)
        ww = np.where(ok, w * w[np.clip(j, 0, N - 1)], 0.0)
        for d in range(-5, 6):
            beta[q + 3, d + 5] = np.sum(ww * np.exp(-2j * np.pi * d * n / N)) / N
    return beta


def test_general_lws_weights_equal_the_1024_256_ones_bit_for_bit():
    from deepvoice3_pytorch_b200 import audio
    old = _lws_weights_1024_256()
    assert np.array_equal(audio._lws_weights_fp64(1024, 256), old)
    assert np.array_equal(audio._lws_weights_fp64(), old)


@pytest.mark.parametrize("N,R", [(800, 200), (1024, 512), (2048, 256), (2400, 600)])
def test_general_lws_weights_and_tables(N, R):
    from deepvoice3_pytorch_b200 import audio
    Q = N // R
    b = audio._lws_weights_fp64(N, R)
    np.testing.assert_allclose(b, G.lws_weights(N, R), rtol=0, atol=1e-15)
    assert b.shape == (2 * Q - 1, 11)
    assert abs(b[Q - 1, 5] - 1.0 / Q) < 1e-15                      # beta_0(0) = sum w^2 / N = 1 / Q
    t = audio._lws_tables_fp64(N, R)
    assert t.shape == ((2 * Q - 1) * 11 + Q,)
    for q in range(-(Q - 1), Q):
        for d in range(-5, 6):
            want = b[q + Q - 1, d + 5] * np.exp(2j * np.pi * d * q / Q)
            assert abs(t[(q + Q - 1) * 11 + d + 5] - want) < 1e-15
    np.testing.assert_allclose(t[-Q:], np.exp(-2j * np.pi * np.arange(Q) / Q), atol=1e-15)


def test_general_lws_oracle_equals_the_1024_256_oracle():
    rng = np.random.RandomState(3)
    T = 17
    x = A.synthetic_clip(2, n=(T - 1) * 256 - 512)
    amp = np.abs(A.lws_stft(x))
    X = amp * np.exp(2j * np.pi * rng.rand(T, 513))
    X[:, [0, 512]] = X[:, [0, 512]].real
    b4, bg = O4.lws_weights(), G.lws_weights(1024, 256)
    assert np.abs(b4 - bg).max() < 1e-15
    scale = np.abs(X).max()
    assert np.abs(O4.lws_local_sum(X, b4) - G.lws_local_sum(X, bg, 4)).max() < 1e-12 * scale
    assert np.abs(O4.lws_iterate(X, amp, b4) - G.lws_iterate(X, amp, bg, 4)).max() < 1e-12 * scale
    assert np.abs(O4.lws_nofuture(amp, b4, 2) - G.lws_nofuture(amp, bg, 4, 2)).max() < 1e-12 * scale
    assert np.abs(O4.lws(amp, 3) - G.lws(amp, 1024, 256, 3)).max() < 1e-12 * np.abs(O4.lws(amp, 3)).max()


@pytest.mark.parametrize("N,R", [(800, 200), (1024, 512), (2048, 256)])
def test_general_lws_weights_are_the_linear_part_of_stft_of_istft(N, R):
    """As tests/test_lws_host.py at 1024 / 256: the complex-linear part of STFT(iSTFT(delta)) at an interior frame is
    beta_q(d) e^{-2 pi i k0 q / Q} at (m0 - q, k0 + d) -- pins the index and sign conventions for any overlap."""
    Q, K = N // R, N // 2 + 1
    beta = G.lws_weights(N, R)
    T, m0 = 24, 12
    Gf = lambda X: A.lws_stft(A.lws_istft(X, N, R), N, R)[:T]
    for k0 in (6, K // 3, K - 7):
        D = np.zeros((T, K), dtype=np.complex128)
        D[m0, k0] = 1.0
        H = (Gf(D) - 1j * Gf(1j * D)) / 2
        for q in range(-(Q - 1), Q):
            for d in range(-5, 6):
                want = beta[q + Q - 1, d + 5] * np.exp(-2j * np.pi * ((k0 * q) % Q) / Q)
                assert abs(H[m0 - q, k0 + d] - want) < 1e-12, (k0, q, d)


def test_general_oracles_reduce_to_the_1024_256_ones():
    h = G.hp(22050, 1024, 256)
    x = A.synthetic_clip(4, n=9000)
    lin, mel = G.process_utterance(x, h)
    rl, rm = A.process_utterance(x)
    assert np.abs(lin - rl).max() < 1e-6 and np.abs(mel - rm).max() < 1e-6
    amp = np.abs(A.lws_stft(x))
    np.testing.assert_allclose(G.griffin_lim(amp, 3, 1024, 256), A.griffin_lim(amp, 3), rtol=0, atol=1e-12)


def test_geom_entry_points_match_the_header():
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import parse_header, LIB_PATH
    _build.build()
    decls = parse_header()
    P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    F = ctypes.c_float
    want = {
        "dv3_stft_num_frames_geom": [I, I, I],
        "dv3_stft_mel_geom": [P, I, P, P, F, P, P, P, P, P, P, I, I, I, I, I, I, I, I, F, F, F, P],
        "dv3_stft_complex_geom": [P, P, LL, P, P, P, I, I, P, I, I, P],
        "dv3_istft_geom": [P, P, P, LL, P, I, I, P, I, I, P],
        "dv3_lws_nofuture_geom": [P, P, P, P, I, I, I, I, I, P],
        "dv3_lws_iterate_geom": [P, P, P, P, P, I, I, I, I, P],
    }
    dll = ctypes.CDLL(LIB_PATH)
    for name, args in want.items():
        assert name in decls, name
        assert [t for t, _ in decls[name][1]] == args, name
        assert decls[name][0] is ctypes.c_int, name
        assert hasattr(dll, name), name
    nf = dll.dv3_stft_num_frames_geom
    nf.argtypes, nf.restype = [I, I, I], I
    for N, R in ((800, 200), (2048, 512), (4096, 1024)):
        for n in (0, 1, R, N, 12345):
            assert nf(n, N, R) == A.num_frames(n, N, R)


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


@pytest.mark.parametrize("src", ["stft_any.cu", "lws_any.cu"])
def test_new_kernels_do_not_spill(tmp_path, src):
    """Every kernel of the general-geometry files: no spills and no stack frame (the FFT radix is a template parameter
    and the plan is held as pass counts, so nothing is indexed at run time)."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    report = r.stdout + r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert len(frames) >= (6 if src == "stft_any.cu" else 2), report
    assert all(f == ("0", "0", "0") for f in frames), report
