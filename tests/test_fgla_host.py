"""CPU: fast Griffin-Lim (audio.griffin_lim_batch with momentum > 0, the csrc/stft_any.cu momentum kernel) -- the fp64
oracle against plain Griffin-Lim, argument checks that fire before any library call, the C ABI of its entry point, and
the ptxas report of its kernel."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import fgla_oracle as F
import stft_geometry_oracle as G
from oracle import audio_oracle as A
from test_stft_geometry_host import CSRC, _nvcc

# Largest mean ratio SC(FGLA-n) / SC(GL-n) over three seeded clips that the GPU must also meet (tests/test_gpu_fgla.py).
# The fp64 oracle measures 0.77 / 0.55 / 0.40 at 1024 / 256 and 0.71 / 0.46 / 0.38 at 2048 / 512 for n = 10 / 30 / 60
# (every clip 0.33 .. 0.79); the bounds leave about 10 % on the larger of the two.
RATIO_BOUND = {10: 0.85, 30: 0.62, 60: 0.45}
GEOMS = [(22050, 1024, 256, 200), (22050, 2048, 512, 120)]


def clip_mags(sr, N, R, T, seeds=(0, 1, 2)):
    """Linear magnitudes (T, K) of seeded synthetic clips that give exactly T frames at (N, R)."""
    n = (T - 1) * R - (N - 2 * R)
    return [np.abs(A.lws_stft(A.synthetic_clip(s, n=n, sr=sr), N, R)) for s in seeds]


@pytest.mark.parametrize("sr,N,R,T", GEOMS, ids=["1024-256", "2048-512"])
def test_zero_momentum_is_griffin_lim(sr, N, R, T):
    amp = clip_mags(sr, N, R, T, seeds=(4,))[0]
    for n in (0, 1, 7):
        got = F.fast_griffin_lim(amp, n, N, R, momentum=0.0)
        want = G.griffin_lim(amp, n, N, R)
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max(), n


@pytest.mark.parametrize("sr,N,R,T", GEOMS, ids=["1024-256", "2048-512"])
def test_fast_griffin_lim_converges_faster(sr, N, R, T):
    """At n = 10, 30 and 60, FGLA-n (momentum 0.99) has a lower spectral convergence than GL-n on every clip, and the
    mean ratio meets RATIO_BOUND."""
    mags = clip_mags(sr, N, R, T)
    sweeps = [F.sc_sweep(a, RATIO_BOUND, N, R) for a in mags]
    for n, bound in RATIO_BOUND.items():
        gl = np.array([G.spectral_convergence(a, G.griffin_lim(a, n, N, R), N, R) for a in mags])
        fg = np.array([s[n] for s in sweeps])
        assert fg.mean() < gl.mean() and (fg < gl).all(), (n, fg, gl)
        assert np.mean(fg / gl) <= bound, (n, fg / gl)


def test_sweep_equals_separate_runs():
    amp = clip_mags(22050, 1024, 256, 60, seeds=(9,))[0]
    sw = F.sc_sweep(amp, (0, 3, 5))
    for n in (0, 3, 5):
        assert sw[n] == G.spectral_convergence(amp, F.fast_griffin_lim(amp, n), 1024, 256), n


def test_beta():
    assert F.beta_of(0.0) == 0.0
    assert F.beta_of(0.99) == 0.99 / 1.99


BAD = [-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf"), "0.5", None, 0.5j, True, [0.5]]


def test_bad_momentum_raises_before_any_library_call(monkeypatch):
    from deepvoice3_pytorch_b200 import audio

    def no_call(*a, **k):
        raise AssertionError("reached a library call")
    monkeypatch.setattr(audio.lib, "call", no_call)
    monkeypatch.setattr(torch.Tensor, "cuda", no_call)
    monkeypatch.setattr(torch.Tensor, "to", no_call)
    mag = torch.zeros(2, 12, 513)                 # a CPU tensor: any later check would raise Dv3Error instead
    spec = np.zeros((513, 12), dtype=np.float32)
    for m in BAD:
        with pytest.raises(ValueError, match="momentum"):
            audio.griffin_lim_batch(mag, [12, 10], 3, momentum=m)
        with pytest.raises(ValueError, match="momentum"):
            audio.griffin_lim(mag[0], momentum=m)
        monkeypatch.setattr(audio.hparams, "griffin_lim_momentum", m)
        with pytest.raises(ValueError, match="momentum"):
            audio.inv_spectrogram(spec, method="fast_griffin_lim")
        with pytest.raises(ValueError, match="momentum"):
            audio.inv_spectrogram_batch([spec, spec], method="fast_griffin_lim")
    monkeypatch.setattr(audio.hparams, "griffin_lim_momentum", 0.99)
    for n_iter in (-1, 2.5, "3"):
        with pytest.raises(ValueError, match="n_iter"):
            audio.inv_spectrogram(spec, n_iter=n_iter, method="fast_griffin_lim")


def test_accepted_momentum_values():
    from deepvoice3_pytorch_b200 import audio
    for m in (0, 0.0, 0.5, np.float32(0.99), np.float64(0.3), 1 - 2 ** -40):
        assert audio._check_momentum(m) == float(m)


def test_hparams_and_methods():
    from deepvoice3_pytorch_b200 import audio
    hp = audio.hparams
    assert hp.griffin_lim_momentum == 0.99 and hp.griffin_lim_iters == 60 and hp.lws_iters == 30
    assert hp.fast_griffin_lim_iters % 5 == 0 and 5 <= hp.fast_griffin_lim_iters < 60
    assert audio.PHASE_METHODS[:2] == ("griffin_lim", "lws") and "fast_griffin_lim" in audio.PHASE_METHODS
    assert audio.check_phase_method("fast_griffin_lim") == "fast_griffin_lim"
    import inspect
    assert inspect.signature(audio.inv_spectrogram).parameters["method"].default == "griffin_lim"
    assert inspect.signature(audio.griffin_lim_batch).parameters["momentum"].default == 0.0


def test_momentum_entry_points_match_the_header():
    """Declared in include/dv3b200.h with the argument types audio.py passes, returning int, exported by the library."""
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import parse_header, LIB_PATH
    _build.build()
    decls = parse_header()
    P, I, L, Fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
    want = {
        "dv3_stft_complex_momentum_geom": [P, P, L, P, P, P, P, I, I, Fl, P, I, I, P],
    }
    dll = ctypes.CDLL(LIB_PATH)
    for name, args in want.items():
        assert name in decls, name
        assert [t for t, _ in decls[name][1]] == args, name
        assert [a for _, a in decls[name][1]][3:6] == ["mag", "prev", "spec"], name
        assert decls[name][0] is ctypes.c_int, name
        assert hasattr(dll, name), name
    # the plain twin is unchanged
    assert [t for t, _ in decls["dv3_stft_complex_geom"][1]] == [P, P, L, P, P, P, I, I, P, I, I, P]


def test_entry_points_refuse_bad_arguments_before_launch():
    """Null mag / prev, and beta outside [0, 1) or NaN, return an error (no device needed: the checks run before any
    CUDA call)."""
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import lib, Dv3Error
    _build.build()
    fake = ctypes.c_void_p(16)                   # never dereferenced: every case fails its host check
    cases = [dict(mag=None), dict(prev=None), dict(beta=-0.5), dict(beta=1.0), dict(beta=float("nan"))]
    for c in cases:
        mag, prev, beta = c.get("mag", fake), c.get("prev", fake), c.get("beta", 0.5)
        with pytest.raises(Dv3Error, match="momentum"):
            lib.call("dv3_stft_complex_momentum_geom", fake, fake, 100, mag, prev, fake, fake, 3, 1, beta, fake, 800,
                     200, None)


@pytest.mark.parametrize("src,kernel", [("stft_any.cu", "stft_complex_momentum_any_kernel")])
def test_momentum_kernels_do_not_spill(tmp_path, src, kernel):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    report = r.stdout + r.stderr
    m = re.search(r"Compiling entry function '\w*%s\w*'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, report, re.S)
    assert m, report
    assert m.groups() == ("0", "0", "0"), report
