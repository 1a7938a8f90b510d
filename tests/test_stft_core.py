"""CPU: the index arithmetic of the STFT kernel (csrc/stft_core.cuh: three radix-8 passes, two warp exchanges, the
even/odd split) compiled with g++ and run lane by lane, against numpy's rfft of the same windowed frame, within the
elementwise bound of tests/audio_bounds.py for this kernel (kernel "stft1024")."""
import os
import subprocess
import numpy as np
import pytest

import audio_bounds as AB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("stft") / "stft_core_harness")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "stft_core_harness.cpp"), "-o", exe])
    return exe


@pytest.mark.parametrize("seed,lim", [(0, 1024), (1, 1024), (2, 1024), (3, 700), (4, 1), (5, 1024), (6, 1024)])
def test_frame_magnitudes_match_rfft(harness, seed, lim):
    """x[-1..1023] raw samples; the harness applies pre-emphasis 0.97 and zeroes the window from sample ``lim`` on
    (the padding after a clip's end), exactly as the kernel's first pass does.  |got - |X|| <= B + 2u (|X| + B)
    (the harness' magnitude is 0.5 sqrt(p4), p4 rounded twice)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(1025).astype(np.float32)
    if seed == 2:
        x[:] = 0; x[4] = 1.0                      # impulse: flat spectrum, exercises every twiddle
    if seed == 5:                                 # tone on bin 37 + DC + Nyquist: sum|x| close to max|X|
        n = np.arange(-1, 1024)
        x = (0.5 * np.cos(2 * np.pi * 37 * n / 1024) + 0.2 + 0.1 * (-1.0) ** n).astype(np.float32)
    if seed == 6:
        x = np.full(1025, 0.7, np.float32)        # DC alone
    c = np.float32(0.97)
    hdr = np.array([c, lim], dtype=np.float32)
    out = subprocess.run([harness], input=hdr.tobytes() + x.tobytes(), stdout=subprocess.PIPE, check=True).stdout
    got = np.frombuffer(out, dtype=np.float32)
    x64 = x.astype(np.float64)
    e = x64[1:] - 0.97 * x64[:-1]
    de = AB.preemphasis_error(x64, 0.97)[1:]
    e[lim:] = 0
    de[lim:] = 0
    w = AB.A.lws_window(1024, 256)
    ref = np.abs(np.fft.rfft(e * w))
    B = AB.frame_bound(np.abs(e), de, "stft1024", 1024, 256)
    assert got.shape == (513,)
    ratio = np.abs(got - ref).max() / (B + 2 * AB.U * (ref.max() + B))
    print("stft_core harness seed %d lim %d: max error / bound %.3g (error %.2f u sum|w e|)"
          % (seed, lim, ratio, np.abs(got - ref).max() / (AB.U * (w * np.abs(e)).sum())))
    assert ratio <= 1.0, ratio
    np.testing.assert_allclose(got, ref, rtol=2e-4, atol=2e-5 * ref.max())     # tighter at the small bins of noise
