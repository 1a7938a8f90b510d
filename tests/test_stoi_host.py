"""No GPU: the fp64 STOI / ESTOI restatement (tests/stoi_oracle.py) on known properties, the band edges against their
closed form, the 10 kHz resampling ratios against scipy and the resampler's shared-memory budget, the C ABI and ptxas
report of csrc/stoi.cu, and the refusals of the intelligibility API before any library call."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

import stoi_oracle as SO
from test_vctk_host import polyphase

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def voiced(n, sr=10000, seed=0):
    """A speech-like test signal: a gliding harmonic tone whose amplitude rises and falls in 0.25 s syllables, with
    short pauses."""
    rng = np.random.RandomState(seed)
    t = np.arange(n) / sr
    f0 = 120 * (1 + 0.15 * np.sin(2 * np.pi * 0.7 * t))
    ph = 2 * np.pi * np.cumsum(f0) / sr
    x = sum(rng.uniform(0.2, 1.0) / h * np.sin(h * ph + rng.uniform(0, 6)) for h in range(1, 25))
    env = np.clip(np.sin(2 * np.pi * 2.0 * t + rng.uniform(0, 6)), 0, None) ** 2
    return (0.3 * x * env).astype(np.float32)


# ---- band edges -------------------------------------------------------------------------------------------------------
def test_band_edges_match_the_closed_form():
    from deepvoice3_pytorch_b200 import intelligibility as I
    lo, hi = I.band_edges()
    olo, ohi = SO.band_edges()
    assert np.array_equal(lo, olo) and np.array_equal(hi, ohi)
    for i in range(15):
        assert lo[i] == round(150 * 2 ** ((2 * i - 1) / 6) * 512 / 10000)
        assert hi[i] == round(150 * 2 ** ((2 * i + 1) / 6) * 512 / 10000)
    assert lo[0] == 7 and hi[-1] == 219 and (hi[:-1] == lo[1:]).all() and (hi > lo).all() and hi.max() < 256
    obm = SO.band_matrix()
    assert obm.shape == (15, 257) and np.array_equal(obm.sum(1), hi - lo)
    assert np.abs(I.window_fp64() - np.hanning(258)[1:-1]).max() < 1e-15
    assert np.array_equal(I.window_fp64(), SO.window())


# ---- oracle properties ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L,F", [(1, 0), (256, 0), (257, 1), (384, 1), (385, 2), (10000, 77)])
def test_frame_count_follows_the_range_rule(L, F):
    from deepvoice3_pytorch_b200 import intelligibility as I
    assert SO.num_frames(L) == I.num_frames(L) == len(range(0, L - 256, 128)) == F
    assert SO.frames(np.ones(L)).shape == (F, 256)


def test_identical_signals_score_one():
    x = voiced(30000)
    r = SO.stoi(x, x)
    assert r["segments"] > 50
    assert abs(r["stoi"] - 1) < 1e-12 and abs(r["estoi"] - 1) < 1e-12


def test_scores_fall_monotonically_with_added_noise():
    x = voiced(40000, seed=1).astype(np.float64)
    noise = np.random.RandomState(7).randn(x.size)
    px, pn = np.mean(x ** 2), np.mean(noise ** 2)
    d, e = [], []
    for snr in (20, 5, 0, -10):
        y = x + noise * math.sqrt(px / pn / 10 ** (snr / 10))
        r = SO.stoi(x, y)
        d.append(r["stoi"])
        e.append(r["estoi"])
    assert all(a > b for a, b in zip(d, d[1:])), d
    assert all(a > b for a, b in zip(e, e[1:])), e
    assert d[0] > 0.9 and d[-1] < 0.7


def test_short_clip_gives_nan_and_no_segments():
    x = voiced(29 * 128 + 256 + 128)          # 30 frames before silence removal: at most 29 envelope frames
    r = SO.stoi(x, x)
    assert r["segments"] == 0 and math.isnan(r["stoi"]) and math.isnan(r["estoi"])
    assert SO.pair_means(np.zeros((0, 2)))[0] != SO.pair_means(np.zeros((0, 2)))[0]


def test_silent_frames_are_removed_before_the_envelopes():
    x = voiced(20000, seed=2).astype(np.float64)
    x[5000:9000] = 0.0
    mask = SO.keep_mask(SO.frame_energies(x))
    assert 0 < mask.sum() < mask.size
    y = SO.overlap_add(x, mask)
    assert y.size == (mask.sum() - 1) * 128 + 256


# ---- resampling to 10 kHz ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", [16000, 22050, 24000, 44100, 48000])
def test_ratios_to_10k_match_resample_poly_and_fit_shared_memory(sr):
    from deepvoice3_pytorch_b200 import audio
    up, down = audio.resample_ratio(sr, 10000)
    assert up * sr == down * 10000 and math.gcd(up, down) == 1
    bank, pre_remove = audio.resample_filter_bank(up, down)
    rng = np.random.RandomState(sr)
    for n in (1, 333, 22050):
        x = rng.uniform(-1, 1, n)
        want = resample_poly(x, up, down)
        got = polyphase(x, bank, pre_remove, up, down)
        assert got.shape == want.shape == (audio.resampled_length(n, up, down),)
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    # csrc/resample.cu: the bank in fp64 plus the fp32 input window of a 4096-output tile, within the 227 KB opt-in
    ntaps = bank.shape[0]
    window = (4095 * down) // up + 2 + ntaps
    assert up * ntaps * 8 + window * 4 <= 227 * 1024
    if sr == 22050:
        assert (up, down) == (200, 441) and bank.shape == (47, 200)


def test_resample_ratio_default_is_the_model_rate():
    from deepvoice3_pytorch_b200 import audio
    assert audio.resample_ratio(48000) == audio.resample_ratio(48000, audio.hparams.sample_rate)


# ---- C ABI and ptxas ----------------------------------------------------------------------------------------------------
NAMES = ("dv3_stoi_frames", "dv3_stoi_overlap_add", "dv3_stoi_bands", "dv3_stoi_segments")


def test_c_abi_declares_and_exports_the_stoi_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {n: [a for _, a in d[n][1]] for n in NAMES}
    assert args["dv3_stoi_frames"] == ["wav", "clips", "n_clips", "win", "energy", "keep", "kept_idx", "kept", "stream"]
    assert args["dv3_stoi_overlap_add"] == ["wav", "clips", "n_clips", "max_samples", "table", "kept_idx", "kept",
                                            "ola", "frames", "stream"]
    assert args["dv3_stoi_bands"] == ["ola", "clips", "blocks", "n_blocks", "table", "bands", "frames", "env", "feat",
                                      "stream"]
    assert args["dv3_stoi_segments"] == ["env", "clips", "pairs", "n_pairs", "blocks", "n_blocks", "path", "steps",
                                         "kept", "seg", "result", "counts", "stream"]
    P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    assert [t for t, _ in d["dv3_stoi_overlap_add"][1]] == [P, P, I, LL, P, P, P, P, P, P]
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in NAMES:
            assert re.search(r"\bT %s\b" % name, nm), name


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "stoi.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 5, rep                    # frames, overlap-add, bands, segments, per-pair reduction
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


# ---- refusals before any library call ---------------------------------------------------------------------------------
@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


def test_stoi_refusals(no_lib):
    from deepvoice3_pytorch_b200 import intelligibility as I
    w = torch.zeros(4000)                                                   # a CPU tensor
    bad = [([], []), ("x", "y"), ([w], []), ([w], [w, w]), ([torch.zeros(0)], [torch.zeros(0)]),
           ([torch.zeros(2, 4000)], [torch.zeros(2, 4000)]),
           ([torch.zeros(4000, dtype=torch.float64)], [torch.zeros(4000, dtype=torch.float64)]),
           ([np.zeros(4000, np.float32)], [np.zeros(4000, np.float32)]),
           ([torch.zeros(5_000_000)], [torch.zeros(5_000_000)]),           # more than 16384 frames at 10 kHz
           ([w], [w])]
    for a, b in bad:
        for fn in (I.stoi, I.stoi_dtw):
            with pytest.raises(ValueError):
                fn(a, b)
    for bad_wavs in ([], [torch.zeros(0)], [w]):
        with pytest.raises(ValueError):
            I.evaluate_vocoder(bad_wavs)
    with pytest.raises(ValueError):
        I.evaluate_vocoder([w], method="wavenet")
    assert no_lib == []


def test_evaluate_intelligibility_refusals(no_lib):
    from deepvoice3_pytorch_b200.intelligibility import evaluate_intelligibility
    from test_mcd_host import _models
    single, multi = _models()
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    wav = np.zeros(4000, np.float32)
    refs = [wav, wav]
    bad_calls = [
        (single, seqs, [wav], None, {}),
        (single, seqs, "wavs", None, {}),
        (single, seqs, [wav, np.zeros(4000)], None, {}),
        (single, seqs, [wav, np.zeros(0, np.float32)], None, {}),
        (single, seqs, [wav, np.zeros(256 * 16400, np.float32)], None, {}),
        (single, seqs, refs, None, {"vocoder": "wavenet"}),
        (single, seqs, refs, [0, 1], {}),
        (multi, seqs, refs, None, {}),
        (multi, seqs, refs, [0, 4], {}),
        (single, [np.array([3, 4]), np.array([], np.int64)], refs, None, {}),
        (single, seqs, refs, None, {"batch_size": 0}),
    ]
    for model, sq, rw, ids, kw in bad_calls:
        with pytest.raises(ValueError):
            evaluate_intelligibility(model, sq, rw, speaker_ids=ids, **kw)
    assert no_lib == []
