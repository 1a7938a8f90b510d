"""No GPU: the fp64 YIN restatement (tests/pitch_oracle.py) on known answers, the frame geometry against the oracle STFT,
the oracle's warping path against a brute force over every monotone path, f0_metrics on hand-built tracks, the
direction-buffer chunks of dtw_path, the C ABI and ptxas report of csrc/pitch.cu, and the refusals of the API before any
library call."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import pitch_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 22050


def _tone(f, n, amp=0.5, harmonics=1):
    t = np.arange(n) / SR
    x = sum(amp / h * np.sin(2 * np.pi * f * h * t + 0.3 * h) for h in range(1, harmonics + 1))
    return x.astype(np.float32)


def _inside(n_frames, n, lo=0, tau_max=368):
    """Frames whose whole span [a_t, a_t + W + tau_max) lies in [lo, n)."""
    a = np.arange(n_frames) * 256 + 256 - 512 - (1024 + tau_max) // 2
    return (a >= lo) & (a + 1024 + tau_max <= n)


# ---- oracle known answers -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [65.0, 82.0, 110.0, 150.0, 220.0, 330.0, 480.0])
def test_oracle_pure_tones_are_voiced_within_a_tenth_of_a_percent(f):
    x = _tone(f, 12000)
    r = PO.yin(x)
    inside = _inside(len(r["f0"]), x.size)
    assert inside.sum() >= 10
    assert r["voiced"][inside].all()
    assert np.abs(r["f0"][inside] / f - 1).max() < 1e-3


@pytest.mark.parametrize("f", [80.0, 125.0, 200.0, 300.0])
def test_oracle_harmonic_tones_are_voiced_within_a_tenth_of_a_percent(f):
    x = _tone(f, 12000, amp=0.3, harmonics=8)
    r = PO.yin(x)
    inside = _inside(len(r["f0"]), x.size)
    assert r["voiced"][inside].all()
    assert np.abs(r["f0"][inside] / f - 1).max() < 1e-3


def test_oracle_noise_is_unvoiced_and_silence_has_aperiodicity_one():
    x = np.random.RandomState(0).randn(12000).astype(np.float32)
    r = PO.yin(x)
    assert not r["voiced"].any() and (r["f0"] == 0).all()
    s = PO.yin(np.zeros(3000, np.float32))
    assert not s["voiced"].any() and (s["aperiodicity"] == 1.0).all() and (s["f0"] == 0).all()


def test_oracle_silence_gate_drops_a_quiet_tone_next_to_a_loud_one():
    loud, quiet = _tone(200.0, 8000, amp=0.5), _tone(200.0, 8000, amp=0.5 * 10 ** (-70 / 20))
    x = np.concatenate([loud, quiet])
    r = PO.yin(x)
    q = _inside(len(r["f0"]), x.size, lo=8000)
    lo_ = _inside(len(r["f0"]), 8000)
    assert q.sum() >= 5 and r["voiced"][q].all()          # periodic, and voiced before the gate
    assert (r["f0"][q] == 0).all() and (r["f0_raw"][q] > 0).all()
    assert (r["f0"][lo_] > 0).all()
    ungated = PO.yin(x, silence_db=-90.0)
    assert (ungated["f0"][q] > 0).all()


# ---- frame geometry ---------------------------------------------------------------------------------------------------
def test_frame_count_and_centres_match_the_oracle_stft():
    from deepvoice3_pytorch_b200 import audio, pitch
    from oracle import audio_oracle as A
    N, R = 1024, 256
    for n in list(range(1, 4 * R + 3)) + [5 * R, 7 * R + 1, 22050]:
        assert PO.num_frames(n) == A.num_frames(n) == audio.num_frames_host(n)
        assert PO.spans(np.zeros(n), N, R, 368).shape[0] == A.num_frames(n)
    # an impulse at p: oracle STFT frame t sees window value w(p - start_t); the frame's centre is start_t + N/2
    n = 3000
    win = A.lws_window(N, R)
    centres = pitch.frame_centres(A.num_frames(n))
    for p in (0, 1, 700, 1500, 2999):
        x = np.zeros(n)
        x[p] = 1.0
        mag = np.abs(A.lws_stft(x, N, R))[:, 0]
        for t, c in enumerate(centres):
            k = p - (c - N // 2)
            assert mag[t] == pytest.approx(win[k] if 0 <= k < N else 0.0, abs=1e-12), (p, t)
    # the oracle's spans are centred there: sample a_t + floor((W + tau_max)/2) is c_t
    x = np.arange(1, n + 1, dtype=np.float64)
    sp = PO.spans(x, N, R, 368)
    for t, c in enumerate(centres):
        if 0 <= c < n:
            assert sp[t, (N + 368) // 2] == x[c]


# ---- warping path -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", range(1, 7))
@pytest.mark.parametrize("M", range(1, 7))
def test_oracle_path_equals_brute_force_with_ties(N, M):
    import mcd_oracle as MO
    rng = np.random.RandomState(N * 10 + M)
    for _ in range(3):
        d = rng.randint(0, 3, (N, M)).astype(np.float64)
        cost, path = PO.dtw_path(d)
        bc, bp = PO.path_brute(d)
        assert cost == bc and np.array_equal(path, bp)
        assert MO.dtw_matrix(d) == (cost, len(path))


def test_oracle_path_stays_in_the_grid_where_the_cost_is_nan():
    """A NaN distance makes the comparisons against it fail, so the recursion can store the diagonal code on row and
    column 1; the walk moves left on row 1 and up on column 1 and still ends at (0, 0) with unit steps."""
    for N, M, bad in ((5, 7, (2, 3)), (7, 5, (0, 4)), (6, 6, (5, 0)), (1, 6, (0, 2)), (6, 1, (3, 0))):
        d = np.ones((N, M))
        d[bad] = np.nan
        cost, path = PO.dtw_path(d)
        assert tuple(path[0]) == (0, 0) and tuple(path[-1]) == (N - 1, M - 1)
        steps = np.diff(path, axis=0)
        assert ((steps == [1, 1]).all(1) | (steps == [1, 0]).all(1) | (steps == [0, 1]).all(1)).all()
        assert (path >= 0).all() and (path[:, 0] < N).all() and (path[:, 1] < M).all()


# ---- metrics ----------------------------------------------------------------------------------------------------------
def test_f0_metrics_on_hand_built_tracks():
    from deepvoice3_pytorch_b200.pitch import f0_metrics
    fa = np.array([0.0, 100.0, 100.0, 200.0, 0.0])
    fb = np.array([0.0, 100.0, 130.0, 100.0 * 2 ** (50 / 1200), 150.0])
    diag = np.stack([np.arange(5)] * 2, 1)
    m = f0_metrics([fa], [fb], [diag])
    # pairs: (0,0) both unvoiced; (1,1) equal; (2,2) 100 vs 130: gross; (3,3) 200 vs 103: gross; (4,4) voicing error
    assert m["vde"][0] == pytest.approx(1 / 5)
    assert m["gpe"][0] == pytest.approx(2 / 3)
    assert m["ffe"][0] == pytest.approx(3 / 5)
    cents = 1200 * np.log2(np.array([1.0, 100 / 130, 200 / fb[3]]))
    assert m["f0_rmse_cents"][0] == pytest.approx(math.sqrt(np.mean(cents ** 2)), rel=1e-12)
    assert m["voiced_fraction"][0].tolist() == [3 / 5, 4 / 5]
    # a path that repeats frames weighs them by their pairs
    path = np.array([[0, 0], [1, 1], [1, 2], [2, 3]])
    m = f0_metrics([np.array([0.0, 100.0, 100.0])], [np.array([0.0, 101.0, 100.0, 0.0])], [path])
    assert m["vde"][0] == pytest.approx(1 / 4) and m["gpe"][0] == 0.0 and m["ffe"][0] == pytest.approx(1 / 4)
    assert m["f0_rmse_cents"][0] == pytest.approx(math.sqrt((1200 * math.log2(100 / 101)) ** 2 / 2))


def test_f0_metrics_nan_where_nothing_is_voiced_on_both_sides():
    from deepvoice3_pytorch_b200.pitch import f0_metrics
    z, v = np.zeros(4), np.full(4, 120.0)
    diag = np.stack([np.arange(4)] * 2, 1)
    m = f0_metrics([z, v, z], [z, z, v], [diag] * 3)
    assert np.isnan(m["gpe"]).all() and np.isnan(m["f0_rmse_cents"]).all()
    assert m["vde"].tolist() == [0.0, 1.0, 1.0] and m["ffe"].tolist() == [0.0, 1.0, 1.0]
    m = f0_metrics([v], [v], [diag])
    assert m["gpe"][0] == 0.0 and m["f0_rmse_cents"][0] == 0.0 and m["vde"][0] == 0.0


def test_f0_metrics_refusals():
    from deepvoice3_pytorch_b200.pitch import f0_metrics
    d = np.stack([np.arange(3)] * 2, 1)
    for a, b, p in (([], [], []), ([np.ones(3)], [np.ones(3)], []), ([np.ones(2)], [np.ones(3)], [d]),
                    ([np.ones(3)], [np.ones(3)], [d[:, :1]]), ([np.ones((3, 1))], [np.ones(3)], [d]),
                    ([np.ones(3)], [np.ones(3)], [d.astype(float)]), ([np.ones(3)], [np.ones(3)], [d[:0]])):
        with pytest.raises(ValueError):
            f0_metrics(a, b, p)


# ---- direction-buffer chunks --------------------------------------------------------------------------------------------
def test_path_chunks_respect_the_budget_and_cover_the_work_list_in_order():
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(3)
    a_lens, b_lens = rng.randint(1, 900, 40).tolist(), rng.randint(1, 900, 40).tolist()
    work, _ = mcd._work_list(list(range(40)), a_lens, list(range(40)), b_lens)
    size = [4 * int(w[2]) * (-(-int(w[4]) // 16)) for w in work]
    for budget in (1, 50_000, 400_000, sum(size), 1 << 30):
        chunks = mcd._path_chunks(work, budget)
        assert chunks[0][0] == 0 and chunks[-1][1] == 40
        assert all(c1 == n0 for (_, c1), (n0, _) in zip(chunks, chunks[1:]))
        for r0, r1 in chunks:
            assert r1 > r0
            assert sum(size[r0:r1]) <= budget or r1 - r0 == 1
            if r1 < 40:
                assert sum(size[r0:r1 + 1]) > budget          # greedy: the next row would not have fit
    assert mcd._path_chunks(work) == [(0, 40)]
    assert 4 * 16384 * (16384 // 16) == 64 << 20 <= mcd.DIR_BUDGET_BYTES


# ---- C ABI and ptxas ----------------------------------------------------------------------------------------------------
def test_c_abi_declares_and_exports_the_pitch_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {n: [a for _, a in d[n][1]] for n in ("dv3_yin_frames_per_cta", "dv3_yin_f0", "dv3_dtw_path",
                                                 "dv3_dtw_backtrace")}
    assert args["dv3_yin_f0"] == ["wav", "blocks", "n_blocks", "clips", "n_clips", "f0", "aperiodicity", "energy",
                                  "diff", "W", "R", "tau_min", "tau_max", "threshold", "gate", "sample_rate", "stream"]
    assert args["dv3_dtw_path"] == ["cep", "K", "work", "path_work", "workspace", "dirs", "cost", "path_len", "P",
                                    "stream"]
    assert args["dv3_dtw_backtrace"] == ["work", "path_work", "dirs", "path", "path_rows", "P", "stream"]
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    assert [t for t, _ in d["dv3_yin_f0"][1]] == [P, P, I, P, I, P, P, P, P, I, I, I, I, F, F, F, P]
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in args:
            assert re.search(r"\bT %s\b" % name, nm), name
        lib = ctypes.CDLL(so)
        assert [lib.dv3_yin_frames_per_cta(t) for t in (0, 1, 368, 416, 417, 832, 833, 1024, 1025)] == \
            [0, 8, 8, 8, 4, 4, 2, 2, 0]


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "pitch.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 11, rep                   # YIN, its gate, the backtrace and the path DTW at K = 8, ..., 64
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


def test_yin_f0_refusals(no_lib):
    from deepvoice3_pytorch_b200 import pitch
    w = torch.zeros(4000)
    bad = [([], {}), ("x", {}), ([torch.zeros(0)], {}), ([torch.zeros(256 * 16400)], {}),
           ([torch.zeros(2, 4000)], {}), ([torch.zeros(4000, dtype=torch.float64)], {}), ([np.zeros(4000)], {}),
           ([w], {}),                                                                   # a CPU tensor
           ([w], {"f0_min": 500.0, "f0_max": 500.0}), ([w], {"f0_min": 300.0, "f0_max": 200.0}),
           ([w], {"f0_min": 0.0}), ([w], {"f0_min": float("nan")}), ([w], {"f0_max": float("inf")}),
           ([w], {"f0_max": 12000.0}),                                                  # tau_min = 1
           ([w], {"f0_min": 21.0}),                                                     # tau_max = 1050
           ([w], {"threshold": 0.0}), ([w], {"threshold": 1.01}), ([w], {"threshold": float("nan")}),
           ([w], {"silence_db": 0.5}), ([w], {"silence_db": float("nan")})]
    for wavs, kw in bad:
        with pytest.raises(ValueError):
            pitch.yin_f0(wavs, **kw)
    assert no_lib == []
    assert pitch.yin_params(60.0, 500.0) == (44, 368, pytest.approx(1e-5))
    assert pitch.yin_params(22050 / 1024.0, 22050 / 2.0, 1.0, 0.0)[:2] == (2, 1024)


def test_dtw_path_refusals(no_lib):
    from deepvoice3_pytorch_b200 import mcd
    z = lambda T, K=24: torch.zeros(T, K)
    for a, b in (([], []), ([z(5)], []), ([z(5)], [z(0)]), ([z(5)], [z(5, 23)]), ([z(5, 65)], [z(5, 65)]),
                 ([z(16385)], [z(5)]), ([z(5)], [z(5)])):
        with pytest.raises(ValueError):
            mcd.dtw_path(a, b)
    assert no_lib == []


def test_evaluate_pitch_refusals(no_lib):
    from deepvoice3_pytorch_b200.pitch import evaluate_pitch
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
        (single, seqs, refs, None, {"n_ceps": 0}),
        (single, seqs, refs, None, {"vocoder": "wavenet"}),
        (single, seqs, refs, [0, 1], {}),
        (multi, seqs, refs, None, {}),
        (multi, seqs, refs, [0, 4], {}),
        (single, [np.array([3, 4]), np.array([], np.int64)], refs, None, {}),
        (single, seqs, refs, None, {"batch_size": 0}),
        (single, seqs, refs, None, {"f0_min": 500.0}),
        (single, seqs, refs, None, {"f0_min": 15.0}),
        (single, seqs, refs, None, {"threshold": 0.0}),
        (single, seqs, refs, None, {"silence_db": 3.0}),
    ]
    for model, sq, rw, ids, kw in bad_calls:
        with pytest.raises(ValueError):
            evaluate_pitch(model, sq, rw, speaker_ids=ids, **kw)
    assert no_lib == []
