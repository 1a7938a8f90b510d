"""No GPU: the fp64 MAS restatement (tests/alignment_oracle.py) against a brute force over every monotone path,
attention_errors on hand-built tracks, the teacher-forced step-count rule against data.collate, the C ABI and ptxas
report of csrc/align.cu, and the refusals of the API before any library call."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import alignment_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the oracle -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", range(1, 10))
@pytest.mark.parametrize("L", range(1, 6))
def test_oracle_equals_brute_force_with_planted_ties(N, L):
    if N < L:
        d, score, path = AO.mas_logp(np.zeros((N, L)))
        assert (d == 0).all() and score == -np.inf and path is None
        return
    rng = np.random.RandomState(10 * N + L)
    for trial in range(4):
        # integer log-probabilities: sums are exact, so equal scores are exact ties; trial 0 is all ties
        lp = np.zeros((N, L)) if trial == 0 else rng.randint(-2, 1, (N, L)).astype(np.float64)
        d, score, path = AO.mas_logp(lp)
        bs, bp = AO.brute_force(lp)
        assert score == bs and np.array_equal(path, bp), (lp, path, bp)
        assert (d >= 1).all() and d.sum() == N and np.array_equal(np.repeat(np.arange(L), d), path)
    # all ties: walking back from the end, the path stays on each token as long as it can, so the last token keeps
    # every spare step
    d, _, _ = AO.mas_logp(np.zeros((N, L)))
    assert d.tolist() == [1] * (L - 1) + [N - L + 1]


def test_oracle_floor_and_nan():
    A = np.array([[np.nan, 0.0], [0.5, 1e-12], [np.nan, 0.7]])
    lp = AO.log_probs(A)
    assert lp[0, 0] == lp[0, 1] == lp[1, 1] == np.log(1e-8)
    d, score, _ = AO.mas(A)
    assert d.tolist() == [2, 1] and score == pytest.approx(np.log(1e-8) + np.log(0.5) + np.log(0.7))


def test_oracle_planted_paths():
    rng = np.random.RandomState(0)
    for N, L in ((1, 1), (7, 1), (6, 6), (40, 9)):
        A, dur = AO.planted(N, L, rng)
        assert np.array_equal(AO.mas(A)[0], dur)


# ---- attention_errors --------------------------------------------------------------------------------------------------
def _errors(p, c, N=None, max_steps=200, m=None, **kw):
    from deepvoice3_pytorch_b200.alignment import attention_errors
    p = np.asarray(p, np.int64)
    m = np.full(p.size, 0.9, np.float32) if m is None else m
    c = np.asarray(c, np.float32)
    got = attention_errors([p], [m], [c], [p.size if N is None else N], max_steps, **kw)
    want = AO.attention_errors(p, m, c, max_steps, **kw)
    for k, v in want.items():
        assert got[k][0] == pytest.approx(v), k
    return {k: v[0] for k, v in got.items()}


def test_attention_errors_clean_diagonal():
    e = _errors(np.repeat(np.arange(10), 3), np.full(10, 2.7))
    assert (e["skips"], e["unreached"], e["repeats"], e["stop_failed"], e["max_dwell"]) == (0, 0, 0, False, 3)
    assert e["focus_rate"] == pytest.approx(0.9) and e["finite"]


def test_attention_errors_one_skip():
    p = [0, 0, 1, 1, 2, 2, 4, 4, 5, 5]                   # token 3 never the argmax
    c = [1.8, 1.8, 1.8, 0.1, 1.8, 1.8]
    e = _errors(p, c)
    assert (e["skips"], e["unreached"], e["repeats"]) == (1, 0, 0)


def test_attention_errors_repeats_need_more_than_the_margin():
    c = np.full(8, 1.5)
    e = _errors([0, 1, 2, 3, 4, 5, 2, 3, 4, 5, 6, 7], c)            # back by 3 from 5, then catching up
    assert e["repeats"] == 1
    e = _errors([0, 1, 2, 3, 4, 5, 4, 5, 6, 7], c)                  # back by exactly repeat_margin = 1
    assert e["repeats"] == 0
    e = _errors([0, 1, 2, 3, 4, 5, 4, 5, 6, 7], c, repeat_margin=0)
    assert e["repeats"] == 1
    e = _errors([0, 1, 2, 3, 4, 5, 1, 2, 3, 4, 6, 1, 7], c)          # two separate returns
    assert e["repeats"] == 2


def test_attention_errors_truncated_tail_and_step_limit():
    e = _errors([0, 1, 2, 3, 4, 5], np.r_[np.ones(6), np.zeros(4)])
    assert (e["unreached"], e["skips"], e["stop_failed"]) == (4, 0, False)
    e = _errors(np.r_[np.arange(5), np.full(196, 4)], np.full(8, 1.0), max_steps=200)
    assert e["stop_failed"] and e["max_dwell"] == 197 and e["unreached"] == 3
    e = _errors(np.r_[np.arange(5), np.full(195, 4)], np.full(8, 1.0), max_steps=200)
    assert not e["stop_failed"]
    e = _errors([0, 1], [1.0, np.nan])
    assert not e["finite"]


def test_attention_errors_refusals():
    from deepvoice3_pytorch_b200.alignment import attention_errors
    p, m, c = np.arange(3), np.ones(3), np.ones(3)
    bad = [([], [], [], [], 10, {}), ([p], [m], [c], [4], 10, {}), ([p], [m[:2]], [c], [3], 10, {}),
           ([p.astype(float)], [m], [c], [3], 10, {}), ([p + 1], [m], [c], [3], 10, {}),
           ([p], [m], [c], [3], 0, {}), ([p], [m], [c], [3], 10, {"skip_coverage": -1.0}),
           ([p], [m], [c], [3], 10, {"skip_coverage": float("nan")}), ([p], [m], [c], [3], 10, {"repeat_margin": -1}),
           ([p], [m], [c], [3], 10, {"repeat_margin": 0.5}), ([p], [m], [c[:0]], [3], 10, {}),
           ([p[:, None]], [m], [c], [3], 10, {}), ((p,), [m], [c], [3], 10, {})]
    for a, mm, cc, s, ms, kw in bad[:-1]:
        with pytest.raises(ValueError):
            attention_errors(a, mm, cc, s, ms, **kw)
    attention_errors(*bad[-1][:5])                      # tuples are lists too


# ---- teacher-forced step counts ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [1, 2, 4])
@pytest.mark.parametrize("ds", [1, 4])
def test_teacher_forced_steps_match_collate(r, ds):
    """Row b's steps are the decoder steps whose input frames [s r ds, (s + 1) r ds) of collate's linear target meet its
    r leading zero frames or its own n frames; its done target is 1 from the last of them on."""
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.alignment import teacher_forced_steps
    rng = np.random.RandomState(r * 10 + ds)
    rd = r * ds                                      # collate needs at least one step's frames
    lens = [rd, rd + 1, rd + 2, 2 * rd - 1, 2 * rd, 31 + rd, 64, 65, 100] + rng.randint(rd, 200, 8).tolist()
    batch = [(np.arange(1, 4), np.ones((n, 4), np.float32), np.ones((n, 3), np.float32)) for n in lens]
    out = data.collate(batch, r=r, downsample_step=ds)
    T_dec = out["frame_positions"].size(1)
    steps = teacher_forced_steps(lens, r, ds)
    y = out["y"][:, :, 0].numpy()
    done = out["done"][:, :, 0].numpy()
    for b, n in enumerate(lens):
        assert 1 <= steps[b] <= T_dec
        nz = np.flatnonzero(y[b])
        assert nz[0] == r and nz[-1] == r + n - 1                       # r leading zero frames, then the target
        assert steps[b] == (r + n - 1) // (r * ds) + 1                  # the step that holds its last frame, counted
        assert (done[b, steps[b] - 1:] == 1).all()
        assert (done[b, :n // rd - 1] == 0).all()


# ---- C ABI and ptxas ----------------------------------------------------------------------------------------------------
def test_c_abi_declares_and_exports_the_alignment_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    names = ("dv3_mas_max_tokens", "dv3_mas_dir_words", "dv3_mas_forward", "dv3_mas_backtrace")
    args = {n: [a for _, a in d[n][1]] for n in names}
    assert args["dv3_mas_forward"] == ["A", "stride_b", "stride_t", "steps", "tokens", "B", "N_max", "L_max",
                                       "dir_off", "dirs", "argmax", "maxv", "coverage", "score", "stream"]
    assert args["dv3_mas_backtrace"] == ["steps", "tokens", "B", "L_max", "dir_off", "dirs", "durations", "stream"]
    P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    assert [t for t, _ in d["dv3_mas_forward"][1]] == [P, LL, LL, P, P, I, I, I, P, P, P, P, P, P, P]
    assert d["dv3_mas_dir_words"][0] == LL
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in names:
            assert re.search(r"\bT %s\b" % name, nm), name
        lib = ctypes.CDLL(so)
        lib.dv3_mas_dir_words.restype = ctypes.c_longlong
        assert lib.dv3_mas_max_tokens() == 1024
        assert [lib.dv3_mas_dir_words(n, l) for n, l in ((1, 1), (10, 32), (10, 33), (4001, 1024), (0, 5), (5, 1025))] \
            == [1, 10, 20, 4001 * 32, 0, 0]


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "align.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert sorted(n for n, *_ in frames) == ["_ZN3dv318mas_forward_kernelEPKfxxPKiS3_iiPKxPjPiPfS8_S8_",
                                             "_ZN3dv320mas_backtrace_kernelEPKiS1_iiPKxPKjPi"], rep
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


def test_monotonic_alignment_refusals(no_lib):
    from deepvoice3_pytorch_b200.alignment import monotonic_alignment
    a = torch.zeros(2, 6, 4)
    bad = [(torch.zeros(6, 4), [6], [4]), (np.zeros((2, 6, 4), np.float32), [6, 6], [4, 4]),
           (a.double(), [6, 6], [4, 4]), (a.half(), [6, 6], [4, 4]), (torch.zeros(1, 6, 1025), [6], [4]),
           (torch.zeros(0, 6, 4), [], []), (a, [6], [4, 4]), (a, [6, 7], [4, 4]), (a, [0, 6], [4, 4]),
           (a, [6, 6], [4, 5]), (a, [6, 6], [0, 4]), (a, [6.0, 6.0], [4, 4]), (a, np.array([[6, 6]]), [4, 4]),
           (a, [6, 6], [4, 4])]                                                      # a CPU tensor
    for x, s, t in bad:
        with pytest.raises(ValueError):
            monotonic_alignment(x, s, t)
    assert no_lib == []


def test_evaluate_attention_refusals(no_lib):
    from deepvoice3_pytorch_b200.alignment import evaluate_attention
    from test_mcd_host import _models
    single, multi = _models()
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    bad_calls = [
        (single, seqs, [0, 1], {}),
        (multi, seqs, None, {}),
        (multi, seqs, [0, 4], {}),
        (multi, seqs, [0], {}),
        (single, [np.array([3, 4]), np.array([], np.int64)], None, {}),
        (single, [np.array([3.0, 4.0])], None, {}),
        (single, [np.arange(1, 70)], None, {}),                    # longer than the position tables
        (single, [], None, {}),
        (single, seqs, None, {"batch_size": 0}),
        (single, seqs, None, {"skip_coverage": -0.5}),
        (single, seqs, None, {"repeat_margin": -1}),
        (single, seqs, None, {"skip_threshold": 0.5}),
    ]
    for model, sq, ids, kw in bad_calls:
        with pytest.raises(ValueError):
            evaluate_attention(model, sq, speaker_ids=ids, **kw)
    assert no_lib == []


def test_teacher_forced_alignment_refusals(no_lib):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.alignment import teacher_forced_alignment
    from test_mcd_host import _models
    single, multi = _models()
    items = [(np.arange(1, 6), np.ones((12, 80), np.float32), np.ones((12, 9), np.float32))]
    batch = data.collate(items, r=1, downsample_step=4)
    for model, b, kw in ((single, {k: v for k, v in batch.items() if k != "y"}, {}), (single, batch, {"layer": 5}),
                         (single, batch, {"layer": -1}), (single, batch, {"layer": 0.5}), (multi, batch, {})):
        with pytest.raises(ValueError):
            teacher_forced_alignment(model, b, **kw)
    with pytest.raises(ValueError):
        teacher_forced_alignment(single.train(), batch)
    single.eval()
    assert no_lib == []
