"""No GPU: the fp64 MCD-DTW restatement (tests/mcd_oracle.py) against a brute force over every monotone path and
against scipy's DCT, the offset-free DCT table of deepvoice3_pytorch_b200/mcd.py, known answers, the host work list,
the C ABI and ptxas report of csrc/mcd.cu, and the refusals of the API before any library call."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from scipy.fft import dct

import mcd_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the oracle's DTW against every monotone path ---------------------------------------------------------------------
@pytest.mark.parametrize("N", range(1, 7))
@pytest.mark.parametrize("M", range(1, 7))
def test_oracle_dtw_equals_brute_force_with_ties(N, M):
    """Small integer distances: costs are exact and ties are everywhere, so the tie rule decides L."""
    rng = np.random.RandomState(N * 10 + M)
    for _ in range(3):
        d = rng.randint(0, 3, (N, M)).astype(np.float64)
        assert MO.dtw_matrix(d) == MO.dtw_brute(d)


@pytest.mark.parametrize("N,M", [(1, 6), (6, 1), (4, 5), (6, 6)])
def test_oracle_dtw_equals_brute_force_on_real_distances(N, M):
    rng = np.random.RandomState(N + 7 * M)
    ca, cb = rng.randn(N, 3), rng.randn(M, 3)
    d = MO.distances(ca, cb)
    cost, L = MO.dtw(ca, cb)
    bc, bL = MO.dtw_brute(d)
    assert cost == pytest.approx(bc, rel=1e-12) and L == bL


def test_tie_rule_prefers_diagonal_then_up_then_left():
    z = np.zeros((2, 2))
    assert MO.dtw_matrix(z) == (0.0, 2)                         # (1,1) -> (2,2) diagonally, not through a corner
    d = np.array([[0.0, 1.0], [1.0, 0.0]])                        # both corners cost 1, the diagonal 0
    assert MO.dtw_matrix(d) == (0.0, 2)
    d = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.0]])              # 2 x 3: one diagonal and one left move
    assert MO.dtw_matrix(d) == (0.0, 3)
    assert MO.monotone_path_count(6, 6) == 1683


# ---- cepstra ------------------------------------------------------------------------------------------------------------
def _mels(rng, T, M):
    return rng.rand(T, M)


@pytest.mark.parametrize("M,K", [(80, 24), (80, 79), (40, 13), (2, 1), (128, 64)])
def test_oracle_cepstrum_is_the_ortho_dct_of_the_denormalised_log_mel(M, K):
    from deepvoice3_pytorch_b200 import audio
    rng = np.random.RandomState(M + K)
    S = _mels(rng, 7, M)
    db = audio._denormalize(S) + audio.hparams.ref_level_db           # 20 log10 A
    want = dct(db * math.log(10.0) / 20.0, type=2, norm="ortho", axis=-1)[:, 1:K + 1]
    np.testing.assert_allclose(MO.cepstra(S, K, audio.hparams.min_level_db, audio.hparams.ref_level_db), want,
                               rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("M,K", [(80, 24), (40, 39), (128, 64)])
def test_offset_only_reaches_c0_so_the_kernel_table_needs_the_scale_alone(M, K):
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(M)
    S = _mels(rng, 9, M)
    a = MO.cepstra(S, K, -100.0, 20.0)
    b = MO.cepstra(S, K, -100.0, -37.5)                               # another offset, the same scale
    np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    table = mcd.dct_basis_fp64(M, K, -100.0)                           # what the kernel multiplies the mels by
    np.testing.assert_allclose(S @ table.T, a, rtol=0, atol=1e-11)
    full = dct(MO.log_amplitude(S), type=2, norm="ortho", axis=-1)
    assert np.abs(full[:, 0] - dct(MO.log_amplitude(S) - MO.log_amplitude(np.zeros_like(S)), type=2, norm="ortho",
                                   axis=-1)[:, 0]).min() > 1.0         # c_0 does carry the offset


# ---- known answers ------------------------------------------------------------------------------------------------------
def test_a_sequence_against_itself_and_against_its_frames_repeated():
    rng = np.random.RandomState(3)
    c = MO.cepstra(_mels(rng, 37, 80), 24)
    cost, L = MO.dtw(c, c)
    assert cost == 0.0 and L == 37
    rep = np.repeat(c, 2, axis=0)
    cost, L = MO.dtw(c, rep)
    assert cost == 0.0 and L == 74
    assert MO.dtw(rep, c) == (0.0, 74)


@pytest.mark.parametrize("N,M", [(5, 5), (3, 8), (11, 4)])
def test_constant_sequences_give_the_closed_form_mcd(N, M):
    """Log mels differing by a known vector v: every cell costs ||DCT(v)_1..K||, the path has max(N, M) cells."""
    rng = np.random.RandomState(N * M)
    Mm, K = 80, 24
    lnA = rng.randn(Mm) * 0.3 - 2.0
    v = rng.randn(Mm) * 0.1
    to_norm = lambda la: (la * 20.0 / math.log(10.0) + 100.0 - 20.0) / 100.0     # inverse of log_amplitude
    a = np.tile(to_norm(lnA), (N, 1))
    b = np.tile(to_norm(lnA + v), (M, 1))
    cost, L = MO.dtw(MO.cepstra(a, K), MO.cepstra(b, K))
    dist = np.linalg.norm(dct(v, type=2, norm="ortho")[1:K + 1])
    assert L == max(N, M)
    assert MO.mcd(cost, L) == pytest.approx(MO.MCD_SCALE * dist, rel=1e-12)


# ---- host work list -----------------------------------------------------------------------------------------------------
def test_work_list_runs_the_longest_recursion_first_with_aligned_workspace():
    from deepvoice3_pytorch_b200 import mcd
    a_lens, b_lens = [10, 900, 33, 1, 64, 64], [900, 10, 33, 1, 64, 65]
    work, ws = mcd._work_list([0, 10, 20, 30, 40, 50], a_lens, [100, 200, 300, 400, 500, 600], b_lens)
    steps = [-(-a_lens[p] // 32) * (b_lens[p] + 31) for p in work[:, 0]]
    assert steps == sorted(steps, reverse=True)
    assert sorted(work[:, 0].tolist()) == list(range(6))
    assert all(w[5] % 32 == 0 for w in work)
    assert ws == sum(2 * (-(-m // 32) * 32) for m in b_lens)
    for w in work:
        p = w[0]
        assert (w[2], w[4]) == (a_lens[p], b_lens[p])


# ---- C ABI and ptxas ----------------------------------------------------------------------------------------------------
def test_c_abi_declares_and_exports_the_mcd_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {n: [a for _, a in d[n][1]] for n in ("dv3_mel_cepstra", "dv3_dtw_mcd", "dv3_mcd_max_frames")}
    assert args["dv3_mel_cepstra"] == ["mels", "lengths", "basis", "cep", "n_seq", "T_max", "M", "K", "stream"]
    assert args["dv3_dtw_mcd"] == ["cep", "K", "work", "workspace", "cost", "path_len", "P", "stream"]
    assert args["dv3_mcd_max_frames"] == []
    P, I = ctypes.c_void_p, ctypes.c_int
    assert [t for t, _ in d["dv3_mel_cepstra"][1]] == [P, P, P, P, I, I, I, I, P]
    assert [t for t, _ in d["dv3_dtw_mcd"][1]] == [P, I, P, P, P, P, I, P]
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in args:
            assert re.search(r"\bT %s\b" % name, nm), name
        from deepvoice3_pytorch_b200 import mcd
        assert ctypes.CDLL(so).dv3_mcd_max_frames() == mcd.MAX_FRAMES


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "mcd.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 9, rep                    # the cepstra kernel and the DTW kernel at K = 8, 16, ..., 64
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


def _z(T, M=80, dtype=torch.float32):
    return torch.zeros(T, M, dtype=dtype)


def test_mel_cepstra_refusals(no_lib):
    from deepvoice3_pytorch_b200 import mcd
    bad = [([], 24), ("x", 24), ([_z(0)], 24), ([_z(16385)], 24), ([_z(5), _z(5, 40)], 24), ([torch.zeros(5)], 24),
           ([_z(5, 1)], 1), ([_z(5, 129)], 24), ([_z(5)], 0), ([_z(5)], 65), ([_z(5, 24)], 24), ([_z(5)], 2.5),
           ([_z(5, dtype=torch.float64)], 24), ([_z(5)], 24)]           # the last: a CPU tensor
    for mels, K in bad:
        with pytest.raises(ValueError):
            mcd.mel_cepstra(mels, K)
    assert no_lib == []


def test_mcd_dtw_and_dtw_refusals(no_lib):
    from deepvoice3_pytorch_b200 import mcd
    for a, b, K in (([], [], 24), ([_z(5)], [], 24), ([_z(5)], [_z(5), _z(6)], 24), ([_z(5)], [_z(0)], 24),
                    ([_z(5)], [_z(16385)], 24), ([_z(5)], [_z(5, 40)], 24), ([_z(5)], [_z(5)], 80),
                    ([_z(5)], [_z(5)], 24)):
        with pytest.raises(ValueError):
            mcd.mcd_dtw(a, b, K)
    for a, b in (([], []), ([_z(5, 24)], []), ([_z(5, 24)], [_z(0, 24)]), ([_z(5, 24)], [_z(5, 23)]),
                 ([_z(5, 65)], [_z(5, 65)]), ([_z(16385, 24)], [_z(5, 24)]), ([_z(5, 24)], [_z(5, 24)])):
        with pytest.raises(ValueError):
            mcd.dtw(a, b)
    assert no_lib == []


def _models():
    from deepvoice3_pytorch_b200 import builder
    kw = dict(n_vocab=40, embed_dim=16, mel_dim=80, linear_dim=9, r=1, downsample_step=4, kernel_size=3,
              encoder_channels=16, decoder_channels=16, converter_channels=16, max_positions=64)
    torch.manual_seed(0)
    ms = builder.deepvoice3_multispeaker(n_speakers=4, speaker_embed_dim=16, speaker_embedding_weight_std=0.2, **kw)
    return builder.deepvoice3(**kw).eval(), ms.eval()


def test_evaluate_synthesis_refusals(no_lib):
    from deepvoice3_pytorch_b200.mcd import evaluate_synthesis
    single, multi = _models()
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    wav = np.zeros(4000, np.float32)
    refs = [wav, wav]
    bad_calls = [
        (single, seqs, [wav], None, {}),                                        # one reference for two sequences
        (single, seqs, refs + [wav], None, {}),
        (single, seqs, "wavs", None, {}),
        (single, seqs, [wav, np.zeros(4000)], None, {}),                        # fp64 reference
        (single, seqs, [wav, np.zeros((2, 4000), np.float32)], None, {}),
        (single, seqs, [wav, np.zeros(0, np.float32)], None, {}),
        (single, seqs, [wav, torch.zeros(4000)], None, {}),
        (single, seqs, [wav, np.zeros(256 * 16400, np.float32)], None, {}),     # more than 16 384 frames
        (single, seqs, refs, None, {"n_ceps": 0}),
        (single, seqs, refs, None, {"n_ceps": 80}),
        (single, seqs, refs, None, {"vocoder": "wavenet"}),
        (single, seqs, refs, [0, 1], {}),                                       # ids for a single-speaker model
        (multi, seqs, refs, None, {}),                                          # no ids for a multi-speaker one
        (multi, seqs, refs, [0, 4], {}),
        (multi, seqs, refs, [0, -1], {}),
        (multi, seqs, refs, [0], {}),
        (single, [np.array([3, 4]), np.array([], np.int64)], refs, None, {}),
        (single, seqs, refs, None, {"batch_size": 0}),
    ]
    for model, sq, rw, ids, kw in bad_calls:
        with pytest.raises(ValueError):
            evaluate_synthesis(model, sq, rw, speaker_ids=ids, **kw)
    assert no_lib == []
