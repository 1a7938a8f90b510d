"""GPU: MCD-DTW (deepvoice3_pytorch_b200/mcd.py, csrc/mcd.cu) against the fp64 restatement of tests/mcd_oracle.py --
cepstra elementwise, DTW cost within a rounding bound and path length exactly, bit for bit on integer cepstra --, batch
independence and run-to-run bits, ``evaluate_synthesis`` on the three presets, and a discrimination check on synthetic
speech-like signals."""
import contextlib
import math

import numpy as np
import pytest
import torch

import mcd_oracle as MO
from test_gpu_synthesis import PRESETS, _model, _sequences

pytestmark = pytest.mark.gpu
U = 2.0 ** -24                    # fp32 unit roundoff


@contextlib.contextmanager
def _conv_math(mode):
    from deepvoice3_pytorch_b200 import ops
    old = ops.conv_math
    ops.conv_math = mode
    try:
        yield
    finally:
        ops.conv_math = old


# ---- cepstra --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K", [(80, 24), (80, 64), (40, 39), (2, 1), (128, 17)])
def test_cepstra_against_the_fp64_oracle(M, K):
    """Each output is one fma chain of M products with table entries rounded once: |err| <= (M + 2) u sum|w||x|."""
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(M * 100 + K)
    lengths = [1, 7, 300, 16, 17]
    mels = [rng.rand(n, M).astype(np.float32) for n in lengths]
    got = mcd.mel_cepstra([torch.from_numpy(m).cuda() for m in mels], K)
    table = np.abs(mcd.dct_basis_fp64(M, K))
    for m, g in zip(mels, got):
        assert tuple(g.shape) == (m.shape[0], K)
        want = MO.cepstra(m, K)
        bound = (M + 2) * U * (m.astype(np.float64) @ table.T) + 1e-30
        err = np.abs(g.cpu().numpy().astype(np.float64) - want)
        assert (err <= bound).all(), float((err / bound).max())


def test_cepstra_read_no_frame_past_a_count_and_write_zeros_there():
    from deepvoice3_pytorch_b200 import mcd
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.ops import _p, _stream
    M, K, T = 80, 24, 40
    rng = np.random.RandomState(2)
    mels = torch.from_numpy(rng.rand(3, T, M).astype(np.float32)).cuda()
    lengths = [40, 1, 23]
    for q, n in enumerate(lengths):
        mels[q, n:] = float("nan")
    cep = torch.full((3, T, K), 7.0, device="cuda")
    lens = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    lib.call("dv3_mel_cepstra", _p(mels), _p(lens), _p(mcd._device_basis(mels.device, M, K)), _p(cep),
             3, T, M, K, _stream())
    alone = mcd.mel_cepstra([mels[q, :n] for q, n in enumerate(lengths)], K)
    for q, n in enumerate(lengths):
        assert torch.equal(cep[q, :n], alone[q])
        assert bool((cep[q, n:] == 0).all())


# ---- DTW --------------------------------------------------------------------------------------------------------------
PAIRS = [(1, 1), (1, 2), (2, 1), (31, 32), (32, 33), (33, 31), (64, 64), (500, 430), (1, 900), (900, 1), (97, 120),
         (200, 65), (33, 1), (1, 33)]


def _warped_pair(rng, N, M, K=24):
    """a: N independent frames; b: a sampled along a random monotone warp plus a little noise -- one clearly best path,
    so the fp32 and fp64 recursions choose the same predecessors on it."""
    a = rng.randn(N, K) * 2.0
    idx = np.sort(rng.randint(0, N, M))
    idx[0], idx[-1] = 0, N - 1
    if M == 1:
        idx = np.array([rng.randint(0, N)])
    b = a[idx] + rng.randn(M, K) * 0.01
    return a.astype(np.float32), b.astype(np.float32)


def _cuda(xs):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]


def test_dtw_against_the_fp64_oracle_on_ragged_pairs():
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(5)
    pairs = [_warped_pair(rng, N, M) for N, M in PAIRS]
    res = mcd.dtw(_cuda([a for a, _ in pairs]), _cuda([b for _, b in pairs]))
    K = 24
    for p, ((a, b), (N, M)) in enumerate(zip(pairs, PAIRS)):
        cost, L = MO.dtw(a, b)
        assert res["path_length"][p] == L, (N, M, res["path_length"][p], L)
        bound = (N + M) * K * U * cost + 1e-6
        assert abs(res["cost"][p] - cost) <= bound, (N, M, res["cost"][p], cost, bound)
        assert res["mcd"][p] == pytest.approx(MO.mcd(res["cost"][p], L), rel=1e-15)


def test_dtw_on_integer_cepstra_is_exact_and_keeps_the_tie_rule():
    """Frames n (3, 4, 0, ...) with small integers n: every distance 5 |n_a - n_b| and every sum is an exact fp32
    integer, and ties are everywhere, so cost and L must equal the oracle's bit for bit."""
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(11)
    shapes = PAIRS + [(6, 6), (40, 70), (70, 40)]
    a_s, b_s = [], []
    for N, M in shapes:
        for side, T in ((a_s, N), (b_s, M)):
            c = np.zeros((T, 24), np.float32)
            n = rng.randint(0, 4, T)
            c[:, 0], c[:, 1] = 3 * n, 4 * n
            side.append(c)
    res = mcd.dtw(_cuda(a_s), _cuda(b_s))
    for p, (a, b) in enumerate(zip(a_s, b_s)):
        cost, L = MO.dtw(a, b)
        assert float(res["cost"][p]) == cost and int(res["path_length"][p]) == L, (shapes[p], res["cost"][p], cost,
                                                                                   res["path_length"][p], L)
        if max(a.shape[0], b.shape[0]) <= 6:
            assert MO.dtw_brute(MO.distances(a, b)) == (cost, L)


@pytest.mark.parametrize("K", [1, 24, 33, 64])
def test_each_pair_alone_in_a_shuffled_batch_and_in_a_second_run_gives_the_same_bits(K):
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(K)
    shapes = [(rng.randint(1, 300), rng.randint(1, 300)) for _ in range(10)] + [(33, 65), (1, 1)]
    a_s = [rng.randn(N, K).astype(np.float32) for N, _ in shapes]
    b_s = [rng.randn(M, K).astype(np.float32) for _, M in shapes]
    batch = mcd.dtw(_cuda(a_s), _cuda(b_s))
    again = mcd.dtw(_cuda(a_s), _cuda(b_s))
    perm = rng.permutation(len(shapes))
    shuffled = mcd.dtw(_cuda([a_s[i] for i in perm]), _cuda([b_s[i] for i in perm]))
    for p in range(len(shapes)):
        alone = mcd.dtw(_cuda([a_s[p]]), _cuda([b_s[p]]))
        q = int(np.where(perm == p)[0][0])
        for key in ("cost", "path_length"):
            vals = [batch[key][p], again[key][p], shuffled[key][q], alone[key][0]]
            assert all(np.asarray(v).tobytes() == np.asarray(vals[0]).tobytes() for v in vals), (p, key, vals)


def test_mcd_dtw_of_mels_matches_the_oracle_and_is_zero_against_itself():
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(8)
    lengths = [(50, 61), (1, 9), (130, 128)]
    a_s = [rng.rand(N, 80).astype(np.float32) for N, _ in lengths]
    b_s = [np.clip(a[np.sort(rng.randint(0, a.shape[0], M))] + rng.randn(M, 80).astype(np.float32) * 0.01, 0, 1)
           for a, (_, M) in zip(a_s, lengths)]
    res = mcd.mcd_dtw(_cuda(a_s), _cuda(b_s))
    for p, (a, b) in enumerate(zip(a_s, b_s)):
        cost, L = MO.dtw(MO.cepstra(a, 24), MO.cepstra(b, 24))
        assert res["path_length"][p] == L
        assert res["mcd"][p] == pytest.approx(MO.mcd(cost, L), rel=1e-4)
    self_res = mcd.mcd_dtw(_cuda(a_s), _cuda(a_s))
    assert (self_res["mcd"] == 0).all() and self_res["path_length"].tolist() == [N for N, _ in lengths]


# ---- evaluate_synthesis ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", PRESETS)
def test_evaluate_synthesis_against_the_models_own_fp32_synthesis(preset, capsys):
    """Reference audio: the model's own earlier fp32 synthesis.  Again in fp32 -> MCD exactly 0 and L = T; in "tc" ->
    small and positive, below 0.05 dB, 10x the largest value measured.  The decoder runs every row to max_decoder_steps, so both sides have the same frame count."""
    from deepvoice3_pytorch_b200.mcd import evaluate_synthesis
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    model = _model(preset, max_steps=40, done_bias=-20.0)
    seqs = _sequences([37, 5, 61])
    spk = [3, 17, 0] if model.n_speakers > 1 else None
    with _conv_math("fp32"):
        refs = [w.astype(np.float32) for w, _, _, _ in tts_batch(model, seqs, spk)]
        stages = []
        same = evaluate_synthesis(model, seqs, refs, speaker_ids=spk,
                                  stage_timer=lambda name: stages.append(name) or contextlib.nullcontext())
    assert stages == ["synthesis", "mel", "mel", "mcd"]
    assert (same["mcd"] == 0).all()
    assert (same["path_length"] == same["frames"][:, 1]).all() and (same["frames"][:, 0] == same["frames"][:, 1]).all()
    assert (same["frame_ratio"] == 1.0).all() and same["mean_mcd"] == 0.0 and same["median_mcd"] == 0.0
    with _conv_math("tc"):
        tc = evaluate_synthesis(model, seqs, refs, speaker_ids=spk)
    with capsys.disabled():
        print("\n%s: tc vs fp32 MCD %s dB, path lengths %s, frames %s" % (preset, np.round(tc["mcd"], 4).tolist(),
                                                                           tc["path_length"].tolist(),
                                                                           tc["frames"].tolist()))
    # measured on an H100: 0.0002 dB (deepvoice3_ljspeech, deepvoice3_vctk) and 0.0023-0.0054 dB (nyanko_ljspeech)
    assert (tc["mcd"] > 0).all() and (tc["mcd"] < 0.05).all(), tc["mcd"]
    assert (tc["frame_ratio"] == 1.0).all()


def test_evaluate_synthesis_single_speaker_model_without_ids():
    from deepvoice3_pytorch_b200.mcd import evaluate_synthesis
    model = _model("nyanko_ljspeech", max_steps=24)
    rng = np.random.RandomState(1)
    refs = [(rng.randn(n) * 0.1).astype(np.float32) for n in (6000, 9000)]
    res = evaluate_synthesis(model, _sequences([12, 30]), refs, n_ceps=13)
    assert res["mcd"].shape == (2,) and np.isfinite(res["mcd"]).all() and (res["mcd"] > 0).all()
    assert res["frames"].shape == (2, 2)
    assert res["mean_mcd"] == pytest.approx(res["mcd"].mean()) and res["median_mcd"] == pytest.approx(
        np.median(res["mcd"]))


# ---- discrimination on speech-like signals ----------------------------------------------------------------------------
def _voiced(f0, formants, seconds, sr=22050, stretch=1.0):
    """A harmonic tone at f0 through formant-like resonances (a sum of Gaussian bumps on the harmonic amplitudes), with a
    slow pitch wobble; ``stretch`` lengthens it in time at the same pitch and envelope."""
    n = int(seconds * stretch * sr)
    t = np.arange(n) / sr
    f = f0 * (1.0 + 0.03 * np.sin(2 * np.pi * 3.0 * t / stretch))
    phase = 2 * np.pi * np.cumsum(f) / sr
    x = np.zeros(n)
    for h in range(1, int(5000 / f0)):
        fh = h * f0
        amp = sum(math.exp(-0.5 * ((fh - c) / w) ** 2) for c, w in formants) + 1e-3
        x += amp * np.sin(h * phase)
    env = np.minimum(1.0, np.minimum(t, t[-1] - t) / 0.02)
    return (0.3 * x / np.abs(x).max() * env).astype(np.float32)


def test_mcd_tells_a_stretched_self_from_a_different_envelope():
    from deepvoice3_pytorch_b200 import audio, mcd
    envelopes = [[(700, 120), (1200, 150), (2600, 200)], [(300, 80), (2300, 150), (3000, 200)],
                 [(500, 100), (900, 120), (2400, 200)], [(400, 90), (1900, 150), (2700, 200)]]
    f0s = [110.0, 180.0, 140.0, 220.0]
    base = [_voiced(f0, env, 0.8) for f0, env in zip(f0s, envelopes)]
    stretched = [_voiced(f0, env, 0.8, stretch=1.3) for f0, env in zip(f0s, envelopes)]
    other = [_voiced(f0, envelopes[(k + 1) % 4], 0.8) for k, f0 in enumerate(f0s)]

    def mels(wavs):
        lens = [len(w) for w in wavs]
        pad = np.zeros((len(wavs), max(lens)), np.float32)
        for k, w in enumerate(wavs):
            pad[k, :lens[k]] = w
        _, m = audio.stft_mel_batch(torch.from_numpy(pad).cuda(), torch.tensor(lens, dtype=torch.int32),
                                    want_linear=False)
        return [m[k, :audio.num_frames(n)] for k, n in enumerate(lens)]

    same = mcd.mcd_dtw(mels(base), mels(stretched))["mcd"]
    diff = mcd.mcd_dtw(mels(base), mels(other))["mcd"]
    assert (same < diff).all(), (same, diff)
