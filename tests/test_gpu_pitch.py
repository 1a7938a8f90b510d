"""GPU: the YIN F0 tracker (deepvoice3_pytorch_b200/pitch.py, csrc/pitch.cu) against the fp64 restatement of
tests/pitch_oracle.py -- d and d' elementwise within a derived fp32 bound, the decision wherever its margins exceed that
bound, f0 within its propagated bound --, its bits alone, in a shuffled batch and in a second run; ``mcd.dtw_path``
against ``mcd.dtw`` bit for bit and against the oracle's path; ``evaluate_pitch`` on the three presets; and a
discrimination check on synthetic speech-like signals."""
import contextlib

import numpy as np
import pytest
import torch

import mcd_oracle as MO
import pitch_oracle as PO
from test_gpu_mcd import _conv_math, _cuda, _voiced, _warped_pair
from test_gpu_synthesis import PRESETS, _model, _sequences

pytestmark = pytest.mark.gpu
SR = 22050
U = 2.0 ** -24


def _signals():
    rng = np.random.RandomState(0)
    t = np.arange(12000) / SR
    tone = lambda f, a=0.5: (a * np.sin(2 * np.pi * f * t + 0.4)).astype(np.float32)
    harm = sum(0.3 / h * np.sin(2 * np.pi * 140.0 * h * t) for h in range(1, 9)).astype(np.float32)
    mixed = np.concatenate([tone(200.0)[:5000], np.zeros(3000, np.float32), rng.randn(4000).astype(np.float32) * 0.1])
    return [tone(65.0), tone(230.0), tone(480.0, 0.01), harm, rng.randn(9000).astype(np.float32) * 0.3,
            np.zeros(2000, np.float32), mixed, _voiced(120.0, [(700, 120), (1200, 150), (2600, 200)], 0.5),
            _voiced(210.0, [(300, 80), (2300, 150), (3000, 200)], 0.4), tone(300.0)[:1], tone(300.0)[:700]]


def _gpu_yin(wavs, silence_db=float("-inf"), **kw):
    from deepvoice3_pytorch_b200 import pitch
    tau_min, tau_max, gate = pitch.yin_params(silence_db=silence_db, **kw)
    clips = _cuda(wavs)
    frames = pitch._check_wavs(clips)
    f0, ap, energy, diff = pitch._yin(clips, frames, tau_min, tau_max, kw.get("threshold", 0.1), gate, want_diff=True)
    offs = np.concatenate([[0], np.cumsum(frames)])
    cut = lambda x: [x[offs[k]:offs[k + 1]].cpu().numpy() for k in range(len(frames))]
    return cut(f0), cut(ap), cut(energy), cut(diff)


# ---- YIN against the oracle ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f0_min,f0_max,threshold", [(60.0, 500.0, 0.1), (50.0, 400.0, 0.15), (100.0, 1000.0, 0.05),
                                                   (25.0, 400.0, 0.1)])      # tau_max 882: three warps a frame
def test_yin_against_the_fp64_oracle(f0_min, f0_max, threshold):
    wavs = _signals()
    kw = dict(f0_min=f0_min, f0_max=f0_max, threshold=threshold)
    f0, ap, energy, diff = _gpu_yin(wavs, **kw)
    W = 1024
    checked = voiced_checked = 0
    for k, x in enumerate(wavs):
        r = PO.yin(x, silence_db=-np.inf, **kw)
        tau_min, tau_max = r["tau_min"], r["tau_max"]
        assert f0[k].shape == (PO.num_frames(x.size),) and diff[k].shape == (f0[k].size, 2, tau_max)
        d, dp = diff[k][:, 0].astype(np.float64), diff[k][:, 1].astype(np.float64)
        assert (np.abs(d - r["d"]) <= PO.d_bound(r["d"], W) + 1e-30).all(), k
        e = PO.dp_bound(r["dp"], W)
        e_dec = e + 2 * U * threshold                      # the kernel compares with threshold rounded to fp32
        assert (np.abs(dp - r["dp"]) <= e + 1e-30).all(), (k, float((np.abs(dp - r["dp"]) / (e + 1e-30)).max()))
        assert (np.abs(energy[k] - r["energy"]) <= (W + 2) * U * r["energy"] + 1e-30).all()
        for t in range(f0[k].size):
            if not PO.stable(r["dp"][t], e_dec[t], tau_min, tau_max, threshold):
                continue
            checked += 1
            assert (f0[k][t] > 0) == r["voiced"][t], (k, t)
            assert ap[k][t] == diff[k][t, 1, r["tau"][t] - 1], (k, t)      # the same tau*
            if r["voiced"][t]:
                b = PO.f0_bound(r["dp"][t], e[t], r["tau"][t], tau_min, tau_max, SR)
                if b is not None:
                    voiced_checked += 1
                    assert abs(f0[k][t] - r["f0"][t]) <= b, (k, t, f0[k][t], r["f0"][t], b)
    assert checked > 200 and voiced_checked > 100, (checked, voiced_checked)


def test_tones_and_silence_gate_on_the_gpu():
    from deepvoice3_pytorch_b200 import pitch
    t = np.arange(12000) / SR
    freqs = [65.0, 97.0, 150.0, 220.0, 330.0, 480.0]
    wavs = [(0.5 * np.sin(2 * np.pi * f * t)).astype(np.float32) for f in freqs]
    quiet = np.concatenate([wavs[3][:8000], wavs[3][:8000] * np.float32(10 ** (-70 / 20))])
    res = pitch.yin_f0(_cuda(wavs + [quiet, np.zeros(3000, np.float32)]))
    for f, (f0, ap) in zip(freqs, res):
        a = np.arange(f0.shape[0]) * 256 + 256 - 512 - (1024 + 368) // 2
        inside = (a >= 0) & (a + 1024 + 368 <= 12000)
        got = f0.cpu().numpy()[inside]
        assert (got > 0).all() and np.abs(got / f - 1).max() < 1e-3, (f, got)
    f0q = res[-2][0].cpu().numpy()
    a = np.arange(f0q.size) * 256 + 256 - 512 - (1024 + 368) // 2
    assert (f0q[(a >= 8000) & (a + 1392 <= 16000)] == 0).all() and (f0q[(a >= 0) & (a + 1392 <= 8000)] > 0).all()
    f0s, aps = res[-1]
    assert (f0s == 0).all() and (aps == 1).all()


def test_each_clip_alone_in_a_shuffled_batch_and_in_a_second_run_gives_the_same_bits():
    from deepvoice3_pytorch_b200 import pitch
    wavs = _signals()
    batch = pitch.yin_f0(_cuda(wavs))
    again = pitch.yin_f0(_cuda(wavs))
    perm = np.random.RandomState(1).permutation(len(wavs))
    shuffled = pitch.yin_f0(_cuda([wavs[i] for i in perm]))
    for k in range(len(wavs)):
        alone = pitch.yin_f0(_cuda([wavs[k]]))[0]
        q = int(np.where(perm == k)[0][0])
        for i in range(2):
            vals = [batch[k][i], again[k][i], shuffled[q][i], alone[i]]
            assert all(v.cpu().numpy().tobytes() == vals[0].cpu().numpy().tobytes() for v in vals), (k, i)


# ---- dtw_path ---------------------------------------------------------------------------------------------------------
PAIRS = [(1, 1), (1, 2), (2, 1), (31, 32), (32, 33), (33, 31), (64, 64), (500, 430), (1, 900), (900, 1), (97, 120),
         (200, 65), (33, 1), (1, 33), (17, 300)]


def _check_path(p, N, M, L):
    assert p.shape == (L, 2) and p.dtype == np.int64
    assert tuple(p[0]) == (0, 0) and tuple(p[-1]) == (N - 1, M - 1)
    steps = np.diff(p, axis=0)
    assert ((steps == [1, 1]).all(1) | (steps == [1, 0]).all(1) | (steps == [0, 1]).all(1)).all()


@pytest.mark.parametrize("K", [1, 24, 64])
def test_dtw_path_cost_and_length_are_dtw_bit_for_bit_and_the_path_sums_to_the_cost(K):
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(K)
    pairs = [_warped_pair(rng, N, M, K) for N, M in PAIRS]
    a, b = _cuda([x for x, _ in pairs]), _cuda([y for _, y in pairs])
    ref = mcd.dtw(a, b)
    res = mcd.dtw_path(a, b)
    for key in ("cost", "path_length", "mcd"):
        assert res[key].tobytes() == ref[key].tobytes(), key
    for p, ((x, y), (N, M)) in enumerate(zip(pairs, PAIRS)):
        path = res["path"][p]
        _check_path(path, N, M, int(res["path_length"][p]))
        d = MO.distances(x, y)
        resum = d[path[:, 0], path[:, 1]].sum()
        assert abs(resum - res["cost"][p]) <= (N + M) * K * U * resum + 1e-6, (N, M)


def test_dtw_path_on_integer_features_is_the_oracles_path():
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(11)
    shapes = PAIRS + [(6, 6), (40, 70), (70, 40), (5, 3)]
    a_s, b_s = [], []
    for N, M in shapes:
        for side, T in ((a_s, N), (b_s, M)):
            c = np.zeros((T, 24), np.float32)
            n = rng.randint(0, 4, T)
            c[:, 0], c[:, 1] = 3 * n, 4 * n
            side.append(c)
    res = mcd.dtw_path(_cuda(a_s), _cuda(b_s))
    for p, (a, b) in enumerate(zip(a_s, b_s)):
        cost, path = PO.dtw_path(MO.distances(a, b))
        assert float(res["cost"][p]) == cost and np.array_equal(res["path"][p], path), shapes[p]
        if max(a.shape[0], b.shape[0]) <= 6:
            assert np.array_equal(PO.path_brute(MO.distances(a, b))[1], path)


def test_dtw_path_with_a_nan_feature_row_stays_in_the_grid():
    """A NaN feature row makes D NaN (or, on a single row or column, +inf) from there on; the comparisons against NaN
    fail and the stored code can be the diagonal on row and column 1.  The backtrace must still walk a monotone unit-step path from corner to corner inside the grid --
    the oracle's, on integer features -- and leave the finite pairs of the batch as they are alone."""
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(12)
    shapes = [(40, 70), (70, 40), (33, 1), (1, 33), (6, 6), (300, 17)]
    a_s, b_s = [], []
    for N, M in shapes:
        for side, T in ((a_s, N), (b_s, M)):
            c = np.zeros((T, 24), np.float32)
            n = rng.randint(0, 4, T)
            c[:, 0], c[:, 1] = 3 * n, 4 * n
            side.append(c)
    bad_a, bad_b = [a.copy() for a in a_s], [b.copy() for b in b_s]
    for k, (N, M) in enumerate(shapes):
        if k % 2:
            bad_b[k][rng.randint(0, M), 5] = np.nan
        else:
            bad_a[k][rng.randint(0, N), 5] = np.nan
    finite = (np.zeros((1, 24), np.float32) + 1, np.zeros((9, 24), np.float32))
    res = mcd.dtw_path(_cuda(bad_a + [finite[0]]), _cuda(bad_b + [finite[1]]))
    for p, (N, M) in enumerate(shapes):
        cost, want = PO.dtw_path(MO.distances(bad_a[p], bad_b[p]))
        assert not np.isfinite(res["cost"][p]) and np.isnan(res["cost"][p]) == np.isnan(cost), (shapes[p], cost)
        path = res["path"][p]
        assert tuple(path[0]) == (0, 0) and tuple(path[-1]) == (N - 1, M - 1)
        steps = np.diff(path, axis=0)
        assert ((steps == [1, 1]).all(1) | (steps == [1, 0]).all(1) | (steps == [0, 1]).all(1)).all()
        assert np.array_equal(path, want), shapes[p]
    alone = mcd.dtw_path(_cuda([finite[0]]), _cuda([finite[1]]))
    assert res["cost"][-1] == alone["cost"][0] and np.array_equal(res["path"][-1], alone["path"][0])
    _check_path(res["path"][-1], 1, 9, int(res["path_length"][-1]))


def test_dtw_path_in_several_budget_chunks_equals_one_launch(monkeypatch):
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(4)
    shapes = [(rng.randint(1, 400), rng.randint(1, 400)) for _ in range(12)] + [(1, 900), (33, 31)]
    a_s = [rng.randn(N, 24).astype(np.float32) for N, _ in shapes]
    b_s = [rng.randn(M, 24).astype(np.float32) for _, M in shapes]
    one = mcd.dtw_path(_cuda(a_s), _cuda(b_s))
    monkeypatch.setattr(mcd, "DIR_BUDGET_BYTES", 40_000)
    work, _ = mcd._work_list(list(range(14)), [N for N, _ in shapes], list(range(14)), [M for _, M in shapes])
    assert len(mcd._path_chunks(work)) >= 4
    many = mcd.dtw_path(_cuda(a_s), _cuda(b_s))
    for key in ("cost", "path_length"):
        assert one[key].tobytes() == many[key].tobytes()
    assert all(np.array_equal(x, y) for x, y in zip(one["path"], many["path"]))


# ---- evaluate_pitch ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", PRESETS)
def test_evaluate_pitch_against_the_models_own_fp32_synthesis(preset, capsys):
    from deepvoice3_pytorch_b200.mcd import evaluate_synthesis
    from deepvoice3_pytorch_b200.pitch import evaluate_pitch
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    model = _model(preset, max_steps=40, done_bias=-20.0)
    seqs = _sequences([37, 5, 61])
    spk = [3, 17, 0] if model.n_speakers > 1 else None
    with _conv_math("fp32"):
        refs = [w.astype(np.float32) for w, _, _, _ in tts_batch(model, seqs, spk)]
        stages = []
        same = evaluate_pitch(model, seqs, refs, speaker_ids=spk,
                              stage_timer=lambda name: stages.append(name) or contextlib.nullcontext())
        mcd_same = evaluate_synthesis(model, seqs, refs, speaker_ids=spk)
    assert stages == ["synthesis", "mel", "mel", "f0", "dtw"]
    assert same["mcd"].tobytes() == mcd_same["mcd"].tobytes()
    assert (same["vde"] == 0).all() and (same["ffe"] == 0).all()
    assert np.all((same["gpe"] == 0) | np.isnan(same["gpe"]))
    assert np.all((same["f0_rmse_cents"] == 0) | np.isnan(same["f0_rmse_cents"]))
    assert (same["path_length"] == same["frames"][:, 1]).all() and (same["frame_ratio"] == 1.0).all()
    assert (same["voiced_fraction"][:, 0] == same["voiced_fraction"][:, 1]).all()
    with _conv_math("tc"):
        tc = evaluate_pitch(model, seqs, refs, speaker_ids=spk)
    with capsys.disabled():
        print("\n%s: tc vs fp32 VDE %s GPE %s FFE %s RMSE %s cents, voiced %s" % (
            preset, tc["vde"].round(4).tolist(), tc["gpe"].round(4).tolist(), tc["ffe"].round(4).tolist(),
            tc["f0_rmse_cents"].round(2).tolist(), tc["voiced_fraction"].round(3).tolist()))
    assert (tc["mcd"] < 0.05).all()
    assert (tc["vde"] <= 0.2).all() and (tc["ffe"] <= 0.25).all()
    assert np.all(np.isnan(tc["gpe"]) | (tc["gpe"] <= 0.2))
    assert np.all(np.isnan(tc["f0_rmse_cents"]) | (tc["f0_rmse_cents"] < 200.0))


# ---- discrimination on speech-like signals ----------------------------------------------------------------------------
def test_pitch_errors_tell_a_stretched_self_from_a_pitch_shift_and_from_noise(capsys):
    from deepvoice3_pytorch_b200 import audio, mcd, pitch
    from deepvoice3_pytorch_b200.synthesis import wav_mels
    envelopes = [[(700, 120), (1200, 150), (2600, 200)], [(300, 80), (2300, 150), (3000, 200)],
                 [(500, 100), (900, 120), (2400, 200)], [(400, 90), (1900, 150), (2700, 200)]]
    f0s = [110.0, 180.0, 140.0, 220.0]
    base = [_voiced(f0, env, 0.8) for f0, env in zip(f0s, envelopes)]
    stretched = [_voiced(f0, env, 0.8, stretch=1.3) for f0, env in zip(f0s, envelopes)]
    shifted = [_voiced(1.3 * f0, env, 0.8) for f0, env in zip(f0s, envelopes)]
    rng = np.random.RandomState(2)
    noise = [(rng.randn(b.size) * 0.1).astype(np.float32) for b in base]
    dev = torch.device("cuda")

    def score(a_w, b_w):
        ma, mb = wav_mels(a_w, dev), wav_mels(b_w, dev)
        paths = mcd.dtw_path(mcd.mel_cepstra(ma), mcd.mel_cepstra(mb))["path"]
        tracks = pitch.yin_f0(_cuda(a_w + b_w))
        return pitch.f0_metrics([f for f, _ in tracks[:4]], [f for f, _ in tracks[4:]], paths)

    same, shift, noisy = score(base, stretched), score(shifted, base), score(base, noise)
    with capsys.disabled():
        print("\nstretched: GPE %s RMSE %s VDE %s; shifted: GPE %s; noise: VDE %s, voiced %s" % (
            same["gpe"].round(4).tolist(), same["f0_rmse_cents"].round(2).tolist(), same["vde"].round(4).tolist(),
            shift["gpe"].round(4).tolist(), noisy["vde"].round(4).tolist(), noisy["voiced_fraction"].round(3).tolist()))
    assert (same["gpe"] < 0.05).all() and (same["f0_rmse_cents"] < 50.0).all()
    assert (shift["gpe"] > 0.9).all()
    # noise is never voiced, so its VDE is the voiced share of the clip's path pairs: 0.36-0.81 against 0.16-0.30 for
    # the stretched self (measured on an H100; the formant-shaped tones are voiced in 36-81 % of their frames)
    assert (noisy["voiced_fraction"][:, 1] == 0).all()
    assert (noisy["vde"] > 0.3).all() and (noisy["vde"] > same["vde"]).all()
    assert audio.hparams.sample_rate == SR
