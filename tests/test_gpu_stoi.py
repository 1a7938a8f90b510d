"""GPU: the STOI / ESTOI kernels of csrc/stoi.cu stage by stage against the fp64 oracle (tests/stoi_oracle.py), each
stage fed the oracle's input to it; the whole measure end to end at 22.05 and 16 kHz; bits independent of the batch and
of the run; the DTW-warped measure; copy synthesis through the three phase-recovery methods; evaluate_intelligibility
on the three presets; and the unchanged launch of resample_batch without sr_to."""
import contextlib
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

import stoi_oracle as SO
from test_gpu_synthesis import PRESETS, _conv_math, _model, _sequences
from test_stoi_host import voiced

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
E2E_BOUND = 1e-4                  # |GPU - oracle| of a pair's STOI and ESTOI


def _cuda(xs):
    return [torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda() for x in xs]


def _speech(n, sr, seed, snr_db=None):
    """``voiced`` at sr, optionally with white noise at snr_db."""
    x = voiced(n, sr, seed).astype(np.float64)
    if snr_db is not None:
        noise = np.random.RandomState(seed + 100).randn(n)
        x = x + noise * math.sqrt(np.mean(x ** 2) / np.mean(noise ** 2) / 10 ** (snr_db / 10))
    return x.astype(np.float32)


@pytest.fixture
def at_10k(monkeypatch):
    """Clips at 10 kHz: resample_batch runs its one-tap identity bank, so every stage sees the clip's own fp32 values."""
    from deepvoice3_pytorch_b200 import audio
    monkeypatch.setattr(audio.hparams, "sample_rate", 10000)


LENGTHS = [4000, 12345, 20000, 30001, 7777]


def _clips(seed=0):
    out = []
    for k, n in enumerate(LENGTHS):
        x = _speech(n, 10000, seed + k, snr_db=[None, 20, 5, 0, 30][k])
        if k == 2:
            x[6000:9000] *= 1e-3                  # a quiet stretch: frames the mask removes
        out.append(x)
    return out


def _margin_ok(e, thr):
    return np.abs(e - thr).min() > 1e-3


# ---- stage by stage ---------------------------------------------------------------------------------------------------
def test_stages_against_the_fp64_oracle(at_10k, capsys):
    from deepvoice3_pytorch_b200 import intelligibility as I
    from deepvoice3_pytorch_b200._lib import lib
    xs = _clips()
    n = len(xs)
    an = I._Analysis(_cuda(xs), list(range(n)))
    torch.cuda.synchronize()
    desc = an.clips.cpu().numpy()
    energy, keep = an.energy.cpu().numpy(), an.keep.cpu().numpy()
    kept, frames = an.kept.cpu().numpy(), an.frames.cpu().numpy()
    ola = an.ola.cpu().numpy()
    worst = {"ola": 0.0, "env": 0.0}
    ola_want, masks = [], []
    for c, x in enumerate(xs):
        F0, fo, oo = SO.num_frames(x.size), int(desc[c, 2]), int(desc[c, 3])
        e = SO.frame_energies(x)
        np.testing.assert_allclose(energy[fo:fo + F0], e, rtol=0, atol=1e-9)
        thr = e.max() - SO.DYN_RANGE
        assert _margin_ok(e, thr), c
        mask = SO.keep_mask(e)
        assert np.array_equal(keep[fo:fo + F0].astype(bool), mask) and kept[c] == mask.sum(), c
        assert frames[c] == mask.sum() - 1
        masks.append(mask)
        # overlap-add: the mask equals the oracle's, so the kernel saw the oracle's input; two products and a sum in fp32
        want = SO.overlap_add(x.astype(np.float64), mask)
        scale = SO.overlap_add(np.abs(x.astype(np.float64)), mask)
        got = ola[oo:oo + want.size]
        err = np.abs(got - want)
        assert (err <= 4 * U * scale + 1e-30).all(), c
        worst["ola"] = max(worst["ola"], float((err / (4 * U * scale + 1e-30)).max()))
        ola_want.append(want.astype(np.float32))
    # band envelopes, fed the oracle's compacted signals rounded to fp32
    for c, y in enumerate(ola_want):
        an.ola[int(desc[c, 3]):int(desc[c, 3]) + y.size] = torch.from_numpy(y).cuda()
    table, _, bands = I._tables(an.ola.device)
    blocks = [(c, t0) for c in range(n) for t0 in range(0, max(an.F0[c] - 1, 0), I.BAND_WARPS)]
    blocks_d = torch.tensor(blocks, dtype=torch.int32).cuda()
    env = torch.full_like(an.env, float("nan"))
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    lib.call("dv3_stoi_bands", p(an.ola), p(an.clips), p(blocks_d), len(blocks), p(table), p(bands), p(an.frames),
             p(env), None, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    env = env.cpu().numpy()
    envs = []
    for c, y in enumerate(ola_want):
        F0, fo, F = an.F0[c], int(desc[c, 2]), int(frames[c])
        want = SO.envelopes(y.astype(np.float64))
        got = env[15 * fo:15 * fo + 15 * F0].reshape(15, F0)[:, :F]
        # the transform's rounding, norm-wise: the input products (u), four radix-4 passes and the split with rounded
        # twiddles (<= 6 u each) -> ||dX|| <= 32 u ||X_512||, ||X_512|| = sqrt(512) ||w y_t||; then the band's
        # <= 45-term fp32 sum and the square root (<= 32 u relative)
        fr = SO.frames(y.astype(np.float64))
        bound = 32 * U * math.sqrt(512) * np.sqrt((fr ** 2).sum(1))[None, :] + 32 * U * want
        assert want.shape == got.shape and (np.abs(got - want) <= bound).all(), c
        worst["env"] = max(worst["env"], float((np.abs(got - want) / bound).max()))
        envs.append(want.astype(np.float32))
    # segments, fed the oracle's envelopes rounded to fp32: fp64 from there on, so 1e-9
    for c, X in enumerate(envs):
        fo, F0 = int(desc[c, 2]), an.F0[c]
        full = np.zeros((15, F0), np.float32)
        full[:, :X.shape[1]] = X
        an.env[15 * fo:15 * fo + 15 * F0] = torch.from_numpy(full.ravel()).cuda()
    # random monotone paths between clips of 54-232 frames.  A path that holds one side on a frame for nearly a whole
    # segment (the 9-frame clip 0 against a long one) makes every normalised row of that side the same step function,
    # so ESTOI's column normalisation divides rounding noise by its own norm: ill-posed, and left out here.
    rng = np.random.RandomState(4)
    pairs, paths = [], []
    for a, b in [(1, 2), (3, 3), (2, 4), (4, 1)]:
        Fa, Fb = envs[a].shape[1], envs[b].shape[1]
        steps = np.sort(rng.choice(Fa + Fb - 2, Fa - 1, replace=False))       # a random monotone path, corner to corner
        moves = np.ones(Fa + Fb - 2, int)
        moves[steps] = 0
        i = np.concatenate([[0], np.cumsum(moves == 0)])
        j = np.concatenate([[0], np.cumsum(moves == 1)])
        pairs.append((a, b))
        paths.append(np.stack([i, j], 1).astype(np.int32))
    L = np.array([len(q) for q in paths], np.int32)
    res, counts, seg = an.segments(pairs, paths, torch.from_numpy(L).cuda(), [max(int(l) - 29, 0) for l in L])
    res, counts, seg = res.cpu().numpy(), counts.cpu().numpy(), seg.cpu().numpy()
    off = 0
    for q, ((a, b), path) in enumerate(zip(pairs, paths)):
        want = SO.segment_values(envs[a], envs[b], path)
        J = want.shape[0]
        assert counts[q, 0] == J and counts[q, 1] == kept[a]
        np.testing.assert_allclose(seg[off:off + J], want, rtol=0, atol=1e-9)
        np.testing.assert_allclose(res[q], SO.pair_means(want), rtol=0, atol=1e-9)
        off += J
    with capsys.disabled():
        print("\nstoi stages: worst error / bound: overlap-add %.3g, envelopes %.3g" % (worst["ola"], worst["env"]))


# ---- end to end -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", [22050, 16000])
def test_end_to_end_against_the_oracle(sr, monkeypatch, capsys):
    from deepvoice3_pytorch_b200 import audio, intelligibility as I
    monkeypatch.setattr(audio.hparams, "sample_rate", sr)
    rng = np.random.RandomState(sr)
    clean, proc = [], []
    for k, (secs, snr) in enumerate([(1.0, 20), (2.5, 5), (3.3, 0), (0.3, 10), (1.7, -5), (2.0, 30)]):
        n = int(secs * sr) + rng.randint(0, 300)
        x = _speech(n, sr, 10 + k)
        y = x + (rng.randn(n) * math.sqrt(np.mean(x.astype(np.float64) ** 2) / 10 ** (snr / 10))).astype(np.float32)
        clean.append(x)
        proc.append(y.astype(np.float32))
    got = I.stoi(_cuda(clean), _cuda(proc))
    worst = 0.0
    for k, (x, y) in enumerate(zip(clean, proc)):
        want = SO.stoi(x, y, sr)
        assert got["segments"][k] == want["segments"] and got["kept_frames"][k] == want["kept_frames"], k
        if want["segments"] == 0:
            assert math.isnan(got["stoi"][k]) and math.isnan(got["estoi"][k])
            continue
        for key in ("stoi", "estoi"):
            err = abs(got[key][k] - want[key])
            worst = max(worst, err)
            assert err <= E2E_BOUND, (k, key, got[key][k], want[key])
    assert np.isnan(got["stoi"]).sum() == 1                      # the 0.3 s clip
    with capsys.disabled():
        print("\nstoi end to end at %d Hz: worst |GPU - oracle| %.3g, stoi %s" % (sr, worst, got["stoi"].round(4)))


# ---- bits -------------------------------------------------------------------------------------------------------------
def test_ragged_batches_give_each_pair_its_own_bits_run_to_run():
    from deepvoice3_pytorch_b200 import intelligibility as I
    rng = np.random.RandomState(1)
    ns = [22050, 5000, 60000, 33333, 12000]
    clean = [_speech(n, 22050, 20 + k) for k, n in enumerate(ns)]
    proc = [(x + 0.05 * rng.randn(x.size)).astype(np.float32) for x in clean]
    other = [_speech(n + 4000 * (k % 2), 22050, 40 + k) for k, n in enumerate(ns)]
    for fn, b in ((I.stoi, proc), (I.stoi_dtw, other)):
        many = fn(_cuda(clean), _cuda(b))
        again = fn(_cuda(clean), _cuda(b))
        order = [3, 0, 4, 2, 1]
        shuffled = fn(_cuda([clean[k] for k in order]), _cuda([b[k] for k in order]))
        for key in many:
            assert many[key].tobytes() == again[key].tobytes(), (fn.__name__, key)
        for k in range(len(ns)):
            alone = fn(_cuda([clean[k]]), _cuda([b[k]]))
            for key in alone:
                assert alone[key][0].tobytes() == many[key][k].tobytes(), (fn.__name__, key, k)
                assert shuffled[key][order.index(k)].tobytes() == many[key][k].tobytes(), (fn.__name__, key, k)


def test_stoi_dtw_of_identical_inputs_is_stoi_bit_for_bit():
    from deepvoice3_pytorch_b200 import intelligibility as I
    rng = np.random.RandomState(2)
    xs = [_speech(n, 22050, 60 + k, snr_db=s) for k, (n, s) in enumerate([(30000, None), (50000, 10), (15000, 0),
                                                                            (3000, None)])]
    xs.append((0.1 * rng.randn(40000)).astype(np.float32))
    a, w = I.stoi(_cuda(xs), _cuda(xs)), I.stoi_dtw(_cuda(xs), _cuda(xs))
    for key in ("stoi", "estoi", "segments", "kept_frames"):
        assert a[key].tobytes() == w[key].tobytes(), key
    ok = a["segments"] > 0
    assert ok.sum() == 4
    assert (w["path_length"][ok] == w["frames"][ok, 0]).all() and (w["frames"][:, 0] == w["frames"][:, 1]).all()
    assert np.all(np.abs(a["stoi"][ok] - 1) < 1e-9) and np.all(np.abs(a["estoi"][ok] - 1) < 1e-9)


def test_stoi_dtw_prefers_a_time_stretched_self_to_an_unrelated_clip(capsys):
    from deepvoice3_pytorch_b200 import intelligibility as I
    clean, stretched, unrelated = [], [], []
    for k in range(3):
        x = _speech(44100 + 5000 * k, 22050, 80 + k, snr_db=30)
        clean.append(x)
        stretched.append(resample_poly(x.astype(np.float64), 11, 10).astype(np.float32))    # 10 % slower
        unrelated.append(_speech(48000 + 3000 * k, 22050, 90 + k, snr_db=30))
    s = I.stoi_dtw(_cuda(clean), _cuda(stretched))
    u = I.stoi_dtw(_cuda(clean), _cuda(unrelated))
    with capsys.disabled():
        print("\nstoi_dtw stretched %s / %s, unrelated %s / %s" % (s["stoi"].round(3), s["estoi"].round(3),
                                                                    u["stoi"].round(3), u["estoi"].round(3)))
    assert (s["stoi"] > u["stoi"]).all() and (s["estoi"] > u["estoi"]).all()
    assert (s["frames"][:, 1] > s["frames"][:, 0]).all() and (s["path_length"] >= s["frames"][:, 1]).all()


# ---- copy synthesis ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["griffin_lim", "lws", "fast_griffin_lim"])
def test_evaluate_vocoder_against_the_oracle_on_its_own_waveforms(method, capsys):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200.intelligibility import evaluate_vocoder
    sr = audio.hparams.sample_rate
    wavs = [_speech(n, sr, 100 + k, snr_db=40) for k, n in enumerate([33000, 41000, 27000])]
    res = evaluate_vocoder(_cuda(wavs), method=method)
    with capsys.disabled():
        print("\n%s copy synthesis: stoi %s estoi %s" % (method, res["stoi"].round(4), res["estoi"].round(4)))
    for key in ("stoi", "estoi"):
        assert np.isfinite(res[key]).all() and (np.abs(res[key]) <= 1).all()
    assert res["mean_stoi"] == pytest.approx(res["stoi"].mean(), abs=1e-15)
    for k, (x, v) in enumerate(zip(wavs, res["vocoded"])):
        v = v.cpu().numpy()
        want = SO.stoi(x[:v.size], v, sr)
        assert abs(res["stoi"][k] - want["stoi"]) <= E2E_BOUND and abs(res["estoi"][k] - want["estoi"]) <= E2E_BOUND


# ---- evaluate_intelligibility -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", PRESETS)
def test_evaluate_intelligibility_is_stoi_dtw_of_the_synthesized_audio(preset):
    from deepvoice3_pytorch_b200.intelligibility import evaluate_intelligibility, stoi_dtw
    from deepvoice3_pytorch_b200.synthesis import synthesized_audio
    model = _model(preset, max_steps=60, done_bias=-20.0)
    seqs = _sequences([37, 5, 61])
    spk = [3, 17, 0] if model.n_speakers > 1 else None
    refs = [_speech(n, 22050, 120 + k, snr_db=30) for k, n in enumerate([30000, 12000, 45000])]
    with _conv_math("fp32"):
        stages = []
        res = evaluate_intelligibility(model, seqs, refs, speaker_ids=spk,
                                       stage_timer=lambda name: stages.append(name) or contextlib.nullcontext())
        wavs, _ = synthesized_audio(model, seqs, spk, "griffin_lim", 16, torch.device("cuda"))
    by_hand = stoi_dtw(_cuda(refs), list(wavs))
    assert stages == ["synthesis", "mel", "stoi", "stoi", "dtw", "stoi"]
    for key in by_hand:
        assert res[key].tobytes() == by_hand[key].tobytes(), key
    ok = ~np.isnan(res["stoi"])
    if ok.any():
        assert res["mean_stoi"] == pytest.approx(float(np.mean(res["stoi"][ok])), abs=1e-15)


# ---- resample_batch without sr_to --------------------------------------------------------------------------------------
def test_resample_batch_without_sr_to_makes_the_same_launch(monkeypatch):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    real = lib.call

    def record(name, *args):
        calls.append((name, list(args[6:11])))              # nclips, bank, up, down, ntaps
        return real(name, *args)
    monkeypatch.setattr(lib, "call", record)
    x = torch.from_numpy(np.random.RandomState(0).uniform(-1, 1, (2, 9600)).astype(np.float32)).cuda()
    a, la = audio.resample_batch(x, [9600, 5000], 48000)
    b, lb = audio.resample_batch(x, [9600, 5000], 48000, sr_to=audio.hparams.sample_rate)
    assert [c[0] for c in calls] == ["dv3_resample_poly_batched"] * 2
    assert [v for v in calls[0][1] if isinstance(v, int)] == [2, 147, 320, 46]
    assert [v for v in calls[0][1] if isinstance(v, int)] == [v for v in calls[1][1] if isinstance(v, int)]
    assert la == lb and torch.equal(a, b)
    c, lc = audio.resample_batch(x, [9600, 5000], 48000, sr_to=10000)
    assert calls[2][1][2:4] == [5, 24] and lc == [2000, 1042]
    want = resample_poly(x[1, :5000].cpu().numpy().astype(np.float64), 5, 24).astype(np.float32)
    assert np.abs(c[1, :lc[1]].cpu().numpy() - want).max() <= 1e-6
