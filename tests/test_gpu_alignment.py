"""GPU: monotonic alignment search and the attention statistics of csrc/align.cu (alignment.py) against the fp64 oracle
(tests/alignment_oracle.py), and evaluate_attention / teacher_forced_alignment on the three presets.

fp32 bounds used below (u = 2^-24):
* logf is accurate to 1 ulp <= 2u |lp|, and each Q(t, j) = fl(lp + max) adds one rounding <= u |Q(t, j)|; max is exact.
  Errors only add along a path, so the fp32 score of any path is within E = u N (2 max|lp| + max|Q|) of its fp64 score,
  and the fp32 Q of every cell within E of its fp64 value (max is 1-Lipschitz).  Hence the GPU path's fp64 score is
  within 2E of the optimum, and where the oracle's two predecessors differ by more than 2E at every cell of its path,
  the GPU takes the same decisions there: the paths are equal.
* coverage: a sum of N fp32 values in order is within gamma_{N-1} sum |A| of the exact sum, gamma_k = k u / (1 - k u).
* argmax and max are comparisons of the same fp32 values: exact."""
import contextlib

import numpy as np
import pytest
import torch

import alignment_oracle as AO
from test_gpu_synthesis import PRESETS, _conv_math, _model, _sequences

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _mas(A_list, steps=None):
    """Pad fp32 numpy alignments (N_b, L_b) into one (B, N, L) CUDA batch -> monotonic_alignment's dict."""
    from deepvoice3_pytorch_b200.alignment import monotonic_alignment
    N = max(a.shape[0] for a in A_list)
    L = max(a.shape[1] for a in A_list)
    pad = np.zeros((len(A_list), N, L), np.float32)
    for b, a in enumerate(A_list):
        pad[b, :a.shape[0], :a.shape[1]] = a
    steps = [a.shape[0] for a in A_list] if steps is None else steps
    return monotonic_alignment(torch.from_numpy(pad).cuda(), steps, [a.shape[1] for a in A_list])


def _softmax(x):
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)


def _fp32_sum(A):
    """Coverage summed in fp32 in increasing t, as the kernel does."""
    c = np.zeros(A.shape[1], np.float32)
    for row in A:
        c = c + row
    return c


def test_planted_paths_are_found_exactly():
    rng = np.random.RandomState(0)
    shapes = [(1, 1), (60, 1), (7, 7), (300, 40), (1200, 1024), (4100, 120), (4000, 1024), (33, 32), (64, 33)]
    A, want = zip(*[AO.planted(N, L, rng) for N, L in shapes])
    res = _mas(list(A))
    for b, (N, L) in enumerate(shapes):
        assert np.array_equal(res["durations"][b, :L], want[b]), (N, L)
        assert (res["durations"][b, L:] == 0).all()
        assert np.isfinite(res["score"][b])


def test_random_softmax_rows_score_within_the_fp32_bound_of_the_optimum():
    rng = np.random.RandomState(1)
    A_list = []
    for k in range(24):
        if k % 2:        # diffuse attention
            N, L = rng.randint(20, 160), rng.randint(2, 50)
            A_list.append(_softmax(rng.randn(max(N, L), L) * 2.0))
        else:            # a sharp, roughly diagonal attention with noise: large margins
            N, L = rng.randint(20, 80), rng.randint(2, 20)
            c = np.linspace(0, L - 1, N)[:, None] + rng.randn(N, 1) * 0.3
            A_list.append(_softmax(-(np.arange(L)[None] - c) ** 2 * 6.0 + rng.randn(N, L) * 1.5))
    res = _mas(A_list)
    equal_checked = 0
    for b, A in enumerate(A_list):
        N, L = A.shape
        lp = AO.log_probs(A)
        d_or, s_or, p_or = AO.mas_logp(lp)
        d = res["durations"][b, :L]
        assert (d >= 1).all() and d.sum() == N
        path = np.repeat(np.arange(L), d)
        s_gpu = AO.path_score(lp, path)
        Q = np.full((N, L), -np.inf)             # oracle Q for the margins
        Q[0, 0] = lp[0, 0]
        for t in range(1, N):
            for j in range(L):
                if j <= t and L - 1 - j <= N - 1 - t:
                    Q[t, j] = lp[t, j] + max(Q[t - 1, j], Q[t - 1, j - 1] if j else -np.inf)
        E = U * N * (2 * np.abs(lp).max() + np.abs(Q[np.isfinite(Q)]).max())
        assert s_or - s_gpu <= 2 * E and s_gpu <= s_or + 1e-9 * abs(s_or), (b, s_or, s_gpu, E)
        assert abs(res["score"][b] - s_gpu) <= E
        margins = [abs(Q[t - 1, j] - Q[t - 1, j - 1]) for t, j in enumerate(p_or) if 0 < j < t]
        if min(margins, default=np.inf) > 2 * E:
            assert np.array_equal(path, p_or), b
            equal_checked += 1
    assert equal_checked >= 6


def test_statistics_exact_and_coverage_within_its_bound():
    rng = np.random.RandomState(2)
    A_list = [_softmax(rng.randn(N, L) * 3.0) for N, L in ((500, 250), (150, 40), (1001, 97), (9, 9))]
    A_list[1][3, 7] = A_list[1][3, 9] = A_list[1][3].max() + 0.25        # a planted tie: the lower token wins
    res = _mas(A_list)
    for b, A in enumerate(A_list):
        p, m, _ = AO.statistics(A)
        assert np.array_equal(res["argmax"][b], p)
        assert np.array_equal(res["max"][b].view(np.int32), m.astype(np.float32).view(np.int32))
        c64 = A.astype(np.float64).sum(0)
        k = A.shape[0] - 1
        gamma = k * U / (1 - k * U)
        assert (np.abs(res["coverage"][b] - c64) <= gamma * np.abs(A).astype(np.float64).sum(0)).all()
        assert np.array_equal(res["coverage"][b], _fp32_sum(A))
    assert res["argmax"][1][3] == 7


def test_degenerate_rows():
    rng = np.random.RandomState(3)
    A = _softmax(rng.randn(80, 20))
    A[10:14] = np.nan
    A[30, 5] = np.nan
    A[:, 17] = np.nan
    short = _softmax(rng.randn(5, 12))
    res = _mas([A, short])
    d = res["durations"][0, :20]
    assert (d >= 1).all() and d.sum() == 80
    assert (res["durations"][1] == 0).all() and res["score"][1] == -np.inf
    assert res["argmax"][1].shape == (5,) and res["coverage"][1].shape == (12,)
    assert not np.isfinite(res["coverage"][0]).all()
    p, m, _ = AO.statistics(A)
    assert np.array_equal(res["argmax"][0], p) and np.array_equal(res["max"][0], m)


def _bits(res, b, L):
    return (res["durations"][b, :L].tobytes(), res["score"][b].tobytes(), res["argmax"][b].tobytes(),
            res["max"][b].tobytes(), res["coverage"][b].tobytes())


def test_bits_do_not_depend_on_the_batch_or_the_run():
    from deepvoice3_pytorch_b200.alignment import monotonic_alignment
    rng = np.random.RandomState(4)
    A_list = [_softmax(rng.randn(rng.randint(40, 400), L) * 2) for L in (3, 31, 32, 33, 250, 64, 100, 1)]
    batch = _mas(A_list)
    again = _mas(A_list)
    alone = [_mas([a]) for a in A_list]
    perm = rng.permutation(len(A_list))
    shuffled = _mas([A_list[i] for i in perm])
    for b, A in enumerate(A_list):
        L = A.shape[1]
        want = _bits(batch, b, L)
        assert _bits(again, b, L) == want and _bits(alone[b], 0, L) == want
        assert _bits(shuffled, int(np.flatnonzero(perm == b)[0]), L) == want
    # a strided layer view and a padded view read in place give the bits of a contiguous copy
    layers = torch.rand(3, 4, 120, 50, device="cuda")
    steps, tokens = [120, 77, 50, 119], [50, 13, 50, 2]
    view = monotonic_alignment(layers[1], steps, tokens)
    copy = monotonic_alignment(layers[1].clone(), steps, tokens)
    wide = torch.zeros(4, 130, 64, device="cuda")
    wide[:, :120, :50] = layers[1]
    padded = monotonic_alignment(wide[:, :120, :50], steps, tokens)
    for b in range(4):
        assert _bits(view, b, 50) == _bits(copy, b, 50) == _bits(padded, b, 50)


def test_direction_buffer_chunks_give_the_same_bits(monkeypatch):
    from deepvoice3_pytorch_b200 import mcd
    rng = np.random.RandomState(5)
    A_list = [_softmax(rng.randn(rng.randint(50, 300), rng.randint(2, 90)) * 2) for _ in range(9)]
    one = _mas(A_list)
    monkeypatch.setattr(mcd, "DIR_BUDGET_BYTES", 2000)           # several launches, each reusing the buffer
    many = _mas(A_list)
    for b, A in enumerate(A_list):
        assert _bits(one, b, A.shape[1]) == _bits(many, b, A.shape[1])


def test_discrimination_on_synthetic_alignments():
    from deepvoice3_pytorch_b200.alignment import attention_errors
    rng = np.random.RandomState(6)
    L = 30
    clean, _ = AO.planted(120, L, rng, durations=np.full(L, 4))
    bad_path = list(range(0, 11)) + list(range(13, 21)) + list(range(15, L))      # skips 11, 12; goes back 20 -> 15
    bad = (rng.random_sample((len(bad_path) * 3, L)) * 0.002).astype(np.float32)    # skipped: coverage < 0.5
    bad[np.arange(bad.shape[0]), np.repeat(bad_path, 3)] = 0.9
    stuck = (rng.random_sample((200, L)) * 0.05).astype(np.float32)
    stuck[np.arange(200), np.minimum(np.arange(200) // 3, 6)] = 0.9
    res = _mas([clean, bad, stuck])
    e = attention_errors(res["argmax"], res["max"], res["coverage"], [120, bad.shape[0], 200], 199)
    assert (e["skips"][0], e["repeats"][0], e["unreached"][0], e["stop_failed"][0]) == (0, 0, 0, False)
    assert e["max_dwell"][0] == 4 and e["focus_rate"][0] == pytest.approx(0.9)
    assert (e["skips"][1], e["repeats"][1], e["unreached"][1]) == (2, 1, 0)
    assert e["max_dwell"][2] >= 150 and e["unreached"][2] == L - 7 and e["stop_failed"][2]


# ---- the presets -------------------------------------------------------------------------------------------------------
def _replay_parent_tts_batch(model, seqs, speaker_ids, batch_size):
    """tts_batch as the parent commit composed it: encoder, decode_ragged, alignment to host, post-net and vocoder."""
    from deepvoice3_pytorch_b200 import incremental, ops, synthesis
    stage = lambda name: contextlib.nullcontext()
    order = sorted(range(len(seqs)), key=lambda i: -seqs[i].size)
    out = [None] * len(seqs)
    for c in range(0, len(order), batch_size):
        idx = order[c:c + batch_size]
        ss = [seqs[i] for i in idx]
        dev = next(model.parameters()).device
        lens = [s.size for s in ss]
        Lm = max(lens)
        text, tpos = np.zeros((len(ss), Lm), np.int64), np.zeros((len(ss), Lm), np.int64)
        for b, s in enumerate(ss):
            text[b, :s.size], tpos[b, :s.size] = s, np.arange(1, s.size + 1)
        text, tpos = torch.from_numpy(text).to(dev), torch.from_numpy(tpos).to(dev)
        text_len = torch.tensor(lens, dtype=torch.int64).to(dev)
        with torch.no_grad():
            ops.rng.begin_forward(False, dev)
            try:
                ids = None if speaker_ids is None else [speaker_ids[i] for i in idx]
                spk = None if ids is None else model._speaker_embedding(torch.tensor(ids).to(dev))
                with ops.length_scope(text_len, Lm):
                    keys, values = model.seq2seq.encoder(text, speaker_embed=spk)
                outputs, aligns, _, states, steps = incremental.decode_ragged(model.seq2seq.decoder, (keys, values),
                                                                              tpos, text_len, spk)
                aligns = aligns.cpu().numpy()
            finally:
                ops.rng.end_forward()
            post = synthesis._postnet_vocode(model, outputs, states, steps, spk, stage)
        for b, (w, lin, mel) in enumerate(post):
            out[idx[b]] = (w, aligns[b, :steps[b], :lens[b]], lin, mel)
    return out


@pytest.mark.parametrize("preset", PRESETS)
def test_presets_evaluate_attention_tts_batch_and_teacher_forcing(preset, monkeypatch):
    from deepvoice3_pytorch_b200 import data, synthesis
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.alignment import evaluate_attention, monotonic_alignment, teacher_forced_alignment
    from deepvoice3_pytorch_b200.train_step import to_device
    from test_gpu_models import preset_kwargs
    model = _model(preset, max_steps=60)
    lengths = [37, 5, 61, 20, 48, 12]
    seqs = _sequences(lengths, seed=11)
    spk = [3, 17, 0, 54, 101, 7] if model.n_speakers > 1 else None
    with _conv_math("fp32"):
        calls = []
        real = lib.call
        monkeypatch.setattr(lib, "call", lambda name, *a: (calls.append(name), real(name, *a))[1])
        got = synthesis.tts_batch(model, seqs, speaker_ids=spk, batch_size=4)
        new_calls, calls[:] = list(calls), []
        want = _replay_parent_tts_batch(model, [np.asarray(s, np.int64) for s in seqs], spk, 4)
        assert new_calls == calls and len(calls) > 0
        monkeypatch.setattr(lib, "call", real)
        for g, w in zip(got, want):
            for a, b in zip(g, w):
                assert a.shape == b.shape and np.array_equal(a, b)
        ev = evaluate_attention(model, seqs, speaker_ids=spk, batch_size=4)
    aligns = [g[1] for g in got]
    assert ev["steps"].tolist() == [a.shape[0] for a in aligns]
    direct = _mas(aligns)
    for k, A in enumerate(aligns):
        p, m, _ = AO.statistics(A)
        want = AO.attention_errors(p, m, _fp32_sum(A), model.seq2seq.decoder.max_decoder_steps)
        for key, v in want.items():
            assert ev[key][k] == pytest.approx(v), (k, key)
        if A.shape[0] >= A.shape[1]:
            assert np.array_equal(ev["durations"][k], direct["durations"][k, :A.shape[1]])
            assert ev["durations"][k].sum() == A.shape[0]
    assert ev["total_skips"] == ev["skips"].sum() and ev["stop_failures"] == ev["stop_failed"].sum()

    # teacher forcing on a collated batch
    _, kw = preset_kwargs(preset)
    r, ds = kw["r"], kw["downsample_step"]
    rng = np.random.RandomState(12)
    items = []
    for k, s in enumerate(seqs[:4]):
        n = int(rng.randint(120, 400))
        item = (s, rng.rand(n, model.mel_dim).astype(np.float32), rng.rand(n, model.linear_dim).astype(np.float32))
        items.append(item + ((spk[k],) if spk else ()))
    batch = to_device(data.collate(items, r=r, downsample_step=ds), "cuda")
    with _conv_math("fp32"):
        tf = teacher_forced_alignment(model, batch)
        tf0 = teacher_forced_alignment(model, batch, layer=0)
    assert tf["frames_per_step"] == r * ds
    for res in (tf, tf0):
        for b, s in enumerate(seqs[:4]):
            if res["steps"][b] >= s.size:
                assert res["durations"][b, :s.size].min() >= 1 and res["durations"][b].sum() == res["steps"][b]
    assert tf["steps"].tolist() == [(r + len(it[1]) - 1) // (r * ds) + 1 for it in items]
    with pytest.raises(ValueError):
        monotonic_alignment(torch.zeros(1, 4, 4, device="cuda"), [5], [4])
