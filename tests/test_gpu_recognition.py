"""GPU: the CTC loss and gradient kernels (csrc/ctc.cu) against the fp64 oracle (tests/ctc_oracle.py) and torch's fp64
CPU ``F.ctc_loss``, greedy decoding and edit distances exactly against the oracle, the independence of every row
from its batch, the token recognizer against an fp64 autograd restatement, its training step (deterministic mode,
graph vs eager, checkpoint resume), learning on a synthetic corpus, and evaluate_recognition end to end.

Bounds of the CTC kernels.  The logits are fp32 and every later operation runs in fp64, so before the final rounding
the kernels and the oracle agree to a few hundred fp64 ulps of the largest intermediate: log-space values reach
about T log V < 1e4, so about 1e4 * 2^-52 * 100 < 3e-10 absolute in nll, and the occupancies exp(alpha + beta -
log p) carry that as a relative error.  The outputs are then rounded once to fp32: nll and the loss within 2^-24
relative of their fp64 values, each dz within 2^-24 |dz| + w_b * 1e-9 (w_b = 1 / (B max(L_b, 1))).  The tests allow
twice the rounding, plus that fp64 term."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ctc_oracle as CO
from speaker_encoder_oracle import _wn
from test_gpu_synthesis import PRESETS, _model, _sequences

U = 2.0 ** -24


@pytest.fixture
def math_mode():
    from deepvoice3_pytorch_b200 import ops
    old = ops.conv_math, ops.deterministic

    def set_(m, det=None):
        ops.conv_math = m
        if det is not None:
            ops.deterministic = det
    yield set_
    ops.conv_math, ops.deterministic = old


def _rows(V, seed):
    """(frames, targets) rows that cover repeats, L = 0, T = L + repeats (feasible) and one frame less (infeasible)."""
    rng = np.random.RandomState(seed)
    rows = [(37, rng.randint(1, V, 12)), (5, np.array([], np.int64)), (1, np.array([], np.int64)),
            (1, np.array([3])), (6, np.array([2, 2, 2, 4])), (5, np.array([2, 2, 2, 4])), (9, np.array([1, 1, 1, 1, 1])),
            (8, np.array([5, 5, 3, 3])), (60, rng.randint(1, V, 25)), (200, rng.randint(1, 4, 70)),
            (64, rng.randint(1, V, 64))]
    return rows


def _pack(rows, T, L):
    B = len(rows)
    tg = np.zeros((B, L), np.int64)
    for b, (_, t) in enumerate(rows):
        tg[b, :t.size] = t
    return (np.array([r[0] for r in rows], np.int32), tg, np.array([r[1].size for r in rows], np.int32))


def _ctc_abi(z, frames, targets, tlen, scale=None):
    """nll, partials, infeasible and dz of one fwd + bwd through the C ABI (d_loss = 1, scale default 1 / B)."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.ops import _p, _stream
    B, V, T = z.shape
    L = targets.shape[1]
    dev = z.device
    fr = torch.from_numpy(frames).to(dev)
    tg = torch.from_numpy(targets.astype(np.int32)).to(dev)
    tl = torch.from_numpy(tlen).to(dev)
    ws = torch.empty(int(lib.raw("dv3_ctc_ws_bytes")(B, T, L)), dtype=torch.uint8, device=dev)
    nll, part = torch.empty(B, device=dev), torch.empty(B, device=dev)
    inf = torch.empty(B, dtype=torch.int32, device=dev)
    lib.call("dv3_ctc_fwd", _p(z), z.stride(0), z.stride(1), _p(fr), _p(tg), L, _p(tl), B, V, T, L, _p(ws), _p(nll),
             _p(part), _p(inf), _p(ops._err_flag(dev)), _stream())
    one = torch.ones(1, device=dev)
    dz = torch.full((B, V, T), float("nan"), device=dev)
    lib.call("dv3_ctc_bwd", _p(z), z.stride(0), z.stride(1), _p(fr), _p(tg), L, _p(tl), B, V, T, L, _p(ws), _p(one),
             1.0 / B if scale is None else scale, _p(dz), _stream())
    torch.cuda.synchronize()
    ops.check_index_errors()
    return nll.cpu().numpy(), part.cpu().numpy(), inf.cpu().numpy(), dz.cpu().numpy()


# ---- CTC loss and gradient ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("V", [6, 149, 1024])
def test_ctc_against_torch_fp64_and_the_oracle(V):
    rows = _rows(V, V)
    T, L = 200, 70
    frames, tg, tl = _pack(rows, T, L)
    B = len(rows)
    z = torch.randn(B, V, T, generator=torch.Generator().manual_seed(V)) * 3
    nll, part, inf, dz = _ctc_abi(z.cuda(), frames, tg, tl)
    # torch fp64 on the CPU
    z64 = z.double().requires_grad_(True)
    lp = F.log_softmax(z64, 1).permute(2, 0, 1)
    want = F.ctc_loss(lp, torch.from_numpy(tg), torch.from_numpy(frames).long(), torch.from_numpy(tl).long(),
                      blank=0, reduction="none", zero_infinity=False)
    finite = torch.isfinite(want).numpy()
    assert np.array_equal(inf == 1, ~finite)
    assert (nll[~finite] == 0).all() and (part[~finite] == 0).all() and (dz[~finite] == 0).all()
    w = want.detach().numpy()
    assert np.all(np.abs(nll[finite] - w[finite]) <= 2 * U * np.abs(w[finite]) + 3e-10)
    lp = F.log_softmax(z64, 1).permute(2, 0, 1)
    F.ctc_loss(lp, torch.from_numpy(tg), torch.from_numpy(frames).long(), torch.from_numpy(tl).long(), blank=0,
               reduction="mean", zero_infinity=True).backward()
    g = z64.grad.numpy()
    wb = 1.0 / (B * np.maximum(tl, 1))[:, None, None]
    assert np.all(np.abs(dz - g) <= 2 * U * np.abs(g) + 1e-9 * wb), np.abs(dz - g).max()
    # the fp64 oracle agrees with torch
    onll, _, odz, oinf = CO.ctc_batch(z.numpy(), frames, tg, tl)
    assert np.array_equal(oinf, ~finite)
    np.testing.assert_allclose(onll[finite], w[finite], rtol=1e-10)
    np.testing.assert_allclose(odz, g, rtol=1e-9, atol=1e-13)


@pytest.mark.gpu
def test_ctc_loss_autograd_is_the_mean_of_the_partials(math_mode):
    from deepvoice3_pytorch_b200 import recognition as R
    V, T, L = 40, 120, 30
    rows = _rows(V, 3)[:8]
    frames, tg, tl = _pack(rows, T, L)
    z = (torch.randn(len(rows), V, T, generator=torch.Generator().manual_seed(5)) * 2).cuda().requires_grad_(True)
    loss, inf = R.ctc_loss(z, frames, tg, tl)
    loss.backward()
    nll, part, inf2, dz = _ctc_abi(z.detach(), frames, tg, tl)
    assert np.array_equal(inf.cpu().numpy(), inf2)
    assert abs(float(loss.detach()) - part.astype(np.float64).mean()) <= 4 * U * np.abs(part).mean()
    assert np.array_equal(z.grad.cpu().numpy(), dz)


# ---- greedy decoding and edit distance ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_greedy_decoding_equals_the_oracle_with_planted_ties():
    from deepvoice3_pytorch_b200.recognition import greedy_decode
    rng = np.random.RandomState(0)
    B, V, T = 9, 37, 300
    z = rng.randint(-3, 3, (B, V, T)).astype(np.float32)      # integer logits: many exact ties
    z[1, :, :] = 0.0                                           # every frame a tie: all blanks
    z[2, 5, :] = 9.0
    z[2, 7, ::2] = 9.0                                         # 5 and 7 tie on even frames: 5 wins, one run of 5
    frames = np.array([300, 300, 300, 1, 17, 299, 64, 33, 250], np.int32)
    got = greedy_decode(torch.from_numpy(z).cuda(), frames)
    want = CO.greedy(z, frames)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert got[1].size == 0 and got[2].tolist() == [5]


@pytest.mark.gpu
def test_edit_distances_equal_the_oracle():
    from deepvoice3_pytorch_b200.recognition import edit_distance
    rng = np.random.RandomState(1)
    hyps, refs = [], []
    for n, m in [(0, 0), (0, 5), (7, 0), (1, 1), (1, 4), (5, 1), (33, 31), (64, 65), (1024, 1000), (1024, 1), (1, 1024),
                 (200, 8000), (1024, 8000), (30, 30)]:
        ref = rng.randint(1, 6, n)
        hyp = ref[rng.rand(n) < 0.8] if m == n else rng.randint(1, 6, m)
        hyps.append(hyp)
        refs.append(ref)
    hyps.append(np.array([1, 2, 3]))
    refs.append(np.array([1, 2, 3]))
    got = edit_distance(hyps, refs)
    small = [k for k, (h, r) in enumerate(zip(hyps, refs)) if h.size * r.size <= 300000]
    for k in small:
        assert tuple(got[k]) == CO.edit(hyps[k], refs[k]), k
    for k in range(len(hyps)):                  # the big ones: the distance by a vectorised DP, S+D+I = distance
        assert got[k, 1:].sum() == got[k, 0] and got[k, 2] - got[k, 3] == refs[k].size - hyps[k].size
    assert tuple(got[0]) == (0, 0, 0, 0) and tuple(got[1]) == (5, 0, 0, 5) and tuple(got[2]) == (7, 0, 7, 0)
    assert tuple(got[-1]) == (0, 0, 0, 0)
    big = [k for k in range(len(hyps)) if k not in small]
    for k in big:
        assert got[k, 0] == _levenshtein(hyps[k], refs[k]), k


def _levenshtein(h, r):
    prev = np.arange(h.size + 1)
    for i in range(1, r.size + 1):
        cur = np.empty_like(prev)
        cur[0] = i
        sub = prev[:-1] + (h != r[i - 1])
        dele = prev[1:] + 1
        best = np.minimum(sub, dele)
        for j in range(1, h.size + 1):
            cur[j] = min(best[j - 1], cur[j - 1] + 1)
        prev = cur
    return int(prev[-1])


@pytest.mark.gpu
def test_edit_distance_tie_rule_on_the_gpu():
    from deepvoice3_pytorch_b200.recognition import edit_distance
    cases = [([1, 2], [2, 1]), ([1], [2, 3]), ([2, 3], [1]), ([1, 1, 2], [1, 2, 2]), ([], [4]), ([5, 6, 7], [6])]
    got = edit_distance([np.array(h) for h, _ in cases], [np.array(r) for _, r in cases])
    for k, (h, r) in enumerate(cases):
        assert tuple(got[k]) == CO.edit(h, r)


# ---- batch independence and determinism -----------------------------------------------------------------------------
@pytest.mark.gpu
def test_rows_alone_shuffled_padded_strided_and_rerun():
    V, T, L = 53, 150, 40
    rows = [r for r in _rows(V, 11) if r[0] <= T and r[1].size <= L]
    frames, tg, tl = _pack(rows, T, L)
    B = len(rows)
    z = torch.randn(B, V, T, generator=torch.Generator().manual_seed(2)).cuda() * 2
    base = _ctc_abi(z, frames, tg, tl)
    again = _ctc_abi(z, frames, tg, tl)
    assert all(np.array_equal(x, y) for x, y in zip(base, again))
    perm = np.random.RandomState(0).permutation(B)
    sh = _ctc_abi(z[perm].contiguous(), frames[perm], tg[perm], tl[perm])
    assert all(np.array_equal(x[perm], y) for x, y in zip(base, sh))
    big = torch.randn(B, V + 7, T + 50).cuda() * 2
    big[:, :V, :T] = z
    view = big[:, :V, :T]                                      # strided: stride_v = T + 50, stride_b = (V + 7)(T + 50)
    tg2 = np.full((B, L + 9), 5, np.int64)                      # padded target slots hold ids, never read
    tg2[:, :L] = tg
    st = _ctc_abi(view, frames, tg2, tl)
    assert all(np.array_equal(x, y) for x, y in zip(base, st))
    for b in range(B):                                        # alone, at the batch's scale 1 / B
        one = _ctc_abi(z[b:b + 1].contiguous(), frames[b:b + 1], tg[b:b + 1], tl[b:b + 1], scale=1.0 / B)
        assert all(np.array_equal(x[0], y[b]) for x, y in zip(one, base)), b


# ---- the recognizer -------------------------------------------------------------------------------------------------
def _recognizer(V=30, C=128, seed=0, **kw):
    from deepvoice3_pytorch_b200.recognition import TokenRecognizer
    torch.manual_seed(seed)
    return TokenRecognizer(V, channels=C, **kw).cuda()


def _forward64(sd, mels, dilations, kernel_size=5):
    x = mels.transpose(1, 2)
    for i in (0, 2):
        x = torch.relu(F.conv1d(x, _wn(sd, "spectral.%d." % i), sd["spectral.%d.bias" % i]))
    for i, d in enumerate(dilations):
        pre = "temporal.%d.conv." % i
        y = F.conv1d(x, _wn(sd, pre), sd[pre + "bias"], padding=(kernel_size - 1) // 2 * d, dilation=d)
        a, gate = y.split(y.shape[1] // 2, dim=1)
        x = (a * torch.sigmoid(gate) + x) * math.sqrt(0.5)
    return F.conv1d(x, _wn(sd, "out.0."), sd["out.0.bias"])


def _close(got, want, rtol, atol, scale=None):
    got = got.detach().double().cpu()
    want = want.detach().double()
    s = float(want.abs().max()) if scale is None else scale
    err = float((got - want).abs().max())
    assert err <= atol * max(s, 1.0) + rtol * s, (err, s)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtol,atol", [("fp32", 1e-4, 1e-5), ("tc", 2e-3, 2e-3)])
def test_recognizer_forward_and_gradients_against_fp64(math_mode, mode, rtol, atol):
    math_mode(mode)
    dil = (1, 2, 4)
    rec = _recognizer(V=30, dilations=dil, seed=1)
    gen = torch.Generator().manual_seed(2)
    B, T = 4, 96
    mels = torch.rand(B, T, 80, generator=gen)
    ml = np.array([96, 80, 50, 96], np.int32)
    toks = np.array([[3, 4, 1, 5, 6, 0], [7, 7, 8, 0, 0, 0], [9, 1, 0, 0, 0, 0], [2, 3, 4, 5, 6, 7]])
    tl = np.array([5, 3, 2, 6])
    logits, loss = rec(mels.cuda(), ml, toks, tl)
    d_ext = torch.randn(logits.shape, generator=gen) * 1e-3
    (loss + (logits * d_ext.cuda()).sum()).backward()
    sd = {k: t.detach().cpu().double().requires_grad_(True) for k, t in rec.state_dict().items()}
    z64 = _forward64(sd, mels.double(), dil)
    stripped, n = rec.strip_batch(toks, tl)
    lp = F.log_softmax(z64, 1).permute(2, 0, 1)
    l64 = F.ctc_loss(lp, torch.from_numpy(stripped).long(), torch.from_numpy(ml).long(), torch.from_numpy(n).long(),
                     reduction="mean", zero_infinity=True)
    (l64 + (z64 * d_ext.double()).sum()).backward()
    _close(logits, z64, rtol, atol)
    _close(loss, l64, rtol, atol)
    scale = max(float(t.grad.abs().max()) for t in sd.values())
    for name, prm in rec.named_parameters():
        _close(prm.grad, sd[name].grad, rtol, atol, scale)


@pytest.mark.gpu
def test_recognized_rows_do_not_depend_on_the_batch(math_mode):
    math_mode("fp32")
    rec = _recognizer(V=12, seed=3)
    rng = np.random.RandomState(4)
    utts = [rng.rand(n, 80).astype(np.float32) for n in (40, 7, 120, 1, 65)]
    got = rec.recognize(utts)
    from deepvoice3_pytorch_b200 import ops
    for j, u in enumerate(utts):
        assert np.array_equal(rec.recognize([u])[0], got[j]), j
    # the logits themselves: bit-identical in fp32, within the tensor-core tolerance in tc
    T = 120
    batch = torch.zeros(len(utts), T, 80).cuda()
    for j, u in enumerate(utts):
        batch[j, :u.shape[0]] = torch.from_numpy(u).cuda()
    lens = torch.tensor([u.shape[0] for u in utts]).cuda()
    for mode in ("fp32", "tc"):
        math_mode(mode)
        rec.eval()
        with torch.no_grad():
            with ops.length_scope(lens, T):
                zb = rec.logits(batch)
            for j, u in enumerate(utts):
                z1 = rec.logits(torch.from_numpy(u)[None].cuda())
                if mode == "fp32":
                    assert torch.equal(z1[0], zb[j, :, :u.shape[0]]), j
                else:
                    _close(z1[0], zb[j, :, :u.shape[0]].cpu(), 2e-3, 2e-3)
        rec.train()


# ---- training step --------------------------------------------------------------------------------------------------
def _batches(n, B=8, T=64, L=12, V=30, seed=0):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        tl = torch.randint(0, L + 1, (B,), generator=gen)
        toks = torch.randint(1, V, (B, L), generator=gen)
        out.append({"mels": torch.rand(B, T, 80, generator=gen), "mel_lengths": torch.randint(T // 2, T + 1, (B,),
                                                                                               generator=gen),
                    "tokens": toks, "token_lengths": tl})
    return out


def _run(steps_of, batches, use_graph, seed=1):
    from deepvoice3_pytorch_b200.recognition import TokenRecognizerStep
    st = TokenRecognizerStep(_recognizer(V=30, seed=seed, dilations=(1, 2)), use_graph=use_graph)
    losses = [st.step(b).clone() for b in batches[:steps_of]]
    torch.cuda.synchronize()
    return st, torch.stack(losses).cpu(), st.arena.flat.clone().cpu(), st.arena.grad.clone().cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
def test_deterministic_mode_is_bit_reproducible(math_mode, use_graph):
    math_mode("tc", "1")
    bs = _batches(4)
    _, la, pa, ga = _run(4, bs, use_graph)
    _, lb, pb, gb = _run(4, bs, use_graph)
    assert torch.equal(la, lb) and torch.equal(pa, pb) and torch.equal(ga, gb)


@pytest.mark.gpu
def test_graph_and_eager_steps_agree_and_checkpoints_resume_bit_exactly(math_mode):
    from deepvoice3_pytorch_b200.recognition import TokenRecognizerStep
    math_mode("tc", "1")
    bs = _batches(6)
    _, le, pe, _ = _run(4, bs, False)
    st_g, lg, pg, _ = _run(4, bs, True)
    assert st_g.launches_per_step is not None and st_g.launches_per_step > 10
    np.testing.assert_allclose(lg.numpy(), le.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pg.numpy(), pe.numpy(), rtol=1e-4, atol=1e-6)
    st, _, _, _ = _run(3, bs, True)
    ckpt = st.state_dict()
    tail = [st.step(b).clone() for b in bs[3:]]
    straight = st.arena.flat.clone().cpu()
    res = TokenRecognizerStep(_recognizer(V=30, seed=9, dilations=(1, 2)), use_graph=True)
    res.load_state_dict(ckpt)
    l2 = [res.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(tail, l2))
    assert torch.equal(res.arena.flat.cpu(), straight) and res.global_step == 6


@pytest.mark.gpu
def test_step_refuses_another_conv_math(math_mode):
    from deepvoice3_pytorch_b200.recognition import TokenRecognizerStep
    math_mode("tc")
    st = TokenRecognizerStep(_recognizer(V=30), use_graph=False)
    math_mode("tc1")
    with pytest.raises(ValueError):
        st.step(_batches(1)[0])


# ---- learning -------------------------------------------------------------------------------------------------------
def _corpus(n, V, rng, templates):
    """Utterances of 6-14 tokens in [2, V) (no EOS); each token its mel template for 2-5 frames, plus noise."""
    out = []
    for _ in range(n):
        toks = rng.randint(2, V, rng.randint(6, 15))
        frames = [templates[t] + 0.1 * rng.randn(rng.randint(2, 6), 80) for t in toks]
        out.append((np.r_[toks, 1], np.concatenate(frames).astype(np.float32)))     # EOS appended, then stripped
    return out


@pytest.mark.gpu
def test_token_error_rate_on_held_out_utterances_after_training(math_mode):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.recognition import TokenRecognizerStep, token_error_rates
    math_mode("tc")
    V = 24
    rng = np.random.RandomState(0)
    templates = rng.rand(V, 80).astype(np.float32)
    train, held = _corpus(400, V, rng, templates), _corpus(40, V, rng, templates)
    rec = _recognizer(V=V, seed=5, dilations=(1, 2, 4))
    st = TokenRecognizerStep(rec, lr=2e-3, use_graph=True)
    B, T, L = 16, 80, 16
    losses = []
    for _ in range(300):
        idx = rng.choice(len(train), B, replace=False)
        mels = np.zeros((B, T, 80), np.float32)
        toks = np.zeros((B, L), np.int64)
        ml, tl = np.zeros(B, np.int64), np.zeros(B, np.int64)
        for b, i in enumerate(idx):
            t, m = train[i]
            n = min(m.shape[0], T)
            mels[b, :n] = m[:n]
            ml[b] = n
            toks[b, :t.size] = t
            tl[b] = t.size
        losses.append(st.step({"mels": torch.from_numpy(mels), "mel_lengths": torch.from_numpy(ml),
                               "tokens": torch.from_numpy(toks), "token_lengths": torch.from_numpy(tl)}).clone())
    losses = torch.stack(losses).cpu().numpy()
    ops.check_index_errors()
    res = token_error_rates(rec, [m for _, m in held], [t for t, _ in held])
    print("recognizer: loss %.4f -> %.4f, held-out corpus TER %.4f" % (float(losses[0]), float(losses[-10:].mean()),
                                                                       res["corpus_ter"]))
    # measured on an H100 ("tc"): loss 6.72 -> 0.028, held-out corpus TER 0.055 (DESIGN 2.21)
    assert float(losses[-10:].mean()) < 0.5 * float(losses[0])
    assert res["corpus_ter"] <= 0.2


# ---- evaluate_recognition -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("preset", PRESETS)
def test_evaluate_recognition_end_to_end(math_mode, preset):
    import contextlib
    from deepvoice3_pytorch_b200.recognition import edit_distance, evaluate_recognition
    from deepvoice3_pytorch_b200.synthesis import synthesized_mels
    math_mode("fp32")
    model = _model(preset, max_steps=40, done_bias=-20.0)
    seqs = _sequences([37, 5, 61])
    spk = [3, 17, 0] if model.n_speakers > 1 else None
    rec = _recognizer(V=149, seed=2)                    # _sequences draws ids in [2, 149)
    stages = []
    res = evaluate_recognition(model, rec, seqs, speaker_ids=spk, word_sep=2,
                               stage_timer=lambda name: stages.append(name) or contextlib.nullcontext())
    assert stages == ["synthesis", "mel", "recognition"]
    n = len(seqs)
    for k in ("distance", "substitutions", "deletions", "insertions", "ref_lengths", "ter", "wer"):
        assert res[k].shape == (n,), k
    assert np.array_equal(res["substitutions"] + res["deletions"] + res["insertions"], res["distance"])
    assert np.array_equal(res["ter"], res["distance"] / res["ref_lengths"])
    assert res["corpus_ter"] == res["distance"].sum() / res["ref_lengths"].sum()
    mels = synthesized_mels(model, seqs, spk, "griffin_lim", 16, torch.device("cuda"))
    hyps = rec.recognize(mels)
    assert all(np.array_equal(a, b) for a, b in zip(hyps, res["hypotheses"]))
    assert np.array_equal(edit_distance(hyps, res["references"])[:, 0], res["distance"])
