"""GPU: the speaker verifier -- its embed and score kernels (csrc/spk_ver.cu) elementwise against the fp64 restatement
(tests/speaker_verifier_oracle.py), the whole verifier against the fp64 oracle's autograd, the independence of every
trial from its batch, the training step (deterministic mode, graph vs eager, checkpoint resume), an EER on unseen
synthetic speakers after training, the cloned-voice evaluation end to end, and the speaker encoder's unchanged launch
sequence."""
import json
import os

import numpy as np
import pytest
import torch

import speaker_verifier_oracle as VO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "speaker_encoder_calls.json")


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


def _verifier(seed=0, **kw):
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier
    torch.manual_seed(seed)
    v = SpeakerVerifier(**kw).cuda()
    with torch.no_grad():                       # S and b start at 0: give the score terms something to check
        v.S.copy_(0.05 * torch.randn(v.embed_dim, v.embed_dim))
        v.b.fill_(0.1)
    return v


def _close(got, want, rtol, atol_rel, scale=None):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    scale = float(want.abs().max()) if scale is None else scale
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=rtol, atol=atol_rel * max(1e-30, scale))


# ---- kernels --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,N,C,D,counts", [(4, 5, 128, 128, [5, 1, 3, 2]), (3, 1, 256, 64, [1, 1, 1]),
                                            (2, 32, 96, 7, [32, 17])])
def test_embed_forward_backward_against_fp64(B, N, C, D, counts):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200 import speaker_verifier as SV
    gen = torch.Generator().manual_seed(B * 100 + N)
    h = torch.randn(B, N, C, generator=gen)
    w, c = torch.randn(D, C, generator=gen) / C ** 0.5, torch.randn(D, generator=gen) * 0.1
    d_out = torch.randn(B, D, generator=gen)
    cnt = torch.tensor(counts, dtype=torch.int32, device="cuda")
    out, hbar = SV.embed_forward(h.cuda(), cnt, w.cuda(), c.cuda())
    d_h = torch.full((B, N, C), float("nan"), device="cuda")
    part = SV.embed_backward(d_out.cuda(), hbar, cnt, w.cuda(), d_h, N)
    g = SV.reduce_rows(part)
    ops.check_index_errors()
    o64, hb64 = VO.embed_fwd(h.double(), counts, w.double(), c.double())
    dh64, dw64, dc64 = VO.embed_bwd(d_out.double(), hb64, counts, w.double(), N)
    _close(out, o64, 1e-5, 1e-6)
    _close(hbar, hb64, 1e-6, 1e-6)
    _close(d_h, dh64, 1e-5, 1e-6)
    for b, n in enumerate(counts):
        assert torch.all(d_h[b, n:] == 0)
    _close(g[:D * C].view(D, C), dw64, 1e-5, 1e-6)
    _close(g[D * C:], dc64, 1e-5, 1e-6)


@pytest.mark.gpu
def test_embed_count_outside_range_sets_the_error_flag():
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200 import speaker_verifier as SV
    ops.check_index_errors()
    w, c = torch.ones(4, 8, device="cuda"), torch.ones(4, device="cuda")
    out, _ = SV.embed_forward(torch.ones(2, 3, 8, device="cuda"), torch.tensor([3, 4], dtype=torch.int32,
                                                                                device="cuda"), w, c)
    with pytest.raises(IndexError):
        ops.check_index_errors()
    assert torch.equal(out.cpu(), torch.tensor([[9.0] * 4, [0.0] * 4]))
    d_h = torch.full((2, 3, 8), float("nan"), device="cuda")
    part = SV.embed_backward(torch.ones(2, 4, device="cuda"), torch.ones(2, 8, device="cuda"),
                             torch.tensor([0, 2], dtype=torch.int32, device="cuda"), w, d_h, 3)
    with pytest.raises(IndexError):
        ops.check_index_errors()
    assert torch.all(d_h[0] == 0) and torch.all(part[0] == 0) and torch.all(d_h[1, :2] == 2.0)     # W^T 1 / 2 = 4 / 2


@pytest.mark.gpu
@pytest.mark.parametrize("B_e,B_t,D,with_ids", [(16, 16, 128, True), (5, 70, 64, True), (40, 3, 16, False),
                                                (33, 65, 128, True)])
def test_score_forward_backward_against_fp64(B_e, B_t, D, with_ids):
    from deepvoice3_pytorch_b200 import speaker_verifier as SV
    gen = torch.Generator().manual_seed(B_e * 1000 + B_t)
    x, y = torch.randn(B_e, D, generator=gen) * 0.3, torch.randn(B_t, D, generator=gen) * 0.3
    S, b = torch.randn(D, D, generator=gen) * 0.05, torch.tensor([0.2])
    ids_e = torch.randint(0, 6, (B_e,), generator=gen)
    ids_t = torch.randint(0, 6, (B_t,), generator=gen)
    ids_e[0], ids_t[0], ids_t[-1] = 1, 1, 7                # both kinds of pair
    d_scores = torch.randn(B_e, B_t, generator=gen)
    ie, it = (ids_e.cuda(), ids_t.cuda()) if with_ids else (None, None)
    scores, lp = SV.score_forward(x.cuda(), y.cuda(), S.cuda(), b.cuda(), ie, it)
    one = torch.ones((), device="cuda")
    dx, dy, part = SV.score_backward(x.cuda(), y.cuda(), S.cuda(), scores, ie, it, d_scores.cuda(),
                                     one if with_ids else None)
    g = SV.reduce_rows(part)
    L64, loss64 = VO.score_fwd(x.double(), y.double(), S.double(), b.double(), *((ids_e, ids_t) if with_ids else ()))
    dx64, dy64, dS64, db64 = VO.score_bwd(x.double(), y.double(), S.double(), L64, *((ids_e, ids_t) if with_ids else
                                                                                    (None, None)),
                                          d_scores.double(), torch.tensor(1.0, dtype=torch.float64))
    _close(scores, L64, 1e-5, 1e-6)
    if with_ids:
        _close(SV.reduce_loss(lp), loss64, 1e-5, 1e-6)
    else:
        assert lp is None
    _close(dx, dx64, 1e-4, 1e-5)
    _close(dy, dy64, 1e-4, 1e-5)
    _close(g[:D * D].view(D, D), dS64, 1e-4, 1e-5)
    _close(g[D * D:], db64, 1e-4, 1e-5)


# ---- whole verifier -------------------------------------------------------------------------------------------------
def _train_batch(B=4, N=5, T=64, seed=2):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(B, N, T, 80, generator=gen), torch.tensor([3, 0, 3, 9][:B] + list(range(10, 10 + B - 4)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtol,atol", [("fp32", 1e-4, 1e-5), ("tc", 2e-3, 2e-3), ("tc1", 2e-2, 2e-2)])
def test_verifier_forward_and_gradients_against_fp64(math_mode, mode, rtol, atol):
    math_mode(mode)
    v = _verifier(seed=1)
    mels, ids = _train_batch()
    scores, loss = v(mels.cuda(), ids.cuda())
    loss.backward()
    sd = {k: t.detach().cpu().double().requires_grad_(True) for k, t in v.state_dict().items()}
    s64, l64 = VO.verifier_forward(sd, mels.double(), ids)
    l64.backward()
    _close(scores, s64, rtol, atol)
    _close(loss, l64, rtol, atol)
    scale = max(float(t.grad.abs().max()) for t in sd.values())
    for name, prm in v.named_parameters():
        _close(prm.grad, sd[name].grad, rtol, atol, scale)


def _ragged(seed, counts=(3, 1, 5)):
    rng = np.random.RandomState(seed)
    return [[rng.rand(rng.randint(20, 90), 80).astype(np.float32) for _ in range(n)] for n in counts]


@pytest.mark.gpu
def test_trials_do_not_depend_on_the_batch(math_mode):
    """fp32: an enrollment row, a test row and a score are bit-identical alone and inside a larger ragged batch, also
    when the frames past each length are garbage rather than zeros."""
    from deepvoice3_pytorch_b200 import speaker_verifier as SV
    math_mode("fp32")
    v = _verifier(seed=3)
    enroll, tests = _ragged(0), [u for spk in _ragged(1, (2, 3)) for u in spk]
    E, Y = v.embed_enrollment(enroll), v.embed_tests(tests)
    scores = v.score(E, Y)
    assert E.shape == (3, 128) and Y.shape == (5, 128) and scores.shape == (3, 5) and v.training
    for k, spk in enumerate(enroll):
        e1 = v.embed_enrollment([spk])
        assert torch.equal(e1[0], E[k]), k
        for j, u in enumerate(tests):
            y1 = v.embed_tests([u])
            assert torch.equal(y1[0], Y[j]) and torch.equal(v.score(e1, y1)[0, 0], scores[k, j]), (k, j)
    # garbage past each length and in the padded slots
    N, T = 5, 90
    mels = torch.rand(3, N, T, 80).cuda()
    lengths = torch.ones(3 * N, dtype=torch.int32)
    for k, spk in enumerate(enroll):
        for j, u in enumerate(spk):
            mels[k, j, :u.shape[0]] = torch.from_numpy(u).cuda()
            lengths[k * N + j] = u.shape[0]
    with torch.no_grad():
        v.eval()
        h = v.pooled(mels, lengths.cuda())
        v.train()
        got, _ = SV.embed_forward(h, torch.tensor([3, 1, 5], dtype=torch.int32, device="cuda"), v.w, v.c)
    assert torch.equal(got, E)


@pytest.mark.gpu
def test_embeddings_within_the_tensor_core_tolerance(math_mode):
    math_mode("tc")
    v = _verifier(seed=3)
    enroll = _ragged(4)
    E = v.embed_enrollment(enroll)
    for k, spk in enumerate(enroll):
        _close(v.embed_enrollment([spk])[0], E[k], 2e-3, 2e-3)


# ---- training step --------------------------------------------------------------------------------------------------
def _batches(n, B=8, N=5, T=64, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return [{"mels": torch.rand(B, N, T, 80, generator=gen), "speaker_ids": torch.randperm(20, generator=gen)[:B]}
            for _ in range(n)]


def _run(steps_of, batches, use_graph, seed=1):
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifierStep
    st = SpeakerVerifierStep(_verifier(seed=seed), use_graph=use_graph)
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
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifierStep
    math_mode("tc", "1")
    bs = _batches(6)
    _, le, pe, _ = _run(4, bs, False)
    st_g, lg, pg, _ = _run(4, bs, True)
    assert st_g.launches_per_step is not None and st_g.launches_per_step > 10
    np.testing.assert_allclose(lg.numpy(), le.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pg.numpy(), pe.numpy(), rtol=1e-4, atol=1e-6)
    st, _, _, _ = _run(3, bs, True)
    ckpt = st.state_dict()
    kept = {k: t.clone() for k, t in ckpt["verifier"].items()}
    tail = [st.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(ckpt["verifier"][k], t) for k, t in kept.items())
    straight = st.arena.flat.clone().cpu()
    res = SpeakerVerifierStep(_verifier(seed=9), use_graph=True)
    res.load_state_dict(ckpt)
    l2 = [res.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(tail, l2))
    assert torch.equal(res.arena.flat.cpu(), straight) and res.global_step == 6


@pytest.mark.gpu
def test_step_refuses_another_conv_math(math_mode):
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifierStep
    math_mode("tc")
    st = SpeakerVerifierStep(_verifier(), use_graph=False)
    math_mode("tc1")
    with pytest.raises(ValueError):
        st.step(_batches(1)[0])


# ---- EER on unseen synthetic speakers -------------------------------------------------------------------------------
def _synthetic_corpus(n_spk, n_utt=10, T=96, seed=0):
    """Per-speaker spectral envelopes of three Gaussian bumps, per-frame gains and noise, clipped to [0, 1]."""
    rng = np.random.RandomState(seed)
    f = np.arange(80)
    corpus = []
    for _ in range(n_spk):
        centers, widths = rng.uniform(0, 80, 3), rng.uniform(4, 16, 3)
        env = sum(np.exp(-0.5 * ((f - c) / w) ** 2) for c, w in zip(centers, widths))
        env = 0.2 + 0.6 * env / env.max()
        utts = []
        for _ in range(n_utt):
            gain = rng.uniform(0.6, 1.2, (T, 1))
            utts.append(np.clip(env[None, :] * gain + 0.05 * rng.randn(T, 80), 0, 1).astype(np.float32))
        corpus.append(utts)
    return corpus


@pytest.mark.gpu
def test_eer_on_unseen_speakers_after_training(math_mode):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifierStep, equal_error_rate
    math_mode("tc")
    corpus = _synthetic_corpus(40)
    train, unseen = corpus[:32], corpus[32:]
    v = _verifier(seed=6)
    st = SpeakerVerifierStep(v, lr=1e-3, use_graph=True)
    rng = np.random.RandomState(7)
    B, N, T = 16, 5, 64
    losses = []
    for _ in range(400):
        spk = rng.choice(len(train), B, replace=False)
        mels = np.empty((B, N, T, 80), np.float32)
        for b, s in enumerate(spk):
            for j, u in enumerate(rng.choice(10, N, replace=False)):
                o = rng.randint(0, 96 - T + 1)
                mels[b, j] = train[s][u][o:o + T]
        losses.append(st.step({"mels": torch.from_numpy(mels), "speaker_ids": torch.from_numpy(spk)}).clone())
    losses = torch.stack(losses).cpu().numpy()
    ops.check_index_errors()
    enroll = v.embed_enrollment([spk[:4] for spk in unseen])
    tests = v.embed_tests([u for spk in unseen for u in spk[4:7]])
    scores = v.score(enroll, tests).cpu().numpy()
    labels = np.arange(8)[:, None] == np.repeat(np.arange(8), 3)[None, :]
    eer, thr = equal_error_rate(scores, labels)
    print("verifier: loss %.4f -> %.4f, EER on 8 unseen speakers (24 tests x 8 enrollments) %.4f at %.3f"
          % (float(losses[0]), float(losses[-10:].mean()), eer, thr))
    # measured on an H100 ("tc"): loss 9.40 -> 0.0000 / 0.0040 in two runs, EER 0.0 both times (DESIGN 2.14)
    assert float(losses[-10:].mean()) < 0.5 * float(losses[0])
    assert eer <= 0.1


# ---- cloned voices end to end ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_verify_cloned_voices_end_to_end(math_mode):
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder, clone_voices
    from deepvoice3_pytorch_b200.speaker_verifier import verify_cloned_voices
    math_mode("tc")
    torch.manual_seed(0)
    model = builder.deepvoice3_multispeaker(
        n_vocab=149, embed_dim=64, mel_dim=80, linear_dim=513, r=1, downsample_step=4, kernel_size=3,
        encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256, n_speakers=4,
        speaker_embed_dim=16, use_memory_mask=True, key_projection=True, value_projection=True,
        speaker_embedding_weight_std=0.3).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = 8
    torch.manual_seed(1)
    enc = SpeakerEncoder().cuda()
    real = _ragged(2, (3, 2))
    ids = clone_voices(model, enc, real)
    v = _verifier(seed=4)
    texts = [np.array([5, 9, 13, 22]), np.array([3, 8, 11]), np.array([7, 7, 2, 30, 4])]
    res = verify_cloned_voices(model, v, [ids[0], ids[1], ids[0]], {ids[0]: real[0], ids[1]: real[1]}, texts)
    assert res["scores"].shape == (2, 3) and np.isfinite(res["scores"]).all()
    assert res["speakers"] == ids
    assert res["labels"].tolist() == [[True, False, True], [False, True, False]]
    assert 0.0 <= res["eer"] <= 1.0


# ---- the speaker encoder launches what it launched before -----------------------------------------------------------
def record_encoder_calls():
    """The lib.call sequence (name and non-pointer arguments) of SpeakerEncoder.forward, embed_batch and one eager and
    one graph SpeakerEncoderStep, "tc", at fixed shapes."""
    import ctypes
    from deepvoice3_pytorch_b200 import builder, ops
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder, SpeakerEncoderStep
    calls, real = [], lib.call

    def rec(name, *a):
        calls.append([name] + [x if isinstance(x, (int, float)) else None for x in a
                               if not isinstance(x, ctypes.c_void_p) and x is not None])
        return real(name, *a)
    old = ops.conv_math
    ops.conv_math = "tc"
    lib.call = rec
    try:
        torch.manual_seed(0)
        enc = SpeakerEncoder().cuda()
        model = builder.deepvoice3_multispeaker(
            n_vocab=149, embed_dim=64, mel_dim=80, linear_dim=513, r=1, downsample_step=4, kernel_size=3,
            encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256, n_speakers=4,
            speaker_embed_dim=16).cuda()
        gen = torch.Generator().manual_seed(0)
        out = {}
        calls.clear()
        with torch.no_grad():
            enc(torch.rand(2, 3, 64, 80, generator=gen).cuda())
        out["forward"] = list(calls)
        calls.clear()
        enc.embed_batch(_ragged(0))
        out["embed_batch"] = list(calls)
        batch = {"mels": torch.rand(4, 3, 64, 80, generator=gen), "speaker_ids": torch.arange(4)}
        for use_graph in (False, True):
            st = SpeakerEncoderStep(enc, model, use_graph=use_graph)
            st.step(batch)
            calls.clear()
            st.step(batch)          # graph mode replays: no calls; the capture happened in the first step
            out["step_graph" if use_graph else "step_eager"] = list(calls)
        calls.clear()
        st = SpeakerEncoderStep(enc, model, use_graph=True)
        st.step(batch)
        out["graph_capture"] = list(calls)
        torch.cuda.synchronize()
        return out
    finally:
        lib.call = real
        ops.conv_math = old


@pytest.mark.gpu
def test_speaker_encoder_launch_sequence_is_unchanged():
    with open(GOLDEN) as f:
        want = json.load(f)
    assert json.loads(json.dumps(record_encoder_calls())) == want
