"""GPU: the speaker classifier -- its logits and gradient kernels (csrc/spk_cls.cu) elementwise against the fp64
restatement (tests/speaker_classifier_oracle.py), the whole classifier against the fp64 oracle's autograd, the
independence of every classified row from its batch, the training step (deterministic mode, graph vs eager, checkpoint
resume), the top-1 accuracy on held-out utterances after training, the cloned-voice evaluation end to end, and the
unchanged launches of verify_cloned_voices."""
import json
import os

import numpy as np
import pytest
import torch

import speaker_classifier_oracle as CO
from test_gpu_speaker_verifier import _ragged, _synthetic_corpus

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "verify_cloned_voices_calls.json")


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


def _classifier(K=10, seed=0, **kw):
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifier
    torch.manual_seed(seed)
    cl = SpeakerClassifier(K, **kw).cuda()
    with torch.no_grad():                       # c starts at 0: give the bias something to check
        cl.c.copy_(0.1 * torch.randn(K))
    return cl


def _close(got, want, rtol, atol_rel, scale=None):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    scale = float(want.abs().max()) if scale is None else scale
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=rtol, atol=atol_rel * max(1e-30, scale))


def _first_max(z):
    """Host ranking: the first class of largest logit of every row."""
    z = z.detach().double().cpu().numpy()
    return np.argmax(z, axis=1)                 # numpy returns the first occurrence of the maximum


# ---- kernels --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("R,C,K,with_labels,with_ext,pad", [(128, 128, 108, True, False, 0), (37, 96, 2, True, True, 7),
                                                             (70, 256, 2484, True, True, 0),
                                                             (33, 5, 65, False, True, 3), (1, 128, 3, True, False, 0),
                                                             (64, 128, 32, True, True, 0)])
def test_head_forward_backward_against_fp64(R, C, K, with_labels, with_ext, pad):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200 import speaker_classifier as SC
    gen = torch.Generator().manual_seed(R * 10000 + K)
    H = torch.randn(R, C + pad, generator=gen)
    w, c = torch.randn(K, C, generator=gen) / C ** 0.5, torch.randn(K, generator=gen) * 0.1
    labels = torch.randint(0, K, (R,), generator=gen)
    d_ext = torch.randn(R, K, generator=gen)
    h = H.cuda()[:, :C]                         # pad > 0: rows pad floats apart past C
    lab = labels.cuda() if with_labels else None
    logits, lse, pred, lp = SC.logits_forward(h, w.cuda(), c.cuda(), lab)
    one = torch.ones((), device="cuda")
    d_h, d_w, d_c = SC.logits_backward(h, w.cuda(), logits, lse, lab, d_ext.cuda() if with_ext else None,
                                       one if with_labels else None, 1.0 / R)
    ops.check_index_errors()
    h64 = H[:, :C].double()
    z64, lse64, loss64 = CO.head_fwd(h64, w.double(), c.double(), labels if with_labels else None)
    dh64, dw64, dc64 = CO.head_bwd(h64, w.double(), z64, lse64, labels if with_labels else None,
                                   d_ext.double() if with_ext else None,
                                   torch.tensor(1.0, dtype=torch.float64) if with_labels else None)
    _close(logits, z64, 1e-5, 1e-6)
    _close(lse, lse64, 1e-5, 1e-6)
    assert pred.dtype == torch.int32 and np.array_equal(pred.cpu().numpy(), _first_max(logits))
    if with_labels:
        _close(SC.mean_loss(lp), loss64, 1e-5, 1e-6)
    else:
        assert lp is None
    _close(d_h, dh64, 1e-4, 1e-5)
    _close(d_w, dw64, 1e-4, 1e-5)
    _close(d_c, dc64, 1e-4, 1e-5)


@pytest.mark.gpu
def test_prediction_ties_go_to_the_lowest_index():
    from deepvoice3_pytorch_b200 import speaker_classifier as SC
    K, C = 700, 8
    w = torch.zeros(K, C, device="cuda")
    c = torch.zeros(K, device="cuda")
    c[[5, 300, 699]] = 1.0                      # row 0: three tied maxima in different threads' slices
    h = torch.zeros(2, C, device="cuda")
    _, _, pred, _ = SC.logits_forward(h, w, c)
    assert pred.tolist() == [5, 5]
    c.zero_()                                   # all equal: class 0
    assert SC.logits_forward(h, w, c)[2].tolist() == [0, 0]


@pytest.mark.gpu
def test_label_outside_range_sets_the_error_flag():
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200 import speaker_classifier as SC
    ops.check_index_errors()
    gen = torch.Generator().manual_seed(3)
    R, C, K = 5, 16, 7
    h, w, c = torch.randn(R, C, generator=gen), torch.randn(K, C, generator=gen), torch.randn(K, generator=gen)
    labels = torch.tensor([0, K, 3, -1, 6])
    logits, lse, _, lp = SC.logits_forward(h.cuda(), w.cuda(), c.cuda(), labels.cuda())
    with pytest.raises(IndexError):
        ops.check_index_errors()
    assert float(lp[1]) == 0.0 and float(lp[3]) == 0.0
    z64, lse64, loss64 = CO.head_fwd(h.double(), w.double(), c.double(), labels)
    _close(SC.mean_loss(lp), loss64, 1e-5, 1e-6)
    d_h, d_w, d_c = SC.logits_backward(h.cuda(), w.cuda(), logits, lse, labels.cuda(), None,
                                       torch.ones((), device="cuda"), 1.0 / R)
    with pytest.raises(IndexError):
        ops.check_index_errors()
    dh64, dw64, dc64 = CO.head_bwd(h.double(), w.double(), z64, lse64, labels, None,
                                   torch.tensor(1.0, dtype=torch.float64))
    _close(d_h, dh64, 1e-4, 1e-5)
    _close(d_w, dw64, 1e-4, 1e-5)
    _close(d_c, dc64, 1e-4, 1e-5)


# ---- whole classifier -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtol,atol", [("fp32", 1e-4, 1e-5), ("tc", 2e-3, 2e-3), ("tc1", 2e-2, 2e-2)])
def test_classifier_forward_and_gradients_against_fp64(math_mode, mode, rtol, atol):
    math_mode(mode)
    cl = _classifier(K=10, seed=1)
    gen = torch.Generator().manual_seed(2)
    B, N, T = 4, 3, 64
    mels = torch.rand(B, N, T, 80, generator=gen)
    ids = torch.tensor([3, 0, 9, 3])
    d_ext = torch.randn(B * N, 10, generator=gen) * 0.1
    logits, loss = cl(mels.cuda(), ids.cuda())
    (loss + (logits * d_ext.cuda()).sum()).backward()
    sd = {k: t.detach().cpu().double().requires_grad_(True) for k, t in cl.state_dict().items()}
    z64, l64 = CO.classifier_forward(sd, mels.double(), ids)
    (l64 + (z64 * d_ext.double()).sum()).backward()
    _close(logits, z64, rtol, atol)
    _close(loss, l64, rtol, atol)
    scale = max(float(t.grad.abs().max()) for t in sd.values())
    for name, prm in cl.named_parameters():
        _close(prm.grad, sd[name].grad, rtol, atol, scale)


@pytest.mark.gpu
def test_classified_rows_do_not_depend_on_the_batch(math_mode):
    """fp32: a row's logits and prediction are bit-identical alone and inside a larger ragged batch, also when the
    frames past each length are garbage rather than zeros."""
    from deepvoice3_pytorch_b200 import speaker_classifier as SC
    math_mode("fp32")
    cl = _classifier(K=40, seed=3)
    utts = [u for spk in _ragged(1, (2, 3, 1)) for u in spk]
    logits, pred = cl.classify(utts)
    assert logits.shape == (6, 40) and pred.dtype == torch.int64 and cl.training
    assert np.array_equal(pred.cpu().numpy(), _first_max(logits))
    for j, u in enumerate(utts):
        l1, p1 = cl.classify([u])
        assert torch.equal(l1[0], logits[j]) and int(p1[0]) == int(pred[j]), j
    T = 100
    mels = torch.rand(len(utts), 1, T, 80).cuda()
    lengths = torch.tensor([u.shape[0] for u in utts], dtype=torch.int32)
    for j, u in enumerate(utts):
        mels[j, 0, :u.shape[0]] = torch.from_numpy(u).cuda()
    with torch.no_grad():
        cl.eval()
        h = cl.pooled(mels, lengths.cuda())
        cl.train()
        got, _, _, _ = SC.logits_forward(h.view(len(utts), -1), cl.w, cl.c)
    assert torch.equal(got, logits)


@pytest.mark.gpu
def test_classified_rows_within_the_tensor_core_tolerance(math_mode):
    math_mode("tc")
    cl = _classifier(K=40, seed=3)
    utts = [u for spk in _ragged(4, (3, 2)) for u in spk]
    logits, _ = cl.classify(utts)
    for j, u in enumerate(utts):
        _close(cl.classify([u])[0][0], logits[j], 2e-3, 2e-3)


# ---- training step --------------------------------------------------------------------------------------------------
def _batches(n, B=8, N=4, T=64, K=20, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return [{"mels": torch.rand(B, N, T, 80, generator=gen), "speaker_ids": torch.randperm(K, generator=gen)[:B]}
            for _ in range(n)]


def _run(steps_of, batches, use_graph, seed=1):
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifierStep
    st = SpeakerClassifierStep(_classifier(K=20, seed=seed), use_graph=use_graph)
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
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifierStep
    math_mode("tc", "1")
    bs = _batches(6)
    _, le, pe, _ = _run(4, bs, False)
    st_g, lg, pg, _ = _run(4, bs, True)
    assert st_g.launches_per_step is not None and st_g.launches_per_step > 10
    np.testing.assert_allclose(lg.numpy(), le.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pg.numpy(), pe.numpy(), rtol=1e-4, atol=1e-6)
    st, _, _, _ = _run(3, bs, True)
    ckpt = st.state_dict()
    kept = {k: t.clone() for k, t in ckpt["classifier"].items()}
    tail = [st.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(ckpt["classifier"][k], t) for k, t in kept.items())
    straight = st.arena.flat.clone().cpu()
    res = SpeakerClassifierStep(_classifier(K=20, seed=9), use_graph=True)
    res.load_state_dict(ckpt)
    l2 = [res.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(tail, l2))
    assert torch.equal(res.arena.flat.cpu(), straight) and res.global_step == 6


@pytest.mark.gpu
def test_step_refuses_another_conv_math(math_mode):
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifierStep
    math_mode("tc")
    st = SpeakerClassifierStep(_classifier(K=20), use_graph=False)
    math_mode("tc1")
    with pytest.raises(ValueError):
        st.step(_batches(1)[0])


# ---- top-1 accuracy on held-out utterances --------------------------------------------------------------------------
@pytest.mark.gpu
def test_top1_accuracy_on_held_out_utterances_after_training(math_mode):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifierStep, top_k_accuracy
    math_mode("tc")
    n_spk = 24
    corpus = _synthetic_corpus(n_spk)
    cl = _classifier(K=n_spk, seed=6)
    st = SpeakerClassifierStep(cl, lr=1e-3, use_graph=True)
    rng = np.random.RandomState(7)
    B, N, T = 16, 4, 64
    losses = []
    for _ in range(300):
        spk = rng.choice(n_spk, B, replace=False)
        mels = np.empty((B, N, T, 80), np.float32)
        for b, s in enumerate(spk):
            for j, u in enumerate(rng.choice(7, N, replace=False)):           # utterances 0..6 train, 7..9 held out
                o = rng.randint(0, 96 - T + 1)
                mels[b, j] = corpus[s][u][o:o + T]
        losses.append(st.step({"mels": torch.from_numpy(mels), "speaker_ids": torch.from_numpy(spk)}).clone())
    losses = torch.stack(losses).cpu().numpy()
    ops.check_index_errors()
    held = [u for spk in corpus for u in spk[7:]]
    targets = np.repeat(np.arange(n_spk), 3)
    logits, pred = cl.classify(held)
    acc = top_k_accuracy(logits, targets, (1, 5))
    assert acc[1] == float((pred.cpu().numpy() == targets).mean())
    print("classifier: loss %.4f -> %.4f, held-out accuracy (72 utterances of 24 speakers) top-1 %.4f top-5 %.4f"
          % (float(losses[0]), float(losses[-10:].mean()), acc[1], acc[5]))
    # measured on an H100 ("tc"): loss 3.22 -> 0.0003, top-1 and top-5 accuracy 1.0 (DESIGN 2.15)
    assert float(losses[-10:].mean()) < 0.5 * float(losses[0])
    assert acc[1] >= 0.9


# ---- cloned voices end to end ---------------------------------------------------------------------------------------
def _ms_model():
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    model = builder.deepvoice3_multispeaker(
        n_vocab=149, embed_dim=64, mel_dim=80, linear_dim=513, r=1, downsample_step=4, kernel_size=3,
        encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256, n_speakers=4,
        speaker_embed_dim=16, use_memory_mask=True, key_projection=True, value_projection=True,
        speaker_embedding_weight_std=0.3).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = 8
    return model


_TEXTS = [np.array([5, 9, 13, 22]), np.array([3, 8, 11]), np.array([7, 7, 2, 30, 4])]


@pytest.mark.gpu
def test_classify_cloned_voices_end_to_end(math_mode):
    from deepvoice3_pytorch_b200.speaker_classifier import classify_cloned_voices
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder, clone_voices
    math_mode("tc", "1")
    model = _ms_model()
    torch.manual_seed(1)
    ids = clone_voices(model, SpeakerEncoder().cuda(), _ragged(2, (3, 2)))
    assert ids == [4, 5]
    cl = _classifier(K=3, seed=4)
    seen, classify = [], cl.classify

    def spy(mels):
        seen.append([m.clone() for m in mels])
        return classify(mels)
    cl.classify = spy
    res = classify_cloned_voices(model, cl, [ids[0], ids[1], ids[0], 2], _TEXTS + [np.array([4, 6, 8])],
                                 targets=[0, 1, 0, 2])
    del cl.classify
    assert res["logits"].shape == (4, 3) and res["predicted"].shape == (4,) and res["targets"] == [0, 1, 0, 2]
    assert torch.isfinite(res["logits"]).all()
    assert len(seen) == 1 and all(m.shape[1] == 80 for m in seen[0])
    logits, pred = cl.classify(seen[0])
    assert torch.equal(res["logits"], logits) and torch.equal(res["predicted"], pred)
    z = res["logits"].double().cpu().numpy()
    t = np.array([0, 1, 0, 2])
    rank = [int((z[i] > z[i, t[i]]).sum() + (z[i, :t[i]] == z[i, t[i]]).sum()) for i in range(4)]
    assert res["accuracy"] == {1: np.mean([r < 1 for r in rank]), 5: 1.0}
    assert np.array_equal(res["predicted"].cpu().numpy(), _first_max(res["logits"]))


# ---- verify_cloned_voices launches what it launched before ----------------------------------------------------------
def record_verify_calls():
    """The lib.call sequence (name and non-pointer arguments) of one verify_cloned_voices call, "tc" in deterministic
    mode, on a small random-weight multi-speaker model with two cloned voices; and its scores."""
    import ctypes
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder, clone_voices
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier, verify_cloned_voices
    calls, real = [], lib.call

    def rec(name, *a):
        calls.append([name] + [x if isinstance(x, (int, float)) else None for x in a
                               if not isinstance(x, ctypes.c_void_p) and x is not None])
        return real(name, *a)
    old = ops.conv_math, ops.deterministic
    ops.conv_math, ops.deterministic = "tc", "1"
    try:
        model = _ms_model()
        torch.manual_seed(1)
        enc = SpeakerEncoder().cuda()
        utts = _ragged(2, (3, 2))
        ids = clone_voices(model, enc, utts)
        torch.manual_seed(4)
        v = SpeakerVerifier().cuda()
        torch.manual_seed(5)
        lib.call = rec
        res = verify_cloned_voices(model, v, [ids[0], ids[1], ids[0]], {ids[0]: utts[0], ids[1]: utts[1]}, _TEXTS)
        torch.cuda.synchronize()
        return {"calls": calls, "scores": res["scores"].tolist()}
    finally:
        lib.call = real
        ops.conv_math, ops.deterministic = old


@pytest.mark.gpu
def test_verify_cloned_voices_launch_sequence_is_unchanged():
    with open(GOLDEN) as f:
        want = json.load(f)
    got = json.loads(json.dumps(record_verify_calls()))
    assert got["calls"] == want["calls"]
    np.testing.assert_allclose(got["scores"], want["scores"], rtol=1e-5, atol=1e-6)
