"""GPU: the speaker encoder -- its pool and attention kernels (csrc/spk_enc.cu) elementwise against the fp64
restatement (tests/speaker_encoder_oracle.py), the whole encoder against the fp64 oracle's autograd, the training step
(deterministic mode, graph vs eager, checkpoint resume), the batch independence of embed_batch, a recovery run on a
synthetic corpus and voice cloning into a multi-speaker model."""
import numpy as np
import pytest
import torch

import speaker_encoder_oracle as SO

S = 16
KW = dict(n_vocab=149, embed_dim=64, mel_dim=80, linear_dim=513, r=1, downsample_step=4, kernel_size=3,
          encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256, n_speakers=4,
          speaker_embed_dim=S, use_memory_mask=True, key_projection=True, value_projection=True,
          speaker_embedding_weight_std=0.3)


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


def _encoder(seed=0, **kw):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder
    torch.manual_seed(seed)
    return SpeakerEncoder(**kw).cuda()


def _ms_model(seed=0, **over):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(seed)
    return builder.deepvoice3_multispeaker(**dict(KW, **over)).cuda()


def _close(got, want, rtol, atol_rel, scale=None):
    """atol = atol_rel * scale (default: max |want|).  Gradients pass the largest gradient of the call as the scale:
    d b_k is 0 in exact arithmetic (the key softmax does not see a shift of every key) and d W_k cancels heavily."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    scale = float(want.abs().max()) if scale is None else scale
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=rtol, atol=atol_rel * max(1e-30, scale))


# ---- kernels --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_pool_forward_backward_ragged_and_row_independent():
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_encoder import masked_mean
    gen = torch.Generator().manual_seed(0)
    R, C, T = 7, 128, 77
    lengths = torch.tensor([77, 1, 31, 32, 33, 64, 50], dtype=torch.int32)
    x = torch.randn(R, C, T, generator=gen)
    xd = x.cuda().requires_grad_(True)
    y = masked_mean(xd, lengths.cuda())
    dy = torch.randn(R, C, generator=gen)
    y.backward(dy.cuda())
    ops.check_index_errors()
    _close(y, SO.pool_fwd(x.double(), lengths), 1e-6, 1e-6)
    assert torch.equal(xd.grad.cpu(), (SO.pool_bwd(dy.double(), lengths, T)).float())
    # a row's bits depend on neither R, T nor the other rows
    alone = masked_mean(x[2:3, :, :31].contiguous().cuda(), lengths[2:3].cuda())
    assert torch.equal(alone, y[2:3].detach())


@pytest.mark.gpu
def test_pool_length_outside_range_sets_the_error_flag():
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_encoder import masked_mean
    ops.check_index_errors()
    y = masked_mean(torch.ones(2, 4, 8, device="cuda"), torch.tensor([8, 9], dtype=torch.int32, device="cuda"))
    with pytest.raises(IndexError):
        ops.check_index_errors()
    assert torch.equal(y.cpu(), torch.tensor([[1.0] * 4, [0.0] * 4]))


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,C,heads,counts", [(3, 5, 128, 2, [5, 2, 1]), (2, 1, 128, 2, [1, 1]),
                                                (2, 32, 256, 4, [32, 17]), (4, 8, 64, 8, [8, 3, 8, 6])])
def test_attention_forward_backward_against_fp64(B, N, C, heads, counts):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_encoder import _ATTN_PARAMS, _AttentionFn
    gen = torch.Generator().manual_seed(B * 1000 + N)
    p = {"w_q": torch.randn(C, C, generator=gen) / C ** 0.5, "w_k": torch.randn(C, C, generator=gen) / C ** 0.5,
         "w_v": torch.randn(C, C, generator=gen) / C ** 0.5, "b_q": torch.randn(C, generator=gen) * 0.1,
         "b_k": torch.randn(C, generator=gen) * 0.1, "b_v": torch.randn(C, generator=gen) * 0.1,
         "w_s": torch.randn(C, generator=gen), "b_s": torch.randn(1, generator=gen) * 0.1,
         "w_e": torch.randn(S, C, generator=gen) / C ** 0.5, "b_e": torch.randn(S, generator=gen) * 0.1}
    h = torch.randn(B, N, C, generator=gen)
    target = torch.randn(B, S, generator=gen) * 0.3
    d_ext = torch.randn(B, S, generator=gen)
    hd = h.cuda().requires_grad_(True)
    pd = {k: v.cuda().requires_grad_(True) for k, v in p.items()}
    out, loss = _AttentionFn.apply(hd, torch.tensor(counts, dtype=torch.int32, device="cuda"), target.cuda(), heads,
                                   *[pd[k] for k in _ATTN_PARAMS])
    (loss + (out * d_ext.cuda()).sum()).backward()
    ops.check_index_errors()
    p64 = {k: v.double() for k, v in p.items()}
    o64, l64, saved = SO.attn_fwd(h.double(), counts, p64, heads, target.double())
    d_h, g = SO.attn_bwd(h.double(), counts, p64, heads, saved, target.double(), d_ext.double(),
                         torch.tensor(1.0, dtype=torch.float64))
    _close(out, o64, 1e-4, 1e-5)
    _close(loss, l64, 1e-5, 1e-6)
    _close(hd.grad, d_h, 1e-3, 1e-5)
    for b, n in enumerate(counts):
        assert torch.all(hd.grad[b, n:] == 0)
    scale = max(float(v.abs().max()) for v in g.values())
    for k in p:
        _close(pd[k].grad, g[k], 1e-3, 1e-5, scale)


# ---- whole encoder --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtol,atol", [("fp32", 1e-4, 1e-5), ("tc", 2e-3, 2e-3), ("tc1", 2e-2, 2e-2)])
def test_encoder_forward_and_gradients_against_fp64(math_mode, mode, rtol, atol):
    math_mode(mode)
    enc = _encoder(seed=1)
    gen = torch.Generator().manual_seed(2)
    mels = torch.rand(4, 8, 64, 80, generator=gen)
    target = torch.randn(4, S, generator=gen) * 0.3
    out = enc(mels.cuda())
    loss = enc.loss(mels.cuda(), target.cuda())
    loss.backward()
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in enc.state_dict().items()}
    o64, _ = SO.encoder_forward(sd, mels.double(), 2, 5, 2)
    _, l64 = SO.encoder_forward(sd, mels.double(), 2, 5, 2, target=target.double())
    l64.backward()
    _close(out, o64, rtol, atol)
    _close(loss, l64, rtol, atol)
    scale = max(float(v.grad.abs().max()) for v in sd.values())
    for name, prm in enc.named_parameters():
        _close(prm.grad, sd[name].grad, rtol, atol, scale)


def _batches(n, B=4, N=8, T=64, n_spk=4, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return [{"mels": torch.rand(B, N, T, 80, generator=gen), "speaker_ids": torch.randperm(n_spk, generator=gen)[:B]}
            for _ in range(n)]


def _run(steps_of, batches, use_graph, seed=1):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep
    enc = _encoder(seed=seed)
    st = SpeakerEncoderStep(enc, _ms_model(), use_graph=use_graph)
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
    math_mode("tc", "1")
    bs = _batches(6)
    st_e, le, pe, _ = _run(4, bs, False)
    st_g, lg, pg, _ = _run(4, bs, True)
    assert st_g.launches_per_step is not None and st_g.launches_per_step > 10
    np.testing.assert_allclose(lg.numpy(), le.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pg.numpy(), pe.numpy(), rtol=1e-4, atol=1e-6)
    # resume: 3 steps, checkpoint, 3 more == 6 straight
    st, _, _, _ = _run(3, bs, True)
    ckpt = st.state_dict()
    kept = {k: v.clone() for k, v in ckpt["encoder"].items()}
    tail = [st.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(ckpt["encoder"][k], v) for k, v in kept.items())     # a copy, not the live arena
    straight = st.arena.flat.clone().cpu()
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep
    res = SpeakerEncoderStep(_encoder(seed=9), _ms_model(), use_graph=True)
    res.load_state_dict(ckpt)
    l2 = [res.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(tail, l2))
    assert torch.equal(res.arena.flat.cpu(), straight) and res.global_step == 6


@pytest.mark.gpu
def test_step_refuses_another_conv_math(math_mode):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep
    math_mode("tc")
    st = SpeakerEncoderStep(_encoder(), _ms_model(), use_graph=False)
    math_mode("tc1")
    with pytest.raises(ValueError):
        st.step(_batches(1)[0])


@pytest.mark.gpu
def test_graph_step_follows_a_speaker_table_that_moved(math_mode):
    """clone_voices installs a new table (add_speakers): the next graph step captures anew and reads the new rows."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep, clone_voices
    math_mode("tc")
    bs = _batches(2)
    model, enc = _ms_model(), _encoder(seed=2)
    st = SpeakerEncoderStep(enc, model, use_graph=True)
    st.step(bs[0])
    clone_voices(model, enc, _ragged_samples(2)[:1])
    with torch.no_grad():
        model.embed_speakers.weight.mul_(2.0)
        table = model.embed_speakers.weight.detach().clone()
        want = enc.loss(bs[1]["mels"].cuda(), table[bs[1]["speaker_ids"].cuda()])
    got = st.step(bs[1])
    ops.check_index_errors()
    assert st.graphs_captured == 2
    torch.testing.assert_close(got, want, rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_forward_with_lengths_sees_each_sample_alone(math_mode):
    math_mode("fp32")
    enc = _encoder(seed=5)
    gen = torch.Generator().manual_seed(3)
    mels = torch.rand(2, 3, 64, 80, generator=gen).cuda()       # frames past each length are garbage, not zeros
    lengths = torch.tensor([64, 40, 17, 33, 1, 64], dtype=torch.int32, device="cuda")
    counts = torch.tensor([3, 2], dtype=torch.int32, device="cuda")
    with torch.no_grad():
        rows = enc(mels, lengths, counts)
        for b in range(2):
            n = int(counts[b])
            T = int(lengths[3 * b:3 * b + n].max())
            alone = torch.zeros(1, n, T, 80, device="cuda")
            for j in range(n):
                L = int(lengths[3 * b + j])
                alone[0, j, :L] = mels[b, j, :L]
            want = enc(alone, lengths[3 * b:3 * b + n].contiguous())
            assert torch.equal(rows[b], want[0]), b
    with pytest.raises(ValueError):
        enc(mels, lengths, counts)


# ---- embed_batch ------------------------------------------------------------------------------------------------------
def _ragged_samples(seed):
    rng = np.random.RandomState(seed)
    counts, out = [3, 1, 5], []
    for n in counts:
        out.append([rng.rand(rng.randint(20, 90), 80).astype(np.float32) for _ in range(n)])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_embed_batch_rows_do_not_depend_on_the_batch(math_mode, mode):
    math_mode(mode)
    enc = _encoder(seed=3)
    samples = _ragged_samples(0)
    rows = enc.embed_batch(samples)
    assert rows.shape == (3, S) and enc.training
    for k, spk in enumerate(samples):
        alone = enc.embed_batch([spk])
        if mode == "fp32":
            assert torch.equal(alone[0], rows[k]), k
        else:
            _close(alone[0], rows[k], 2e-3, 2e-3)


# ---- recovery on a synthetic corpus ---------------------------------------------------------------------------------
def _synthetic_corpus(n_spk=8, n_utt=10, T=96, seed=0):
    """Per-speaker spectral envelopes, per-frame gains and noise, clipped to [0, 1] (the normalised mel range)."""
    rng = np.random.RandomState(seed)
    f = np.arange(80)
    corpus = []
    for s in range(n_spk):
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
def test_recovery_on_a_synthetic_corpus(math_mode):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep
    math_mode("tc")
    corpus = _synthetic_corpus()
    torch.manual_seed(5)
    table = torch.randn(108, S) * 0.3          # a deepvoice3_vctk-sized table (108 speakers x 16)
    model = _ms_model(n_speakers=108)
    with torch.no_grad():
        model.embed_speakers.weight.copy_(table.cuda())
    enc = _encoder(seed=6)
    st = SpeakerEncoderStep(enc, model, lr=1e-3, use_graph=True)
    rng = np.random.RandomState(7)
    B, N, T = 8, 4, 64
    losses = []
    for step in range(400):
        mels = np.empty((B, N, T, 80), np.float32)
        for s in range(B):
            for j, u in enumerate(rng.choice(8, N, replace=False)):     # utterances 8, 9 held out
                o = rng.randint(0, 96 - T + 1)
                mels[s, j] = corpus[s][u][o:o + T]
        losses.append(st.step({"mels": torch.from_numpy(mels), "speaker_ids": torch.arange(B)}).clone())
    losses = torch.stack(losses).cpu().numpy()
    ops.check_index_errors()
    first, last = float(losses[0]), float(losses[-10:].mean())
    held = enc.embed_batch([[corpus[s][8], corpus[s][9]] for s in range(8)]).cpu()
    dist = torch.cdist(held, table[:8])
    # measured on an H100: L1 0.381 -> 0.0125, held-out distances to the own row 0.05-0.10, all nearest (DESIGN 2.13)
    print("recovery: L1 %.4f -> %.4f, held-out distance to own row %s, nearest %s"
          % (first, last, dist.diagonal().numpy().round(3), dist.argmin(1).tolist()))
    assert last < 0.25 * first
    assert dist.argmin(1).tolist() == list(range(8))


# ---- cloning ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_clone_voices_appends_rows_that_synthesis_and_adaptation_accept(math_mode):
    from deepvoice3_pytorch_b200 import data, ops, synthesis
    from deepvoice3_pytorch_b200.speaker_encoder import clone_voices
    from deepvoice3_pytorch_b200.train_step import TrainStep, to_device
    math_mode("fp32")
    model = _ms_model().eval()
    enc = _encoder(seed=4)
    samples = _ragged_samples(1)[:2]
    old = model.embed_speakers.weight.detach().clone()
    want = enc.embed_batch(samples)
    ids = clone_voices(model, enc, samples)
    assert ids == [4, 5]
    table = model.embed_speakers.weight.detach()
    assert torch.equal(table[:4], old) and torch.equal(table[4:], want)
    model.seq2seq.decoder.max_decoder_steps = 8
    texts = [np.array([5, 9, 13, 22], dtype=np.int64), np.array([3, 8, 11], dtype=np.int64)]
    out = synthesis.tts_batch(model, texts, speaker_ids=ids)
    assert len(out) == 2 and all(np.isfinite(o[0]).all() for o in out)
    math_mode("tc")
    rng = np.random.RandomState(0)
    utt = [(rng.randint(2, 149, n).astype(np.int32), (0.05 + 0.9 * rng.rand(t, 80)).astype(np.float32),
            (0.05 + 0.9 * rng.rand(t, 513)).astype(np.float32), s) for n, t, s in ((12, 40, 4), (9, 32, 5))]
    st = TrainStep(model.train(), adapt_speakers=ids, lr_schedule=None)
    loss = st.step(to_device(data.collate(utt), "cuda"))
    ops.check_index_errors()
    assert np.isfinite(float(loss))
    assert torch.equal(model.embed_speakers.weight.detach()[:4], old)
