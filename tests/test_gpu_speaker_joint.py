"""GPU: fine-tuning a speaker encoder through the multi-speaker model's training loss (TrainStep(speaker_encoder=...),
DESIGN.md section 2.16) -- both modes' gradients against the plain multi-speaker step and the adaptation step on a model
whose table holds the encoder's rows, what each mode leaves untouched, graph capture with buckets, deterministic
replays, checkpoint resume, a recovery run on a synthetic corpus and the refusals."""
import copy

import numpy as np
import pytest
import torch

N_VOCAB, LIN, S, M = 149, 129, 16, 80
KW = dict(n_vocab=N_VOCAB, embed_dim=64, mel_dim=M, linear_dim=LIN, r=1, downsample_step=4, kernel_size=3,
          encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256, n_speakers=4,
          speaker_embed_dim=S, use_memory_mask=True, key_projection=True, value_projection=True,
          speaker_embedding_weight_std=0.3)
N_CLONE, T_CROP = 3, 32


@pytest.fixture
def modes():
    from deepvoice3_pytorch_b200 import ops
    old = ops.conv_math, ops.deterministic

    def set_(m, det=None):
        ops.conv_math = m
        if det is not None:
            ops.deterministic = det
    yield set_
    ops.conv_math, ops.deterministic = old


def _model(dropout=0.05, seed=0, **over):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(seed)
    return builder.deepvoice3_multispeaker(dropout=dropout, **dict(KW, **over)).cuda().train()


def _encoder(seed=1, **over):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder
    torch.manual_seed(seed)
    return SpeakerEncoder(**dict(dict(mel_dim=M, speaker_embed_dim=S, channels=128, heads=2, max_samples=4),
                                 **over)).cuda()


def _utterances(spk, text_lens=(23, 17, 9), frame_lens=(70, 51, 33), seed=0):
    rng = np.random.RandomState(seed)
    return [(rng.randint(2, N_VOCAB, n).astype(np.int32), (0.05 + 0.9 * rng.rand(t, M)).astype(np.float32),
             (0.05 + 0.9 * rng.rand(t, LIN)).astype(np.float32), s) for n, t, s in zip(text_lens, frame_lens, spk)]


def _batch(seed=0, spk=(1, 3, 1), n=N_CLONE, **kw):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    b = data.collate(_utterances(spk, seed=seed, **kw))
    b["speaker_mels"] = torch.from_numpy(np.random.RandomState(100 + seed).rand(len(spk), n, T_CROP, M)
                                         .astype(np.float32))
    return to_device(b, "cuda")


def _copy_with_table(model, e):
    """A model with n_speakers = B, the same parameters as ``model`` and the table e."""
    ref = _model(n_speakers=e.shape[0], seed=9)
    sd = {k: v for k, v in model.state_dict().items() if k != "embed_speakers.weight"}
    sd["embed_speakers.weight"] = e.detach().clone()
    ref.load_state_dict(sd, strict=True)
    return ref


def _grads(module, names=None):
    return {k: p.grad.detach().clone() for k, p in module.named_parameters()
            if p.grad is not None and (names is None or k in names)}


def _max_rel(got, want):
    worst = 0.0
    for k, w in want.items():
        g = got[k]
        scale = max(float(w.abs().max()), 1e-30)
        worst = max(worst, float((g - w).abs().max()) / scale)
    return worst


def _assert_grads(got, want, rtol, what):
    assert set(got) == set(want), (what, set(got) ^ set(want))
    for k, w in want.items():
        scale = float(w.abs().max())
        torch.testing.assert_close(got[k], w, rtol=rtol, atol=rtol * scale, msg=lambda m: "%s %s: %s" % (what, k, m))


# ---- gradient identities ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("math,rtol", [("fp32", 1e-5), ("tc", 1e-3)])
def test_joint_gradients_equal_the_table_step_on_the_encoders_rows(modes, math, rtol):
    """Joint step == the plain multi-speaker step on a model whose table is e = encoder(speaker_mels), ids arange(B):
    every model gradient but the table's, and the encoder's gradient == autograd of e against that table gradient."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    modes(math, True)
    model, enc = _model(), _encoder()
    batch = _batch()
    st = TrainStep(model, speaker_encoder=enc, lr_schedule=None)
    ops.rng.manual_seed(11, torch.device("cuda"))
    st._forward_backward(batch)
    got_model = _grads(model)
    got_enc = _grads(enc)
    assert "embed_speakers.weight" not in got_model
    e = enc(batch["speaker_mels"])
    ref = _copy_with_table(model, e)
    rs = TrainStep(ref, lr_schedule=None)
    ops.rng.manual_seed(11, torch.device("cuda"))
    rs._forward_backward(dict(batch, speaker_ids=torch.arange(3, device="cuda")))
    want_model = _grads(ref)
    d_table = want_model.pop("embed_speakers.weight")
    want_enc = dict(zip([k for k, _ in enc.named_parameters()],
                        torch.autograd.grad(e, list(enc.parameters()), d_table)))
    print("joint %s: largest relative difference model %.3g, encoder %.3g"
          % (math, _max_rel(got_model, want_model), _max_rel(got_enc, want_enc)))
    _assert_grads(got_model, want_model, rtol, "model")
    _assert_grads(got_enc, want_enc, rtol, "encoder")
    # joint mode: the encoder's layers were banked (tensor-core weight norm) and sank their gradients into the arena
    flat = st.arena.grad
    lo, hi = flat.data_ptr(), flat.data_ptr() + 4 * flat.numel()
    assert all(lo <= p.grad.data_ptr() < hi for p in enc.parameters())
    if math == "tc":                        # the temporal blocks' convs, as the model's own blocks
        banked = set(st.bank.layers)
        convs = [blk.conv.weight_v for blk in enc.temporal]
        assert convs and all(v.data_ptr() in banked for v in convs)


@pytest.mark.gpu
@pytest.mark.parametrize("math,rtol", [("fp32", 1e-5), ("tc", 1e-3)])
def test_frozen_gradients_equal_the_adaptation_step_on_the_encoders_rows(modes, math, rtol):
    """Encoder-only step: the encoder's gradient == autograd of e against the rows' gradient of an adaptation step
    (adapt_speakers = range(B)) on a model whose table is e; every model parameter and buffer keeps its bits over
    several steps, and no encoder conv comes from the frozen-weight cache."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    modes(math, True)
    model, enc = _model(), _encoder()
    before = {k: v.detach().clone() for k, v in model.state_dict().items()}
    batch = _batch()
    st = TrainStep(model, speaker_encoder=enc, train_model=False, lr_schedule=None, init_lr=1e-2)
    ops.rng.manual_seed(11, torch.device("cuda"))
    st._forward_backward(batch)
    got_enc = _grads(enc)
    e = enc(batch["speaker_mels"])
    ref = _copy_with_table(model, e)
    rs = TrainStep(ref, adapt_speakers=list(range(3)), lr_schedule=None)
    ops.rng.manual_seed(11, torch.device("cuda"))
    rs._forward_backward(dict(batch, speaker_ids=torch.arange(3, device="cuda")))
    rows = rs.arena.grad.view(3, S).clone()
    want_enc = dict(zip([k for k, _ in enc.named_parameters()], torch.autograd.grad(e, list(enc.parameters()), rows)))
    print("frozen %s: largest relative difference encoder %.3g" % (math, _max_rel(got_enc, want_enc)))
    _assert_grads(got_enc, want_enc, rtol, "encoder")
    for i in range(3):
        st.step(_batch(seed=i))
    torch.cuda.synchronize()
    ops.check_index_errors()
    after = model.state_dict()
    for k, v in before.items():
        assert torch.equal(after[k], v), k
    enc_ptrs = {p.data_ptr() for p in enc.parameters()}
    assert st.adapt.frozen.entries
    assert not [e_ for e_ in st.adapt.frozen.entries.values() if e_[1].data_ptr() in enc_ptrs]


@pytest.mark.gpu
def test_joint_mode_keeps_the_table_and_gives_it_no_state(modes):
    from deepvoice3_pytorch_b200.train_step import TrainStep
    modes("tc", False)
    model, enc = _model(), _encoder()
    table = model.embed_speakers.weight
    t0 = table.detach().clone()
    st = TrainStep(model, speaker_encoder=enc, lr_schedule=None, init_lr=1e-3)
    w0 = {k: v.detach().clone() for k, v in enc.state_dict().items()}
    for i in range(3):
        st.step(_batch(seed=i))
    torch.cuda.synchronize()
    assert torch.equal(table.detach(), t0) and table.grad is None
    trainable = list(model.get_trainable_parameters())
    ti = next(i for i, p in enumerate(trainable) if p is table)
    ck = st.state_dict()
    assert ti not in ck["optimizer"]["state"] and len(ck["optimizer"]["param_groups"][0]["params"]) == len(trainable)
    assert len(ck["speaker_encoder"]["optimizer"]["state"]) == len(list(enc.parameters()))
    assert any(not torch.equal(v, w0[k]) for k, v in enc.state_dict().items())
    assert ck["train_model"] is True
    fresh = _model(seed=5)
    fresh.load_state_dict(ck["state_dict"], strict=True)


# ---- graphs, buckets, determinism, checkpoints ----------------------------------------------------------------------
def _batches():
    return [_batch(seed=0), _batch(seed=1, text_lens=(15, 12, 30), frame_lens=(40, 66, 90)),
            _batch(seed=2, text_lens=(11, 10, 9), frame_lens=(30, 31, 29)), _batch(seed=3)]


def _run(train_model, use_graph, order, batches, ckpt_at=None):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    model, enc = _model(dropout=0.0), _encoder()
    ops.rng.manual_seed(3, torch.device("cuda"))
    st = TrainStep(model, speaker_encoder=enc, train_model=train_model, use_graph=use_graph)
    losses, ck = [], None
    for n, i in enumerate(order):
        if n == ckpt_at:
            ck = copy.deepcopy(st.state_dict())
        losses.append(float(st.step(batches[i])))
    torch.cuda.synchronize()
    return st, losses, st.arena.flat.clone(), ck


@pytest.mark.gpu
@pytest.mark.parametrize("train_model", [True, False])
def test_graph_buckets_determinism_and_resume(modes, train_model):
    """Graph steps over variable-length batches replayed out of order: bit-identical run to run (deterministic
    mode), within 1e-5 of eager steps; a checkpoint after 3 graph steps resumes to the bits of 6 straight steps."""
    from deepvoice3_pytorch_b200.train_step import TrainStep
    modes("tc", True)
    batches = _batches()
    order = [0, 1, 2, 1, 3, 2]
    _, le, pe, _ = _run(train_model, False, order, batches)
    st1, l1, p1, _ = _run(train_model, True, order, batches)
    _, l2, p2, _ = _run(train_model, True, order, batches)
    assert st1.graphs_captured >= 3
    assert l1 == l2 and torch.equal(p1, p2)
    np.testing.assert_allclose(l1, le, rtol=1e-5)
    torch.testing.assert_close(p1, pe, rtol=1e-5, atol=1e-6)
    # resume; the order keeps every batch on the same kind of graph (exact or bucket) in both runs
    order = [0, 1, 2, 0, 1, 2]
    st, straight, p_straight, ck = _run(train_model, True, order, batches, ckpt_at=3)
    assert ck["global_step"] == 3 and ck["train_model"] is train_model
    model, enc = _model(dropout=0.0, seed=7), _encoder(seed=8)
    res = TrainStep(model, speaker_encoder=enc, train_model=train_model, use_graph=True)
    res.load_state_dict(ck)
    tail = [float(res.step(batches[i])) for i in order[3:]]
    torch.cuda.synchronize()
    assert tail == straight[3:]
    assert torch.equal(res.arena.flat, p_straight) and res.global_step == 6


# ---- recovery on a synthetic corpus ---------------------------------------------------------------------------------
def _synthetic_corpus(n_spk=10, n_utt=10, T=96, seed=0):
    """Per-speaker spectral envelopes, per-frame gains and noise, clipped to [0, 1] (the normalised mel range)."""
    rng = np.random.RandomState(seed)
    f = np.arange(M)
    corpus = []
    for s in range(n_spk):
        centers, widths = rng.uniform(0, M, 3), rng.uniform(4, 16, 3)
        env = sum(np.exp(-0.5 * ((f - c) / w) ** 2) for c, w in zip(centers, widths))
        env = 0.2 + 0.6 * env / env.max()
        utts = []
        for _ in range(n_utt):
            gain = rng.uniform(0.6, 1.2, (T, 1))
            utts.append(np.clip(env[None, :] * gain + 0.05 * rng.randn(T, M), 0, 1).astype(np.float32))
        corpus.append(utts)
    return corpus


def _tts_batch(corpus, speakers, rng, n=4, t_crop=64):
    """One TTS batch whose row b speaks as speakers[b] (a random text, one of its utterances as the mel target, the
    linear target derived from it), with n cloning crops of its other utterances."""
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    items, clones = [], []
    for s in speakers:
        u = rng.randint(0, 8)
        mel = corpus[s][u]
        lin = np.concatenate([mel, mel[:, :LIN - M]], 1)
        items.append((rng.randint(2, N_VOCAB, rng.randint(10, 25)).astype(np.int32), mel, lin, s))
        others = [j for j in range(8) if j != u]
        crops = []
        for j in rng.choice(others, n, replace=False):
            o = rng.randint(0, mel.shape[0] - t_crop + 1)
            crops.append(corpus[s][j][o:o + t_crop])
        clones.append(np.stack(crops))
    b = data.collate(items)
    b["speaker_mels"] = torch.from_numpy(np.stack(clones))
    return to_device(b, "cuda")


def _held_out_loss(model, enc, corpus, speakers):
    """Teacher-forced loss of one utterance of each held-out speaker, that speaker cloned by the encoder from its
    utterances 0-7."""
    from deepvoice3_pytorch_b200.train_step import fused_training_loss
    rng = np.random.RandomState(1)
    b = _tts_batch(corpus, speakers, rng)
    e = enc.embed_batch([[corpus[s][j] for j in range(8)] for s in speakers])
    model.eval()
    try:
        with torch.no_grad():
            outs = model(b["x"], b["mel"], speaker_embed=e, text_positions=b["text_positions"],
                         frame_positions=b["frame_positions"], input_lengths=b["input_lengths_dev"])
            return float(fused_training_loss(outs, b))
    finally:
        model.train()


def _pool_loss(model, enc, pool):
    """Mean training loss over the batches of ``pool`` with the encoder's current embeddings, no update."""
    from deepvoice3_pytorch_b200.train_step import fused_training_loss
    with torch.no_grad():
        losses = []
        for b in pool:
            outs = model(b["x"], b["mel"], speaker_embed=enc(b["speaker_mels"]), text_positions=b["text_positions"],
                         frame_positions=b["frame_positions"], input_lengths=b["input_lengths_dev"])
            losses.append(float(fused_training_loss(outs, b)))
    return float(np.mean(losses))


@pytest.mark.gpu
@pytest.mark.parametrize("train_model,lr", [(True, 1e-3), (False, 3e-3)])
def test_recovery_on_a_synthetic_corpus(modes, train_model, lr):
    """Stage 2 (SpeakerEncoderStep, 100 steps), then 200 graph steps of the mode on four fixed batches.  Against the
    mean loss of those batches before fine-tuning (the pretrained encoder, no update): every 20-step mean of the
    training loss stays below it (the loss falls without first blowing up), and the last one is below 0.8x of it
    (deterministic mode: the same bits every run).  The teacher-forced loss of two held-out speakers cloned by the
    encoder is recorded, not bounded: with random weights it need not show generalisation (DESIGN.md section 2.16)."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep
    from deepvoice3_pytorch_b200.train_step import TrainStep
    modes("tc", True)
    corpus = _synthetic_corpus()
    model, enc = _model(n_speakers=8, dropout=0.0), _encoder(seed=6, max_samples=8)
    pre = SpeakerEncoderStep(enc, model, lr=1e-3, use_graph=True)
    rng = np.random.RandomState(7)
    for _ in range(100):                         # stage 2: regress the table rows of the 8 training speakers
        mels = np.stack([np.stack([corpus[s][j][o:o + 64] for j, o in zip(rng.choice(8, 4, replace=False),
                                                                        rng.randint(0, 33, 4))]) for s in range(8)])
        pre.step({"mels": torch.from_numpy(mels), "speaker_ids": torch.arange(8)})
    held = [8, 9]
    before = _held_out_loss(model, enc, corpus, held)
    pool = [_tts_batch(corpus, list(rng.permutation(8)[:4]), rng) for _ in range(4)]
    base = _pool_loss(model, enc, pool)
    st = TrainStep(model, speaker_encoder=enc, train_model=train_model, use_graph=True, init_lr=lr,
                   lr_schedule=None, clip_thresh=0.0)
    losses = [st.step(pool[i % 4]).clone() for i in range(200)]
    losses = torch.stack(losses).cpu().numpy()
    ops.check_index_errors()
    windows = losses.reshape(10, 20).mean(1)
    after = _held_out_loss(model, enc, corpus, held)
    print("recovery train_model=%s: loss before %.4f, 20-step means %s (last %.3fx), pool loss after %.4f, held-out "
          "cloned loss %.4f -> %.4f" % (train_model, base, [round(float(w), 4) for w in windows], windows[-1] / base,
                                        _pool_loss(model, enc, pool), before, after))
    assert windows.max() < base
    assert windows[-1] < 0.8 * base
    assert np.isfinite(after)


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_before_any_launch(modes, monkeypatch):
    import torch.distributed as dist
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.train_step import TrainStep
    modes("tc", False)
    model, enc = _model(), _encoder()
    n0 = lib.raw("dv3_launch_count")()
    torch.manual_seed(0)
    single = builder.deepvoice3(**{k: v for k, v in KW.items() if k not in ("n_speakers", "speaker_embed_dim",
                                                                             "speaker_embedding_weight_std")}).cuda()
    for train_model in (True, False):
        for m, e, kw in ((single, enc, {}), (model, _encoder(speaker_embed_dim=8), {}),
                         (model, _encoder(mel_dim=40), {}), (model, enc, dict(train_postnet=False)),
                         (model, enc, dict(train_seq2seq=False)), (model, enc, dict(adapt_speakers=[3]))):
            with pytest.raises(ValueError):
                TrainStep(m, speaker_encoder=e, train_model=train_model, **kw)
    with monkeypatch.context() as mp:
        mp.setattr(dist, "is_initialized", lambda: True)
        mp.setattr(dist, "get_world_size", lambda *a: 2)
        with pytest.raises(ValueError):
            TrainStep(model, speaker_encoder=enc)
    assert lib.raw("dv3_launch_count")() == n0
    for train_model in (True, False):
        st = TrainStep(_model(), speaker_encoder=_encoder(), train_model=train_model, use_graph=True)
        n0 = lib.raw("dv3_launch_count")()
        good = _batch()
        bad = [_batch(n=5),                                                    # N > max_samples
               {k: v for k, v in good.items() if k != "speaker_mels"},         # missing
               dict(good, speaker_mels=good["speaker_mels"].double()),
               dict(good, speaker_mels=good["speaker_mels"][:2]),              # rows != B
               dict(good, speaker_mels=good["speaker_mels"][..., :40]),        # mel_dim
               dict(good, speaker_mels=good["speaker_mels"][0])]               # 3-D
        for b in bad:
            with pytest.raises(ValueError):
                st.step(b)
        assert lib.raw("dv3_launch_count")() == n0 and st.global_step == 0
        st.step(good)
        n1 = lib.raw("dv3_launch_count")()
        with pytest.raises(ValueError):                                        # one shape for the life of the step
            st.step(_batch(n=2))
        assert lib.raw("dv3_launch_count")() == n1 and st.global_step == 1


# ---- the plain step is unchanged ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_plain_multispeaker_step_launches_what_it_launched_before(modes):
    """deepvoice3_vctk, graph mode: the captured step of a TrainStep without a speaker encoder launches as many
    kernels as before this feature existed (measured on the previous code, in "tc", deterministic mode off, B = 4,
    T_text 64, T_mel 256)."""
    from bench import PRESETS
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.train_step import TrainStep, make_synthetic_batch, to_device
    modes("tc", False)
    name, kw, extra = PRESETS["deepvoice3_vctk"]
    torch.manual_seed(0)
    model = getattr(builder, name)(**kw).cuda().train()
    st = TrainStep(model, use_graph=True, **extra)
    st.step(to_device(make_synthetic_batch(B=4, T_text=64, T_mel=256, n_speakers=kw["n_speakers"], linear_dim=513),
                      "cuda"))
    assert st.launches_per_step == 566          # 579 at B = 16, T_text 128, T_mel 800 (DESIGN.md section 2.12)
