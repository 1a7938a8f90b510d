"""CPU: the host side of TrainStep's training modes and optimizer settings -- the learning-rate schedules, the hparams
mapping, the refusals, the partial arena and bucket plan, and FlatAdam's torch.optim.Adam checkpoint format."""
import math

import numpy as np
import pytest
import torch


def _lrschedule(name, init_lr, step, **kw):
    """reference lrschedule.py:14-35, restated."""
    if name == "step_learning_rate_decay":
        return init_lr * kw.get("anneal_rate", 0.98) ** (step // kw.get("anneal_interval", 30000))
    TdivM = kw["T"] // kw["M"]
    return init_lr / 2.0 * (np.cos(np.pi * ((step - 1) % TdivM) / TdivM) + 1.0)


@pytest.mark.parametrize("name,kw", [("step_learning_rate_decay", {}),
                                     ("step_learning_rate_decay", dict(anneal_rate=0.5, anneal_interval=7)),
                                     ("cyclic_cosine_annealing", dict(T=1000, M=4)),
                                     ("cyclic_cosine_annealing", dict(T=97, M=3))])
def test_schedules_match_reference(name, kw):
    from deepvoice3_pytorch_b200 import train_step
    f = getattr(train_step, name)
    for step in list(range(0, 300)) + [29999, 30000, 30001, 10 ** 6]:
        want = _lrschedule(name, 5e-4, step, **kw)
        assert f(5e-4, step, **kw) == pytest.approx(want, rel=1e-12, abs=0), (name, step)


def test_train_step_kwargs_maps_optimizer_settings_and_schedules():
    from deepvoice3_pytorch_b200 import hparams, train_step
    hp = dict(initial_learning_rate=1e-3, adam_beta1=0.5, adam_beta2=0.9, adam_eps=1e-6, clip_thresh=0.1,
              outputs_per_step=1, downsample_step=4, masked_loss_weight=0.5, binary_divergence_weight=0.1,
              guided_attention_sigma=0.2, use_guided_attention=True, weight_decay=1e-6, amsgrad=True,
              lr_schedule="cyclic_cosine_annealing", lr_schedule_kwargs=dict(T=100, M=2))
    ts = hparams.train_step_kwargs(hp)
    assert ts["weight_decay"] == 1e-6 and ts["amsgrad"] is True
    for step in (0, 1, 49, 50, 51):
        assert ts["lr_schedule"](1e-3, step) == train_step.cyclic_cosine_annealing(1e-3, step, T=100, M=2)
    ts = hparams.train_step_kwargs(dict(hp, lr_schedule="step_learning_rate_decay", lr_schedule_kwargs={}))
    assert ts["lr_schedule"] is train_step.step_learning_rate_decay
    ts = hparams.train_step_kwargs({k: v for k, v in hp.items() if k not in ("weight_decay", "amsgrad")})
    assert ts["weight_decay"] == 0.0 and ts["amsgrad"] is False


def _model(use_decoder_state=False, n_speakers=1):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    kw = dict(n_vocab=30, embed_dim=16, mel_dim=8, linear_dim=17, r=1, downsample_step=4, kernel_size=3,
              encoder_channels=16, decoder_channels=16, converter_channels=16, max_positions=64,
              use_decoder_state_for_postnet_input=use_decoder_state)
    if n_speakers > 1:
        return builder.deepvoice3_multispeaker(n_speakers=n_speakers, speaker_embed_dim=4, **kw)
    return builder.deepvoice3(**kw)


def test_training_mode_refusals():
    from deepvoice3_pytorch_b200.train_step import TrainStep
    with pytest.raises(ValueError, match="both False"):
        TrainStep(_model(), train_seq2seq=False, train_postnet=False)
    for mode in (dict(train_postnet=False), dict(train_seq2seq=False)):
        with pytest.raises(ValueError, match="single-speaker"):
            TrainStep(_model(n_speakers=3), **mode)
    with pytest.raises(ValueError, match="use_decoder_state_for_postnet_input"):
        TrainStep(_model(use_decoder_state=True), train_seq2seq=False)
    with pytest.raises(ValueError, match="weight_decay"):
        from deepvoice3_pytorch_b200.train_step import FlatAdam, ParameterArena
        FlatAdam(ParameterArena(_model()), weight_decay=-1.0)


@pytest.mark.parametrize("mode", ["seq2seq", "postnet"])
def test_partial_arena_and_bucket_plan(mode):
    from deepvoice3_pytorch_b200.train_step import ParameterArena, arena_parts, gradient_buckets
    model = _model()
    part = getattr(model, mode)
    trainable = list(model.get_trainable_parameters())
    own = {id(p) for p in part.parameters()}
    sub = [p for p in trainable if id(p) in own]
    other = [p.detach().clone() for p in model.parameters() if id(p) not in own]
    arena = ParameterArena(model, sub)
    assert arena.numel == sum((p.numel() + 3) // 4 * 4 for p in sub)
    assert all(p.grad is None for p in model.parameters() if id(p) not in own)
    assert all(torch.equal(a, b) for a, b in zip(other, [p for p in model.parameters() if id(p) not in own]))
    assert arena_parts(model, arena) == [(0, arena.numel)]
    tagged, rest = gradient_buckets(model, arena)
    if mode == "postnet":
        assert tagged == {"postnet": (0, arena.numel)} and rest == []
    else:
        assert "postnet" not in tagged and set(tagged) == {"encoder_hi", "encoder_mid"}
        spans = sorted(list(tagged.values()) + rest)
        assert spans[0][0] == 0 and spans[-1][1] == arena.numel
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def test_joint_arena_parts():
    from deepvoice3_pytorch_b200.train_step import ParameterArena, arena_parts
    model = _model(n_speakers=3)
    arena = ParameterArena(model)
    parts = arena_parts(model, arena)
    assert parts[0] == arena.range_of(list(model.seq2seq.parameters()))
    assert parts[1] == arena.range_of(list(model.postnet.parameters()))
    assert parts[2] == (parts[1][1], arena.numel)           # the speaker embedding


def _adam_steps(opt, params, n, seed):
    gen = torch.Generator().manual_seed(seed)
    for _ in range(n):
        for p in params:
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()


def test_partial_flat_adam_state_round_trips_with_torch_amsgrad():
    """A postnet-only FlatAdam state (indices over all of get_trainable_parameters(), state for the postnet only,
    max_exp_avg_sq, the real weight_decay / amsgrad) loads into torch.optim.Adam(amsgrad=True) and back; a joint
    FlatAdam resumes the postnet at its step and the seq2seq at step 0."""
    from deepvoice3_pytorch_b200.train_step import FlatAdam, ParameterArena, arena_parts
    model = _model()
    trainable = list(model.get_trainable_parameters())
    own = {id(p) for p in model.postnet.parameters()}
    index = [i for i, p in enumerate(trainable) if id(p) in own]
    ref = torch.optim.Adam([trainable[i] for i in index], lr=1e-3, betas=(0.5, 0.9), eps=1e-6, weight_decay=1e-4,
                           amsgrad=True)
    _adam_steps(ref, [trainable[i] for i in index], 3, seed=1)
    local = ref.state_dict()
    # the reference's full-list indexing: state only for the trained parameters
    full = {"state": {index[j]: s for j, s in local["state"].items()},
            "param_groups": [dict(local["param_groups"][0], params=list(range(len(trainable))))]}

    arena = ParameterArena(model, [trainable[i] for i in index])
    flat = FlatAdam(arena, weight_decay=1e-4, amsgrad=True, index=index, n_index=len(trainable))
    flat.load_state_dict(full)
    assert flat.part_t == [3]
    out = flat.state_dict()
    assert sorted(out["state"]) == index
    g = out["param_groups"][0]
    assert g["weight_decay"] == 1e-4 and g["amsgrad"] is True and g["params"] == list(range(len(trainable)))
    back = torch.optim.Adam(trainable, lr=1.0, weight_decay=1e-4, amsgrad=True)
    back.load_state_dict(out)
    for j, i in enumerate(index):
        for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.equal(back.state_dict()["state"][i][key], local["state"][j][key]), key
        assert float(back.state_dict()["state"][i]["step"]) == 3.0
    with pytest.raises(ValueError, match="amsgrad"):
        FlatAdam(arena, weight_decay=1e-4, index=index, n_index=len(trainable)).load_state_dict(full)
    with pytest.raises(ValueError, match="weight_decay"):
        FlatAdam(arena, amsgrad=True, index=index, n_index=len(trainable)).load_state_dict(full)

    # the joint model resumes from the partial state: postnet part at step 3, everything else at step 0
    model2 = _model()
    arena2 = ParameterArena(model2)
    joint = FlatAdam(arena2, weight_decay=1e-4, amsgrad=True, parts=arena_parts(model2, arena2))
    joint.load_state_dict(full)
    assert joint.part_t == [0, 3] and joint.t == 3
    assert sorted(joint.state_dict()["state"]) == index
    # two parts with different clocks are held separately; a part whose parameters disagree cannot be represented
    bad = {"state": dict(full["state"]), "param_groups": full["param_groups"]}
    bad["state"][index[0]] = dict(bad["state"][index[0]], step=torch.tensor(5.0))
    with pytest.raises(ValueError, match="step counts differ"):
        joint.load_state_dict(bad)
    assert math.isfinite(joint.lr)


def test_partial_flat_adam_keeps_the_other_parts_state():
    """A postnet-only FlatAdam loading a joint torch.optim.Adam state keeps the seq2seq entries as they are and writes
    them back: its state_dict() holds state for every parameter, as the reference's checkpoint does."""
    from deepvoice3_pytorch_b200.train_step import FlatAdam, ParameterArena
    model = _model()
    trainable = list(model.get_trainable_parameters())
    ref = torch.optim.Adam(trainable, lr=1e-3, betas=(0.5, 0.9), eps=1e-6)
    _adam_steps(ref, trainable, 2, seed=3)
    full = ref.state_dict()
    own = {id(p) for p in model.postnet.parameters()}
    index = [i for i, p in enumerate(trainable) if id(p) in own]
    flat = FlatAdam(ParameterArena(model, [trainable[i] for i in index]), index=index, n_index=len(trainable))
    flat.load_state_dict(full)
    out = flat.state_dict()
    assert sorted(out["state"]) == sorted(full["state"])
    for i, st in full["state"].items():
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(out["state"][i][key], st[key]), (i, key)
        assert float(out["state"][i]["step"]) == 2.0
    torch.optim.Adam(trainable, lr=1.0).load_state_dict(out)
