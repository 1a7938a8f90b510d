"""GPU parity of the full models (builder API) against the golden vectors of the live reference and,
at the BASELINE.json preset sizes, against the CPU oracle.  rtol=1e-3 / atol=1e-4 (north_star)."""
import json
import os

import numpy as np
import pytest
import torch

import golden_util as G
from test_gpu_blocks import close, grad_close

pytestmark = pytest.mark.gpu
MODELS = G.load("models.npz")


def _build(kw):
    from deepvoice3_pytorch_b200 import builder
    kw = dict(kw)
    name = kw.pop("builder")
    return getattr(builder, name)(**kw)


@pytest.mark.parametrize("name", list(MODELS))
def test_model_golden(name):
    case = MODELS[name]
    model = _build(G.kwargs_of(case)).cuda()
    missing = model.load_state_dict(G.tensors(case["sd"]), strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    model.train()          # dropout=0 in the fixture configs
    ins = G.tensors(case["in"], "cuda")
    ins["mel"].requires_grad_(True)
    outs = model(ins["text"], ins["mel"], speaker_ids=ins.get("speaker_ids"),
                 text_positions=ins["text_positions"], frame_positions=ins["frame_positions"],
                 input_lengths=case["meta"]["input_lengths"])
    for i, o in enumerate(outs):
        close(o, case["out"][str(i)], what="%s out%d" % (name, i))
    loss = sum((o * G.loss_weights(o.shape, i, "cuda")).sum() for i, o in enumerate(outs))
    loss.backward()
    params = dict(model.named_parameters())
    for k, ref in case["gsd"].items():
        assert params[k].grad is not None, k
        grad_close(params[k].grad, ref, what="%s grad %s" % (name, k))
    grad_close(ins["mel"].grad, case["gin"]["mel"], what="grad mel")
    from deepvoice3_pytorch_b200 import ops
    ops.check_index_errors()


def preset_kwargs(name):
    """The train.py:812-840 hparams -> builder kwargs mapping for the three BASELINE.json presets."""
    base = dict(n_vocab=149, mel_dim=80, linear_dim=513, r=1, downsample_step=4, padding_idx=0, kernel_size=3,
                use_memory_mask=True, trainable_positional_encodings=False, force_monotonic_attention=True,
                use_decoder_state_for_postnet_input=True, freeze_embedding=False, window_ahead=3,
                window_backward=1, speaker_embed_dim=16)
    if name == "deepvoice3_ljspeech":
        return "deepvoice3", dict(base, n_speakers=1, embed_dim=256, encoder_channels=512, decoder_channels=256,
                                  converter_channels=256, max_positions=512, key_projection=True,
                                  value_projection=True, speaker_embedding_weight_std=0.01)
    if name == "nyanko_ljspeech":
        return "nyanko", dict(base, n_speakers=1, embed_dim=128, encoder_channels=256, decoder_channels=256,
                              converter_channels=256, max_positions=512, key_projection=False,
                              value_projection=False, speaker_embedding_weight_std=0.01)
    if name == "deepvoice3_vctk":
        return "deepvoice3_multispeaker", dict(base, n_speakers=108, embed_dim=256, encoder_channels=512,
                                               decoder_channels=256, converter_channels=256, max_positions=1024,
                                               key_projection=True, value_projection=True,
                                               speaker_embedding_weight_std=0.05)
    raise ValueError(name)


def synthetic_batch(B, T_text, T_dec, n_speakers, seed, ragged=True):
    gen = torch.Generator().manual_seed(seed)
    text = torch.randint(2, 149, (B, T_text), generator=gen)
    lengths = torch.randint(T_text // 2, T_text + 1, (B,), generator=gen).numpy() if ragged \
        else np.full(B, T_text)
    lengths[0] = T_text
    tpos = torch.arange(1, T_text + 1)[None].repeat(B, 1)
    for b in range(B):
        text[b, lengths[b]:] = 0
        tpos[b, lengths[b]:] = 0
    mel = torch.rand(B, T_dec, 80, generator=gen)
    fpos = torch.arange(1, T_dec + 1)[None].repeat(B, 1)
    spk = torch.randint(0, n_speakers, (B,), generator=gen) if n_speakers > 1 else None
    return text, mel, tpos, fpos, lengths, spk


_ORACLE_CACHE = {}


def _preset_case(preset, B):
    """Model weights, batch and the CPU oracle's outputs / gradients (fp32 = parity target, fp64 = error yardstick),
    computed once per preset and shared by the arithmetic modes."""
    key = (preset, B)
    if key in _ORACLE_CACHE:
        return _ORACLE_CACHE[key]
    from deepvoice3_pytorch_b200 import builder
    from oracle import dv3_oracle as O
    from oracle.specs import spec_from_builder
    bname, kw = preset_kwargs(preset)
    kw["dropout"] = 0.0
    torch.manual_seed(11)
    model = getattr(builder, bname)(**kw)
    with torch.no_grad():       # move g / bias off their init so the fixtures exercise them
        gen = torch.Generator().manual_seed(5)
        for n, p in model.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(1 + 0.1 * torch.randn(p.shape, generator=gen))
            elif n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=gen))
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    batch = synthetic_batch(B, 128, 200, kw["n_speakers"], 77)
    text, mel, tpos, fpos, lengths, spk = batch
    spec = spec_from_builder(bname, **kw)

    def run_oracle(dtype):
        leaves = {k: (v.detach().to(dtype).requires_grad_(True) if v.is_floating_point() else v)
                  for k, v in sd.items()}
        outs_o = O.model_forward(leaves, spec, text, mel.to(dtype), spk, tpos, fpos, lengths)
        loss_o = sum((o * G.loss_weights(o.shape, i, dtype=dtype)).sum() / o.numel() ** 0.5
                     for i, o in enumerate(outs_o))
        loss_o.backward()
        return [o.detach() for o in outs_o], {k: v.grad for k, v in leaves.items()
                                              if torch.is_tensor(v) and v.grad is not None}

    outs_ref, grads32 = run_oracle(torch.float32)
    _, grads64 = run_oracle(torch.float64)
    _ORACLE_CACHE[key] = (bname, kw, sd, batch, outs_ref, grads32, grads64)
    return _ORACLE_CACHE[key]


_FP32_MODE_ERR = {}        # (preset, parameter) -> relative L2 gradient error of the exact-fp32 mode (filled by the fp32 rows)


@pytest.mark.parametrize("math", ["fp32", "tc"])          # fp32 rows first: the tc rows compare against their errors
@pytest.mark.parametrize("preset", ["deepvoice3_ljspeech", "nyanko_ljspeech", "deepvoice3_vctk"])
def test_preset_model_vs_oracle(preset, math, monkeypatch):
    """The three BASELINE.json presets at the benchmark size -- B=16, T_text=128, T_mel=800 (T_dec=200) -- forward +
    every parameter gradient, in both ConvBlock arithmetic modes (wgmma fp16/bf16 operand pairs = the benched mode;
    exact-fp32 CUDA cores), at north_star's tolerance: rtol=1e-3 / atol=1e-4 on every output."""
    from deepvoice3_pytorch_b200 import builder, ops
    monkeypatch.setattr(ops, "conv_math", math)
    B = 16
    bname, kw, sd, (text, mel, tpos, fpos, lengths, spk), outs_ref, grads32, grads64 = _preset_case(preset, B)
    model = getattr(builder, bname)(**kw)
    model.load_state_dict(sd)
    model = model.cuda().train()
    outs = model(text.cuda(), mel.cuda(), speaker_ids=None if spk is None else spk.cuda(),
                 text_positions=tpos.cuda(), frame_positions=fpos.cuda(), input_lengths=lengths)
    names = ["mel", "linear", "alignments", "done"]
    for i, (o, r) in enumerate(zip(outs, outs_ref)):
        assert o.shape == r.shape
        close(o, r, rtol=1e-3, atol=1e-4, what="%s %s (%s)" % (preset, names[i], math))
    loss = sum((o * G.loss_weights(o.shape, i, "cuda")).sum() / o.numel() ** 0.5 for i, o in enumerate(outs))
    loss.backward()
    # Gradients here are sums of ~1e5-1e7 signed terms (the projection loss above cancels heavily), which makes them
    # ILL-CONDITIONED functions of the forward values: a 1e-6 perturbation of the activations moves some of them by
    # 1e-3 (measured: switching the gradient GEMMs from 16-bit to 22-bit operands changed no error below in the 4th
    # digit -- the forward rounding, not the backward arithmetic, sets them).  At B=16 the exact-fp32 CUDA-core mode
    # itself sits at 2e-3 (ljspeech) .. 2.5e-2 (nyanko) relative L2 against fp64 on its worst tensor, single-scalar
    # parameters (the position-rate projections' bias / weight_g, sums of ~1e6 cancelling terms) at 4e-2, and
    # parameters with an exactly-zero true gradient (the key-projection bias: softmax is shift invariant) carry pure
    # noise.  Yardsticks:
    #  (1) both modes: relative L2 error against the fp64 oracle <= 1e-2 (<= 1e-1 for tensors of <= 16 elements), or
    #      <= 8x the CPU fp32 oracle's own error on that tensor;
    #  (2) the tensor-core mode is as good as the exact-fp32 mode: per tensor err_tc <= max(1e-2, 4 * err_exact_fp32);
    #  frozen tensors (the position tables: not in get_trainable_parameters(), their gradients are never used) are skipped.
    worst = 0.0
    trainable = {id(p) for p in model.get_trainable_parameters()}
    for k, p in model.named_parameters():
        if k not in grads64 or id(p) not in trainable:
            continue
        assert p.grad is not None, k
        truth = grads64[k]
        norm = float(truth.norm())
        if norm < 1e-10:
            continue
        err = float((p.grad.cpu().double() - truth).norm()) / norm
        err32 = float((grads32[k].double() - truth).norm()) / norm
        worst = max(worst, err)
        floor = 1e-2 if truth.numel() > 16 else 1e-1
        assert err < max(floor, 8 * err32), "%s (%s): relative L2 gradient error %.3e (cpu fp32: %.3e)" % (k, math, err,
                                                                                                           err32)
        if math == "fp32":
            _FP32_MODE_ERR[(preset, k)] = err
        elif (preset, k) in _FP32_MODE_ERR and truth.numel() > 16:
            ref = _FP32_MODE_ERR[(preset, k)]
            assert err < max(1e-2, 4 * ref), "%s: tensor-core mode %.3e vs exact-fp32 mode %.3e" % (k, err, ref)
    print("worst relative L2 gradient error vs fp64 (%s, %s): %.3e" % (preset, math, worst))
