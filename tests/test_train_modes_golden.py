"""Seq2seq-only / postnet-only losses pinned to the reference's own ``train()``: tests/golden/train_modes.npz was produced
by running train.py (tests/golden/make_train_modes_golden.py) in both partial modes and jointly on a stand-in model.
The torch-ops loss (CPU) and the fused loss kernels with their per-term slots (GPU) must give every logged scalar
and d(loss)/d(outputs)."""
import numpy as np
import pytest
import torch

import golden_util as G

MODES = G.load("train_modes.npz")
TAGS = {"mel_l1_loss": "TERM_MEL_L1", "mel_binary_div_loss": "TERM_MEL_BD", "linear_l1_loss": "TERM_LIN_L1",
        "linear_binary_div_loss": "TERM_LIN_BD", "done_loss": "TERM_DONE", "attn_loss": "TERM_ATTN"}
NAMES = ("mel_out", "lin_out", "attn", "done_hat")


def _inputs(case, device):
    """-> (outputs of the trained part as leaves, None elsewhere; batch dict; loss kwargs)."""
    w, bw, pw, guided, pfreq, sr, sigma, r, ds, s2s, post = case["meta"]["cfg"]
    r, ds = int(r), int(ds)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in case["in"].items()}
    run = {"mel_out": s2s, "lin_out": post, "attn": s2s, "done_hat": s2s}
    outs = [t[k].clone().requires_grad_(True) if run[k] else None for k in NAMES]
    batch = {"mel": t["mel"][:, 0::ds, :].contiguous() if ds > 1 else t["mel"], "y": t["y"], "done": t["done"],
             "target_lengths": t["target_lengths"], "input_lengths_dev": t["input_lengths"]}
    kw = dict(r=r, downsample_step=ds, masked_loss_weight=w, binary_divergence_weight=bw, guided_attention_sigma=sigma,
              use_guided_attention=bool(guided), priority_freq=pfreq, priority_freq_weight=pw, sample_rate=sr)
    return outs, batch, kw


def _check_grads(case, outs, rtol):
    for o, k in zip(outs, NAMES):
        want = case["out"]["grad_" + k]
        got = o.grad.detach().cpu().numpy() if o is not None and o.grad is not None else np.zeros_like(want)
        np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-9, err_msg=k)


@pytest.mark.parametrize("name", sorted(MODES))
def test_torch_loss_matches_reference_partial_modes(name):
    from deepvoice3_pytorch_b200.train_step import training_loss
    case = MODES[name]
    outs, batch, kw = _inputs(case, "cpu")
    loss = training_loss(outs, batch, **kw)
    loss.backward()
    np.testing.assert_allclose(float(loss), float(case["out"]["loss"]), rtol=2e-6)
    _check_grads(case, outs, 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODES))
def test_fused_loss_terms_match_reference_partial_modes(name):
    """The *_terms kernels: total, every logged per-term value the mode has (and zero in the slots of the part that
    does not run), "mel loss" / "linear_loss" as their weighted sums, and d(loss)/d(outputs)."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import fused_training_loss
    case = MODES[name]
    outs, batch, kw = _inputs(case, "cuda")
    terms = torch.zeros(ops.TERM_COUNT, device="cuda")
    loss = fused_training_loss(outs, batch, terms=terms, **kw)
    loss.backward()
    out = case["out"]
    np.testing.assert_allclose(float(loss), float(out["loss"]), rtol=2e-5)
    t = terms.cpu().double().numpy()
    for tag, slot in TAGS.items():
        want = float(out[tag]) if tag in out else 0.0
        np.testing.assert_allclose(t[getattr(ops, slot)], want, rtol=2e-5, atol=1e-7, err_msg=tag)
    w = kw["binary_divergence_weight"]
    if "mel_loss" in out:
        np.testing.assert_allclose((1 - w) * t[ops.TERM_MEL_L1] + w * t[ops.TERM_MEL_BD], float(out["mel_loss"]),
                                   rtol=2e-5)
    if "linear_loss" in out:
        np.testing.assert_allclose((1 - w) * t[ops.TERM_LIN_L1] + w * t[ops.TERM_LIN_BD], float(out["linear_loss"]),
                                   rtol=2e-5)
    _check_grads(case, outs, 2e-4)
