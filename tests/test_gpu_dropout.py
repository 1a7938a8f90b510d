"""GPU: training-mode dropout of every kernel that applies the counter-based mask or rebuilds it in a backward pass,
against an fp64 reference (computed on the device with plain torch ops) that applies the same mask explicitly.

The mask comes from oracle/dropout_mask.py, which restates the device hash; test_dropout_mask_bit_exact pins that
restatement to the device bit for bit, every other test here relies on it.  Procedure: ``ops.rng.manual_seed`` +
``ops.rng.start_forward`` and one call with ``training=True``, so the call site draws salt 1.

Discrimination guard: every comparison is repeated against the reference under the mask of salt 2 and under no mask;
both must miss the tolerance by at least 10x on every guarded tensor, so the tolerance can tell the right mask from a
wrong one.
"""
import numpy as np
import pytest
import torch

import golden_util as G
import test_gpu_attention as A
from test_gpu_blocks import ATOL, RTOL
from test_gpu_fp32_conv import gamma

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 10.0


def excess(got, want, grad=False):
    """max |got - want| / (atol + rtol |want|): <= 1 is the bar of test_gpu_blocks.close (grad=False) /
    grad_close (grad=True, atol scaled by the tensor's magnitude)."""
    got, want = got.detach().double(), want.detach().double()
    atol = ATOL * 10 * max(1.0, float(want.abs().max())) if grad else ATOL
    return float(((got - want).abs() / (atol + RTOL * want.abs())).max())


def check(got, refs, grad_names, guarded, what):
    """got {name: tensor}; refs {"mask": {...}, "salt+1": {...}, "none": {...}} of fp64 references."""
    ok = {n: excess(got[n], refs["mask"][n], n in grad_names) for n in got}
    bad = [n for n, r in ok.items() if r > 1]
    assert not bad, "%s: error / tolerance %s" % (what, ok)
    for wrong in ("salt+1", "none"):
        miss = {n: excess(got[n], refs[wrong][n], n in grad_names) for n in guarded}
        weak = [n for n, r in miss.items() if r < GUARD]
        assert not weak, "%s: the %s reference is within %gx of the tolerance: %s" % (what, wrong, GUARD, miss)
        ok["guard " + wrong] = min(miss.values())
    return ok


def _seed_and_salt(seed):
    from deepvoice3_pytorch_b200 import ops
    ops.rng.manual_seed(seed, torch.device(DEV))
    ops.rng.start_forward()
    return ops.rng


def _mask(rng, salt, p, shape):
    from oracle import dropout_mask as DM
    return torch.from_numpy(DM.mask(DM.seed_u64(rng.seed), salt, p, shape)).to(DEV)


# ---- standalone dropout: pins oracle/dropout_mask.py to the device hash ------------------------------------------
@pytest.mark.parametrize("p", [0.05, 0.25, 0.5, 0.9])
def test_dropout_mask_bit_exact(p):
    from deepvoice3_pytorch_b200 import ops
    from oracle import dropout_mask as DM
    n = 100_003                                          # odd numel
    gen = torch.Generator().manual_seed(int(p * 100))
    x = (torch.randn(n, generator=gen) + 0.1).to(DEV).requires_grad_(True)
    dy = torch.randn(n, generator=gen).to(DEV)
    seeds = [("small", 1234, 0), ("high32", 0x7654321089ABCDEF, 0), ("wrapped", 0x7000000000000000, 3)]
    for name, seed, advances in seeds:
        for salt in (1, 0xFFFFFFF0):
            rng = _seed_and_salt(seed)
            for _ in range(advances):
                rng.advance()
            if advances:
                assert int(rng.seed.item()) < 0, "advance() should have wrapped the int64 seed"
            rng.salt = salt - 1                          # the next call site draws ``salt``
            y = ops.dropout(x, p, True)
            assert rng.salt == salt
            m = torch.from_numpy(DM.mask(DM.seed_u64(rng.seed), salt, p, (n,))).to(DEV)
            assert torch.equal(y, x.detach() * m), "forward %s salt %#x" % (name, salt)
            (gx,) = torch.autograd.grad(y, x, dy)
            assert torch.equal(gx, dy * m), "backward %s salt %#x" % (name, salt)
            kept = float((m > 0).double().mean())
            assert abs(kept - (1 - p)) < 5 * (p * (1 - p) / n) ** 0.5 + 1e-4, kept
            other = DM.mask(DM.seed_u64(rng.seed), salt + 1, p, (n,))
            assert not np.array_equal(other, m.cpu().numpy())


def test_dropout_mask_edges():
    """CPU-side properties the device relies on: p <= 0 is a no-op, the threshold clamps, the scale is fp32."""
    from oracle import dropout_mask as DM
    assert (DM.mask(1, 1, 0.0, (7,)) == 1).all()
    assert DM.threshold(1.0) == 0xFFFFFFFF and DM.threshold(0.5) == 0x80000000
    assert DM.scale(0.05) == np.float32(1) / (np.float32(1) - np.float32(0.05))
    assert DM.seed_u64(-1) == 2 ** 64 - 1


# ---- ConvBlock (GLU +- residual, highway; speaker addend) ----------------------------------------------------------
def _block_params(B, C, T, k, seed):
    gen = torch.Generator().manual_seed(seed)
    v = torch.randn(2 * C, C, k, generator=gen) * (4.0 / (k * C)) ** 0.5
    g = v.pow(2).sum((1, 2), keepdim=True).sqrt() * (1 + 0.2 * torch.randn(2 * C, 1, 1, generator=gen))
    bias = 0.1 * torch.randn(2 * C, generator=gen)
    x = torch.randn(B, C, T, generator=gen)
    z = torch.randn(B, T, C, generator=gen)            # pre-softsign speaker addend
    return v, g, bias, x, z


def _block_ref(v, g, bias, x, z, drop, k, d, causal, mode, residual, R):
    """fp64 oracle forward + backward on the device -> {y, dx, dv, dg, dbias[, dz]}."""
    from oracle import dv3_oracle as O
    C = x.shape[1]
    sd = {"m.conv.weight_v": v.double().requires_grad_(True), "m.conv.weight_g": g.double().requires_grad_(True),
          "m.conv.bias": bias.double().requires_grad_(True)}
    xr = x.double().requires_grad_(True)
    zr = None
    if z is not None:        # identity speaker projection: the oracle adds softsign(z), the device's spk input
        sd["m.speaker_proj.weight_v"] = torch.eye(C, device=DEV, dtype=torch.float64)
        sd["m.speaker_proj.weight_g"] = torch.ones(C, 1, device=DEV, dtype=torch.float64)
        sd["m.speaker_proj.bias"] = torch.zeros(C, device=DEV, dtype=torch.float64)
        zr = z.double().requires_grad_(True)
    dr = None if drop is None else drop.double()
    if mode == "hw":
        y = O.highway_conv1d(sd, "m", xr, k, d, causal, drop=dr)
    else:
        y = O.conv1d_glu(sd, "m", xr, k, d, causal, residual, zr, drop=dr)
    leaves = [xr, sd["m.conv.weight_v"], sd["m.conv.weight_g"], sd["m.conv.bias"]] + ([zr] if z is not None else [])
    grads = torch.autograd.grad((y * R.double()).sum(), leaves)
    out = dict(zip(["dx", "dv", "dg", "dbias", "dz"], grads))
    out["y"] = y.detach()
    return out


BLOCK_CASES = [
    # mode, B, C, T, k, d, causal, residual, p
    ("glu", 3, 128, 37, 3, 27, True, True, 0.5),        # causal halo 54 >= T, one partial time tile
    ("glu", 1, 256, 131, 5, 9, False, False, 0.05),     # k = 5, T = 128 + 3
    ("hw", 3, 384, 200, 3, 1, False, True, 0.5),
    ("hw", 16, 256, 200, 3, 27, True, True, 0.05),      # bench-size highway layer
    ("glu", 16, 512, 800, 3, 9, False, True, 0.05),     # bench-size encoder / converter layer
    ("glu", 3, 128, 800, 5, 27, True, False, 0.5),
    ("glu", 1, 512, 37, 5, 27, False, True, 0.05),      # non-causal halo 54 per side >= T
    ("hw", 1, 128, 131, 5, 9, True, True, 0.5),
    ("glu", 3, 80, 131, 3, 9, True, True, 0.5),         # C the tensor-core path refuses
    ("hw", 16, 80, 37, 5, 1, False, True, 0.05),
]


def _run_block_case(math, mode, B, C, T, k, d, causal, residual, p, spk, monkeypatch):
    from deepvoice3_pytorch_b200 import ops
    monkeypatch.setattr(ops, "conv_math", math)
    assert ops.tc_supported(B, C, T, k) == (C % 128 == 0)
    v, g, bias, x, z = _block_params(B, C, T, k, B * 7919 + C + T + k + d)
    if not spk:
        z = None
    R = G.loss_weights((B, C, T), 0, DEV)
    vc, gc, bc, xc = [t.to(DEV).requires_grad_(True) for t in (v, g, bias, x)]
    zc = None if z is None else z.to(DEV).requires_grad_(True)
    spk_in = None if zc is None else ops.transpose12(torch.nn.functional.softsign(zc))
    rng = _seed_and_salt(4242 + C)
    y = ops.convblock(xc, vc, gc, bc, spk_in, k, d, causal, ops.MODE_GLU if mode == "glu" else ops.MODE_HIGHWAY,
                      residual, p_drop=p, training=True)
    assert rng.salt == 1
    leaves = [xc, vc, gc, bc] + ([zc] if zc is not None else [])
    grads = torch.autograd.grad((y * R).sum(), leaves)
    got = dict(zip(["dx", "dv", "dg", "dbias", "dz"], grads))
    got["y"] = y
    args = (x.to(DEV), z if z is None else z.to(DEV))
    refs = {name: _block_ref(v.to(DEV), g.to(DEV), bias.to(DEV), *args, drop, k, d, causal, mode, residual, R)
            for name, drop in (("mask", _mask(rng, 1, p, (B, C, T))), ("salt+1", _mask(rng, 2, p, (B, C, T))),
                               ("none", None))}
    what = "%s %s B=%d C=%d T=%d k=%d d=%d causal=%s res=%s p=%g spk=%s" % (math, mode, B, C, T, k, d, causal,
                                                                          residual, p, spk)
    r = check(got, refs, {"dx", "dv", "dg", "dbias", "dz"}, ("y", "dx", "dv"), what)
    print("%s: %s" % (what, " ".join("%s %.3g" % kv for kv in sorted(r.items()))))


@pytest.mark.parametrize("math", ["tc", "fp32"])
@pytest.mark.parametrize("mode,B,C,T,k,d,causal,residual,p", BLOCK_CASES)
def test_convblock_dropout_vs_fp64(mode, B, C, T, k, d, causal, residual, p, math, monkeypatch):
    _run_block_case(math, mode, B, C, T, k, d, causal, residual, p, False, monkeypatch)


@pytest.mark.parametrize("math", ["tc", "fp32"])
@pytest.mark.parametrize("B,C,T,d,causal,residual,p", [(3, 128, 200, 9, True, True, 0.5),
                                                       (2, 256, 131, 1, False, False, 0.05)])
def test_convblock_speaker_dropout_vs_fp64(B, C, T, d, causal, residual, p, math, monkeypatch):
    """The speaker addend of the gated block (spk, and dspk rebuilt from the bf16 gradient planes on the tensor-core
    path) with dropout on; dz is the gradient through softsign(z) = spk."""
    _run_block_case(math, "glu", B, C, T, 3, d, causal, residual, p, True, monkeypatch)


# ---- attention core -------------------------------------------------------------------------------------------------
def _attn_ref(q, k, v, mask, drop, Wout, Wp):
    from oracle import dv3_oracle as O
    qr, kr, vr = [t.double().requires_grad_(True) for t in (q, k, v)]
    ctx, probs = O.attention_core(qr.transpose(1, 2), kr, vr.transpose(1, 2), mask,
                                  None if drop is None else drop.double())
    out = ctx.transpose(1, 2)
    loss = (out * Wout.double()).sum() + (0 if Wp is None else (probs * Wp.double()).sum())
    dq, dk, dv = torch.autograd.grad(loss, (qr, kr, vr))
    return {"out": out.detach(), "probs": probs.detach(), "dq": dq, "dk": dk, "dv": dv,
            "dropmask": None if drop is None else drop.double()}


ATTN_CASES = [
    # path, B, E, Td, Ts, key mask, dprobs, p
    ("tc", 16, 256, 200, 128, True, True, 0.05),         # bench shape: 2 row tiles, 2 key slabs, 2 cols CTAs
    ("tc", 3, 128, 200, 100, True, False, 0.5),
    ("tc", 2, 144, 37, 13, False, True, 0.5),
    ("tc", 1, 64, 129, 65, False, False, 0.05),
    ("simt", 3, 128, 200, 100, True, True, 0.05),
    ("simt", 2, 64, 37, 13, False, False, 0.5),
    ("auto", 3, 128, 131, 129, True, True, 0.5),         # Ts > 128: automatic fallback
    ("auto", 2, 256, 64, 200, False, False, 0.05),
]


@pytest.mark.parametrize("path,B,E,Td,Ts,masked,use_dprobs,p", ATTN_CASES)
def test_attention_dropout_vs_fp64(path, B, E, Td, Ts, masked, use_dprobs, p, monkeypatch):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    monkeypatch.setattr(ops, "conv_math", "tc")
    monkeypatch.setattr(ops, "tc_attention", path != "simt")
    assert bool(lib.raw("dv3_tc_attn_supported")(B, E, Td, Ts)) == (path != "auto")
    gen = torch.Generator().manual_seed(B + E + Td + Ts)
    s = 1.2 * E ** -0.25
    q, k = s * torch.randn(B, E, Td, generator=gen), s * torch.randn(B, E, Ts, generator=gen)
    v = torch.randn(B, E, Ts, generator=gen)
    q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
    mask = None
    if masked:
        lengths = torch.tensor([Ts - (13 * b) % max(Ts // 2, 1) for b in range(B)])
        lengths[-1] = min(33, Ts)                           # crosses the 32-key boundary
        mask = (torch.arange(Ts)[None, :] >= lengths[:, None]).to(DEV)
    Wout = G.loss_weights((B, E, Td), 0, DEV)
    Wp = G.loss_weights((B, Td, Ts), 1, DEV) if use_dprobs else None
    qc, kc, vc = [t.clone().requires_grad_(True) for t in (q, k, v)]
    rng = _seed_and_salt(999 + Ts)
    out, probs = ops.attention_core(qc, kc, vc, mask, p, True)
    assert rng.salt == 1
    loss = (out * Wout).sum() + (0 if Wp is None else (probs * Wp).sum())
    dq, dk, dv = torch.autograd.grad(loss, (qc, kc, vc))
    got = {"out": out, "probs": probs, "dq": dq, "dk": dk, "dv": dv}
    refs = {name: _attn_ref(q, k, v, mask, drop, Wout, Wp)
            for name, drop in (("mask", _mask(rng, 1, p, (B, Td, Ts))), ("salt+1", _mask(rng, 2, p, (B, Td, Ts))),
                               ("none", None))}
    what = "%s B=%d E=%d Td=%d Ts=%d mask=%s dprobs=%s p=%g" % (path, B, E, Td, Ts, masked, use_dprobs, p)
    # The context is scale * Pd.V with scale = sqrt(Ts): its absolute error grows with sqrt(Ts) sum|V| Pd, which the
    # fixed atol of ``close`` does not follow (the 16-bit operand split of the tensor-core GEMM alone reaches ~1e-4
    # at Ts = 100, p = 0.5).  Its bar is the elementwise bound derived from the arithmetic (test_gpu_attention.py), with
    # the exact-fp32 GEMM coefficient on the bgemm + softmax path.
    tc = path != "simt" and bool(lib.raw("dv3_tc_attn_supported")(B, E, Td, Ts))
    _, _, _, bout = A.ref_forward(q.double(), k.double(), v.double(), mask, refs["mask"]["dropmask"],
                                  c=A.c_gemm if tc else gamma)
    r_out = {name: A.bound_ratio(out, refs[name]["out"], bout) for name in refs}
    assert r_out["mask"] <= 1, "%s: out error / bound %.3g" % (what, r_out["mask"])
    assert min(r_out["salt+1"], r_out["none"]) >= GUARD, "%s: out guard %s" % (what, r_out)
    del got["out"]
    # probs are returned before dropout: not guarded
    r = check(got, refs, {"dq", "dk", "dv"}, ("dq", "dk", "dv"), what)
    r.update({"out/bound": r_out["mask"], "out guard": min(r_out["salt+1"], r_out["none"])})
    print("%s: %s" % (what, " ".join("%s %.3g" % kv for kv in sorted(r.items()))))


# ---- model level: tensor-core vs exact-fp32 mode with dropout on ----------------------------------------------------
def _models():
    base = dict(n_vocab=149, mel_dim=80, linear_dim=129, r=1, downsample_step=4, kernel_size=3, encoder_channels=128,
                decoder_channels=128, converter_channels=128, use_memory_mask=True, max_positions=256)
    return [("deepvoice3", dict(base, embed_dim=64, key_projection=True, value_projection=True), 1),
            ("nyanko", dict(base, embed_dim=128), 1),
            ("deepvoice3_multispeaker", dict(base, embed_dim=64, n_speakers=4, speaker_embed_dim=16), 4)]


@pytest.mark.parametrize("bname,kw,n_speakers", _models(), ids=[m[0] for m in _models()])
def test_model_dropout_tc_vs_fp32(bname, kw, n_speakers, monkeypatch):
    """One training forward (dropout=0.3 at every site: ConvBlocks, attention, embeddings; the plain convs, ReLU convs
    and ConvTranspose layers draw no salt) and the fused-loss backward, from the same seed in both arithmetic modes:
    same salt sequence, really dropped, and outputs / parameter gradients at the bars of
    test_gpu_models.test_preset_model_vs_oracle."""
    from deepvoice3_pytorch_b200 import builder, ops
    from deepvoice3_pytorch_b200.train_step import fused_training_loss, make_synthetic_batch, to_device
    host = make_synthetic_batch(B=3, T_text=40, T_mel=128, linear_dim=129, n_speakers=n_speakers, seed=21)
    lengths = [40, 33, 17]
    host["input_lengths_dev"] = torch.tensor(lengths)
    for b, n in enumerate(lengths):
        host["x"][b, n:] = 0
        host["text_positions"][b, n:] = 0
    batch = to_device(host, DEV)
    torch.manual_seed(0)
    model = getattr(builder, bname)(**dict(kw, dropout=0.3)).to(DEV).train()
    plain = getattr(builder, bname)(**dict(kw, dropout=0.0)).to(DEV).train()
    plain.load_state_dict(model.state_dict())

    def run(m, math):
        monkeypatch.setattr(ops, "conv_math", math)
        m.zero_grad(set_to_none=True)
        ops.rng.manual_seed(31337, torch.device(DEV))
        outs = m(batch["x"], batch["mel"], speaker_ids=batch.get("speaker_ids"),
                 text_positions=batch["text_positions"], frame_positions=batch["frame_positions"],
                 input_lengths=batch["input_lengths_dev"])
        salt = ops.rng.salt
        fused_training_loss(outs, batch).backward()
        return [o.detach() for o in outs], {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}, \
            salt

    outs_tc, g_tc, salt_tc = run(model, "tc")
    outs_32, g_32, salt_32 = run(model, "fp32")
    outs_plain, _, salt_plain = run(plain, "tc")
    assert salt_tc == salt_32 > 0 and salt_plain == 0, (salt_tc, salt_32, salt_plain)
    names = ["mel", "linear", "alignments", "done"]
    for n, a, b, c in zip(names, outs_tc, outs_32, outs_plain):
        assert excess(a, b) <= 1, "%s: tc vs fp32 %.3g x tolerance" % (n, excess(a, b))
        assert excess(a, c) >= GUARD, "%s: dropout=0.3 output within %gx of the dropout-free one" % (n, GUARD)
    trainable = {id(p) for p in model.get_trainable_parameters()}
    worst = 0.0
    for n, p in model.named_parameters():
        if id(p) not in trainable or n.endswith("key_projection.bias"):
            continue        # softmax is shift invariant: the key-projection bias has an exactly-zero true gradient
        assert n in g_tc and n in g_32, n
        norm = float(g_32[n].norm())
        if norm < 1e-10:
            continue
        err = float((g_tc[n] - g_32[n]).double().norm()) / norm
        worst = max(worst, err)
        assert err < (1e-2 if p.numel() > 16 else 1e-1), "%s: relative L2 tc vs fp32 %.3e" % (n, err)
    print("%s: salts %d, worst relative L2 gradient difference tc vs fp32 %.3e" % (bname, salt_tc, worst))
