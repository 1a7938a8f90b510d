"""GPU parity of the C-ABI block kernels against (a) the golden vectors of the live reference and
(b) the CPU oracle at BASELINE.json sizes.  Tolerance is north_star's: rtol=1e-3, atol=1e-4 (fp32)."""
import numpy as np
import pytest
import torch

import golden_util as G

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4


def close(a, b, rtol=RTOL, atol=ATOL, what=""):
    a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.detach().float().cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol, err_msg=what)


def grad_close(a, b, what=""):
    """Gradients are sums over up to B*T terms: compare relative to the tensor's scale."""
    b = np.asarray(b)
    scale = max(1.0, float(np.abs(b).max()))
    close(a, b, rtol=RTOL, atol=ATOL * scale * 10, what=what)


BLOCKS = G.load("blocks.npz")


def _run_block(case, fn):
    """fn(sd, ins) -> output tensor (on cuda); checks outputs and all gradients against the golden case."""
    dev = "cuda"
    sd = G.tensors(case["sd"], dev)
    for v in sd.values():
        v.requires_grad_(True)
    ins = G.tensors(case["in"], dev)
    for v in ins.values():
        if v.is_floating_point():
            v.requires_grad_(True)
    out = fn(sd, ins)
    outs = out if isinstance(out, tuple) else (out,)
    for i, o in enumerate(outs):
        close(o, case["out"][str(i)], what="out%d" % i)
    loss = sum((o * G.loss_weights(o.shape, i, dev)).sum() for i, o in enumerate(outs))
    loss.backward()
    for k, ref in case.get("gsd", {}).items():
        assert sd[k].grad is not None, k
        grad_close(sd[k].grad, ref, what="grad " + k)
    for k, ref in case.get("gin", {}).items():
        grad_close(ins[k].grad, ref, what="grad in " + k)


@pytest.mark.parametrize("name", [n for n in BLOCKS if n.startswith("glu") and "spk" not in n])
def test_conv1d_glu_golden(name):
    from deepvoice3_pytorch_b200 import ops
    case = BLOCKS[name]
    m = {k: G.meta_scalar(case, k) for k in ("k", "d", "causal", "residual")}
    _run_block(case, lambda sd, ins: ops.convblock(
        ins["x"], sd["conv.weight_v"], sd["conv.weight_g"], sd["conv.bias"], None, m["k"], m["d"],
        bool(m["causal"]), ops.MODE_GLU, bool(m["residual"])))


@pytest.mark.parametrize("name", [n for n in BLOCKS if n.startswith("hw")])
def test_highway_golden(name):
    from deepvoice3_pytorch_b200 import ops
    case = BLOCKS[name]
    m = {k: G.meta_scalar(case, k) for k in ("k", "d", "causal")}
    _run_block(case, lambda sd, ins: ops.convblock(
        ins["x"], sd["conv.weight_v"], sd["conv.weight_g"], sd["conv.bias"], None, m["k"], m["d"],
        bool(m["causal"]), ops.MODE_HIGHWAY, True))


@pytest.mark.parametrize("name", ["conv1x1_0", "conv1x1_1"])
def test_conv1x1_golden(name):
    from deepvoice3_pytorch_b200 import ops
    _run_block(BLOCKS[name], lambda sd, ins: ops.conv1d(ins["x"], sd["weight_v"], sd["weight_g"], sd["bias"]))


def test_conv_ramp_known_answer():
    """reference tests/test_conv.py: weights 1, bias 0, ramp input, causal -- exact integers expected."""
    from deepvoice3_pytorch_b200 import ops
    ramp = G.load("conv_ramp.npz")
    for name, case in ramp.items():
        B, T, C, k, d = [int(v) for v in case["meta"]["BTCkd"]]
        v = torch.ones(2 * C, C, k, device="cuda")
        g = torch.full((2 * C, 1, 1), float(C * k) ** 0.5, device="cuda")
        x = (torch.zeros(B, C, T) + torch.arange(0, T).float()).cuda()
        y = ops.conv1d(x, v, g, torch.zeros(2 * C, device="cuda"), k=k, dilation=d, causal=True)
        close(y, case["out"]["0"], rtol=1e-6, atol=1e-5, what=name)


@pytest.mark.parametrize("math", ["fp32", "tc"])
@pytest.mark.parametrize("Cin,Cout,T,kind", [(256, 512, 128, "conv_relu"), (80, 256, 200, "conv"), (512, 513, 800, "conv"),
                                            (513, 513, 400, "conv"), (256, 256, 200, "convT")])
def test_plain_conv_canonical_vs_oracle(Cin, Cout, T, kind, math, monkeypatch):
    """1x1 Conv1d (+ReLU) and ConvTranspose1d(k=2,s=2) at preset shapes (incl. the odd 513 width and the 80-wide mel
    input) in the exact-fp32 and tensor-core modes, against the CPU oracle."""
    from deepvoice3_pytorch_b200 import ops
    from oracle import dv3_oracle as O
    import torch.nn.functional as F
    monkeypatch.setattr(ops, "conv_math", math)
    B = 4
    gen = torch.Generator().manual_seed(Cin + Cout + T)
    x = torch.randn(B, Cin, T, generator=gen)
    if kind == "convT":
        v = torch.randn(Cin, Cout, 2, generator=gen) * (1.0 / (2 * Cin)) ** 0.5
        g = v.pow(2).sum((1, 2), keepdim=True).sqrt() * (1 + 0.2 * torch.randn(Cin, 1, 1, generator=gen))
    else:
        v = torch.randn(Cout, Cin, 1, generator=gen) * (1.0 / Cin) ** 0.5
        g = v.pow(2).sum((1, 2), keepdim=True).sqrt() * (1 + 0.2 * torch.randn(Cout, 1, 1, generator=gen))
    bias = 0.1 * torch.randn(Cout, generator=gen)
    sd = {"m.weight_v": v.clone().requires_grad_(True), "m.weight_g": g.clone().requires_grad_(True),
          "m.bias": bias.clone().requires_grad_(True)}
    xr = x.clone().requires_grad_(True)
    if kind == "convT":
        yr = O.conv_transpose1d(sd, "m", xr)
    else:
        yr = O.conv1d(sd, "m", xr)
        if kind == "conv_relu":
            yr = F.relu(yr + 0.3)                  # shift the kink away from 0-crossing noise... still a ReLU test
    R = G.loss_weights(yr.shape, 0)
    (yr * R).sum().backward()
    vc, gc, bc, xc = [t.cuda().requires_grad_(True) for t in (v, g, bias, x)]
    if kind == "convT":
        y = ops.conv_transpose1d_k2s2(xc, vc, gc, bc)
    elif kind == "conv_relu":
        y = ops.conv1d(xc, vc, gc, bc + 0.3, relu=True)
    else:
        y = ops.conv1d(xc, vc, gc, bc)
    close(y, yr, what="y")
    (y * R.cuda()).sum().backward()
    grad_close(xc.grad, xr.grad.numpy(), "dx")
    grad_close(vc.grad, sd["m.weight_v"].grad.numpy(), "dv")
    grad_close(gc.grad, sd["m.weight_g"].grad.numpy(), "dg")
    grad_close(bc.grad, sd["m.bias"].grad.numpy(), "dbias")


# ---- BASELINE.json canonical shapes against the CPU oracle ---------------------------------------
@pytest.mark.parametrize("B,C,T,k,d,causal,residual,mode", [
    (3, 128, 37, 3, 9, True, True, "glu"),           # ragged: T odd, single partial tile, halo > T/2
    (2, 256, 131, 5, 3, False, True, "hw"),          # k=5, T = 128 + 3
    (16, 256, 200, 3, 27, True, False, "glu"),
    (16, 512, 128, 3, 9, False, True, "glu"),
    (4, 256, 800, 3, 3, False, True, "glu"),
    (2, 512, 800, 3, 1, False, True, "glu"),
    (16, 256, 200, 3, 9, True, True, "hw"),
])
@pytest.mark.parametrize("math", ["fp32", "tc"])
def test_convblock_canonical_vs_oracle(B, C, T, k, d, causal, residual, mode, math, monkeypatch):
    """Both arithmetic modes of the ConvBlock -- exact-fp32 CUDA cores and the wgmma split-bf16 path --
    must meet the same parity bar against the CPU oracle."""
    from deepvoice3_pytorch_b200 import ops
    from oracle import dv3_oracle as O
    monkeypatch.setattr(ops, "conv_math", math)
    if math != "fp32":
        assert ops.tc_supported(B, C, T, k), "canonical shapes must run on the tensor-core path"
    gen = torch.Generator().manual_seed(B * 1000 + C + T + d)
    v = torch.randn(2 * C, C, k, generator=gen) * (4.0 / (k * C)) ** 0.5
    g = v.pow(2).sum((1, 2), keepdim=True).sqrt() * (1 + 0.2 * torch.randn(2 * C, 1, 1, generator=gen))
    bias = 0.1 * torch.randn(2 * C, generator=gen)
    x = torch.randn(B, C, T, generator=gen)
    sd = {"m.conv.weight_v": v.clone().requires_grad_(True), "m.conv.weight_g": g.clone().requires_grad_(True),
          "m.conv.bias": bias.clone().requires_grad_(True)}
    xr = x.clone().requires_grad_(True)
    if mode == "glu":
        yr = O.conv1d_glu(sd, "m", xr, k, d, causal, residual)
    else:
        yr = O.highway_conv1d(sd, "m", xr, k, d, causal)
    R = G.loss_weights(yr.shape, 0)
    (yr * R).sum().backward()

    vc, gc, bc, xc = [t.cuda().requires_grad_(True) for t in (v, g, bias, x)]
    y = ops.convblock(xc, vc, gc, bc, None, k, d, causal,
                      ops.MODE_GLU if mode == "glu" else ops.MODE_HIGHWAY, residual)
    close(y, yr, what="y")
    (y * R.cuda()).sum().backward()
    grad_close(xc.grad, xr.grad.numpy(), "dx")
    grad_close(vc.grad, sd["m.conv.weight_v"].grad.numpy(), "dv")
    grad_close(gc.grad, sd["m.conv.weight_g"].grad.numpy(), "dg")
    grad_close(bc.grad, sd["m.conv.bias"].grad.numpy(), "dbias")


@pytest.mark.parametrize("math,C", [("fp32", 64), ("tc", 128)])
def test_convblock_dropout_statistics_and_consistency(math, C, monkeypatch):
    """In-kernel dropout: keep-rate ~ 1-p, scale 1/(1-p), and the backward regenerates the same mask."""
    from deepvoice3_pytorch_b200 import ops
    monkeypatch.setattr(ops, "conv_math", math)
    B, T, k = 4, 256, 1
    p = 0.25
    # identity-like block: v = [I ; 0] so a = dropout(x), b = 0 -> s = 0.5 -> y = 0.5*dropout(x)
    v = torch.zeros(2 * C, C, k, device="cuda")
    v[:C, :, 0] = torch.eye(C)
    v[C:, :, 0] = 1e-3 * torch.eye(C)       # keep ||v|| > 0
    g = v.pow(2).sum((1, 2), keepdim=True).sqrt()
    g[C:] = 0.0                             # b rows scaled to exactly 0
    bias = torch.zeros(2 * C, device="cuda")
    x = (torch.rand(B, C, T, device="cuda") + 0.5).requires_grad_(True)
    ops.rng.manual_seed(1234, x.device)
    ops.rng.start_forward()
    y = ops.convblock(x, v, g, bias, None, k, 1, False, ops.MODE_GLU, False, p_drop=p, training=True)
    ratio = (y / (0.5 * x)).detach()
    kept = ratio > 0
    rate = kept.float().mean().item()
    assert abs(rate - (1 - p)) < 0.01, rate
    close(ratio[kept], torch.full_like(ratio[kept], 1 / (1 - p)), rtol=2e-4, atol=1e-5)
    y.sum().backward()
    # dx = 0.5 * mask/(1-p)
    close(x.grad, 0.5 * kept.float() / (1 - p), rtol=2e-4, atol=1e-5)
    # different salt / seed -> different mask
    ops.rng.start_forward()
    ops.rng.advance()
    y2 = ops.convblock(x, v, g, bias, None, k, 1, False, ops.MODE_GLU, False, p_drop=p, training=True)
    assert ((y2 > 0) != (y > 0)).float().mean().item() > 0.2
    # eval: no dropout
    y3 = ops.convblock(x, v, g, bias, None, k, 1, False, ops.MODE_GLU, False, p_drop=p, training=False)
    close(y3, 0.5 * x, rtol=2e-4, atol=1e-6)
