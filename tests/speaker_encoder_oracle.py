"""fp64 restatement of the speaker encoder (deepvoice3_pytorch_b200/speaker_encoder.py, csrc/spk_enc.cu).

pool_* and attn_* spell out the forward and the hand-derived backward the kernels implement, per speaker over its
n valid samples (the host tests check the backward against torch autograd with gradcheck); ``encoder_forward`` is the
whole encoder as plain torch fp64 autograd code over a state_dict (weight-normed convs, GLU blocks, pool, attention).
"""
import math

import torch
import torch.nn.functional as F

ATTN = ("w_q", "b_q", "w_k", "b_k", "w_v", "b_v", "w_s", "b_s", "w_e", "b_e")


def pool_fwd(x, lengths):
    """x (R, C, T), lengths (R,) -> (R, C) means over t < lengths[r]."""
    T = x.shape[2]
    mask = (torch.arange(T)[None, :] < torch.as_tensor(lengths)[:, None]).to(x.dtype)
    return (x * mask[:, None, :]).sum(-1) / torch.as_tensor(lengths, dtype=x.dtype)[:, None]


def pool_bwd(dy, lengths, T):
    mask = (torch.arange(T)[None, :] < torch.as_tensor(lengths)[:, None]).to(dy.dtype)
    return dy[:, :, None] * mask[:, None, :] / torch.as_tensor(lengths, dtype=dy.dtype)[:, None, None]


def _speaker_fwd(h, p, heads):
    """h (n, C) -> (out (S,), saved dict)."""
    n, C = h.shape
    dh = C // heads
    q, k, v = h @ p["w_q"].T + p["b_q"], h @ p["w_k"].T + p["b_k"], h @ p["w_v"].T + p["b_v"]
    qh, kh, vh = (t.view(n, heads, dh).transpose(0, 1) for t in (q, k, v))       # (H, n, dh)
    P = torch.softmax(qh @ kh.transpose(1, 2) / math.sqrt(dh), dim=-1)           # (H, n, n)
    o = (P @ vh).transpose(0, 1).reshape(n, C)
    s = o @ p["w_s"] + p["b_s"]
    a = torch.softmax(s, dim=0)
    e = h @ p["w_e"].T + p["b_e"]
    out = a @ e
    return out, dict(q=qh, k=kh, v=vh, P=P, o=o, a=a, e=e, out=out)


def attn_fwd(h, counts, p, heads, target=None):
    """h (B, N, C), counts (B,) -> (out (B, S), L1 loss or None, per-speaker saved)."""
    outs, saved = [], []
    for b in range(h.shape[0]):
        o, sv = _speaker_fwd(h[b, :int(counts[b])], p, heads)
        outs.append(o)
        saved.append(sv)
    out = torch.stack(outs)
    loss = None if target is None else (out - target).abs().mean()
    return out, loss, saved


def attn_bwd(h, counts, p, heads, saved, target=None, d_out=None, d_loss=None):
    """The kernels' backward, by hand: -> (d_h (B, N, C), {name: gradient})."""
    B, N, C = h.shape
    S = p["w_e"].shape[0]
    dh_ = C // heads
    scale = 1.0 / math.sqrt(dh_)
    d_h = torch.zeros_like(h)
    g = {k: torch.zeros_like(v) for k, v in p.items()}
    for b in range(B):
        n = int(counts[b])
        sv, hb = saved[b], h[b, :n]
        dout = torch.zeros(S, dtype=h.dtype) if d_out is None else d_out[b].clone()
        if target is not None and d_loss is not None:
            dout = dout + d_loss * torch.sign(sv["out"] - target[b]) / (B * S)
        a, e, o = sv["a"], sv["e"], sv["o"]
        da = e @ dout
        ds = a * (da - (a * da).sum())
        g["b_s"] += ds.sum()
        g["w_s"] += ds @ o
        g["w_e"] += torch.outer(dout, a @ hb)
        g["b_e"] += a.sum() * dout
        dO = torch.outer(ds, p["w_s"]).view(n, heads, dh_).transpose(0, 1)          # (H, n, dh)
        P, qh, kh, vh = sv["P"], sv["q"], sv["k"], sv["v"]
        dP = dO @ vh.transpose(1, 2)
        dZ = P * (dP - (P * dP).sum(-1, keepdim=True))
        dvh = P.transpose(1, 2) @ dO
        dqh = scale * dZ @ kh
        dkh = scale * dZ.transpose(1, 2) @ qh
        dq, dk, dv = (t.transpose(0, 1).reshape(n, C) for t in (dqh, dkh, dvh))
        for name, d in (("q", dq), ("k", dk), ("v", dv)):
            g["w_" + name] += d.T @ hb
            g["b_" + name] += d.sum(0)
        d_h[b, :n] = dq @ p["w_q"] + dk @ p["w_k"] + dv @ p["w_v"] + torch.outer(a, dout) @ p["w_e"]
    return d_h, g


def _wn(sd, prefix):
    v, gw = sd[prefix + "weight_v"], sd[prefix + "weight_g"]
    return gw * v / v.pow(2).sum(tuple(range(1, v.dim())), keepdim=True).sqrt()


def encoder_forward(sd, mels, heads, kernel_size, n_conv, lengths=None, counts=None, target=None):
    """The whole encoder in torch fp64 autograd over a state_dict of fp64 leaves: mels (B, N, T, M) -> (out, loss)."""
    B, N, T, M = mels.shape
    x = mels.reshape(B * N, T, M).transpose(1, 2)
    for i in (0, 2):
        x = torch.relu(F.conv1d(x, _wn(sd, "spectral.%d." % i), sd["spectral.%d.bias" % i]))
    for i in range(n_conv):
        pre = "temporal.%d.conv." % i
        res = x
        y = F.conv1d(x, _wn(sd, pre), sd[pre + "bias"], padding=(kernel_size - 1) // 2)
        a, gate = y.split(y.shape[1] // 2, dim=1)
        x = (a * torch.sigmoid(gate) + res) * math.sqrt(0.5)
    if lengths is None:
        lengths = torch.full((B * N,), T)
    if counts is None:
        counts = torch.full((B,), N)
    h = pool_fwd(x, lengths).view(B, N, -1)
    out, loss, _ = attn_fwd(h, counts, {k: sd[k] for k in ATTN}, heads, target)
    return out, loss
