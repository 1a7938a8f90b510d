"""fp64 restatement of the speaker verifier (deepvoice3_pytorch_b200/speaker_verifier.py, csrc/spk_ver.cu).

embed_* and score_* spell out the forward and the hand-derived backward the kernels implement (the host tests check the
backward against torch autograd with gradcheck); ``verifier_forward`` is the whole verifier as plain torch fp64
autograd code over a state_dict (weight-normed convs, GLU blocks, pool, embeddings, scores, balanced loss).
"""
import math

import torch
import torch.nn.functional as F


def embed_fwd(h, counts, w, c):
    """h (B, N, C), counts (B,) -> (out (B, D) = W mean_{i < n_b} h_{b,i} + c, hbar (B, C))."""
    hbar = torch.stack([h[b, :int(n)].mean(0) for b, n in enumerate(counts)])
    return hbar @ w.T + c, hbar


def embed_bwd(d_out, hbar, counts, w, N):
    """-> (d_h (B, N, C) with rows >= counts[b] 0, d_w, d_c)."""
    B, C = hbar.shape
    d_h = torch.zeros(B, N, C, dtype=d_out.dtype)
    for b, n in enumerate(counts):
        d_h[b, :int(n)] = (d_out[b] @ w) / int(n)
    return d_h, d_out.T @ hbar, d_out.sum(0)


def _same(ids_e, ids_t):
    return torch.as_tensor(ids_e)[:, None] == torch.as_tensor(ids_t)[None, :]


def score_fwd(x, y, S, b, ids_e=None, ids_t=None):
    """-> (scores (B_e, B_t), balanced BCE loss or None)."""
    qx = torch.einsum("ei,ij,ej->e", x, S, x)
    qy = torch.einsum("ti,ij,tj->t", y, S, y)
    L = x @ y.T - qx[:, None] - qy[None, :] + b
    if ids_e is None:
        return L, None
    same = _same(ids_e, ids_t)
    return L, 0.5 * F.softplus(-L[same]).mean() + 0.5 * F.softplus(L[~same]).mean()


def score_bwd(x, y, S, scores, ids_e=None, ids_t=None, d_scores=None, d_loss=None):
    """The kernels' backward, by hand: -> (dx, dy, dS, db)."""
    G = torch.zeros_like(scores) if d_scores is None else d_scores.clone()
    if ids_e is not None and d_loss is not None:
        same = _same(ids_e, ids_t)
        n_same, n_diff = int(same.sum()), int((~same).sum())
        dl = torch.where(same, -torch.sigmoid(-scores) / (2 * max(n_same, 1)),
                         torch.sigmoid(scores) / (2 * max(n_diff, 1)))
        G = G + d_loss * dl
    gx, gy = G.sum(1), G.sum(0)
    SS = S + S.T
    dx = G @ y - gx[:, None] * (x @ SS)
    dy = G.T @ x - gy[:, None] * (y @ SS)
    dS = -(x.T * gx) @ x - (y.T * gy) @ y
    return dx, dy, dS, G.sum().reshape(1)


def _wn(sd, prefix):
    v, gw = sd[prefix + "weight_v"], sd[prefix + "weight_g"]
    return gw * v / v.pow(2).sum(tuple(range(1, v.dim())), keepdim=True).sqrt()


def pooled(sd, mels, kernel_size, n_conv):
    """The trunk: mels (B, N, T, M) -> (B, N, C) frame means (fixed-length samples)."""
    B, N, T, M = mels.shape
    x = mels.reshape(B * N, T, M).transpose(1, 2)
    for i in (0, 2):
        x = torch.relu(F.conv1d(x, _wn(sd, "spectral.%d." % i), sd["spectral.%d.bias" % i]))
    for i in range(n_conv):
        pre = "temporal.%d.conv." % i
        y = F.conv1d(x, _wn(sd, pre), sd[pre + "bias"], padding=(kernel_size - 1) // 2)
        a, gate = y.split(y.shape[1] // 2, dim=1)
        x = (a * torch.sigmoid(gate) + x) * math.sqrt(0.5)
    return x.mean(-1).view(B, N, -1)


def verifier_forward(sd, mels, ids, kernel_size=5, n_conv=2):
    """The whole verifier over a training batch (row b: N - 1 enrollment samples, then the test sample) in torch fp64
    autograd -> (scores (B, B), loss)."""
    h = pooled(sd, mels, kernel_size, n_conv)
    x = h[:, :-1].mean(1) @ sd["w"].T + sd["c"]
    y = h[:, -1] @ sd["w"].T + sd["c"]
    return score_fwd(x, y, sd["S"], sd["b"], ids, ids)
