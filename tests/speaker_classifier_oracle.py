"""fp64 restatement of the speaker classifier (deepvoice3_pytorch_b200/speaker_classifier.py, csrc/spk_cls.cu).

head_fwd / head_bwd spell out the forward and the hand-derived backward the kernels implement (the host tests check the
backward against torch autograd with gradcheck); ``classifier_forward`` is the whole classifier as plain torch fp64
autograd code over a state_dict (the verifier oracle's trunk, then the head and its loss).
"""
import torch

from speaker_verifier_oracle import pooled


def head_fwd(h, w, c, labels=None):
    """h (R, C), w (K, C), c (K,) -> (logits (R, K), lse (R,), mean cross-entropy or None).  A label outside [0, K)
    adds 0 to the loss (the mean is still over all R rows)."""
    z = h @ w.T + c
    lse = torch.logsumexp(z, 1)
    if labels is None:
        return z, lse, None
    lab = torch.as_tensor(labels)
    ok = (lab >= 0) & (lab < z.shape[1])
    picked = z[torch.arange(z.shape[0]), lab.clamp(0, z.shape[1] - 1)]
    return z, lse, torch.where(ok, lse - picked, torch.zeros_like(lse)).mean()


def grad_logits(z, lse, labels=None, d_logits=None, d_loss=None):
    """G = d_logits + d_loss / R * (softmax - onehot), the onehot only for labels inside [0, K)."""
    G = torch.zeros_like(z) if d_logits is None else d_logits.clone()
    if labels is not None and d_loss is not None:
        R, K = z.shape
        lab = torch.as_tensor(labels)
        onehot = (torch.arange(K)[None, :] == lab[:, None]).to(z.dtype)
        G = G + d_loss / R * (torch.exp(z - lse[:, None]) - onehot)
    return G


def head_bwd(h, w, z, lse, labels=None, d_logits=None, d_loss=None):
    """The kernels' backward, by hand: -> (d_h, d_w, d_c)."""
    G = grad_logits(z, lse, labels, d_logits, d_loss)
    return G @ w, G.T @ h, G.sum(0)


def classifier_forward(sd, mels, ids, kernel_size=5, n_conv=2):
    """The whole classifier over a training batch (row b: N utterances of class ids[b]) in torch fp64 autograd ->
    (logits (B*N, K), loss)."""
    B, N = mels.shape[:2]
    h = pooled(sd, mels, kernel_size, n_conv).reshape(B * N, -1)
    z, _, loss = head_fwd(h, sd["w"], sd["c"], torch.as_tensor(ids).repeat_interleave(N))
    return z, loss
