"""fp64 restatements of the neural vocoder (deepvoice3_pytorch_b200/vocoder.py, csrc/vocoder.cu): the multi-resolution
STFT loss, its per-bin gradient, the STFT adjoint and the generator, built on oracle.audio_oracle.lws_stft."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.audio_oracle import lws_stft, lws_window, num_frames

FLOOR = 1e-7


def stft(x, N, R):
    """(F, N/2 + 1) complex128 STFT of a 1-D signal: sqrt-Hann window, N - R zeros each side, num_frames frames."""
    return lws_stft(np.asarray(x, np.float64), N, R)


def mag(X):
    return np.sqrt(np.maximum(X.real ** 2 + X.imag ** 2, FLOOR))


def clip_terms(X, Y):
    """(sc, mag) of one clip at one resolution: X the generated, Y the target spectrum."""
    a, b = mag(X), mag(Y)
    return np.linalg.norm(b - a) / np.linalg.norm(b), np.mean(np.abs(np.log(b) - np.log(a)))


def clip_losses(ys, xs, resolutions):
    """[(1/M) sum_m (sc + mag) of clip c] for lists of 1-D waveforms."""
    out = []
    for y, x in zip(ys, xs):
        out.append(np.mean([sum(clip_terms(stft(y, N, R), stft(x, N, R))) for N, R in resolutions]))
    return np.array(out)


def loss(ys, xs, resolutions):
    return float(np.mean(clip_losses(ys, xs, resolutions)))


def grad_spec(X, Y, w):
    """dL/dX (complex: d/dRe + i d/dIm) of w * (sc + mag) of one clip at one resolution."""
    p = X.real ** 2 + X.imag ** 2
    a, b = mag(X), mag(Y)
    num, den = np.linalg.norm(b - a), np.linalg.norm(b)
    da = ((a - b) / (num * den) if num > 0 else 0.0) + np.sign(np.log(a) - np.log(b)) / (a.size * a)
    return np.where(p > FLOOR, w * da * X / a, 0.0)


def stft_adjoint(G, N, R, n):
    """STFT^H G by its definition: dL/dy[t] = sum_f w(t - fR + N - R) sum_k Re(G[f, k] e^{2 pi i k (t - fR + N - R) / N})
    over the frames covering t, for t in [0, n)."""
    G = np.asarray(G, np.complex128)
    w = lws_window(N, R)
    k = np.arange(N // 2 + 1)
    j = np.arange(N)
    E = np.exp(2j * np.pi * np.outer(k, j) / N)
    frames = np.real(G @ E) * w[None]
    y = np.zeros((G.shape[0] - 1) * R + N)
    for f in range(G.shape[0]):
        y[f * R:f * R + N] += frames[f]
    pad = N - R
    return y[pad:pad + n]


def adjoint_spectrum(G, N):
    """The spectrum whose inverse STFT (irfft with 1/N, window, overlap-add) is STFT^H G: N G / 2 at interior bins,
    N Re(G) at bins 0 and N/2."""
    S = np.asarray(G, np.complex128) * (N / 2.0)
    S[:, 0] = N * G[:, 0].real
    S[:, -1] = N * G[:, -1].real
    return S


def istft(S, N, R, n):
    """irfft (1/N) * window, overlap-added, samples [N - R, N - R + n)."""
    frames = np.fft.irfft(S, n=N, axis=1) * lws_window(N, R)[None]
    y = np.zeros((S.shape[0] - 1) * R + N)
    for f in range(S.shape[0]):
        y[f * R:f * R + N] += frames[f]
    return y[N - R:N - R + n]


def grad_wave(ys, xs, resolutions, d_loss=1.0):
    """dL/dy of ``loss`` for each clip, through grad_spec and stft_adjoint."""
    M, B = len(resolutions), len(ys)
    out = []
    for y, x in zip(ys, xs):
        g = np.zeros(len(y))
        for N, R in resolutions:
            G = grad_spec(stft(y, N, R), stft(x, N, R), d_loss / (M * B))
            g += stft_adjoint(G, N, R, len(y))
        out.append(g)
    return out


def torch_loss(ys, xs, resolutions):
    """The same loss in torch fp64 (explicit framing + rfft), for autograd."""
    tot = 0.0
    for y, x in zip(ys, xs):
        c = 0.0
        for N, R in resolutions:
            w = torch.from_numpy(lws_window(N, R))
            nf = num_frames(len(y), N, R)
            L = (nf - 1) * R + N

            def spec(s):
                s = F.pad(s, (N - R, L - (N - R) - s.numel()))
                return torch.fft.rfft(s.unfold(0, N, R)[:nf] * w, dim=1)
            X, Y = spec(y), spec(x)
            a = torch.sqrt(torch.clamp_min(X.real ** 2 + X.imag ** 2, FLOOR))
            b = torch.sqrt(torch.clamp_min(Y.real ** 2 + Y.imag ** 2, FLOOR))
            c = c + torch.linalg.norm(b - a) / torch.linalg.norm(b) + torch.mean(torch.abs(torch.log(b) - torch.log(a)))
        tot = tot + c / len(resolutions)
    return tot / len(ys)


# ---- generator ----
def _wn(v, g):
    """weight_norm dim=0: g * v / ||v[r]|| over every dim but 0."""
    return g * v / v.pow(2).sum(tuple(range(1, v.dim())), keepdim=True).sqrt()


def vocoder_forward(sd, vocoder, cond):
    """fp64 restatement of NeuralVocoder.forward from its state_dict sd (fp64 leaves): cond (B, K, T) -> (B, T R)."""
    from deepvoice3_pytorch_b200 import conv as C, modules as Mo
    x = cond
    layers = list(vocoder.layers)
    i = 0
    while i < len(layers):
        f, p = layers[i], "layers.%d." % i
        if isinstance(f, C.Conv1d):
            w = _wn(sd[p + "weight_v"], sd[p + "weight_g"])
            d = f.dilation[0]
            x = F.conv1d(x, w, sd[p + "bias"], padding=(f.kernel_size[0] - 1) // 2 * d, dilation=d)
        elif isinstance(f, torch.nn.ReLU):
            x = torch.relu(x)
        elif isinstance(f, Mo.Conv1dGLU):
            c = f.conv
            w = _wn(sd[p + "conv.weight_v"], sd[p + "conv.weight_g"])
            d = c.dilation[0]
            h = F.conv1d(x, w, sd[p + "conv.bias"], padding=(c.kernel_size[0] - 1) // 2 * d, dilation=d)
            a, b = h.split(h.shape[1] // 2, dim=1)
            x = (a * torch.sigmoid(b) + x) * np.sqrt(0.5)
        elif isinstance(f, C.ConvTranspose1d):
            w = _wn(sd[p + "weight_v"], sd[p + "weight_g"])
            x = F.conv_transpose1d(x, w, sd[p + "bias"], stride=f.stride[0])
        else:
            raise TypeError(type(f))
        i += 1
    return x.reshape(x.shape[0], -1)
