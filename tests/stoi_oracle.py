"""fp64 numpy restatement of the intelligibility measures of deepvoice3_pytorch_b200/intelligibility.py (DESIGN.md
section 2.20): STOI (Taal et al. 2011) and ESTOI (Jensen & Taal 2016) as the module docstring defines them, stage by
stage with the kernels' boundaries, so that a GPU test can feed each kernel the oracle's input to that stage:

    resample -> frame_energies -> keep_mask -> overlap_add -> envelopes -> segment_values -> pair_means
"""
import math

import numpy as np
from scipy.signal import resample_poly

FS = 10000
FRAME, NFFT, HOP = 256, 512, 128
BANDS, MIN_FREQ = 15, 150.0
N_SEG = 30
BETA_DB = -15.0
DYN_RANGE = 40.0
EPS = 2.220446049250313e-16
CLIP = 1.0 + 10.0 ** (-BETA_DB / 20.0)


def window():
    """w(n) = 0.5 - 0.5 cos(2 pi (n + 1) / 257), n < 256: np.hanning(258)[1:-1]."""
    n = np.arange(FRAME)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * (n + 1) / (FRAME + 1))


def resample(x, sr):
    """scipy's resample_poly of the fp64 clip from sr to 10 kHz."""
    g = math.gcd(int(sr), FS)
    return resample_poly(np.asarray(x, np.float64), FS // g, int(sr) // g)


def num_frames(L):
    """len(range(0, L - 256, 128))."""
    return len(range(0, int(L) - FRAME, HOP))


def frames(x):
    """(F, 256) windowed frames starting at 0, 128, ... while start < L - 256."""
    x = np.asarray(x, np.float64)
    F = num_frames(x.size)
    idx = np.arange(F)[:, None] * HOP + np.arange(FRAME)[None, :]
    return x[idx] * window()[None, :] if F else np.zeros((0, FRAME))


def frame_energies(x):
    """e_t = 20 log10(||w x_t||_2 + eps)."""
    f = frames(x)
    return 20.0 * np.log10(np.sqrt(np.sum(f * f, axis=1)) + EPS)


def keep_mask(e):
    """Frames within the 40 dB dynamic range of the loudest one: e > max(e) - 40."""
    e = np.asarray(e, np.float64)
    return e > e.max() - DYN_RANGE if e.size else np.zeros(0, bool)


def overlap_add(x, mask):
    """The kept windowed frames overlap-added at hop 128: (K - 1) 128 + 256 samples (none when K = 0)."""
    f = frames(x)[np.asarray(mask, bool)]
    K = f.shape[0]
    if K == 0:
        return np.zeros(0)
    y = np.zeros((K - 1) * HOP + FRAME)
    for k in range(K):
        y[k * HOP:k * HOP + FRAME] += f[k]
    return y


def band_edges():
    """pystoi's thirdoct: for band i the bins nearest 150 * 2^((2i - 1)/6) and 150 * 2^((2i + 1)/6) on the grid
    f_k = k * 10000 / 512 -> (lo, hi) int arrays; band i sums bins [lo, hi)."""
    f = np.arange(NFFT // 2 + 1) * FS / NFFT
    k = np.arange(BANDS, dtype=np.float64)
    lo = [int(np.argmin((f - MIN_FREQ * 2.0 ** ((2 * i - 1) / 6)) ** 2)) for i in k]
    hi = [int(np.argmin((f - MIN_FREQ * 2.0 ** ((2 * i + 1) / 6)) ** 2)) for i in k]
    return np.array(lo), np.array(hi)


def band_matrix():
    """(15, 257) 0/1 matrix of the bands."""
    lo, hi = band_edges()
    obm = np.zeros((BANDS, NFFT // 2 + 1))
    for i in range(BANDS):
        obm[i, lo[i]:hi[i]] = 1.0
    return obm


def envelopes(y):
    """(15, F) band envelopes of a (compacted) signal: X[i, t] = sqrt(sum over band i's bins of |rfft_512(w y_t)|^2)."""
    f = frames(y)
    if f.shape[0] == 0:
        return np.zeros((BANDS, 0))
    spec = np.fft.rfft(f, NFFT, axis=1)
    return np.sqrt(band_matrix() @ (np.abs(spec) ** 2).T)


def segment_values(X, Y, path=None):
    """Per segment s < J = L - 29 of the path (identity when None: L = X's frames) -> (J, 2): (sum over the 15 bands
    of the STOI correlation, ESTOI's d_seg).  X, Y: (15, F) envelopes; path: (L, 2) frame pairs (i of X, j of Y)."""
    X, Y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
    if path is None:
        path = np.stack([np.arange(X.shape[1])] * 2, 1)
    path = np.asarray(path)
    J = max(path.shape[0] - N_SEG + 1, 0)
    out = np.zeros((J, 2))
    for s in range(J):
        x = X[:, path[s:s + N_SEG, 0]]
        y = Y[:, path[s:s + N_SEG, 1]]
        alpha = np.sqrt(np.sum(x * x, 1, keepdims=True)) / (np.sqrt(np.sum(y * y, 1, keepdims=True)) + EPS)
        yp = np.minimum(alpha * y, CLIP * x)
        xc = x - x.mean(1, keepdims=True)
        yc = yp - yp.mean(1, keepdims=True)
        xn = xc / (np.sqrt(np.sum(xc * xc, 1, keepdims=True)) + EPS)
        yn = yc / (np.sqrt(np.sum(yc * yc, 1, keepdims=True)) + EPS)
        out[s, 0] = np.sum(xn * yn)
        out[s, 1] = np.sum(_row_col(x) * _row_col(y)) / N_SEG
    return out


def _row_col(m):
    m = m - m.mean(1, keepdims=True)
    m = m / (np.sqrt(np.sum(m * m, 1, keepdims=True)) + EPS)
    m = m - m.mean(0, keepdims=True)
    return m / (np.sqrt(np.sum(m * m, 0, keepdims=True)) + EPS)


def pair_means(seg):
    """(J, 2) segment values -> (stoi, estoi): the means over the J * 15 (segment, band) pairs and over the J segments;
    NaN when J = 0."""
    J = seg.shape[0]
    if J == 0:
        return float("nan"), float("nan")
    return float(seg[:, 0].sum() / (BANDS * J)), float(seg[:, 1].sum() / J)


def stoi(clean, processed, sr=FS):
    """Aligned STOI / ESTOI of two equal-length clips at sr -> dict(stoi, estoi, segments, kept_frames)."""
    x, y = resample(clean, sr), resample(processed, sr)
    assert x.size == y.size
    mask = keep_mask(frame_energies(x))
    X, Y = envelopes(overlap_add(x, mask)), envelopes(overlap_add(y, mask))
    seg = segment_values(X, Y)
    d, e = pair_means(seg)
    return {"stoi": d, "estoi": e, "segments": seg.shape[0], "kept_frames": int(mask.sum())}
