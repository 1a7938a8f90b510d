"""TEST INFRASTRUCTURE ONLY.  fp64 numpy restatement of Local Weighted Sums phase recovery (Le Roux et al., DAFx 2010)
on the STFT frame of oracle/audio_oracle.py (N = 1024, hop R = 256, sqrt-Hann analysis = synthesis window, 513 bins),
the algorithm csrc/lws.cu implements (DESIGN.md section 7).

PARITY UNPINNED.  The reference calls ``lws.run_lws``; the ``lws`` package's source is absent, so what is restated here
is the published algorithm, not that package:

* weights  beta_q(d) = (1/N) sum_n w(n) w(n - qR) e^{-2 pi i d n / N},  q in [-3, 3], d in [-L, L], L = 5;
* local weighted sum  Y(m,k) = sum_{(q,d) != (0,0)} beta_q(d) (-i)^{k'q} X(m+q, k'),  k' = k - d  (hop = N/4 turns the
  frame shift into the factor (-i)^{k'q}); bins k' < 0 read conj X(m, -k'), bins k' > 512 read conj X(m, 1024 - k'),
  and the factor keeps the unreduced k';
* frames outside [0, T) contribute 0.  Exact away from the clip's ends; in the first and last 3 frames it ignores that
  the inverse STFT crops the 768 padding samples;
* update  X <- A Y / |Y|  (A + 0i where Y == 0); bins 0 and 512 are real: A sign(Re Y), +A where Re Y == 0;
* batch iteration: every bin reads the previous iterate (Jacobi);
* no-future initialisation: frames in order, each from the sum over its 3 past frames, then ``init_iters`` in-frame
  Jacobi passes that add the beta_0(d) terms of its own bins.
"""
import numpy as np

from oracle import audio_oracle as A

N, R, K, L, Q = 1024, 256, 513, 5, 3


def lws_weights(L=L, fsize=N, fshift=R):
    """-> (7, 2L+1) complex128, [q + 3, d + L] = beta_q(d)."""
    w = A.lws_window(fsize, fshift)
    n = np.arange(fsize)
    beta = np.zeros((2 * Q + 1, 2 * L + 1), dtype=np.complex128)
    for q in range(-Q, Q + 1):
        ok = (n - q * fshift >= 0) & (n - q * fshift < fsize)
        ww = np.where(ok, w * w[np.clip(n - q * fshift, 0, fsize - 1)], 0.0)
        for d in range(-L, L + 1):
            beta[q + Q, d + L] = np.sum(ww * np.exp(-2j * np.pi * d * n / fsize)) / fsize
    return beta


def _extend(X):
    """(T, 513) -> (T + 6, 523): frames -3..T+2 (zero outside the clip), bins -5..517 (conjugate mirror)."""
    T = X.shape[0]
    Xe = np.zeros((T + 2 * Q, K + 2 * L), dtype=np.complex128)
    Xe[Q:Q + T, L:L + K] = X
    for j in range(1, L + 1):
        Xe[Q:Q + T, L - j] = np.conj(X[:, j])                   # k' = -j
        Xe[Q:Q + T, L + K - 1 + j] = np.conj(X[:, K - 1 - j])   # k' = 512 + j -> 1024 - k' = 512 - j
    return Xe


def _phase(q, kp):
    return (-1j) ** ((kp * q) % 4)


def lws_local_sum(X, beta, qs=range(-Q, Q + 1)):
    """Y(m, k) summed over the frame offsets qs (all (q, d) except (0, 0))."""
    T = X.shape[0]
    Xe = _extend(np.asarray(X, dtype=np.complex128))
    k = np.arange(K)
    Y = np.zeros((T, K), dtype=np.complex128)
    for q in qs:
        for d in range(-L, L + 1):
            if q == 0 and d == 0:
                continue
            kp = k - d
            Y += beta[q + Q, d + L] * _phase(q, kp)[None, :] * Xe[Q + q:Q + q + T, kp + L]
    return Y


def _project(Amag, Y):
    a = np.abs(Y)
    X = np.where(a > 0, Amag * Y / np.where(a > 0, a, 1.0), Amag + 0j)
    for k in (0, K - 1):
        X[..., k] = np.where(Y[..., k].real >= 0, Amag[..., k], -Amag[..., k])
    return X


def lws_iterate(X, Amag, beta):
    """One Jacobi iteration over every bin."""
    return _project(np.asarray(Amag, dtype=np.float64), lws_local_sum(X, beta))


def lws_nofuture_frame(Am, past_frames, beta, init_iters=1):
    """Frame m of the no-future scan from its 3 past frames past_frames = (X(m-3), X(m-2), X(m-1)) (zeros before the
    clip) -> X(m, :)."""
    Am = np.asarray(Am, dtype=np.float64)
    ctx = np.concatenate([np.asarray(past_frames, dtype=np.complex128), np.zeros((1, K), np.complex128)])
    past = lws_local_sum(ctx, beta, qs=(-3, -2, -1))[Q]
    x = _project(Am, past)
    for _ in range(init_iters):
        own = np.zeros((2 * Q + 1, K), np.complex128)
        own[Q] = x
        x = _project(Am, past + lws_local_sum(own, beta, qs=(0,))[Q])
    return x


def lws_nofuture(Amag, beta, init_iters=1):
    Amag = np.asarray(Amag, dtype=np.float64)
    T = Amag.shape[0]
    X = np.zeros((T + Q, K), dtype=np.complex128)        # 3 leading zero frames
    for m in range(T):
        X[m + Q] = lws_nofuture_frame(Amag[m], X[m:m + Q], beta, init_iters)
    return X[Q:]


def lws_spectrum(Amag, n_iter=30, init_iters=1):
    beta = lws_weights()
    X = lws_nofuture(Amag, beta, init_iters)
    for _ in range(n_iter):
        X = lws_iterate(X, Amag, beta)
    return X


def lws(Amag, n_iter=30, init_iters=1):
    """Magnitude (T, 513) -> waveform (before de-emphasis), as audio.lws."""
    return A.lws_istft(lws_spectrum(Amag, n_iter, init_iters))


def spectral_convergence(Amag, x):
    """||A - |STFT(x)||| / ||A|| over the clip's frames."""
    Amag = np.asarray(Amag, dtype=np.float64)
    S = np.abs(A.lws_stft(np.asarray(x, dtype=np.float64)))[:Amag.shape[0]]
    return float(np.linalg.norm(Amag - S) / np.linalg.norm(Amag))
