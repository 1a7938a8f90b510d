"""TEST INFRASTRUCTURE ONLY.  fp64 numpy restatements for any STFT frame (N = fft_size, R = hop_size, Q = N / R an
integer in [2, 8], K = N / 2 + 1 bins): the reference front-end (linear / mel), Griffin-Lim, the inverse spectrogram and
Local Weighted Sums phase recovery -- the algorithms csrc/stft_any.cu and csrc/lws_any.cu implement.  At N = 1024,
R = 256 they reduce to oracle/audio_oracle.py and tests/lws_oracle.py (checked on the CPU in
tests/test_stft_geometry_host.py).  Parity with the reference's lws package is unpinned, as for those oracles.

LWS for general Q: weights beta_q(d) for |q| <= Q - 1, |d| <= L = 5; the frame shift gives the phase factor
e^{-2 pi i k'q/Q} with k' = k - d unreduced; bins k' < 0 read conj X(m, -k'), bins k' > N/2 read conj X(m, N - k');
frames outside [0, T) contribute 0; bins 0 and N/2 are projected onto the real axis."""
import numpy as np

from oracle import audio_oracle as A

L = 5


def hp(sr, N, R, num_mels=80, fmin=125, fmax=7600):
    return dict(sample_rate=sr, fft_size=N, hop_size=R, num_mels=num_mels, fmin=fmin, fmax=fmax, preemphasis=0.97,
                min_level_db=-100, ref_level_db=20)


def process_utterance(wav, h):
    """(T, K) linear and (T, num_mels) mel, float64, as audio_oracle.process_utterance for the frame of h."""
    D = np.abs(A.lws_stft(A.preemphasis(wav, h["preemphasis"]), h["fft_size"], h["hop_size"]))
    lin = A._normalize(A._amp_to_db(D, h["min_level_db"]) - h["ref_level_db"], h["min_level_db"])
    basis = A.mel_basis(h["sample_rate"], h["fft_size"], h["num_mels"], h["fmin"], h["fmax"]).astype(np.float64)
    mel = A._normalize(A._amp_to_db(D @ basis.T, h["min_level_db"]) - h["ref_level_db"], h["min_level_db"])
    return lin, mel


def griffin_lim(mag, n_iter, N, R):
    mag = np.asarray(mag, dtype=np.float64)
    x = A.lws_istft(mag.astype(np.complex128), N, R)
    for _ in range(n_iter):
        X = A.lws_stft(x, N, R)[:mag.shape[0]]
        a = np.abs(X)
        X = np.where(a > 0, mag * X / np.maximum(a, 1e-300), mag)
        x = A.lws_istft(X, N, R)
    return x


def lws_weights(N, R):
    """-> (2Q - 1, 2L + 1) complex128, [q + Q - 1, d + L] = beta_q(d)."""
    Q = N // R
    w = A.lws_window(N, R)
    n = np.arange(N)
    beta = np.zeros((2 * Q - 1, 2 * L + 1), dtype=np.complex128)
    for q in range(-(Q - 1), Q):
        ok = (n - q * R >= 0) & (n - q * R < N)
        ww = np.where(ok, w * w[np.clip(n - q * R, 0, N - 1)], 0.0)
        for d in range(-L, L + 1):
            beta[q + Q - 1, d + L] = np.sum(ww * np.exp(-2j * np.pi * d * n / N)) / N
    return beta


def _extend(X, H):
    """(T, K) -> (T + 2H, K + 2L): frames -H..T+H-1 (zero outside the clip), bins -L..K-1+L (conjugate mirror)."""
    T, K = X.shape
    Xe = np.zeros((T + 2 * H, K + 2 * L), dtype=np.complex128)
    Xe[H:H + T, L:L + K] = X
    for j in range(1, L + 1):
        Xe[H:H + T, L - j] = np.conj(X[:, j])
        Xe[H:H + T, L + K - 1 + j] = np.conj(X[:, K - 1 - j])
    return Xe


def _phase(q, kp, Q):
    return np.exp(-2j * np.pi * ((kp * q) % Q) / Q)


def lws_local_sum(X, beta, Q, qs=None):
    T, K = X.shape
    H = Q - 1
    Xe = _extend(np.asarray(X, dtype=np.complex128), H)
    k = np.arange(K)
    Y = np.zeros((T, K), dtype=np.complex128)
    for q in (range(-H, H + 1) if qs is None else qs):
        for d in range(-L, L + 1):
            if q == 0 and d == 0:
                continue
            kp = k - d
            Y += beta[q + H, d + L] * _phase(q, kp, Q)[None, :] * Xe[H + q:H + q + T, kp + L]
    return Y


def _project(Amag, Y):
    a = np.abs(Y)
    X = np.where(a > 0, Amag * Y / np.where(a > 0, a, 1.0), Amag + 0j)
    K = Y.shape[-1]
    for k in (0, K - 1):
        X[..., k] = np.where(Y[..., k].real >= 0, Amag[..., k], -Amag[..., k])
    return X


def lws_iterate(X, Amag, beta, Q):
    return _project(np.asarray(Amag, dtype=np.float64), lws_local_sum(X, beta, Q))


def lws_nofuture_frame(Am, past_frames, beta, Q, init_iters=1):
    """Frame m from its Q - 1 past frames (X(m-Q+1) .. X(m-1), zeros before the clip) -> X(m, :)."""
    H = Q - 1
    Am = np.asarray(Am, dtype=np.float64)
    K = Am.shape[0]
    ctx = np.concatenate([np.asarray(past_frames, dtype=np.complex128).reshape(H, K), np.zeros((1, K), np.complex128)])
    past = lws_local_sum(ctx, beta, Q, qs=range(-H, 0))[H]
    x = _project(Am, past)
    for _ in range(init_iters):
        own = np.zeros((1, K), np.complex128)
        own[0] = x
        x = _project(Am, past + lws_local_sum(own, beta, Q, qs=(0,))[0])
    return x


def lws_nofuture(Amag, beta, Q, init_iters=1):
    Amag = np.asarray(Amag, dtype=np.float64)
    T, K = Amag.shape
    H = Q - 1
    X = np.zeros((T + H, K), dtype=np.complex128)
    for m in range(T):
        X[m + H] = lws_nofuture_frame(Amag[m], X[m:m + H], beta, Q, init_iters)
    return X[H:]


def lws(Amag, N, R, n_iter=30, init_iters=1):
    """Magnitude (T, K) -> waveform (before de-emphasis), as audio.lws at the frame (N, R)."""
    Q = N // R
    beta = lws_weights(N, R)
    X = lws_nofuture(Amag, beta, Q, init_iters)
    for _ in range(n_iter):
        X = lws_iterate(X, Amag, beta, Q)
    return A.lws_istft(X, N, R)


def spectral_convergence(Amag, x, N, R):
    Amag = np.asarray(Amag, dtype=np.float64)
    S = np.abs(A.lws_stft(np.asarray(x, dtype=np.float64), N, R))[:Amag.shape[0]]
    return float(np.linalg.norm(Amag - S) / np.linalg.norm(Amag))
