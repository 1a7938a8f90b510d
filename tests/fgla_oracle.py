"""TEST INFRASTRUCTURE ONLY.  fp64 numpy restatement of fast Griffin-Lim (FGLA: Perraudin, Balazs & Sondergaard, "A fast
Griffin-Lim algorithm", WASPAA 2013), the algorithm of audio.griffin_lim_batch(momentum > 0), on the STFT, inverse STFT
and spectral convergence of tests/stft_geometry_oracle.py (any supported frame N = fft_size, R = hop_size).

From the zero-phase start x = istft(A), prev = 0, each iteration is
    X = stft(x);  C = X - beta prev;  prev = X;  spec = A C / |C| (A + 0i where C == 0);  x = istft(spec)
with beta = momentum / (1 + momentum), the form of librosa.griffinlim and torchaudio's GriffinLim.  At momentum 0 this
is stft_geometry_oracle.griffin_lim step for step."""
import numpy as np

from stft_geometry_oracle import A, spectral_convergence  # noqa: F401  (re-exported for the tests)


def beta_of(momentum):
    """The momentum coefficient of C = X - beta prev, in fp64 (audio.griffin_lim_batch rounds it to fp32 once)."""
    return momentum / (1.0 + momentum)


def project(mag, C):
    """mag C / |C|, and mag + 0i where C == 0 (the kernels' projection)."""
    a = np.abs(C)
    return np.where(a > 0, mag * C / np.maximum(a, 1e-300), mag + 0j)


def step(x, prev, mag, beta, N=1024, R=256):
    """One iteration from the waveform x and prev (T, K) -> (X, C, spec): X the new prev, spec the projection of C."""
    X = A.lws_stft(np.asarray(x, dtype=np.float64), N, R)[:mag.shape[0]]
    C = X - beta * prev
    return X, C, project(mag, C)


def fast_griffin_lim(mag, n_iter, N=1024, R=256, momentum=0.99, beta=None):
    """Magnitude (T, K) -> waveform (before de-emphasis) after n_iter FGLA iterations.  beta: use this coefficient
    instead of beta_of(momentum) (e.g. the fp32 value the kernels receive)."""
    mag = np.asarray(mag, dtype=np.float64)
    b = beta_of(momentum) if beta is None else float(beta)
    x = A.lws_istft(mag.astype(np.complex128), N, R)
    prev = np.zeros(mag.shape, dtype=np.complex128)
    for _ in range(n_iter):
        prev, _, spec = step(x, prev, mag, b, N, R)
        x = A.lws_istft(spec, N, R)
    return x


def sc_sweep(mag, ns, N=1024, R=256, momentum=0.99):
    """{n: spectral convergence of FGLA-n} for every n in ns, from one run of max(ns) iterations."""
    mag = np.asarray(mag, dtype=np.float64)
    b = beta_of(momentum)
    ns = sorted(set(int(n) for n in ns))
    x = A.lws_istft(mag.astype(np.complex128), N, R)
    prev = np.zeros(mag.shape, dtype=np.complex128)
    out = {}
    for i in range(ns[-1] + 1):
        if i in ns:
            out[i] = spectral_convergence(mag, x, N, R)
        if i < ns[-1]:
            prev, _, spec = step(x, prev, mag, b, N, R)
            x = A.lws_istft(spec, N, R)
    return out
