"""fp64 restatement of the YIN F0 tracker of deepvoice3_pytorch_b200/pitch.py (DESIGN.md section 2.18) from its
definition, the fp32 error bounds the GPU tests compare it with, the DTW warping path by a full cost matrix and its
backtrace, and a brute force over every monotone path for small sizes."""
import math

import numpy as np

U = 2.0 ** -24                    # fp32 unit roundoff


def num_frames(n, N=1024, R=256):
    """Frames of the padded STFT (oracle/audio_oracle.py): ceil((n + 2 (N - R) - N) / R) + 1."""
    return int(math.ceil((n + 2 * (N - R) - N) / float(R))) + 1


def taus(sr=22050, f0_min=60.0, f0_max=500.0):
    return int(math.floor(sr / f0_max)), int(math.ceil(sr / f0_min))


def spans(x, N=1024, R=256, tau_max=368):
    """(F, N + tau_max) fp64: the samples x[a_t + m] each frame reads, a_t = t R + R - N/2 - floor((N + tau_max)/2),
    zero outside the clip."""
    x = np.asarray(x, np.float64)
    F = num_frames(x.size, N, R)
    a = np.arange(F) * R + R - N // 2 - (N + tau_max) // 2
    idx = a[:, None] + np.arange(N + tau_max)[None, :]
    ok = (idx >= 0) & (idx < x.size)
    return np.where(ok, x[np.clip(idx, 0, max(x.size - 1, 0))], 0.0)


def difference(sp, W, tau_max):
    """(F, tau_max) d(tau) = sum_{j < W} (x_j - x_{j + tau})^2, tau = 1 .. tau_max, evaluated directly."""
    d = np.empty((sp.shape[0], tau_max))
    for tau in range(1, tau_max + 1):
        diff = sp[:, :W] - sp[:, tau:tau + W]
        d[:, tau - 1] = np.einsum("fj,fj->f", diff, diff)
    return d


def cmndf(d):
    """d'(tau) = tau d(tau) / sum_{j <= tau} d(j); 1 where the sum is 0."""
    S = np.cumsum(d, axis=1)
    tau = np.arange(1, d.shape[1] + 1)[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(S == 0, 1.0, tau * d / np.where(S == 0, 1.0, S))


def decide(dp, tau_min, tau_max, threshold):
    """One frame's d' (index tau - 1) -> (voiced, tau*): the absolute threshold and the walk, else the argmin."""
    for tau in range(tau_min, tau_max + 1):
        if dp[tau - 1] < threshold:
            while tau < tau_max and dp[tau] < dp[tau - 1]:
                tau += 1
            return True, tau
    rng = dp[tau_min - 1:tau_max]
    return False, tau_min + int(np.argmin(rng))


def parabolic(dp, tau, tau_min, tau_max):
    """delta of the parabola through d'(tau - 1, tau, tau + 1), clamped to [-1, 1]; 0 without both neighbours or with a
    curvature <= 0."""
    if tau - 1 < tau_min or tau + 1 > tau_max:
        return 0.0
    y0, y1, y2 = dp[tau - 2], dp[tau - 1], dp[tau]
    c = (y0 + y2) - 2.0 * y1
    if not c > 0:
        return 0.0
    return min(1.0, max(-1.0, (y0 - y2) / (2.0 * c)))


def yin(x, sr=22050, N=1024, R=256, f0_min=60.0, f0_max=500.0, threshold=0.1, silence_db=-50.0):
    """-> dict of per-frame arrays: "d", "dp" (F, tau_max), "voiced", "tau" (tau*), "delta", "f0" (gated),
    "f0_raw" (before the gate), "aperiodicity", "energy", and "tau_min", "tau_max", "gate"."""
    tau_min, tau_max = taus(sr, f0_min, f0_max)
    sp = spans(x, N, R, tau_max)
    d = difference(sp, N, tau_max)
    dp = cmndf(d)
    F = sp.shape[0]
    voiced = np.zeros(F, bool)
    tau_s = np.zeros(F, np.int64)
    delta = np.zeros(F)
    f0 = np.zeros(F)
    for t in range(F):
        voiced[t], tau_s[t] = decide(dp[t], tau_min, tau_max, threshold)
        if voiced[t]:
            delta[t] = parabolic(dp[t], tau_s[t], tau_min, tau_max)
            f0[t] = sr / (tau_s[t] + delta[t])
    energy = np.einsum("fj,fj->f", sp[:, :N], sp[:, :N])
    gate = 10.0 ** (silence_db / 10.0)
    gated = np.where(energy < gate * energy.max(), 0.0, f0)
    return {"d": d, "dp": dp, "voiced": voiced, "tau": tau_s, "delta": delta, "f0": gated, "f0_raw": f0,
            "aperiodicity": dp[np.arange(F), tau_s - 1], "energy": energy, "tau_min": tau_min, "tau_max": tau_max,
            "gate": gate}


# ---- fp32 bounds ----------------------------------------------------------------------------------------------------
def d_bound(d, W):
    """|d_fp32 - d| <= (W + 3) u d: W nonnegative terms, each a rounded difference squared by an fma."""
    return (W + 3) * U * d


def dp_bound(dp, W):
    """|d'_fp32 - d'| <= (2 W + tau + 10) u d': d, the sequential prefix S and the product and quotient."""
    tau = np.arange(1, dp.shape[-1] + 1)
    return (2 * W + tau + 10) * U * dp


def stable(dp, e, tau_min, tau_max, threshold):
    """Is the decision (voicing and tau*) of a frame the same for every d' within +-e of this one?  The margins to the
    threshold before and at the first crossing, along the walk and at its stop, or (unvoiced) to the runner-up of the
    argmin, must all exceed the bound."""
    lo, hi = dp - e, dp + e
    voiced, tau = decide(dp, tau_min, tau_max, threshold)
    if voiced:
        first = next(t for t in range(tau_min, tau_max + 1) if dp[t - 1] < threshold)
        if not all(lo[t - 1] >= threshold for t in range(tau_min, first)) or not hi[first - 1] < threshold:
            return False
        for t in range(first, tau):
            if not hi[t] < lo[t - 1]:
                return False
        return tau == tau_max or lo[tau] >= hi[tau - 1]
    if not all(lo[t - 1] >= threshold for t in range(tau_min, tau_max + 1)):
        return False
    others = np.delete(lo[tau_min - 1:tau_max], tau - tau_min)
    return others.size == 0 or hi[tau - 1] < others.min()


def f0_bound(dp, e, tau, tau_min, tau_max, sr):
    """Bound on |f0_fp32 - f0| of a voiced frame whose decision is stable, or None where the interpolation's branch
    (neighbours, curvature sign, clamp) could differ."""
    f0 = sr / tau
    if tau - 1 < tau_min or tau + 1 > tau_max:
        return 2 * U * f0
    y0, y1, y2 = dp[tau - 2], dp[tau - 1], dp[tau]
    e0, e1, e2 = e[tau - 2], e[tau - 1], e[tau]
    c = (y0 + y2) - 2.0 * y1
    ec = e0 + 2 * e1 + e2 + 4 * U * (abs(y0 + y2) + abs(c))
    if abs(c) <= ec:
        return None
    if c < 0:
        return 2 * U * f0
    num = y0 - y2
    en = e0 + e2 + U * abs(num)
    delta = num / (2 * c)
    ed = (en + abs(delta) * 2 * ec) / (2 * (c - ec)) + 2 * U * abs(delta)
    if abs(abs(delta) - 1.0) <= ed:
        return None
    if abs(delta) > 1.0:
        return 2 * U * f0 * 2
    den = tau + delta
    return sr * ed / (den * (den - ed)) + 3 * U * sr / den


# ---- DTW warping path -------------------------------------------------------------------------------------------------
def dtw_path(d):
    """(N, M) frame distances -> (D(N, M), path (L, 2) of 0-based (i, j)): the full cost matrix with the tie rule of
    tests/mcd_oracle.py (diagonal, then (i-1, j), then (i, j-1)) and its backtrace.  On row 1 the walk moves left and on
    column 1 up: the codes a finite D gives there, and a walk that stays in the grid where D is NaN (every comparison
    fails, so the stored code is the diagonal)."""
    N, M = d.shape
    D = np.full((N + 1, M + 1), np.inf)
    code = np.zeros((N + 1, M + 1), np.int64)
    D[0, 0] = 0.0
    for i in range(1, N + 1):
        for j in range(1, M + 1):
            best, c = D[i - 1, j - 1], 0
            if D[i - 1, j] < best:
                best, c = D[i - 1, j], 1
            if D[i, j - 1] < best:
                best, c = D[i, j - 1], 2
            D[i, j] = d[i - 1, j - 1] + best
            code[i, j] = c
    i, j, path = N, M, []
    while True:
        path.append((i - 1, j - 1))
        if (i, j) == (1, 1):
            break
        c = 2 if i == 1 else 1 if j == 1 else code[i, j]        # row 1 moves left, column 1 up, whatever D says
        i, j = (i - 1, j - 1) if c == 0 else (i - 1, j) if c == 1 else (i, j - 1)
    return float(D[N, M]), np.array(path[::-1], np.int64)


def path_brute(d):
    """Every monotone path from (0, 0) to (N-1, M-1): the least cost and, among the paths of least cost, the one whose
    moves read backwards from the end are lexicographically first with diagonal < (i-1, j) < (i, j-1) -> (cost, path)."""
    N, M = d.shape
    best = None

    def walk(i, j, cost, moves, cells):
        nonlocal best
        if (i, j) == (N - 1, M - 1):
            key = (cost, tuple(reversed(moves)))
            if best is None or key < best[0]:
                best = (key, list(cells))
            return
        for rank, (di, dj) in ((0, (1, 1)), (1, (1, 0)), (2, (0, 1))):
            if i + di < N and j + dj < M:
                walk(i + di, j + dj, cost + d[i + di, j + dj], moves + [rank], cells + [(i + di, j + dj)])

    walk(0, 0, d[0, 0], [], [(0, 0)])
    return best[0][0], np.array(best[1], np.int64)
