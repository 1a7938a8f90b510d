"""fp64 numpy restatement of deepvoice3_pytorch_b200/alignment.py: monotonic alignment search with the same floor and
tie rule, a brute force over every monotone path, the per-step statistics and the attention-error counts."""
import itertools

import numpy as np

FLOOR = 1e-8


def log_probs(A):
    """lp = log(max(A, 1e-8)) in fp64; np.fmax takes a NaN cell to the floor, as fmaxf does."""
    return np.log(np.fmax(np.asarray(A, np.float64), FLOOR))


def mas_logp(lp):
    """MAS over log-probabilities lp (N, L) -> (durations int64 (L,), score, path (N,) token per step).  Q(0,0) = lp(0,0),
    Q(t,j) = lp(t,j) + max(Q(t-1,j), Q(t-1,j-1)); the backtrace from (N-1, L-1) stays on the token where the two
    predecessors tie.  N < L: zero durations, score -inf, no path (None)."""
    lp = np.asarray(lp, np.float64)
    N, L = lp.shape
    if N < L:
        return np.zeros(L, np.int64), -np.inf, None
    Q = np.full((N, L), -np.inf)
    Q[0, 0] = lp[0, 0]
    for t in range(1, N):
        for j in range(L):
            if j > t or L - 1 - j > N - 1 - t:
                continue
            stay = Q[t - 1, j]
            diag = Q[t - 1, j - 1] if j > 0 else -np.inf
            Q[t, j] = lp[t, j] + (diag if diag > stay else stay)
    path = np.zeros(N, np.int64)
    j = L - 1
    for t in range(N - 1, -1, -1):
        path[t] = j
        if t > 0 and j > 0 and (j >= t or Q[t - 1, j - 1] > Q[t - 1, j]):
            j -= 1
    return np.bincount(path, minlength=L).astype(np.int64), Q[N - 1, L - 1], path


def mas(A):
    """MAS of one alignment (N, L) (any float dtype) with the floor of ``log_probs``."""
    return mas_logp(log_probs(A))


def path_score(lp, path):
    """Sum of lp along a path (token per step), in increasing t, fp64."""
    s = 0.0
    for t, j in enumerate(path):
        s += lp[t, j]
    return s


def brute_force(lp):
    """Every monotone path from (0, 0) to (N-1, L-1) with unit token steps: -> (best score, path) where among equal
    scores the path whose token sequence read from the last step backwards is largest wins (the backtrace that stays on
    the token at ties picks that one)."""
    lp = np.asarray(lp, np.float64)
    N, L = lp.shape
    best = None
    for moves in itertools.combinations(range(1, N), L - 1):
        path = np.zeros(N, np.int64)
        for t in moves:
            path[t:] += 1
        key = (path_score(lp, path), tuple(path[::-1]))
        if best is None or key > best:
            best = key
    return best[0], np.array(best[1][::-1], np.int64)


def statistics(A):
    """Per-step argmax (lowest index at ties; NaN as -inf) and max of fp32 values, and fp64 coverage sum_t A[t, j]."""
    A = np.asarray(A)
    masked = np.where(np.isnan(A), -np.inf, A)
    return np.argmax(masked, axis=1), masked.max(axis=1), np.asarray(A, np.float64).sum(axis=0)


def attention_errors(argmax, maxv, coverage, max_decoder_steps, skip_coverage=0.5, repeat_margin=1):
    """One utterance's counts (alignment.attention_errors), restated with explicit loops."""
    p = [int(x) for x in argmax]
    N, L = len(p), len(coverage)
    run_max, m = [], -1
    for x in p:
        m = x if x > m else m
        run_max.append(m)
    repeats, inside = 0, False
    for t in range(1, N):
        back = p[t] < run_max[t - 1] - repeat_margin
        if back and not inside:
            repeats += 1
        inside = back
    dwell = best = 1
    for t in range(1, N):
        dwell = dwell + 1 if p[t] == p[t - 1] else 1
        best = max(best, dwell)
    last = run_max[-1]
    return {"focus_rate": float(np.mean(np.asarray(maxv, np.float64))),
            "skips": sum(1 for j in range(last + 1) if coverage[j] < skip_coverage),
            "unreached": L - 1 - last, "repeats": repeats, "max_dwell": best,
            "stop_failed": N == max_decoder_steps + 1, "finite": bool(np.isfinite(coverage).all())}


def planted(N, L, rng, durations=None, on=0.9, noise=0.05):
    """An (N, L) fp32 alignment with a planted monotone path: ``on`` on the path and uniform noise in [0, noise)
    elsewhere -> (A, durations).  durations: given, or random >= 1 summing to N."""
    if durations is None:
        cuts = np.sort(rng.choice(np.arange(1, N), L - 1, replace=False)) if L > 1 else np.array([], np.int64)
        durations = np.diff(np.concatenate([[0], cuts, [N]]))
    durations = np.asarray(durations, np.int64)
    A = (rng.random_sample((N, L)) * noise).astype(np.float32)
    path = np.repeat(np.arange(L), durations)
    A[np.arange(N), path] = on
    return A, durations
