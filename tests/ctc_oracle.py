"""fp64 numpy restatement of csrc/ctc.cu: the CTC loss and its gradient with respect to the logits, greedy CTC
decoding, and the Levenshtein distance with the S/D/I counts of the tie rule (diagonal, then deletion, then insertion).
Also brute force over every alignment and every edit path, for short inputs."""
import itertools

import numpy as np


def log_softmax(z):
    """z (V, T) -> fp64 log-softmax over V."""
    z = np.asarray(z, np.float64)
    m = z.max(0, keepdims=True)
    return z - (m + np.log(np.exp(z - m).sum(0, keepdims=True)))


def _lse(*xs):
    m = max(xs)
    if m == -np.inf:
        return m
    return m + np.log(sum(np.exp(x - m) for x in xs))


def feasible(T, labels):
    labels = list(labels)
    reps = sum(1 for a, b in zip(labels[:-1], labels[1:]) if a == b)
    return T >= len(labels) + reps


def ctc(z, labels):
    """z (V, T) logits of one row, labels (L,) in [1, V) -> (nll = -log p, dz (V, T) of nll, infeasible).  An
    infeasible row gives (0, 0, True) as torch's zero_infinity does."""
    lp = log_softmax(z)
    V, T = lp.shape
    ext = [0]
    for l in labels:
        ext += [int(l), 0]
    S = len(ext)
    if not feasible(T, labels):
        return 0.0, np.zeros((V, T)), True
    NEG = -np.inf
    alpha = np.full((T, S), NEG)
    alpha[0, 0] = lp[0, 0]
    if S > 1:
        alpha[0, 1] = lp[ext[1], 0]
    for t in range(1, T):
        for s in range(S):
            a = alpha[t - 1, s]
            b = alpha[t - 1, s - 1] if s >= 1 else NEG
            c = alpha[t - 1, s - 2] if s >= 2 and ext[s] != 0 and ext[s] != ext[s - 2] else NEG
            alpha[t, s] = lp[ext[s], t] + _lse(a, b, c)
    beta = np.full((T, S), NEG)                  # suffix after t, emissions of t excluded
    beta[T - 1, S - 1] = 0.0
    if S > 1:
        beta[T - 1, S - 2] = 0.0
    for t in range(T - 2, -1, -1):
        for s in range(S):
            q = lambda u: beta[t + 1, u] + lp[ext[u], t + 1]
            a = q(s)
            b = q(s + 1) if s + 1 < S else NEG
            c = q(s + 2) if s + 2 < S and ext[s + 2] != 0 and ext[s + 2] != ext[s] else NEG
            beta[t, s] = _lse(a, b, c)
    logp = _lse(alpha[T - 1, S - 1], alpha[T - 1, S - 2]) if S > 1 else alpha[T - 1, 0]
    occ = np.zeros((V, T))
    gam = np.exp(alpha + beta - logp)
    for s in range(S):
        occ[ext[s]] += gam[:, s]
    return -logp, np.exp(lp) - occ, False


def ctc_batch(z, frames, targets, target_lengths):
    """z (B, V, T) -> (per-row nll (B,), mean loss over rows of nll / max(L, 1), dz (B, V, T) of that mean,
    infeasible (B,) bool)."""
    z = np.asarray(z, np.float64)
    B, V, T = z.shape
    nll, dz, inf = np.zeros(B), np.zeros((B, V, T)), np.zeros(B, bool)
    for b in range(B):
        Tb, Lb = int(frames[b]), int(target_lengths[b])
        n, g, f = ctc(z[b, :, :Tb], np.asarray(targets[b])[:Lb])
        nll[b], inf[b] = n, f
        dz[b, :, :Tb] = g / max(Lb, 1) / B
    return nll, float(np.mean(nll / np.maximum(np.asarray(target_lengths, np.float64), 1))), dz, inf


def brute_force_nll(z, labels):
    """-log of the sum over every frame labelling that collapses to ``labels`` (V**T paths: small inputs only)."""
    lp = log_softmax(z)
    V, T = lp.shape
    tot = -np.inf
    for path in itertools.product(range(V), repeat=T):
        if collapse(path) == list(labels):
            tot = _lse(tot, sum(lp[v, t] for t, v in enumerate(path)))
    return -tot


def collapse(path):
    out, prev = [], None
    for v in path:
        if v != prev and v != 0:
            out.append(int(v))
        prev = v
    return out


def greedy(z, frames):
    """z (B, V, T) -> list of hypotheses: per-frame argmax (first of the largest), collapsed, blanks dropped."""
    return [np.array(collapse(np.argmax(np.asarray(z[b])[:, :int(frames[b])], axis=0)), np.int64)
            for b in range(len(frames))]


def edit(hyp, ref):
    """-> (distance, substitutions, deletions, insertions) along the path that prefers the diagonal, then a deletion
    (i - 1, j), then an insertion (i, j - 1) among predecessors of equal cost; rows i index ref, columns j hyp."""
    N, M = len(ref), len(hyp)
    D = np.zeros((N + 1, M + 1), np.int64)
    C = np.zeros((N + 1, M + 1, 2), np.int64)              # (S, D) carried
    for i in range(1, N + 1):
        D[i, 0] = i
        C[i, 0] = (0, i)
    for j in range(1, M + 1):
        D[0, j] = j
    for i in range(1, N + 1):
        for j in range(1, M + 1):
            mis = int(ref[i - 1] != hyp[j - 1])
            best, c = D[i - 1, j - 1] + mis, C[i - 1, j - 1] + (mis, 0)
            if D[i - 1, j] + 1 < best:
                best, c = D[i - 1, j] + 1, C[i - 1, j] + (0, 1)
            if D[i, j - 1] + 1 < best:
                best, c = D[i, j - 1] + 1, C[i, j - 1]
            D[i, j], C[i, j] = best, c
    d, (s, dl) = int(D[N, M]), C[N, M]
    return d, int(s), int(dl), d - int(s) - int(dl)


def brute_force_distance(hyp, ref):
    """The edit distance by enumerating every edit script (short strings only): the minimum over alignments."""
    hyp, ref = list(hyp), list(ref)

    def go(i, j):
        if i == len(ref):
            return len(hyp) - j
        if j == len(hyp):
            return len(ref) - i
        return min(go(i + 1, j + 1) + (ref[i] != hyp[j]), go(i + 1, j) + 1, go(i, j + 1) + 1)
    return go(0, 0)
