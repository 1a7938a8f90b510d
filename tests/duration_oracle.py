"""fp64 numpy oracle of duration-guided synthesis (DESIGN.md section 2.22): the speaking-rate rule, the guided token
path, and the duration predictor's loss with its gradient, each restated from its definition with plain loops."""
import math

import numpy as np


def scale_durations(d, speed):
    """B_0 = 0, B_j = max(B_{j-1} + 1, round-half-even(C_j / speed)), d'_j = B_j - B_{j-1} (Python floats: fp64)."""
    out, prev, c = [], 0, 0
    for x in d:
        c += int(x)
        b = max(prev + 1, int(round(c / float(speed))))
        out.append(b - prev)
        prev = b
    return np.array(out, np.int64)


def path(durations, steps):
    """-> int64 (B, steps): token j of row b for the steps S_j <= t < S_{j+1}, the row's last token from its total on."""
    out = np.zeros((len(durations), steps), np.int64)
    for b, d in enumerate(durations):
        t = 0
        for j, n in enumerate(d):
            for _ in range(int(n)):
                if t < steps:
                    out[b, t] = j
                t += 1
        for u in range(t, steps):
            out[b, u] = len(d) - 1
    return out


def loss(y, d, lengths):
    """y (B, L) float, d (B, L) integer, lengths (B,) -> (loss, dloss/dy (B, L)) in fp64:
    mean_b (1/n_b) sum_{j < n_b} (y - log d)^2."""
    B, L = y.shape
    total, grad = 0.0, np.zeros((B, L))
    for b in range(B):
        n = int(lengths[b])
        s = 0.0
        for j in range(n):
            e = float(y[b, j]) - math.log(float(d[b, j]))
            s += e * e
            grad[b, j] = 2.0 * e / (n * B)
        total += s / n
    return total / B, grad
