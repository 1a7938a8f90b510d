"""fp64 restatement of MCD-DTW (deepvoice3_pytorch_b200/mcd.py, DESIGN.md section 2.17): mel cepstra from the
definition (denormalise, natural-log amplitude, orthonormal DCT-II, c_1..c_K), the DTW recursion with its tie rule
vectorised over anti-diagonals, and a brute force over every monotone path for small sizes."""
import math

import numpy as np
from scipy.fft import dct

MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)


def log_amplitude(S, min_level_db=-100.0, ref_level_db=20.0):
    """Normalised mel rows -> natural-log amplitude: (S (-min_level_db) + min_level_db + ref_level_db) ln10 / 20."""
    S = np.asarray(S, np.float64)
    return (S * -min_level_db + min_level_db + ref_level_db) * math.log(10.0) / 20.0


def cepstra(S, K, min_level_db=-100.0, ref_level_db=20.0):
    """(T, M) normalised mels -> (T, K): c_1..c_K of DCT-II_ortho(ln A), the definition."""
    return dct(log_amplitude(S, min_level_db, ref_level_db), type=2, norm="ortho", axis=-1)[:, 1:K + 1]


def distances(ca, cb):
    """(N, K), (M, K) -> (N, M) fp64 Euclidean distances."""
    ca, cb = np.asarray(ca, np.float64), np.asarray(cb, np.float64)
    d = np.empty((ca.shape[0], cb.shape[0]))
    for i0 in range(0, ca.shape[0], 64):
        diff = ca[i0:i0 + 64, None, :] - cb[None, :, :]
        d[i0:i0 + 64] = np.sqrt(np.einsum("ijk,ijk->ij", diff, diff))
    return d


def dtw_matrix(d):
    """(N, M) frame distances -> (D(N, M), L): the recursion, ties to the diagonal, then (i-1, j), then (i, j-1)."""
    N, M = d.shape
    D = np.full((N + 1, M + 1), np.inf)
    L = np.zeros((N + 1, M + 1), np.int64)
    D[0, 0] = 0.0
    for s in range(2, N + M + 1):                     # anti-diagonal i + j = s
        i = np.arange(max(1, s - M), min(N, s - 1) + 1)
        j = s - i
        best, bl = D[i - 1, j - 1].copy(), L[i - 1, j - 1].copy()
        up = D[i - 1, j] < best
        best[up], bl[up] = D[i - 1, j][up], L[i - 1, j][up]
        left = D[i, j - 1] < best
        best[left], bl[left] = D[i, j - 1][left], L[i, j - 1][left]
        D[i, j] = d[i - 1, j - 1] + best
        L[i, j] = bl + 1
    return float(D[N, M]), int(L[N, M])


def dtw(ca, cb):
    return dtw_matrix(distances(ca, cb))


def mcd(cost, L):
    return MCD_SCALE * cost / L


def dtw_brute(d):
    """Every monotone path from (1, 1) to (N, M) with steps (1, 1), (1, 0), (0, 1): the least cost, and among the paths
    of least cost the one whose moves, read backwards from (N, M), are lexicographically first with diagonal < (i-1, j)
    < (i, j-1) -- the path the recursion's tie rule picks.  -> (cost, L)."""
    N, M = d.shape
    best = None

    def walk(i, j, cost, moves, cells):
        nonlocal best
        if (i, j) == (N - 1, M - 1):
            key = (cost, tuple(reversed(moves)))
            if best is None or key < best[0]:
                best = (key, cells)
            return
        for rank, (di, dj) in ((0, (1, 1)), (1, (1, 0)), (2, (0, 1))):
            if i + di < N and j + dj < M:
                walk(i + di, j + dj, cost + d[i + di, j + dj], moves + [rank], cells + 1)

    walk(0, 0, d[0, 0], [], 1)
    return best[0][0], best[1]


def monotone_path_count(N, M):
    """Delannoy number D(N - 1, M - 1): how many paths ``dtw_brute`` walks."""
    a, b = N - 1, M - 1
    return sum(math.comb(a, k) * math.comb(b, k) * 2 ** k for k in range(min(a, b) + 1))

