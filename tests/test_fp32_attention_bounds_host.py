"""CPU: the bounds of tests/test_gpu_fp32_attention.py have teeth.  An fp32 emulation of the kernels' arithmetic sits
inside each bound at the GPU test's shapes: the GEMM as a serial chain of exact (fp64) products, each add rounded to
fp32 (csrc/gemm_simt.cuh tile_mma), the softmax with its lane-strided partial sums and butterfly (csrc/elementwise.cu).
Each defect below, applied to that emulation, leaves the bound by more than a factor of two on at least one element
(or, for the GEMM, on the norm-wise bar), so a kernel within its bounds cannot carry it."""
import math

import torch

import test_gpu_attention as A
import test_gpu_fp32_attention as FA
from test_gpu_fp32_conv import U, gamma, norm_ratio, ratio, tf32

FACTOR = 2.0
F32 = torch.float32


def _report(what, factors):
    print("\n%s: defect / bound" % what)
    for k, v in sorted(factors.items(), key=lambda kv: kv[1]):
        print("  %-40s %10.3g" % (k, v))
    print("  smallest factor %.3g" % min(factors.values()))
    for k, v in factors.items():
        assert v > FACTOR, (k, v)


# ---- emulations of the kernels' fp32 arithmetic -----------------------------------------------------------------------
def gemm_fp32(a, b, alpha, c0=None, drop_last_chunk=False):
    """a (batch, M, K), b (batch, K, N) fp32 -> C: acc = fmaf(a, b, acc) over k in order (the fp64 product is exact,
    the add rounds to fp32), then fp32(alpha) * acc (+ c0)."""
    K = a.shape[-1]
    if drop_last_chunk:
        K = (K - 1) // 16 * 16
    ad, bd = a.double(), b.double()
    acc = torch.zeros(a.shape[0], a.shape[1], b.shape[2], dtype=F32)
    for k in range(K):
        acc = (acc.double() + ad[:, :, k, None] * bd[:, None, k, :]).float()
    v = torch.tensor(alpha, dtype=F32) * acc
    return v if c0 is None else c0 + v


def _lanes(x):
    """(rows, L) -> (rows, ceil(L/32), 32): key i on lane i % 32, zero past L."""
    rows, L = x.shape
    n = -(-L // 32)
    return torch.nn.functional.pad(x, (0, 32 * n - L)).view(rows, n, 32)


def _warp_sum(part):
    """common.cuh warp_sum: the xor butterfly over 32 lanes (every lane ends with the same fp32 sum)."""
    for o in (16, 8, 4, 2, 1):
        part = part + part[:, torch.arange(32) ^ o]
    return part[:, 0]


def softmax_fp32(s, keymask, rows_per_b, defect=None):
    rows, L = s.shape
    r = torch.arange(rows)
    mrow = r // rows_per_b
    if defect == "mask row of the neighbouring batch":
        mrow = ((r + 1) // rows_per_b).clamp(max=keymask.shape[0] - 1)
    v = s.masked_fill(keymask[mrow], -math.inf)
    mx = v.max(-1, keepdim=True).values
    e = torch.exp((v - mx).double()).float()                # fp32 argument, exp rounded once
    x = _lanes(e)
    part = torch.zeros(rows, 32, dtype=F32)
    for j in range(x.shape[1]):
        part = part + x[:, j]
    if defect == "one lane's partial sum dropped":
        part[:, (L - 1) % 32] = 0.0
    inv = torch.ones(rows, dtype=F32) / _warp_sum(part)
    return e * inv[:, None]


def softmax_bwd_fp32(P, dpd, drop, dprobs, defect=None):
    g = torch.zeros_like(P)
    if dpd is not None:
        g = dpd if drop is None else dpd * drop
    if dprobs is not None:
        g = g + dprobs
    gl, pl = _lanes(g), _lanes(P)
    part = torch.zeros(P.shape[0], 32, dtype=F32)
    for j in range(gl.shape[1]):
        part = (part.double() + gl[:, j].double() * pl[:, j].double()).float()
    dot = _warp_sum(part)
    if defect == "softmax backward without its dot term":
        dot = torch.zeros_like(dot)
    return P * (g - dot[:, None])


def drop_values(seed, salt, p, shape):
    from oracle import dropout_mask as DM
    return torch.from_numpy(DM.mask(seed, salt, p, shape))


# ---- GEMM ------------------------------------------------------------------------------------------------------------
def test_bgemm_bounds():
    factors = {"TF32 operands": 0.0, "last 16-wide K chunk dropped": 0.0}
    worst = 0.0
    for batch, M, N, K, _, _, _, _ in FA.GEMM_CASES:
        g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
        a, b = FA.randn_full((batch, M, K), g), FA.randn_full((batch, K, N), g)
        for alpha, acc in ((1.0, False), (-0.5, True)):
            c0 = 0.25 * math.sqrt(K) * torch.randn(batch, M, N, generator=g) if acc else None
            R, bound = FA.bgemm_ref(a, b, alpha, c0)
            got = gemm_fp32(a, b, alpha, c0)
            r = max(ratio(got, R, bound), norm_ratio(got, R))
            assert r <= 1, ((batch, M, N, K), alpha, r)
            worst = max(worst, r)
            for name, bad in (("TF32 operands", gemm_fp32(tf32(a), tf32(b), alpha, c0)),
                              ("last 16-wide K chunk dropped", gemm_fp32(a, b, alpha, c0, drop_last_chunk=True))):
                factors[name] = max(factors[name], ratio(bad, R, bound), norm_ratio(bad, R))
    print("\nbgemm emulation: worst error / bound %.3g" % worst)
    _report("bgemm", factors)


# ---- softmax ---------------------------------------------------------------------------------------------------------
def test_softmax_bounds():
    defects = ("mask row of the neighbouring batch", "one lane's partial sum dropped")
    factors = dict.fromkeys(defects + ("dropout mask of salt + 1", "softmax backward without its dot term"), 0.0)
    worst = {}
    for L in FA.SOFTMAX_LS:
        g = torch.Generator().manual_seed(L)
        s, mask = FA.softmax_inputs(L, g)
        rows = s.shape[0]
        P, bP = FA.softmax_ref(s, mask, FA.TD)
        probs = softmax_fp32(s, mask, FA.TD)
        worst["probs"] = max(worst.get("probs", 0.0), ratio(probs, P, bP))
        for d in defects:
            if L > 1 or d != "one lane's partial sum dropped":     # L = 1: the only partial, the sum would be 0
                factors[d] = max(factors[d], ratio(softmax_fp32(s, mask, FA.TD, defect=d), P, bP))
        dpd, dprobs = torch.randn(rows, L, generator=g), torch.randn(rows, L, generator=g)
        for p in (0.0, 0.05, 0.5):
            drop = drop_values(FA.SEED0 + L, FA.SALT, p, (rows, L)) if p > 0 else None
            if drop is not None:
                other = drop_values(FA.SEED0 + L, FA.SALT + 1, p, (rows, L))
                factors["dropout mask of salt + 1"] = max(factors["dropout mask of salt + 1"],
                                                          ratio(probs * other, P * drop, (bP + U * P) * drop))
            for name, a, b in (("dpd", dpd, None), ("dprobs", None, dprobs), ("both", dpd, dprobs)):
                want, bound = FA.softmax_bwd_ref(probs, a, drop, b)
                worst["ds " + name] = max(worst.get("ds " + name, 0.0),
                                          ratio(softmax_bwd_fp32(probs, a, drop, b), want, bound))
                bad = softmax_bwd_fp32(probs, a, drop, b, defect="softmax backward without its dot term")
                factors["softmax backward without its dot term"] = max(
                    factors["softmax backward without its dot term"], ratio(bad, want, bound))
    print("\nsoftmax emulation: worst error / bound %s" % " ".join("%s %.3g" % kv for kv in sorted(worst.items())))
    assert max(worst.values()) <= 1, worst
    _report("softmax", factors)


# ---- attention core of a bucketed batch ------------------------------------------------------------------------------
def attention_fp32(q, k, v, keymask, scale):
    """ops._AttentionCoreFn's forward on the emulated kernels: scores, softmax (one mask row per batch), context."""
    B, E, Td = q.shape
    Ts = k.shape[2]
    scores = gemm_fp32(q.transpose(1, 2), k, 1.0)
    probs = softmax_fp32(scores.reshape(B * Td, Ts), keymask, Td).view(B, Td, Ts)
    return probs, gemm_fp32(v, probs.transpose(1, 2), scale)


def test_context_scale_bounds():
    """The composed forward bound of tests/test_gpu_attention.py with gamma (test_attention_fallback_vs_fp64 and the
    buckets of tests/test_gpu_fp32_attention.py) holds the emulation at the logical context scale and refuses the
    padded Ts's."""
    B, E, Td = 3, 64, 37
    worst, factor = 0.0, 0.0
    for ts_log, Ts in FA.BUCKETS:
        g = torch.Generator().manual_seed(ts_log + Ts)
        sd = 1.2 * E ** -0.25
        q, k = sd * torch.randn(B, E, Td, generator=g), sd * torch.randn(B, E, Ts, generator=g)
        v = torch.randn(B, E, Ts, generator=g)
        lengths = torch.tensor([ts_log, ts_log - 19, 97])
        key = torch.arange(Ts)[None, :]
        mask = key >= lengths[:, None]
        P, out, bP, bout = A.ref_forward(q.double(), k[..., :ts_log].double(), v[..., :ts_log].double(),
                                         mask[:, :ts_log], c=gamma)
        for t, name in ((ts_log, "logical"), (Ts, "padded")):
            probs, got = attention_fp32(q, k, v, mask | (key >= ts_log), float(A._scale(t)))
            r = ratio(got, out, bout)
            if name == "logical":
                worst = max(worst, r, ratio(probs[..., :ts_log], P, bP))
                assert bool((probs[..., ts_log:] == 0).all())
            else:
                factor = max(factor, r)
    print("\nattention emulation at the logical scale: worst error / bound %.3g" % worst)
    assert worst <= 1
    _report("attention core", {"context scale of the padded Ts": factor})
