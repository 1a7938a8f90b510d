"""GPU: the exact-fp32 attention path at kernel level, through the C ABI: dv3_bgemm / dv3_bgemm_ctx_scale (csrc/bgemm.cu
on the gemm_simt_kernel mainloop of csrc/gemm_simt.cuh) and dv3_softmax_fwd / dv3_softmax_bwd (csrc/elementwise.cu),
the kernels ops._AttentionCoreFn runs.  They carry the attention under DV3_CONV_MATH=fp32, with DV3_TC_ATTN=0, and in
the default mode for every shape dv3_tc_attn_supported refuses (E % 16 != 0, E > 256, Ts > 128): every training batch
whose longest text is longer than 128 symbols, padded to a bucket inside ops.extent_scope or not.

Bounds (u = 2^-24, gamma(K) = K u / (1 - K u); every reference is fp64 on the operands the kernel reads):
  GEMM, C = alpha sum_k a b (+ C0 when accumulating): each output is one serial fmaf chain over k in 16-wide chunks
    (zero operands past K leave the accumulator unchanged), so |acc - D| <= gamma(K) S with S = sum |a||b|; the product
    by alpha and the add onto C0 round once each:
      |C - R| <= |alpha| gamma(K) S (1 + u) + u |alpha D|   (+ u (|R| + that) when accumulating).
    Three checks per launch, as tests/test_gpu_fp32_conv.py makes them:
      (a) exact: integer operands in [-8, 8], alpha a power of two (or 0), integer C0: every partial sum is an integer
          below 2^24, so the kernel matches fp64 bit for bit.  Catches a missing, duplicated or misplaced term.
      (b) elementwise, random operands: the bound above.
      (c) norm-wise: ||C - R||_2 <= 2^-16 ||R||_2.  Its control: the fp64 result of the TF32-rounded operands misses it
          by >= 10x on every launch.  The random operands carry 0x0FFF in their 13 low mantissa bits (bits TF32 drops,
          just under half its last place), so the control's miss does not depend on the draw, even for one element.
    Operands sit in NaN-filled buffers (leading-dimension padding, batch-stride gaps): a read outside the operand
    poisons the output.  Outputs sit in sentinel-filled buffers: the ldc - N columns and the batch gaps stay untouched,
    every element inside is written.  Batch z launched alone is bit-identical to batch z inside the whole launch.
  Softmax forward, one warp per row of L keys: exact max; d = fl(s - max) (u |d|); expf at 2 ulp (the library is built
    without fast math): relative eta = 2^-22 + u |s - max|; the row sum is ceil(L/32) - 1 lane-strided adds and 5
    butterfly adds, gamma(ceil(L/32) + 4); one reciprocal and one product:
      |p - P| <= P (eta + sum_j P_j eta_j + gamma(ceil(L/32) + 4) + 2u) (1 + that) + 2^-149.
    pd = probs * dropout scale is one fp32 product: bit-identical to probs times oracle/dropout_mask.py's mask.
  Softmax backward, against the fp64 backward of the kernel's own fp32 probs P: g = fl(fl(dpd m) + dprobs) (u each),
    dot = lane-strided fmaf partials of ceil(L/32) terms and 5 butterfly adds, gamma(ceil(L/32) + 5) sum |g| P, then
    one subtraction and one product (softmax_bwd_ref).  Where a result falls below 2^-126 its rounding is absolute,
    at most 2^-150: the product once, the n + 6 roundings before it scaled by P <= 1.  That floor is needed: a key with
    p ~ 2e-34 whose gradient was dropped gets ds = -p dot ~ -2e-41 (L = 32, p_drop = 0.5).
  Attention core (ops.attention_core on this path): tests/test_gpu_attention.py composes the bounds, gamma in place of
    the tensor-core c_gemm, in test_attention_fallback_vs_fp64; here the buckets: inside ops.extent_scope the keys past
    the logical text length get p = 0 exactly, and with dropout off the valid region is bit-identical to the unpadded
    call (a masked key adds +0 to every sum, fmaf(x, 0, acc) leaves a non-negative-zero accumulator unchanged, key i
    stays on lane i % 32 and the K order of every chain does not depend on K).
The largest error / bound ratio of every tensor is printed (run with -s).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import test_gpu_attention as A
from test_gpu_fp32_conv import MUTANT_MARGIN, U, check_norm, gamma, ratio, tf32
from test_gpu_tc1 import _call, _p, _st
from test_gpu_tc_pairs import GUARD, SENT32, assert_written_inside_only, guarded

pytestmark = pytest.mark.gpu

SALT = 7
SEED0 = 0x5EED0000      # dropout seed of the softmax tests: SEED0 + L
LOW_BITS = 0x0FFF


# ---- bounds (device-agnostic fp64 torch: tests/test_fp32_attention_bounds_host.py checks them on the CPU) -------------
def bgemm_ref(a, b, alpha, c0=None):
    """fp64 R = alpha a.b (+ c0) of a (batch, M, K) and b (batch, K, N), and its elementwise bound."""
    a, b = a.double(), b.double()
    K = a.shape[-1]
    D = a @ b
    S = a.abs() @ b.abs()
    al = abs(alpha)
    R = alpha * D
    bound = al * gamma(K) * S * (1 + U) + U * al * D.abs()
    if c0 is not None:
        R = R + c0.double()
        bound = bound + U * (R.abs() + bound)
    return R, bound


def softmax_ref(s, keymask, rows_per_b):
    """s (rows, L) fp32 scores, keymask (rows / rows_per_b, L) bool (True = masked) or None -> fp64 P and its bound."""
    rows, L = s.shape
    S = s.double()
    m = None
    if keymask is not None:
        m = keymask.repeat_interleave(rows_per_b, 0)
        S = S.masked_fill(m, -math.inf)
    P = torch.softmax(S, -1)
    mx = S.max(-1, keepdim=True).values
    eta = 2.0 ** -22 + U * (S - mx).abs()
    if m is not None:
        eta = eta.masked_fill(m, 0.0)
    rel = eta + (P * eta).sum(-1, keepdim=True) + gamma(-(-L // 32) + 4) + 2 * U
    return P, P * rel * (1 + rel) + 2.0 ** -149


def softmax_bwd_ref(P, dpd, drop, dprobs):
    """fp64 dS = P (g - <g, P>), g = dpd * drop + dprobs, of the fp32 probs P the kernel reads, and its bound.  dpd or
    dprobs may be None; drop is the dropout mask's fp32 values (None: dropout off, the product is exact)."""
    L = P.shape[-1]
    P = P.double()
    t, bt = torch.zeros_like(P), torch.zeros_like(P)
    if dpd is not None:
        t = dpd.double() * (1.0 if drop is None else drop.double())
        if drop is not None:
            bt = U * t.abs()
    G = t + (0.0 if dprobs is None else dprobs.double())
    bg = bt + (U * (G.abs() + bt) if dpd is not None and dprobs is not None else 0.0)
    dot = (G * P).sum(-1, keepdim=True)
    bdot = gamma(-(-L // 32) + 5) * ((G.abs() + bg) * P).sum(-1, keepdim=True) + (bg * P).sum(-1, keepdim=True)
    dS = P * (G - dot)
    sub = 2.0 ** -150 * (1 + (-(-L // 32) + 6) * P)
    return dS, P * ((bg + bdot) + 2 * U * ((G - dot).abs() + bg + bdot)) * (1 + 4 * U) + sub


# ---- operands and launches --------------------------------------------------------------------------------------------
def ints(shape, g):
    return torch.randint(-8, 9, shape, generator=g, device=g.device).float()


def randn_full(shape, g):
    """N(0, 1) with the 13 low mantissa bits set to 0x0FFF: TF32 rounding drops just under half a last place."""
    x = torch.randn(shape, generator=g, device=g.device)
    return ((x.view(torch.int32) & ~0x1FFF) | LOW_BITS).view(torch.float32)


def place(x, kmajor, gap):
    """Logical (batch, R, K) operand -> (NaN-filled flat buffer holding it, strides (batch, row, k)).  Unit stride along
    K when kmajor, else along R; with gap > 0 the other stride is padded by 3 and the batch stride by gap."""
    bt, R, K = x.shape
    pad = 3 if gap else 0
    if kmajor:
        s_r, s_k = K + pad, 1
        span = (R - 1) * s_r + K
    else:
        s_r, s_k = 1, R + pad
        span = (K - 1) * s_k + R
    s_b = span + gap
    buf = torch.full((bt * s_b,), math.nan, device="cuda")
    torch.as_strided(buf, x.shape, (s_b, s_r, s_k)).copy_(x)
    return buf, (s_b, s_r, s_k)


def views(abuf, sA, bbuf, sB, batch, M, N, K):
    """The logical (batch, M, K) and (batch, K, N) operands of one launch (sA = (sAb, sAm, sAk), sB = (sBb, sBk, sBn))."""
    return (torch.as_strided(abuf, (batch, M, K), sA), torch.as_strided(bbuf, (batch, K, N), sB))


def launch(abuf, sA, bbuf, sB, batch, M, N, K, alpha, ldc=None, sCb=None, c0=None, ts=None, z0=0):
    """One dv3_bgemm (ts None: alpha) or dv3_bgemm_ctx_scale (ts: int64 key count on the device) launch of batches
    z0 .. z0 + batch - 1 into a sentinel-filled C of leading dimension ldc and batch stride sCb, accumulating onto c0 when
    given.  Checks the write extent; returns C (batch, M, N)."""
    ldc = N if ldc is None else ldc
    sCb = M * ldc if sCb is None else sCb
    n = (batch - 1) * sCb + (M - 1) * ldc + N
    buf, c = guarded(n)
    inside = torch.as_strided(c, (batch, M, N), (sCb, ldc, 1))
    if c0 is not None:
        inside.copy_(c0)
    a = ctypes.c_void_p(abuf.data_ptr() + 4 * z0 * sA[0])
    b = ctypes.c_void_p(bbuf.data_ptr() + 4 * z0 * sB[0])
    if ts is None:
        _call("dv3_bgemm", a, *sA, b, *sB, _p(c), sCb, ldc, batch, M, N, K, alpha, int(c0 is not None), _st())
    else:
        _call("dv3_bgemm_ctx_scale", a, *sA, b, *sB, _p(c), sCb, ldc, batch, M, N, K, _p(ts), int(c0 is not None),
              _st())
    torch.cuda.synchronize()
    written = torch.zeros(n, dtype=torch.bool, device="cuda")
    torch.as_strided(written, (batch, M, N), (sCb, ldc, 1)).fill_(True)
    assert bool((c.view(torch.int32)[~written] == SENT32).all()), "write into an ldc or batch gap"
    check = buf.clone()
    check[GUARD:GUARD + n][~written] = 0.0
    assert_written_inside_only(check, n)
    return inside.clone()


def launch_count():
    from deepvoice3_pytorch_b200._lib import lib
    return int(lib.raw("dv3_launch_count")())


# ---- 1. bgemm through the C ABI ---------------------------------------------------------------------------------------
GEMM_CASES = [
    # (batch, M, N, K, A unit stride along K, B unit stride along K, batch gap, ldc - N): M, N, K around the 128 x 64
    # CTA tile, the 16-wide K chunk and the 4 x 8 transposed-load pattern; every <A_KMAJOR, B_KMAJOR> instantiation
    (1, 1, 1, 1, False, False, 0, 0),
    (3, 15, 17, 16, True, True, 5, 3),
    (3, 16, 63, 17, False, True, 5, 0),
    (1, 17, 64, 15, True, False, 0, 7),
    (16, 63, 65, 63, False, False, 1, 1),
    (3, 64, 15, 64, True, True, 5, 2),
    (1, 65, 129, 65, False, True, 0, 0),
    (3, 127, 16, 127, True, False, 5, 1),
    (16, 128, 1, 128, False, False, 3, 0),
    (1, 129, 200, 129, True, True, 0, 5),
    (3, 200, 127, 200, False, True, 7, 0),
    (1, 257, 128, 257, True, False, 0, 0),
    (3, 1, 257, 1000, False, False, 5, 3),
    (1, 200, 257, 1000, True, True, 2, 1),
]
ALPHAS = (1.0, -0.5, 0.0)


def _gemm_id(c):
    return "b%d_M%d_N%d_K%d_%s%s_gap%d_ldc+%d" % (c[:4] + ("k" if c[4] else "d", "k" if c[5] else "d") + c[6:])


def check_launches(name, abuf, sA, bbuf, sB, batch, M, N, K, a_int, b_int, g, ldc=None, sCb=None):
    """(a) on the integer operands, (b) and (c) on the random ones, for every alpha with and without accumulation, and
    batch invariance.  The buffers hold the integer operands first, then are refilled with the random ones."""
    av, bv = views(abuf, sA, bbuf, sB, batch, M, N, K)
    av.copy_(a_int)
    bv.copy_(b_int)
    assert K * 64 < 2 ** 24
    for alpha in ALPHAS:
        for acc in (False, True):
            c0 = ints((batch, M, N), g) if acc else None
            got = launch(abuf, sA, bbuf, sB, batch, M, N, K, alpha, ldc, sCb, c0)
            R, _ = bgemm_ref(av, bv, alpha, c0)
            assert torch.equal(got.double(), R), (name, "exact", alpha, acc)
    av.copy_(randn_full(av.shape, g))
    bv.copy_(randn_full(bv.shape, g))
    D_tf32 = tf32(av).double() @ tf32(bv).double()
    worst, c, cm = 0.0, 0.0, math.inf
    for alpha in ALPHAS:
        for acc in (False, True):
            c0 = 0.25 * math.sqrt(K) * torch.randn(batch, M, N, generator=g, device="cuda") if acc else None
            got = launch(abuf, sA, bbuf, sB, batch, M, N, K, alpha, ldc, sCb, c0)
            R, bound = bgemm_ref(av, bv, alpha, c0)
            if alpha != 0:
                mut = alpha * D_tf32 + (0.0 if c0 is None else c0.double())
                cc, cmm = check_norm((name, alpha, acc), got, R, mut)
                c, cm = max(c, cc), min(cm, cmm)
            r = ratio(got, R, bound)
            assert r <= 1, (name, alpha, acc, r)
            worst = max(worst, r)
            if alpha == 1.0 and not acc and batch > 1:
                for z in sorted({0, batch // 2, batch - 1}):
                    one = launch(abuf, sA, bbuf, sB, 1, M, N, K, alpha, ldc, None, None, z0=z)
                    assert torch.equal(one[0].view(torch.int32), got[z].view(torch.int32)), (name, "batch", z)
    return worst, c, cm


@pytest.mark.parametrize("case", GEMM_CASES, ids=_gemm_id)
def test_bgemm(case):
    batch, M, N, K, ak, bk, gap, ldc_pad = case
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a_int, bt_int = ints((batch, M, K), g), ints((batch, N, K), g)
    abuf, (sAb, sAr, sAk) = place(a_int, ak, gap)
    bbuf, (sBb, sBr, sBk) = place(bt_int, bk, gap)
    sA, sB = (sAb, sAr, sAk), (sBb, sBk, sBr)
    ldc = N + ldc_pad
    sCb = M * ldc + gap
    worst, c, cm = check_launches(_gemm_id(case), abuf, sA, bbuf, sB, batch, M, N, K, a_int,
                                  bt_int.transpose(1, 2), g, ldc, sCb)
    print("bgemm %s: (b) %.3g, (c) %.3g, TF32 control %.3g" % (_gemm_id(case), worst, c, cm))


def test_gemm_cases_reach_every_instantiation():
    """The launcher picks <A_KMAJOR, B_KMAJOR> = <sAm != 1, sBn != 1>.  The six contractions of ops reach <0,0>, <1,1>
    and <1,0> only; the generic cases reach all four."""
    seen = set()
    for batch, M, N, K, ak, bk, gap, ldc_pad in GEMM_CASES:
        sAm = (K + (3 if gap else 0)) if ak else 1
        sBn = (K + (3 if gap else 0)) if bk else 1
        seen.add((sAm != 1, sBn != 1))
    assert seen == {(False, False), (False, True), (True, False), (True, True)}, seen


def attention_contractions(B, E, Td, Ts):
    """The six contractions of ops._AttentionCoreFn with exactly the strides it passes: (name, A operand, (sAb, sAm,
    sAk), B operand, (sBb, sBk, sBn), M, N, K, whether ops scales it by the context scale).  Operands are the dense
    tensors q, dout (B,E,Td); k, v (B,E,Ts); pd, ds (B,Td,Ts)."""
    return [
        ("scores", "q", (E * Td, 1, Td), "k", (E * Ts, Ts, 1), Td, Ts, E, False),
        ("context", "v", (E * Ts, Ts, 1), "pd", (Td * Ts, 1, Ts), E, Td, Ts, True),
        ("dPd", "dout", (E * Td, 1, Td), "v", (E * Ts, Ts, 1), Td, Ts, E, True),
        ("dV", "dout", (E * Td, Td, 1), "pd", (Td * Ts, Ts, 1), E, Ts, Td, True),
        ("dQ", "k", (E * Ts, Ts, 1), "ds", (Td * Ts, 1, Ts), E, Td, Ts, False),
        ("dK", "q", (E * Td, Td, 1), "ds", (Td * Ts, Ts, 1), E, Ts, Td, False),
    ]


ATTN_GEMM_SHAPES = [(3, 40, 129, 257), (2, 272, 31, 200), (1, 16, 1, 129), (16, 256, 200, 200)]


@pytest.mark.parametrize("B,E,Td,Ts", ATTN_GEMM_SHAPES)
def test_bgemm_attention_contractions(B, E, Td, Ts):
    """Each contraction as ops issues it: checks (a)-(c) and batch invariance; the context-scaled ones also through
    dv3_bgemm_ctx_scale at a key count below Ts, bit-identical to dv3_bgemm with that count's fp32 scale."""
    g = torch.Generator(device="cuda").manual_seed(B + E + Td + Ts)
    shapes = {"q": (B, E, Td), "dout": (B, E, Td), "k": (B, E, Ts), "v": (B, E, Ts), "pd": (B, Td, Ts),
              "ds": (B, Td, Ts)}
    t_log = Ts - 7
    ts = torch.tensor([t_log], dtype=torch.int64, device="cuda")
    scale = float(np.float32(t_log * math.sqrt(1.0 / t_log)))
    for name, an, sA, bn, sB, M, N, K, scaled in attention_contractions(B, E, Td, Ts):
        abuf = torch.empty(math.prod(shapes[an]), device="cuda")
        bbuf = torch.empty(math.prod(shapes[bn]), device="cuda")
        a_int, b_int = ints((B, M, K), g), ints((B, K, N), g)
        worst, c, cm = check_launches(name, abuf, sA, bbuf, sB, B, M, N, K, a_int, b_int, g)
        if scaled:
            want = launch(abuf, sA, bbuf, sB, B, M, N, K, scale)
            got = launch(abuf, sA, bbuf, sB, B, M, N, K, None, ts=ts)
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, "ctx scale")
        print("bgemm %s B%d E%d Td%d Ts%d: (b) %.3g, (c) %.3g, TF32 control %.3g" % (name, B, E, Td, Ts, worst, c, cm))


def test_ctx_scale_every_key_count():
    """One-hot operands (C = alpha): dv3_bgemm_ctx_scale gives fp32(t sqrt(1/t)) for every t in 0..1024 (t = 0 read as
    1), and that equals the host scale Ts * (1/Ts) ** 0.5 that ops passes outside an extent scope, rounded to fp32 as
    the C ABI's float argument rounds it."""
    n = 1025
    ts = torch.arange(n, dtype=torch.int64, device="cuda")
    one = torch.ones(1, device="cuda")
    buf, c = guarded(n)
    for t in range(n):
        _call("dv3_bgemm_ctx_scale", _p(one), 1, 1, 1, _p(one), 1, 1, 1, ctypes.c_void_p(c.data_ptr() + 4 * t), 1, 1,
              1, 1, 1, 1, ctypes.c_void_p(ts.data_ptr() + 8 * t), 0, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(buf, n)
    got = c.cpu().numpy()
    want = np.array([np.float32(max(t, 1) * math.sqrt(1.0 / max(t, 1))) for t in range(n)], np.float32)
    host = np.array([np.float32(t * (1.0 / t) ** 0.5) for t in range(1, n)], np.float32)
    assert np.array_equal(got, want), np.nonzero(got != want)
    assert np.array_equal(got[1:], host), np.nonzero(got[1:] != host)


def test_bgemm_refusals():
    """Batch 0, batch 65536, an operand without a unit stride, a NULL key count: Dv3Error and no launch."""
    from deepvoice3_pytorch_b200._lib import Dv3Error
    x = torch.ones(64, device="cuda")
    c = torch.zeros(64, device="cuda")
    ts = torch.tensor([5], dtype=torch.int64, device="cuda")
    n0 = launch_count()
    bad = [  # (sA, sB, batch)
        ((4, 1, 2), (4, 2, 1), 0),
        ((4, 1, 2), (4, 2, 1), 65536),
        ((4, 2, 2), (4, 2, 1), 1),
        ((4, 1, 2), (4, 2, 2), 1),
    ]
    for sA, sB, batch in bad:
        with pytest.raises(Dv3Error):
            _call("dv3_bgemm", _p(x), *sA, _p(x), *sB, _p(c), 4, 2, batch, 2, 2, 2, 1.0, 0, _st())
        with pytest.raises(Dv3Error):
            _call("dv3_bgemm_ctx_scale", _p(x), *sA, _p(x), *sB, _p(c), 4, 2, batch, 2, 2, 2, _p(ts), 0, _st())
    with pytest.raises(Dv3Error):
        _call("dv3_bgemm_ctx_scale", _p(x), 4, 1, 2, _p(x), 4, 2, 1, _p(c), 4, 2, 1, 2, 2, 2, None, 0, _st())
    assert launch_count() == n0
    assert bool((c == 0).all())


# ---- 2. softmax through the C ABI -------------------------------------------------------------------------------------
SOFTMAX_LS = [1, 2, 31, 32, 33, 64, 65, 129, 192, 257]
NB, TD = 4, 5          # batches of TD rows: batch 0 all keys, 1 a single key, 2 a prefix, 3 a scattered mask


def softmax_inputs(L, g):
    """(NB*TD, L) scores and the (NB, L) key mask.  Row 0 of a batch: spread 0.5, row 1: exact ties (three values, the
    largest repeated), row 2: uniform over [max - 80, max], rows 3, 4: spreads 4 and 8 (|s - max| stays below ~80, so
    every p is a normal fp32 number)."""
    rows, dev = NB * TD, g.device
    s = torch.randn(rows, L, generator=g, device=dev)
    s = s * torch.tensor([0.5, 1.0, 1.0, 4.0, 8.0], device=dev).repeat(NB)[:, None]
    s[1::TD] = torch.randint(0, 3, (NB, L), generator=g, device=dev).float() * 0.75
    s[2::TD] = -80.0 * torch.rand(NB, L, generator=g, device=dev)
    s[2::TD, 0] = 0.0
    key = torch.arange(L, device=dev)
    mask = torch.stack([key < 0, key >= 1, key >= L // 2 + 1,
                        (torch.rand(L, generator=g, device=dev) < 0.4) & (key > 0)])
    return s, mask


def softmax_fwd(s, mask, rows_per_b, p, seed, want_pd=True):
    rows, L = s.shape
    n = rows * L
    (pbuf, probs), (dbuf, pd) = guarded(n), guarded(n)
    m8 = None if mask is None else mask.to(torch.uint8).contiguous()
    _call("dv3_softmax_fwd", _p(s), _p(m8), _p(probs), _p(pd) if want_pd else None, rows, L, rows_per_b, p, _p(seed),
          SALT, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(pbuf, n)
    if want_pd:
        assert_written_inside_only(dbuf, n)
    else:
        assert bool((dbuf.view(torch.int32) == SENT32).all()), "pd written without a pd buffer"
    return probs.view(rows, L), pd.view(rows, L)


def softmax_bwd(probs, dpd, dprobs, p, seed):
    rows, L = probs.shape
    n = rows * L
    buf, ds = guarded(n)
    _call("dv3_softmax_bwd", _p(probs), _p(dpd), _p(dprobs), _p(ds), rows, L, p, _p(seed), SALT, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(buf, n)
    return ds.view(rows, L)


def drop_values(seed, p, shape):
    from oracle import dropout_mask as DM
    return torch.from_numpy(DM.mask(DM.seed_u64(seed), SALT, p, shape)).cuda()


@pytest.mark.parametrize("L", SOFTMAX_LS)
def test_softmax(L):
    g = torch.Generator(device="cuda").manual_seed(L)
    s, mask = softmax_inputs(L, g)
    rows = NB * TD
    P, bP = softmax_ref(s, mask, TD)
    m = mask.repeat_interleave(TD, 0)
    seed = torch.tensor([SEED0 + L], dtype=torch.int64, device="cuda")
    dpd = torch.randn(rows, L, generator=g, device="cuda")
    dprobs = torch.randn(rows, L, generator=g, device="cuda")
    worst = {}
    for p in (0.0, 0.05, 0.5):
        sd = seed if p > 0 else None
        probs, pd = softmax_fwd(s, mask, TD, p, sd)
        r = ratio(probs, P, bP)
        assert r <= 1, ("probs", p, r)
        worst["probs"] = max(worst.get("probs", 0.0), r)
        assert bool((probs[m] == 0).all()) and bool((pd[m] == 0).all()), "masked key p != 0"
        single = probs[TD:2 * TD]
        assert bool((single[:, 0] == 1).all()) and bool((single[:, 1:] == 0).all()), "single valid key"
        drop = drop_values(sd, p, (rows, L)) if p > 0 else None
        assert torch.equal(pd.view(torch.int32), (probs if drop is None else probs * drop).view(torch.int32)), p
        probs_only, _ = softmax_fwd(s, mask, TD, p, sd, want_pd=False)
        assert torch.equal(probs_only.view(torch.int32), probs.view(torch.int32)), "probs depend on the pd buffer"
        for name, a, b in (("dpd", dpd, None), ("dprobs", None, dprobs), ("both", dpd, dprobs)):
            ds = softmax_bwd(probs, a, b, p, sd)
            want, bound = softmax_bwd_ref(probs, a, drop, b)
            r = ratio(ds, want, bound)
            assert r <= 1, (name, p, r)
            assert bool((ds[m] == 0).all()), "masked key ds != 0"
            worst["ds " + name] = max(worst.get("ds " + name, 0.0), r)
    print("softmax L=%d: %s" % (L, " ".join("%s %.3g" % kv for kv in sorted(worst.items()))))


def test_softmax_without_mask_takes_any_row_count():
    """No mask: rows_per_b is not read, rows need not be whole batches."""
    g = torch.Generator(device="cuda").manual_seed(3)
    s = torch.randn(7, 45, generator=g, device="cuda") * 3
    probs, _ = softmax_fwd(s, None, 3, 0.0, None)
    P, bP = softmax_ref(s, None, 3)
    assert ratio(probs, P, bP) <= 1


def test_softmax_refusals():
    """rows < 1, L < 1, rows past one int-indexed warp each, rows_per_b < 1, a mask with rows not whole batches of
    rows_per_b: Dv3Error and no launch."""
    from deepvoice3_pytorch_b200._lib import Dv3Error
    x = torch.zeros(64, device="cuda")
    m8 = torch.zeros(64, dtype=torch.uint8, device="cuda")
    huge = 2 ** 31 // 32
    n0 = launch_count()
    for rows, L, rpb, mask in ((0, 4, 1, None), (4, 0, 1, None), (huge, 1, 1, None), (4, 4, 0, None),
                               (4, 4, 0, m8), (6, 4, 4, m8), (-1, 4, 1, None)):
        with pytest.raises(Dv3Error):
            _call("dv3_softmax_fwd", _p(x), _p(mask), _p(x), None, rows, L, rpb, 0.0, None, 0, _st())
    for rows, L in ((0, 4), (4, 0), (huge, 1), (-3, 2)):
        with pytest.raises(Dv3Error):
            _call("dv3_softmax_bwd", _p(x), _p(x), None, _p(x), rows, L, 0.0, None, 0, _st())
    assert launch_count() == n0


# ---- 3. bucketed batches on the fallback ------------------------------------------------------------------------------
BUCKETS = [(150, 160), (129, 192), (131, 144)]      # (logical text length, padded Ts)


def attend(q, k, v, mask, dout, dprobs, called):
    """ops.attention_core forward and backward (dropout off) -> out, probs, {dq, dk, dv}, the entry points it called."""
    from deepvoice3_pytorch_b200 import ops
    called.clear()
    qg, kg, vg = [t.clone().requires_grad_(True) for t in (q, k, v)]
    out, probs = ops.attention_core(qg, kg, vg, mask, 0.0, False)
    ((out * dout).sum() + (probs * dprobs).sum()).backward()
    torch.cuda.synchronize()
    return out.detach(), probs.detach(), {"dq": qg.grad, "dk": kg.grad, "dv": vg.grad}, set(called)


def spy_calls(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    called = []
    real = lib.call

    def spy(name, *args):
        called.append(name)
        return real(name, *args)
    monkeypatch.setattr(lib, "call", spy)
    return called


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("memory_mask", [False, True], ids=["no_mask", "memory_mask"])
@pytest.mark.parametrize("ts_log,Ts", BUCKETS)
def test_bucketed_attention(ts_log, Ts, memory_mask, monkeypatch):
    """ops.attention_core inside ops.extent_scope with a logical text length below the padded Ts (default mode: Ts > 128
    takes the exact-fp32 path): forward and backward within the fp64 bounds at the logical context scale (the padded
    Ts's scale misses them), p, dk and dv exactly 0 at the padded keys, and the valid region bit-identical to the
    unpadded call at Ts = ts_log."""
    from deepvoice3_pytorch_b200 import ops
    B, E, Td = 3, 64, 37
    called = spy_calls(monkeypatch)
    q, k, v, dout, dprobs, _ = A.inputs(B, E, Td, Ts, ts_log + Ts + memory_mask)
    mask = None
    if memory_mask:
        mask = (torch.arange(Ts)[None, :] >= torch.tensor([ts_log, ts_log - 19, 97])[:, None]).cuda()
    ext = torch.tensor([Td, ts_log, Td, Td], dtype=torch.int64, device="cuda")
    with ops.extent_scope(ext, (Td, Ts, Td, Td)):
        out, probs, grads, names = attend(q, k, v, mask, dout, dprobs, called)
    assert "dv3_bgemm_ctx_scale" in names and not [n for n in names if n.startswith("dv3_tc_attn")], names
    what = "bucket %d -> %d mask=%s" % (ts_log, Ts, memory_mask)
    # padded keys
    assert bool((probs[..., ts_log:] == 0).all()), what + ": p at a padded key"
    assert bool((grads["dk"][..., ts_log:] == 0).all()) and bool((grads["dv"][..., ts_log:] == 0).all()), what
    # fp64 at the logical scale
    kl, vl = k[..., :ts_log], v[..., :ts_log]
    ml = None if mask is None else mask[:, :ts_log]
    P, out_r, bP, bout = A.ref_forward(q.double(), kl.double(), vl.double(), ml, c=gamma)
    ratios = A.check_forward(probs[..., :ts_log], out, P, out_r, bP, bout, ml, what)
    ref = A.ref_backward(q.double(), kl.double(), vl.double(), probs[..., :ts_log].double(), dout.double(),
                         dprobs[..., :ts_log].double(), c=gamma)
    got = {"dq": grads["dq"], "dk": grads["dk"][..., :ts_log], "dv": grads["dv"][..., :ts_log]}
    ratios.update(A.check_backward(got, ref, what))
    # negative control: the padded Ts's context scale
    control = A.bound_ratio(out, out_r * (A._scale(Ts) / A._scale(ts_log)), bout)
    assert control >= MUTANT_MARGIN, (what, control)
    # bit for bit against the unpadded call
    out1, probs1, grads1, names1 = attend(q, kl.contiguous(), vl.contiguous(), ml, dout,
                                          dprobs[..., :ts_log].contiguous(), called)
    assert "dv3_bgemm" in names1 and "dv3_bgemm_ctx_scale" not in names1, names1
    assert same_bits(out, out1), what + ": out"
    assert same_bits(probs[..., :ts_log], probs1), what + ": probs"
    assert same_bits(grads["dq"], grads1["dq"]), what + ": dq"
    for n in ("dk", "dv"):
        assert same_bits(grads[n][..., :ts_log], grads1[n]), what + ": " + n
    print("%s: %s, padded-scale control %.3g" % (what, " ".join("%s %.3g" % kv for kv in sorted(ratios.items())),
                                                 control))


@pytest.mark.parametrize("math_mode", ["tc", "fp32"])
def test_bucketed_training_step_on_the_fallback(math_mode, monkeypatch):
    """One training step of deepvoice3 on texts of 150, 131 and 97 symbols (Ts > 128: the attention takes the
    exact-fp32 path in both modes), unpadded and padded to 160 text positions: loss, gradient arena and grad norm
    within tests/test_gpu_train_ragged.py's tolerance.  The padded step scales its context through
    dv3_bgemm_ctx_scale, the unpadded one does not, and no tensor-core attention kernel runs."""
    from test_gpu_train_ragged import TOL, _batches, _excess, _train
    rtol, atol = TOL[math_mode]
    called = spy_calls(monkeypatch)
    plain, padded = _batches("deepvoice3", extra_text=10, text_lens=(150, 131, 97))
    assert plain["x"].shape[1] == 150 and padded["x"].shape[1] == 160
    l_ref, g_ref, n_ref, _, _ = _train("deepvoice3", [plain], math_mode)
    plain_calls = set(called)
    called.clear()
    l_pad, g_pad, n_pad, _, _ = _train("deepvoice3", [padded], math_mode)
    pad_calls = set(called)
    assert "dv3_bgemm_ctx_scale" in pad_calls and "dv3_bgemm_ctx_scale" not in plain_calls
    assert not [n for n in plain_calls | pad_calls if n.startswith("dv3_tc_attn")]
    assert float(g_ref.abs().max()) > 0
    assert _excess(l_pad, l_ref, rtol, atol) <= 1, (l_pad, l_ref)
    assert _excess(n_pad, n_ref, rtol, atol) <= 1, (n_pad, n_ref)
    torch.testing.assert_close(g_pad, g_ref, rtol=rtol, atol=atol)
    print("%s: loss %.6g / %.6g, grad arena excess %.3g" % (math_mode, l_pad[0], l_ref[0],
                                                            _excess(g_pad, g_ref, rtol, atol)))
