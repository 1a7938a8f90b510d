"""GPU: the exact-fp32 CUDA-core conv kernels (csrc/conv.cu on the gemm_simt_kernel mainloop of csrc/gemm_simt.cuh) at
kernel level, through the C ABI.  They run the whole model under DV3_CONV_MATH=fp32, every shape the tensor-core path
declines in the default mode, the set-up projections of incremental decoding, and they carry the batched-synthesis
guarantee (a batched result is bit-identical to the one-utterance result).

Every GEMM launch gets three checks against an fp64 contraction of the operands the kernel reads (x * dropout mask is
one fp32 multiply in the kernel and in the reference, so both see the same operand):
  (a) exact: integer operands in [-8, 8] (dropout p = 0.5, scale 2).  Every partial sum is an integer below 2^24, so
      fp32 accumulation is exact in any order and the kernel must match fp64 bit for bit.  Catches any missing,
      duplicated or misplaced term: a wrong tap offset, a dropped K chunk, a wrong gate half, a wrong split boundary.
  (b) elementwise, random fp32 operands: |out - R| <= gamma(K) sum |a||b| with gamma(K) = K u / (1 - K u), u = 2^-24,
      K the taps x channels that reach the output (the split's samples for a weight gradient), plus the rounding of
      each epilogue operation and 6 u of the sigmoid (expf is 2 ulp without fast math, then an add and a division).
  (c) norm-wise, full 24-bit mantissas: ||out - R||_2 <= 2^-16 ||R||_2 (fp32 accumulation is ~u sqrt(K/2)).  (a)
      cannot see a GEMM that drops to TF32- or bf16-class operands (small integers are exact in both), and (b) only
      while its worst-case bound stays tighter than the operand rounding; (c) sees it at any K, and each launch proves
      it: the fp64 result of the TF32-rounded operands misses the bound by >= 10x.  (c) is asserted before (b).
Every output is a view into a sentinel-filled buffer: nothing outside it changes and every element inside is written.
"""
import math

import numpy as np
import pytest
import torch

from test_gpu_tc1 import _call, _p, _st, ref_conv
from test_gpu_tc_pairs import GUARD, SENT32, assert_written_inside_only, guarded

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NORM_TOL = 2.0 ** -16
MUTANT_MARGIN = 10.0
SQRT_HALF = 0.7071067811865476
SALT = 11


def gamma(K):
    return K * U / (1 - K * U)


def ints(shape, g):
    return torch.randint(-8, 9, shape, generator=g, device="cuda").float()


def tf32(x):
    """x rounded as cvt.rna.tf32.f32 rounds it: 10 explicit mantissa bits, ties away from zero."""
    return ((x.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def drop_mask(seed, p, shape):
    from oracle import dropout_mask as DM
    return torch.from_numpy(DM.mask(seed, SALT, p, shape)).cuda()


def seed_of(p, value):
    return torch.tensor([value], dtype=torch.int64, device="cuda") if p > 0 else None


def exact_premise(K, scale=1.0):
    """Integer operands in [-8, 8]: every partial sum stays an exactly representable integer."""
    assert K * 8 * 8 * scale < 2 ** 24, K


def ratio(got, want, bound):
    err = (got.double() - want).abs()
    return float((err / bound.clamp_min(1e-300)).max())


def norm_ratio(got, want):
    return float((got.double() - want).norm()) / (NORM_TOL * float(want.norm()))


def check_norm(what, got, want, mutant):
    """(c): the kernel within 2^-16 of ||R||; the TF32-operand mutant at least 10x outside it."""
    c, cm = norm_ratio(got, want), norm_ratio(mutant, want)
    assert c <= 1, (what, c)
    assert cm >= MUTANT_MARGIN, (what, cm)
    return c, cm


def padl(k, dil, causal):
    return (k - 1) * dil if causal else (k - 1) // 2 * dil


def conv_ref(x, w_f, k, dil, causal):
    """fp64 y[b,co,t] = sum_{j,ci} w_f[j,ci,co] x[b,ci,t+off_j]: x (B,Cin,T), w_f [k][Cin][Cout] -> (B,Cout,T)."""
    return ref_conv(x.double().transpose(1, 2), w_f.double().permute(0, 2, 1), k, dil, causal, False)


def dgrad_ref(dab, w_b, k, dil, causal):
    """fp64 dx[b,ci,t] = sum_{j,m} w_b[j,m,ci] dab[b,m,t+padl-j*dil]: dab (B,M,T), w_b [k][M][Cin] -> (B,Cin,T)."""
    return ref_conv(dab.double().transpose(1, 2), w_b.double().permute(0, 2, 1), k, dil, causal, True)


def taps_in_range(T, k, dil, causal, transpose):
    """(T,) fp64: how many of the k taps of output frame t land inside [0, T)."""
    ones = torch.ones(1, T, 1, dtype=torch.float64, device="cuda")
    return ref_conv(ones, torch.ones(k, 1, 1, dtype=torch.float64, device="cuda"), k, dil, causal, transpose)[0, 0]


# ---- tile width: csrc/gemm_simt.cuh pick_bn, with the device's SM count as conv.cu num_sms() reads it ----------------
def pick_bn(n_cols, m_tiles, z=1):
    slots = 2 * torch.cuda.get_device_properties(0).multi_processor_count
    c128 = -(-n_cols // 128) * m_tiles * z
    c64 = -(-n_cols // 64) * m_tiles * z
    w128 = -(-c128 // slots) * 128
    w64 = -(-c64 // slots) * 68
    return 64 if w64 < w128 else 128


def plain_bn(B, Mout, T):
    return pick_bn(B * T, -(-Mout // 128))


def gated_bn(B, C, T):
    return pick_bn(B * T, -(-C // 64))


# ---- launchers ------------------------------------------------------------------------------------------------------
def launch_fwd(x, w_f, bias, k, dil, causal, relu):
    B, Cin, T = x.shape
    Cout = w_f.shape[2]
    n = B * Cout * T
    buf, y = guarded(n)
    _call("dv3_conv1d_fwd", _p(x), _p(w_f), _p(bias), _p(y), B, Cin, Cout, T, k, dil, int(causal), int(relu), _st())
    torch.cuda.synchronize()
    assert_written_inside_only(buf, n)
    return y.view(B, Cout, T)


def launch_gated(x, w_f, bias, spk, k, dil, causal, mode, residual, p, seed):
    B, C, T = x.shape
    n = B * C * T
    (ybuf, y), (abuf, a), (sbuf, s) = guarded(n), guarded(n), guarded(n)
    _call("dv3_convblock_fwd", _p(x), _p(w_f), _p(bias), _p(spk), _p(y), _p(a), _p(s), B, C, T, k, dil, int(causal),
          mode, int(residual), p, _p(seed), SALT, _st())
    torch.cuda.synchronize()
    for buf in (ybuf, abuf, sbuf):
        assert_written_inside_only(buf, n)
    return y.view(B, C, T), a.view(B, C, T), s.view(B, C, T)


def launch_dgrad(dab, w_b, k, dil, causal, p, seed, addmode=0, e1=None, e2=None, alpha=0.0):
    B, M, T = dab.shape
    Cin = w_b.shape[2]
    n = B * Cin * T
    buf, dx = guarded(n)
    _call("dv3_conv1d_dgrad", _p(dab), _p(w_b), _p(dx), B, M, Cin, T, k, dil, int(causal), p, _p(seed), SALT, addmode,
          _p(e1), _p(e2), alpha, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(buf, n)
    return dx.view(B, Cin, T)


# ---- 1. plain conv forward ------------------------------------------------------------------------------------------
FWD_CASES = [
    # (B, Cin, Cout, T, k, dilation, causal)
    (1, 80, 256, 37, 1, 1, False),       # mel input: the default mode's small-T route
    (2, 17, 130, 131, 3, 9, False),      # BK tail (Cin % 16), Cout % 128 = 2, odd T: scalar epilogue
    (3, 513, 513, 64, 2, 1, False),      # even k: asymmetric padding; float4 epilogue
    (1, 64, 200, 20, 8, 3, True),        # k = MAX_TAPS, causal halo 21 > T
    (4, 33, 64, 5, 5, 27, False),        # halo wider than T on both sides
    (16, 256, 512, 200, 1, 1, False),    # large N
    (32, 256, 512, 200, 3, 1, False),    # enough tiles for 128-column tiles
]


def _fwd_id(c):
    return "B%d_Cin%d_Cout%d_T%d_k%d_d%d%s" % (c[:6] + ("_causal" if c[6] else "",))


@pytest.mark.parametrize("case", FWD_CASES, ids=_fwd_id)
def test_conv1d_fwd(case):
    B, Cin, Cout, T, k, dil, causal = case
    g = torch.Generator(device="cuda").manual_seed(Cin * 7 + Cout + T + k)
    # (a) exact
    x, w = ints((B, Cin, T), g), ints((k, Cin, Cout), g)
    exact_premise(k * Cin)
    y = launch_fwd(x, w, None, k, dil, causal, False)
    assert torch.equal(y.double(), conv_ref(x, w, k, dil, causal)), "exact forward"
    # (b), (c)
    x = torch.randn(B, Cin, T, device="cuda", generator=g)
    w = torch.randn(k, Cin, Cout, device="cuda", generator=g) * (k * Cin) ** -0.5
    bias = torch.randn(Cout, device="cuda", generator=g) * 0.1
    D = conv_ref(x, w, k, dil, causal)
    bD = gamma(Cin * taps_in_range(T, k, dil, causal, False)) * conv_ref(x.abs(), w.abs(), k, dil, causal)
    mut = conv_ref(tf32(x), tf32(w), k, dil, causal)
    worst, c, cm = 0.0, 0.0, math.inf
    for has_bias in (False, True):
        for relu in (False, True):
            y = launch_fwd(x, w, bias if has_bias else None, k, dil, causal, relu)
            bv = bias.double()[None, :, None] if has_bias else torch.zeros((), dtype=torch.float64, device="cuda")
            want, mwant = D + bv, mut + bv
            bound = bD * (1 + U) + U * want.abs()
            if relu:
                want, mwant = want.clamp_min(0.0), mwant.clamp_min(0.0)
            cc, cmm = check_norm((has_bias, relu), y, want, mwant)
            r = ratio(y, want, bound)
            assert r <= 1, (has_bias, relu, r)
            worst = max(worst, r)
            c, cm = max(c, cc), min(cm, cmm)
    print("conv1d_fwd %s BN %d: (b) %.3g, (c) %.3g, TF32 mutant %.3g" % (case, plain_bn(B, Cout, T), worst, c, cm))


# ---- 2. gated forward -----------------------------------------------------------------------------------------------
GATED_CASES = [
    # (B, C, T, k, dilation, causal, mode, residual, speaker addend, p_drop): mode 0 = GLU, 1 = highway
    (2, 80, 37, 3, 1, False, 0, True, False, 0.0),      # Cg % 64 = 16, odd T
    (3, 96, 128, 5, 2, True, 0, False, True, 0.05),     # Cg % 64 = 32, float4 epilogue
    (4, 64, 4, 8, 3, False, 1, False, False, 0.5),      # k = MAX_TAPS, halo > T, T = 4
    (2, 128, 131, 2, 1, False, 1, False, True, 0.0),    # even k: asymmetric padding
    (1, 200, 200, 3, 9, True, 0, True, True, 0.5),      # one row, Cg % 64 = 8
    (2, 64, 37, 8, 1, True, 0, False, False, 0.05),     # k = MAX_TAPS causal
    (3, 200, 4, 5, 1, False, 1, False, True, 0.05),     # halo > T on both sides
    (32, 200, 200, 5, 1, False, 0, True, False, 0.05),  # enough tiles for 128-column tiles
]


def _gated_id(c):
    return "B%d_C%d_T%d_k%d_d%d%s_%s%s%s_p%g" % (c[0], c[1], c[2], c[3], c[4], "_causal" if c[5] else "",
                                                "glu" if c[6] == 0 else "highway", "_res" if c[7] else "",
                                                "_spk" if c[8] else "", c[9])


def gated_ref(D, bD, bias, spk, x, mode, residual):
    """fp64 (a, s, y) of the gated epilogue on the GEMM result D (B, 2C, T) and their elementwise bounds, given the
    GEMM bound bD: each fp32 operation adds u of its result, the sigmoid 6 u."""
    C = x.shape[1]
    bd = bias.double()[None, :, None]
    sp = spk.double() if spk is not None else torch.zeros_like(D[:, :C])
    a = D[:, :C] + bd[:, :C] + sp
    ea = bD[:, :C] + 2 * U * (D[:, :C].abs() + bd[:, :C].abs() + sp.abs() + bD[:, :C])
    z = D[:, C:] + bd[:, C:]
    ez = bD[:, C:] + U * (z.abs() + bD[:, C:])
    s = torch.sigmoid(z)
    es = (s * (1 - s) + ez) * ez + 6 * U * s        # |sigmoid''| < 0.1, so s (1 - s) + ez bounds the slope nearby
    r = x.double()
    if mode == 0:
        y = a * s
        ey = s * ea + a.abs() * es + ea * es + U * (y.abs() + s * ea + a.abs() * es)
        if residual:
            t = y + r
            et = ey + U * (t.abs() + ey)
            y = t * SQRT_HALF                          # the kernel's constant is sqrt(0.5) rounded to fp32 (0.3 u)
            ey = SQRT_HALF * (et + 2.5 * U * (t.abs() + et))
    else:
        y = s * a + (1 - s) * r
        ey = s * ea + (a - r).abs() * es + ea * es + 4 * U * ((s * a).abs() + ((1 - s) * r).abs() + ea + es * r.abs())
    return a, ea, s, es, y, ey


@pytest.mark.parametrize("case", GATED_CASES, ids=_gated_id)
def test_convblock_fwd(case):
    B, C, T, k, dil, causal, mode, residual, has_spk, p = case
    g = torch.Generator(device="cuda").manual_seed(C * 5 + T + 13 * k)
    K = C * taps_in_range(T, k, dil, causal, False)
    # (a) exact: save_a = conv(x * mask)[:C] + bias + speaker addend, all integers
    pe = 0.5 if p > 0 else 0.0
    seed = seed_of(pe, 777 + C)
    x, w = ints((B, C, T), g), ints((k, C, 2 * C), g)
    bias, spk = ints((2 * C,), g), ints((B, C, T), g) if has_spk else None
    exact_premise(k * C, 2.0 if pe else 1.0)
    _, a, _ = launch_gated(x, w, bias, spk, k, dil, causal, mode, residual, pe, seed)
    xm = x * drop_mask(seed, pe, (B, C, T))
    want = conv_ref(xm, w, k, dil, causal)[:, :C] + bias.double()[None, :C, None]
    if has_spk:
        want += spk.double()
    assert torch.equal(a.double(), want), "exact save_a"
    # (b), (c)
    seed = seed_of(p, 4242 + T)
    x = torch.randn(B, C, T, device="cuda", generator=g)
    w = torch.randn(k, C, 2 * C, device="cuda", generator=g) * (k * C) ** -0.5
    bias = torch.randn(2 * C, device="cuda", generator=g) * 0.1
    spk = torch.randn(B, C, T, device="cuda", generator=g) * 0.3 if has_spk else None
    y, a, s = launch_gated(x, w, bias, spk, k, dil, causal, mode, residual, p, seed)
    xm = x * drop_mask(seed, p, (B, C, T))
    D = conv_ref(xm, w, k, dil, causal)
    bD = gamma(K) * conv_ref(xm.abs(), w.abs(), k, dil, causal)
    a_ref, ea, s_ref, es, y_ref, ey = gated_ref(D, bD, bias, spk, x, mode, residual)
    mut = conv_ref(tf32(xm), tf32(w), k, dil, causal)[:, :C] + (a_ref - D[:, :C])
    c, cm = check_norm("save_a", a, a_ref, mut)
    ra, rs, ry = ratio(a, a_ref, ea), ratio(s, s_ref, es), ratio(y, y_ref, ey)
    assert ra <= 1 and rs <= 1 and ry <= 1, (ra, rs, ry)
    print("convblock_fwd %s BN %d: (b) a %.3g s %.3g y %.3g, (c) %.3g, TF32 mutant %.3g" % (
        case, gated_bn(B, C, T), ra, rs, ry, c, cm))


# ---- 3. data gradient -----------------------------------------------------------------------------------------------
DGRAD_CASES = [(B, Cout, Cin, T, k, dil, causal) for B, Cin, Cout, T, k, dil, causal in FWD_CASES]


def _dgrad_id(c):
    return "B%d_M%d_Cin%d_T%d_k%d_d%d%s" % (c[:6] + ("_causal" if c[6] else "",))


@pytest.mark.parametrize("case", DGRAD_CASES, ids=_dgrad_id)
def test_conv1d_dgrad(case):
    B, M, Cin, T, k, dil, causal = case
    g = torch.Generator(device="cuda").manual_seed(M * 3 + Cin + T + k)
    # (a) exact, with and without the output dropout (scale 2)
    dab, w = ints((B, M, T), g), ints((k, M, Cin), g)
    D = dgrad_ref(dab, w, k, dil, causal)
    for pe in (0.0, 0.5):
        exact_premise(k * M, 2.0 if pe else 1.0)
        seed = seed_of(pe, 99 + M)
        dx = launch_dgrad(dab, w, k, dil, causal, pe, seed)
        assert torch.equal(dx.double(), D * drop_mask(seed, pe, (B, Cin, T)).double()), ("exact dgrad", pe)
    # (b), (c): addmode 0 / 1 (alpha = sqrt(0.5)) / 2, dropout off, 0.5, 0.05 (mask index (b*Cin+ci)*T+t)
    dab = torch.randn(B, M, T, device="cuda", generator=g)
    w = torch.randn(k, M, Cin, device="cuda", generator=g) * (k * M) ** -0.5
    # addend below the GEMM term (which can be one tap of k), so that (c) still weighs the GEMM
    e1 = torch.randn(B, Cin, T, device="cuda", generator=g) * 0.25
    e2 = torch.rand(B, Cin, T, device="cuda", generator=g)
    D = dgrad_ref(dab, w, k, dil, causal)
    bD = gamma(M * taps_in_range(T, k, dil, causal, True)) * dgrad_ref(dab.abs(), w.abs(), k, dil, causal)
    mut = dgrad_ref(tf32(dab), tf32(w), k, dil, causal)
    alpha = float(np.float32(SQRT_HALF))
    worst, c, cm = 0.0, 0.0, math.inf
    for addmode in (0, 1, 2):
        for p in (0.0, 0.5, 0.05):
            seed = seed_of(p, 31 * addmode + T)
            dx = launch_dgrad(dab, w, k, dil, causal, p, seed, addmode, e1 if addmode else None,
                              e2 if addmode == 2 else None, SQRT_HALF if addmode == 1 else 0.0)
            m = drop_mask(seed, p, (B, Cin, T)).double()
            t = (alpha * e1.double() if addmode == 1 else e1.double() * (1 - e2.double()) if addmode == 2
                 else torch.zeros_like(D))
            want = D * m + t
            bound = m * bD * (1 + 2 * U) + 2 * U * (D * m).abs() + 3 * U * t.abs()
            cc, cmm = check_norm((addmode, p), dx, want, mut * m + t)
            r = ratio(dx, want, bound)
            assert r <= 1, (addmode, p, r)
            worst = max(worst, r)
            c, cm = max(c, cc), min(cm, cmm)
    print("conv1d_dgrad %s BN %d: (b) %.3g, (c) %.3g, TF32 mutant %.3g" % (case, plain_bn(B, Cin, T), worst, c, cm))


# ---- 4. weight gradient ---------------------------------------------------------------------------------------------
WGRAD_CASES = [
    # (B, M, Cin, T, k, dilation, causal, layout, p_drop): layout "v" = (M, Cin, k) as ops._wgrad_conv,
    # "convT" = ConvTranspose1d's v (Cin, Cout, 2) with M = 2 * Cout rows ordered (j, co), as ops._CONVT
    (2, 64, 80, 37, 3, 2, False, "v", 0.0),         # B*T = 74 < 128: nsplit = 1; B*T % 16 != 0
    (4, 128, 96, 131, 5, 1, True, "v", 0.05),       # nsplit > 1, B*T % 16 != 0
    (16, 256, 128, 200, 3, 1, False, "v", 0.5),     # many splits
    (3, 130, 17, 64, 8, 3, False, "v", 0.0),        # even k = MAX_TAPS, M % 128 = 2, Cin % 64 = 17, halo > T
    (8, 160, 256, 50, 1, 1, False, "convT", 0.0),   # ConvTranspose layout, nsplit > 1
    (1, 512, 513, 37, 1, 1, False, "convT", 0.0),   # ConvTranspose layout, nsplit = 1
]


def _wgrad_id(c):
    return "B%d_M%d_Cin%d_T%d_k%d_d%d%s_%s_p%g" % (c[:6] + ("_causal" if c[6] else "",) + c[7:])


def shifted_rows(x, k, dil, causal):
    """x (B,C,T) fp64 -> [k] of (B*T, C): row b*T+t of tap j holds x[b, :, t + off_j] (zero outside [0, T))."""
    B, C, T = x.shape
    rows = []
    for j in range(k):
        off = j * dil - padl(k, dil, causal)
        sh = torch.zeros_like(x)
        lo, hi = max(0, -off), min(T, T - off)
        if hi > lo:
            sh[:, :, lo:hi] = x[:, :, lo + off:hi + off]
        rows.append(sh.transpose(1, 2).reshape(B * T, C))
    return rows


def wgrad_ref(dab, x, k, dil, causal, n0, n1):
    """fp64 (M, Cin, k) = sum over samples n = b*T + t in [n0, n1) of dab[b,m,t] x[b,ci,t+off_j]."""
    B, M, T = dab.shape
    a = dab.double().transpose(1, 2).reshape(B * T, M)[n0:n1]
    return torch.stack([a.t() @ xs[n0:n1] for xs in shifted_rows(x.double(), k, dil, causal)], dim=2)


def run_wgrad(dab, x, k, dil, causal, layout, p, seed):
    """Launch into a sentinel-guarded [nsplit][numel] workspace -> (slots (nsplit, M, Cin, k), split n-ranges)."""
    from deepvoice3_pytorch_b200._lib import lib
    B, M, T = dab.shape
    Cin = x.shape[1]
    nsplit = lib.raw("dv3_conv1d_wgrad_nsplit")(B, M, Cin, T, k)
    chunks = -(-B * T // 16)                                       # 16-sample K chunks, split as the launcher splits
    cps = -(-chunks // nsplit)
    ranges = [(min(B * T, s * cps * 16), min(B * T, (s + 1) * cps * 16)) for s in range(nsplit)]
    numel = M * Cin * k
    if layout == "v":
        ms, s_m, s_mh, s_n, s_j = M, Cin * k, 0, k, 1
    else:
        assert k == 1 and M % 2 == 0
        ms, s_m, s_mh, s_n, s_j = M // 2, 2, 1, M, 0
    buf, parts = guarded(nsplit * numel)
    _call("dv3_conv1d_wgrad", _p(dab), _p(x), _p(parts), numel, B, M, Cin, T, k, dil, int(causal), p, _p(seed), SALT,
          ms, s_m, s_mh, s_n, s_j, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(buf, nsplit * numel)
    m = torch.arange(M, device="cuda")[:, None, None]
    n = torch.arange(Cin, device="cuda")[None, :, None]
    j = torch.arange(k, device="cuda")[None, None, :]
    idx = (m % ms) * s_m + (m // ms) * s_mh + n * s_n + j * s_j
    return parts.view(nsplit, numel)[:, idx], ranges


@pytest.mark.parametrize("case", WGRAD_CASES, ids=_wgrad_id)
def test_conv1d_wgrad(case):
    B, M, Cin, T, k, dil, causal, layout, p = case
    g = torch.Generator(device="cuda").manual_seed(M + 3 * Cin + T + k)
    # (a) exact, every split slot
    pe = 0.5 if p > 0 else 0.0
    seed = seed_of(pe, 555 + Cin)
    dab, x = ints((B, M, T), g), ints((B, Cin, T), g)
    slots, ranges = run_wgrad(dab, x, k, dil, causal, layout, pe, seed)
    xm = x * drop_mask(seed, pe, (B, Cin, T))
    for s, (n0, n1) in enumerate(ranges):
        exact_premise(n1 - n0, 2.0 if pe else 1.0)
        assert torch.equal(slots[s].double(), wgrad_ref(dab, xm, k, dil, causal, n0, n1)), ("exact slot", s)
    # (b) per slot, (c) on the sum of the slots
    seed = seed_of(p, 808 + T)
    dab = torch.randn(B, M, T, device="cuda", generator=g)
    x = torch.randn(B, Cin, T, device="cuda", generator=g)
    slots, ranges = run_wgrad(dab, x, k, dil, causal, layout, p, seed)
    xm = x * drop_mask(seed, p, (B, Cin, T))
    N = B * T
    c, cm = check_norm("wgrad", slots.double().sum(0), wgrad_ref(dab, xm, k, dil, causal, 0, N),
                       wgrad_ref(tf32(dab), tf32(xm), k, dil, causal, 0, N))
    worst = 0.0
    for s, (n0, n1) in enumerate(ranges):
        want = wgrad_ref(dab, xm, k, dil, causal, n0, n1)
        bound = gamma(n1 - n0) * wgrad_ref(dab.abs(), xm.abs(), k, dil, causal, n0, n1)
        r = ratio(slots[s], want, bound)
        assert r <= 1, (s, r)
        worst = max(worst, r)
    print("conv1d_wgrad %s nsplit %d: (b) %.3g, (c) %.3g, TF32 mutant %.3g" % (case, len(ranges), worst, c, cm))


# ---- 5. tile widths and batch invariance ----------------------------------------------------------------------------
def test_case_lists_reach_both_tile_widths():
    plain = {plain_bn(c[0], c[2], c[3]) for c in FWD_CASES}
    gated = {gated_bn(c[0], c[1], c[2]) for c in GATED_CASES}
    assert plain == {64, 128} and gated == {64, 128}, (plain, gated)


ROWS = (0, 17, 31)


def test_batch_invariance():
    """Row b of a 32-row launch is bit-identical to row b launched alone, for the plain forward, the gated forward and
    the data gradient, on shapes where the 32-row launch takes 128-column tiles and the single row 64-column tiles:
    the kernel-level basis of the batched-synthesis guarantee."""
    g = torch.Generator(device="cuda").manual_seed(5)
    B, T, k = 32, 200, 3
    # plain forward (+ bias, ReLU)
    Cin, Cout = 256, 512
    assert plain_bn(B, Cout, T) == 128 and plain_bn(1, Cout, T) == 64
    x = torch.randn(B, Cin, T, device="cuda", generator=g)
    w = torch.randn(k, Cin, Cout, device="cuda", generator=g) * (k * Cin) ** -0.5
    bias = torch.randn(Cout, device="cuda", generator=g)
    y = launch_fwd(x, w, bias, k, 1, False, True)
    for b in ROWS:
        assert torch.equal(y[b:b + 1], launch_fwd(x[b:b + 1].contiguous(), w, bias, k, 1, False, True)), ("fwd", b)
    # gated forward (GLU + residual + speaker addend)
    C = 200
    assert gated_bn(B, C, T) == 128 and gated_bn(1, C, T) == 64
    x = torch.randn(B, C, T, device="cuda", generator=g)
    w = torch.randn(k, C, 2 * C, device="cuda", generator=g) * (k * C) ** -0.5
    bias = torch.randn(2 * C, device="cuda", generator=g) * 0.1
    spk = torch.randn(B, C, T, device="cuda", generator=g) * 0.3
    outs = launch_gated(x, w, bias, spk, k, 1, True, 0, True, 0.0, None)
    for b in ROWS:
        one = launch_gated(x[b:b + 1].contiguous(), w, bias, spk[b:b + 1].contiguous(), k, 1, True, 0, True, 0.0, None)
        for name, full, single in zip(("y", "a", "s"), outs, one):
            assert torch.equal(full[b:b + 1], single), ("gated", name, b)
    # data gradient (highway addend)
    M, Cin = 256, 512
    assert plain_bn(B, Cin, T) == 128 and plain_bn(1, Cin, T) == 64
    dab = torch.randn(B, M, T, device="cuda", generator=g)
    w = torch.randn(k, M, Cin, device="cuda", generator=g) * (k * M) ** -0.5
    e1 = torch.randn(B, Cin, T, device="cuda", generator=g)
    e2 = torch.rand(B, Cin, T, device="cuda", generator=g)
    dx = launch_dgrad(dab, w, k, 1, False, 0.0, None, 2, e1, e2)
    for b in ROWS:
        one = launch_dgrad(dab[b:b + 1].contiguous(), w, k, 1, False, 0.0, None, 2, e1[b:b + 1].contiguous(),
                           e2[b:b + 1].contiguous())
        assert torch.equal(dx[b:b + 1], one), ("dgrad", b)


# ---- 6. gate backward, bias backward --------------------------------------------------------------------------------
def prefilled(values):
    """A sentinel-guarded buffer whose inside holds `values` (a bias gradient accumulates into it)."""
    buf, v = guarded(values.numel())
    v.copy_(values)
    return buf, v


def check_row_sums(got, pre, v, ev, what):
    """got = pre + sum over (b, t) of v (B, R, T) in any order, each term within ev of v."""
    n = v.shape[0] * v.shape[2] + 1
    want = pre.double() + v.sum((0, 2))
    bound = gamma(n) * (pre.double().abs() + (v.abs() + ev).sum((0, 2))) + ev.sum((0, 2))
    r = ratio(got, want, bound)
    assert r <= 1, (what, r)
    return r


GATE_BWD_CASES = [
    # (B, C, T, mode, residual)
    (2, 80, 37, 0, 1),
    (3, 96, 128, 0, 0),
    (2, 200, 131, 1, 0),
    (1, 64, 33, 1, 1),      # highway ignores the residual flag
]


@pytest.mark.parametrize("case", GATE_BWD_CASES, ids=lambda c: "B%d_C%d_T%d_%s%s" % (
    c[0], c[1], c[2], "glu" if c[3] == 0 else "highway", "_res" if c[4] else ""))
def test_convblock_gate_bwd(case):
    B, C, T, mode, residual = case
    g = torch.Generator(device="cuda").manual_seed(C + T + mode)
    dy, a, x = (torch.randn(B, C, T, device="cuda", generator=g) for _ in range(3))
    s = torch.rand(B, C, T, device="cuda", generator=g)
    pre = torch.randn(2 * C, device="cuda", generator=g)
    n = B * 2 * C * T
    dbuf, dab = guarded(n)
    bbuf, dbias = prefilled(pre)
    _call("dv3_convblock_gate_bwd", _p(dy), _p(a), _p(s), _p(x), _p(dab), _p(dbias), B, C, T, mode, residual, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(dbuf, n)
    assert_written_inside_only(bbuf, 2 * C)
    gs = SQRT_HALF if mode == 0 and residual else 1.0
    gd, sd = dy.double() * gs, s.double()
    da = gd * sd
    db = gd * (a.double() if mode == 0 else a.double() - x.double()) * sd * (1 - sd)
    dab = dab.view(B, 2 * C, T)
    eda, edb = 3 * U * da.abs(), 7 * U * db.abs()     # the fp32 sqrt(0.5) (0.3 u) and one u per operation
    ra, rb = ratio(dab[:, :C], da, eda), ratio(dab[:, C:], db, edb)
    assert ra <= 1 and rb <= 1, (ra, rb)
    rbias = check_row_sums(dbias, pre, torch.cat([da, db], 1), torch.cat([eda, edb], 1), "dbias")
    print("gate_bwd %s: da %.3g db %.3g dbias %.3g" % (case, ra, rb, rbias))


@pytest.mark.parametrize("relu", [1, 0])
def test_bias_act_bwd(relu):
    B, C, T = 3, 130, 101
    g = torch.Generator(device="cuda").manual_seed(7 + relu)
    dy, y = (torch.randn(B, C, T, device="cuda", generator=g) for _ in range(2))
    r = torch.rand(B, C, T, device="cuda", generator=g)
    y = torch.where(r < 0.05, 0.0, torch.where(r < 0.1, -0.0, y))        # +0 and -0 do not pass the ReLU
    pre = torch.randn(C, device="cuda", generator=g)
    dy0 = dy.clone()
    bbuf, dbias = prefilled(pre)
    n = B * C * T
    if relu:
        rbuf, dyr = guarded(n)
        _call("dv3_bias_act_bwd", _p(dy), _p(y), _p(dyr), _p(dbias), B, C, T, 1, _st())
        torch.cuda.synchronize()
        assert_written_inside_only(rbuf, n)
        v = torch.where(y > 0, dy, 0.0)
        assert torch.equal(dyr.view(B, C, T).view(torch.int32), v.view(torch.int32)), "dyr"
    else:
        # the ConvTranspose call: no ReLU, dyr = y = NULL; writes nothing but dbias
        _call("dv3_bias_act_bwd", _p(dy), None, None, _p(dbias), B, C, T, 0, _st())
        torch.cuda.synchronize()
        v = dy
        # and with a dyr buffer, no ReLU leaves it untouched
        rbuf, dyr = guarded(n)
        bbuf2, dbias2 = prefilled(pre)
        _call("dv3_bias_act_bwd", _p(dy), _p(y), _p(dyr), _p(dbias2), B, C, T, 0, _st())
        torch.cuda.synchronize()
        assert bool((rbuf.view(torch.int32) == SENT32).all()), "dyr written without ReLU"
        assert_written_inside_only(bbuf2, C)
        check_row_sums(dbias2, pre, dy.double(), torch.zeros_like(dy, dtype=torch.float64), "dbias, dyr given")
    assert torch.equal(dy, dy0), "dy written"
    assert_written_inside_only(bbuf, C)
    rb = check_row_sums(dbias, pre, v.double(), torch.zeros_like(v, dtype=torch.float64), "dbias")
    print("bias_act_bwd relu=%d: dbias %.3g" % (relu, rb))


# ---- 7. ConvTranspose time interleave -------------------------------------------------------------------------------
def test_interleave2():
    B, C, T = 3, 37, 41
    g = torch.Generator(device="cuda").manual_seed(17)
    n = B * 2 * C * T
    x = torch.randn(B, 2 * C, T, device="cuda", generator=g)          # rows ordered (j, co)
    want = x.view(B, 2, C, T).permute(0, 2, 3, 1).reshape(B, C, 2 * T)  # out[b, co, 2t + j] = in[b, j*C + co, t]
    obuf, out = guarded(n)
    _call("dv3_interleave2", _p(x), _p(out), B, C, T, 0, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(obuf, n)
    assert torch.equal(out.view(B, C, 2 * T).view(torch.int32), want.view(torch.int32)), "forward"
    back_buf, back = guarded(n)
    _call("dv3_interleave2", _p(out), _p(back), B, C, T, 1, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(back_buf, n)
    assert torch.equal(back.view(B, 2 * C, T).view(torch.int32), x.view(torch.int32)), "round trip"
    z = torch.randn(B, C, 2 * T, device="cuda", generator=g)
    ibuf, inv = guarded(n)
    _call("dv3_interleave2", _p(z), _p(inv), B, C, T, 1, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(ibuf, n)
    want = z.view(B, C, T, 2).permute(0, 3, 1, 2).reshape(B, 2 * C, T)
    assert torch.equal(inv.view(B, 2 * C, T).view(torch.int32), want.view(torch.int32)), "inverse"
