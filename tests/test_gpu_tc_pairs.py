"""GPU: the default two-plane tensor-core mode (ops.conv_math = "tc", DESIGN.md section 2.1) at kernel level, the NPL = 2
counterpart of tests/test_gpu_tc1.py.  Calls the C ABI directly.

Splits: dv3_tc_split_input (fp16 pair + bf16 pair of x * dropout mask), dv3_tc_gate_bwd_split_npl and
dv3_tc_grad_split_npl with npl = 2, bit for bit against common.cuh split_pair restated in torch (split_pair below):
hi = rn16(clamp(x)), lo = rn16((x - hi) * 2^11), clamp to +-65504 in the fp16 pair only.  Pad columns come out zero, the
logical extent zeroes frames t >= tmult * tlen, nothing past the planes is written.

GEMMs: every NPL = 2 instantiation of tc_conv_kernel (gated <2,64,32>, conv <1,128,32>, <1,64,64>, <1,64,32>) and
tc_wgrad_mn_kernel<2>, on pair planes of random fp32 data, against the fp64 value of the three products the kernel
issues, R = A_hi.W_hi + 2^-11 (A_hi.W_lo + A_lo.W_hi) (16-bit products are exact in fp64; lo.lo is not part of the
arithmetic), with the launch's epilogue applied in fp64.  Two checks per launch:
  (a) elementwise, the worst-case bound of tests/test_gpu_tc1.py on each accumulator plus the truncation compensation:
      |out - R| <= c1(K) (|A_hi||W_hi| + 2^-11 (|A_hi||W_lo| + |A_lo||W_hi|)) + (gamma n_mma + 2^-23) |R|,
      n_mma computed as the launcher computes it, gamma as capi.cu reads it (DV3_TC_GAMMA);
  (b) norm-wise, the cross-term discriminator: ||out - R||_2 <= min(||2^-11 A_hi.W_lo||_2, ||2^-11 A_lo.W_hi||_2) / 20.
      (a) alone cannot see a missing, mis-scaled or mis-fed cross MMA (its slack is larger than either cross term);
      (b) fails for each of those.
Every output is a view into a sentinel-filled buffer: nothing outside (B, Nc, T) (or outside the nsplit weight-gradient
slots) changes, and every element inside is written.  One case per instantiation with pad columns (Kc % 8 != 0; the
gated kernel and <1,64,64> take C % 128 == 0 / Kc % 64 == 0, so they have none) reruns with NaN in every pad column of
both planes and must give the same bits.

Truncation compensation: the systematic bias <out - R, R> / <R, R> of long contractions (the metric of
tools/trunc_bias.py) stays within a quarter of the uncompensated shrink gamma0 n_mma; a subprocess with DV3_TC_GAMMA=0
shows the shrink (more than half of gamma0 n_mma), so the compensation is there, once, with the right sign and count.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_tc1 import _call, _p, _st, c1, ratio, ref_conv

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
U = 2.0 ** -24
LO = 2.0 ** -11
GAMMA0 = 0.56 * 2.0 ** -25                 # capi.cu default (units of 2^-25 per MMA)
NAN16 = {F16: 0x7E00, BF16: 0x7FC0}        # quiet NaN bit patterns of the two plane formats
SENT16 = 0x7A5B                            # plane sentinel (int16)
SENT32 = 0x7FC00BAD                        # output sentinel (a NaN with a payload, int32)
GUARD = 64                                 # sentinel elements on each side of an output


def gamma():
    """The per-MMA compensation coefficient as capi.cu reads it: DV3_TC_GAMMA in units of 2^-25, default 0.56."""
    e = os.environ.get("DV3_TC_GAMMA")
    return (0.56 if e is None else float(e or 0)) * 2.98023224e-8


def pad8(n):
    return (n + 7) // 8 * 8


def split_pair(x, f16):
    """common.cuh split_pair on fp32 x -> [2, *x.shape] 16-bit planes (hi, lo)."""
    if f16:
        x = x.clamp(-65504.0, 65504.0)
    dt = F16 if f16 else BF16
    hi = x.to(dt)
    return torch.stack([hi, ((x - hi.float()) * 2048.0).to(dt)])


def pair_planes(x, f16):
    """(..., K) fp32 -> [2][...][pad8(K)] pair planes, pad columns zero."""
    p = torch.zeros(2, *x.shape[:-1], pad8(x.shape[-1]), dtype=F16 if f16 else BF16, device=x.device)
    p[..., :x.shape[-1]] = split_pair(x, f16)
    return p


# ---- launcher configuration (tc_gemm.cu dv3_tc_conv / dv3_tc_convblock_fwd with npl = 2) -----------------------------
STAGES = {(2, 64, 32): 4, (1, 128, 32): 4, (1, 64, 64): 3, (1, 64, 32): 6}     # (NBOX, BR, BK) -> ring depth (TcCfg)


def conv_config(B, Kc, Nc, T, k):
    """(NBOX, BR, BK), K-iterations per tile, n_mma of the compensation, number of tiles."""
    t_tiles = -(-T // 128)
    tiles128 = t_tiles * -(-Nc // 128) * B
    narrow = Nc > 64 and (k == 1 or Nc % 64 == 0) and tiles128 < 100
    bk = 64 if narrow and Kc % 64 == 0 else 32
    br = 64 if narrow else 128
    kb_n = -(-Kc // bk)
    return (1, br, bk), k * kb_n, k * kb_n * bk // 16, t_tiles * -(-Nc // br) * B


def gated_config(B, C, T, k):
    kb_n = C // 32
    return (2, 64, 32), k * kb_n, k * kb_n * 2, -(-T // 128) * (C // 64) * B


# ---- helpers ----------------------------------------------------------------------------------------------------------
def guarded(n):
    """A sentinel-filled fp32 buffer and the n-element view of it a launch writes into."""
    buf = torch.full((n + 2 * GUARD,), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    return buf, buf[GUARD:GUARD + n]


def assert_written_inside_only(buf, n):
    bits = buf.view(torch.int32)
    assert bool((bits[:GUARD] == SENT32).all()) and bool((bits[GUARD + n:] == SENT32).all()), "write outside"
    assert bool(torch.isfinite(buf[GUARD:GUARD + n]).all()), "element left unwritten"


def sentinel_planes(*shape, dtype, extra=256):
    """16-bit sentinel buffer with `extra` elements past the planes (checked untouched by planes_untouched_past)."""
    n = math.prod(shape)
    buf = torch.full((n + extra,), SENT16, dtype=torch.int16, device="cuda")
    return buf, buf[:n].view(dtype).view(*shape)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def pair_reference(a, w, fn):
    """fp64 R, the two cross terms (scaled), and the |.| term of the bound, from pair planes (pad columns sliced off)."""
    Ah, Al, Wh, Wl = a[0].double(), a[1].double(), w[0].double(), w[1].double()
    x1, x2 = LO * fn(Ah, Wl), LO * fn(Al, Wh)
    R = fn(Ah, Wh) + x1 + x2
    absb = fn(Ah.abs(), Wh.abs()) + LO * (fn(Ah.abs(), Wl.abs()) + fn(Al.abs(), Wh.abs()))
    return R, x1, x2, absb


def discriminator(err, x1, x2):
    """||err||_2 over min(||x1||_2, ||x2||_2) / 20: <= 1 only if both cross products are there, each once."""
    return float(err.norm()) / (min(float(x1.norm()), float(x2.norm())) / 20.0)


def poison_pads(p, K):
    """A copy of pair planes p with NaN in every pad column [K, pad8(K))."""
    q = p.clone()
    q.view(torch.int16)[..., K:] = NAN16[p.dtype]
    return q


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 1. split kernels, bit for bit ------------------------------------------------------------------------------------
def _special_values(x, g):
    """Sprinkle x with values past the fp16 range and in its subnormal range (~1e-6), and fp16 range edges."""
    r = torch.rand(x.shape, device="cuda", generator=g)
    x = torch.where(r < 0.05, x * 4e4, x)                   # about half of these land past +-65504
    x = torch.where((r >= 0.05) & (r < 0.1), x * 1e-6, x)
    flat = x.view(-1)
    edge = torch.tensor([65504.0, -65504.0, 65519.0, 65520.0, -7e4, 1e6, 65500.0, 2.0 ** -24 * 1.5, -1e-7, 0.0],
                        device="cuda")
    flat[:edge.numel()] = edge
    return x


SPLIT_INPUT_CASES = [
    # (B, C, T, p_drop, ext): channel tails (C % 64, C % 8), T % 4 == 0 (float4 loads) or not (scalar loads)
    (2, 8, 64, 0.0, False),
    (3, 16, 37, 0.3, False),
    (2, 80, 100, 0.3, True),
    (3, 136, 101, 0.0, True),
    (2, 513, 203, 0.3, False),
    (2, 513, 128, 0.0, True),
]


@pytest.mark.parametrize("case", SPLIT_INPUT_CASES, ids=lambda c: "B%d_C%d_T%d_p%g%s" % (
    c[0], c[1], c[2], c[3], "_ext" if c[4] else ""))
def test_split_input_pairs(case):
    from oracle import dropout_mask as DM
    B, C, T, p, ext = case
    g = torch.Generator(device="cuda").manual_seed(C * 3 + T)
    x = _special_values(torch.randn(B, C, T, device="cuda", generator=g), g)
    seed = torch.tensor([2024 + C], dtype=torch.int64, device="cuda")
    Cp = pad8(C)
    hbuf, btc = sentinel_planes(2, B, T, Cp, dtype=F16)
    wbuf, bct = sentinel_planes(2, B, T, Cp, dtype=BF16)
    tmult, tlen = 4, torch.tensor([T // 6], dtype=torch.int64, device="cuda")
    if ext:
        _call("dv3_tc_split_input_ext", _p(x), _p(btc), 2, _p(bct), B, C, T, p, _p(seed), 7, _p(tlen), tmult, _st())
    else:
        _call("dv3_tc_split_input", _p(x), _p(btc), 2, _p(bct), B, C, T, 3, 1, 0, p, _p(seed), 7, _st())
    torch.cuda.synchronize()
    m = torch.from_numpy(DM.mask(seed, 7, p, (B, C, T))).cuda()
    xm = x * m                                               # the kernel's one fp32 multiply (x * 1 without dropout)
    if ext:
        xm[:, :, tmult * int(tlen):] = 0.0
    v = xm.transpose(1, 2)
    assert same_bits(btc[..., :C], split_pair(v, True)), "fp16 pair"
    assert same_bits(bct[..., :C], split_pair(v, False)), "bf16 pair"
    for pl in (btc, bct):
        assert bool((pl[..., C:].view(torch.int16) == 0).all()), "pad columns must be +0"
    for buf in (hbuf, wbuf):
        assert bool((buf[2 * B * T * Cp:] == SENT16).all()), "write past the planes"
    # the data reached the clamp (fp16 pair only) and the fp16 subnormal range
    assert bool((v.abs() > 65504.0).any()) and bool(((v.abs() < 2.0 ** -14) & (v != 0)).any())


GATE_CASES = [
    # (B, C, T, mode, residual, ext): mode 0 = GLU, 1 = highway
    (2, 136, 37, 0, 1, False),
    (3, 64, 100, 0, 0, True),
    (2, 136, 101, 1, 0, False),
    (2, 256, 64, 1, 0, True),
]


@pytest.mark.parametrize("case", GATE_CASES, ids=lambda c: "B%d_C%d_T%d_%s%s%s" % (
    c[0], c[1], c[2], "glu" if c[3] == 0 else "highway", "_res" if c[4] else "", "_ext" if c[5] else ""))
def test_gate_bwd_split_pairs(case):
    B, C, T, mode, residual, ext = case
    g = torch.Generator(device="cuda").manual_seed(C + 5 * T)
    dy, a, x = (torch.randn(B, C, T, device="cuda", generator=g) for _ in range(3))
    s = torch.rand(B, C, T, device="cuda", generator=g)
    tmult, tlen = 2, torch.tensor([T // 3], dtype=torch.int64, device="cuda")
    buf, planes = sentinel_planes(2, B, T, 2 * C, dtype=BF16)
    dbias = torch.zeros(2 * C, device="cuda")
    _call("dv3_tc_gate_bwd_split_npl", _p(dy), _p(a), _p(s), _p(x) if mode else None, _p(planes), 2, None, _p(dbias),
          B, C, T, mode, residual, _p(tlen) if ext else None, tmult, _st())
    torch.cuda.synchronize()
    # the kernel's fp32 expressions in its order: products only, so no contraction applies
    gs = torch.tensor(0.70710678118654752 if mode == 0 and residual else 1.0, dtype=torch.float32, device="cuda")
    gg = dy * gs
    da = gg * s
    db = ((gg * (a if mode == 0 else a - x)) * s) * (1.0 - s)
    if ext:
        da[:, :, tmult * int(tlen):] = 0.0
        db[:, :, tmult * int(tlen):] = 0.0
    assert same_bits(planes[..., :C], split_pair(da.transpose(1, 2), False)), "da pair"
    assert same_bits(planes[..., C:], split_pair(db.transpose(1, 2), False)), "db pair"
    assert bool((buf[2 * B * T * 2 * C:] == SENT16).all()), "write past the planes"
    v = torch.cat([da, db], 1).double()
    want = v.sum((0, 2))
    bound = B * T * U * v.abs().sum((0, 2))
    assert bool(((dbias.double() - want).abs() <= bound).all()), "dbias"


GRAD_CASES = [
    # (B, C, T, relu, ext)
    (2, 136, 101, 1, False),
    (3, 513, 64, 1, True),
    (2, 80, 37, 0, False),
    (2, 8, 130, 0, True),
]


@pytest.mark.parametrize("case", GRAD_CASES, ids=lambda c: "B%d_C%d_T%d%s%s" % (
    c[0], c[1], c[2], "_relu" if c[3] else "", "_ext" if c[4] else ""))
def test_grad_split_pairs(case):
    B, C, T, relu, ext = case
    g = torch.Generator(device="cuda").manual_seed(C + 7 * T)
    dy, y = (torch.randn(B, C, T, device="cuda", generator=g) for _ in range(2))
    r = torch.rand(B, C, T, device="cuda", generator=g)
    y = torch.where(r < 0.05, 0.0, y)
    y = torch.where((r >= 0.05) & (r < 0.1), -0.0, y)
    y = torch.where((r >= 0.1) & (r < 0.15), float("nan"), y)
    assert bool((y.view(torch.int32) == -2 ** 31).any())                     # -0 is present
    tmult, tlen = 3, torch.tensor([T // 5], dtype=torch.int64, device="cuda")
    Cp = pad8(C)
    buf, planes = sentinel_planes(2, B, T, Cp, dtype=BF16)
    dbias = torch.zeros(C, device="cuda")
    _call("dv3_tc_grad_split_npl", _p(dy), _p(y) if relu else None, _p(planes), 2, None, _p(dbias), B, C, T, relu,
          _p(tlen) if ext else None, tmult, _st())
    torch.cuda.synchronize()
    v = torch.where(y > 0, dy, 0.0) if relu else dy.clone()                 # 0, -0 and NaN all mask
    if ext:
        v[:, :, tmult * int(tlen):] = 0.0
    assert same_bits(planes[..., :C], split_pair(v.transpose(1, 2), False))
    assert bool((planes[..., C:].view(torch.int16) == 0).all()), "pad columns must be +0"
    assert bool((buf[2 * B * T * Cp:] == SENT16).all()), "write past the planes"
    vd = v.double()
    assert bool(((dbias.double() - vd.sum((0, 2))).abs() <= B * T * U * vd.abs().sum((0, 2))).all()), "dbias"


# ---- 2./3. the GEMMs against fp64 on the exact operand planes ---------------------------------------------------------
CONV_CASES = [
    # (B, Kc, Nc, T, k, dilation, causal, transpose_taps, epilogue, NaN pad rerun)
    # <1,128,32>: 128-column tiles
    (16, 80, 513, 800, 1, 1, False, False, "none", False),     # 560 tiles, 3 K-iterations on a 4-stage ring
    (16, 513, 80, 800, 1, 1, False, True, "none", True),       # data gradient, Nc = 80 on a 128-wide tile, Kc tail
    (3, 8, 16, 37, 1, 1, False, False, "bias_relu", False),    # Kc = 8, Nc = 16
    (2, 16, 16, 1, 1, 1, False, True, "add1", False),          # T = 1
    (16, 256, 256, 400, 3, 2, True, False, "drop", False),     # k = 3, dilated, causal
    (16, 128, 512, 203, 5, 3, False, True, "add2", False),     # k = 5, dilated
    (100, 64, 128, 50, 8, 16, False, True, "none", False),     # k = 8: halo > T, taps wholly outside [0, T)
    (20, 96, 768, 128, 1, 1, False, False, "add1", False),     # T = 128
    (32, 513, 256, 129, 1, 1, False, True, "bias_relu", False),
    # <1,64,64>: 64-column tiles, Kc % 64 == 0
    (4, 320, 384, 800, 1, 1, False, False, "none", False),     # 168 tiles, 5 K-iterations on a 3-stage ring
    (2, 128, 256, 37, 3, 2, True, True, "bias_relu", False),
    (4, 64, 128, 50, 8, 16, False, False, "drop", False),
    (3, 256, 513, 129, 1, 1, False, True, "add2", False),
    (2, 192, 80, 1, 1, 1, False, False, "add1", False),
    (5, 128, 256, 128, 5, 1, False, False, "none", False),
    (2, 64, 128, 203, 1, 1, False, True, "none", False),
    # <1,64,32>: 64-column tiles, Kc % 64 != 0
    (4, 513, 384, 800, 1, 1, False, False, "none", True),      # 168 tiles, 17 K-iterations on a 6-stage ring
    (2, 80, 513, 37, 1, 1, False, True, "bias_relu", False),
    (3, 8, 80, 129, 1, 1, False, False, "add1", False),
    (2, 16, 256, 1, 3, 2, True, True, "add2", False),
    (2, 96, 128, 50, 8, 16, False, True, "drop", False),
    (4, 160, 256, 128, 5, 3, False, False, "none", False),
    (2, 80, 128, 203, 1, 1, False, False, "none", False),
]


def conv_epilogue(D, bD, m, bias, relu, addmode, e1, e2, alpha):
    """fp64 dv3_tc_conv epilogue (out = D * mask + bias + addend, ReLU) and its bound: the GEMM bound through the mask,
    plus the fp32 rounding of at most four operations on the terms."""
    out, S, bound = D * m, (D * m).abs(), bD * m
    if bias is not None:
        bv = bias.double()[None, :, None]
        out, S = out + bv, S + bv.abs()
    if addmode:
        t = float(alpha) * e1.double() if addmode == 1 else e1.double() * (1.0 - e2.double())
        out, S = out + t, S + t.abs()
    if relu:
        out = out.clamp_min(0.0)
    return out, bound + 4 * U * S


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "B%d_K%d_N%d_T%d_k%d_d%d%s%s_%s%s" % (
    c[0], c[1], c[2], c[3], c[4], c[5], "_causal" if c[6] else "", "_dgrad" if c[7] else "", c[8],
    "_nanpad" if c[9] else ""))
def test_conv_pairs(case):
    from oracle import dropout_mask as DM
    B, Kc, Nc, T, k, dil, causal, tr, epi, nanpad = case
    f16 = not tr
    cfg, n_iters, n_mma, tiles = conv_config(B, Kc, Nc, T, k)
    g = torch.Generator(device="cuda").manual_seed(Kc * 11 + Nc + T + k)
    A = torch.randn(B, T, Kc, device="cuda", generator=g)
    W = torch.randn(k, Nc, Kc, device="cuda", generator=g) * (k * Kc) ** -0.5
    a, w = pair_planes(A, f16), pair_planes(W, f16)
    bias = torch.randn(Nc, device="cuda", generator=g) * 0.1 if epi == "bias_relu" else None
    addmode = {"add1": 1, "add2": 2}.get(epi, 0)
    e1 = torch.randn(B, Nc, T, device="cuda", generator=g) if addmode else None
    e2 = torch.rand(B, Nc, T, device="cuda", generator=g) if addmode == 2 else None
    alpha = 0.37 if addmode == 1 else 0.0
    p = 0.3 if epi == "drop" else 0.0
    seed = torch.tensor([4321 + T], dtype=torch.int64, device="cuda")
    n = B * Nc * T

    def launch(a, w):
        buf, out = guarded(n)
        _call("dv3_tc_conv", _p(a), _p(w), 2, _p(out), B, Kc, Nc, T, k, dil, int(causal), int(tr), _p(bias),
              int(epi == "bias_relu"), p, _p(seed) if p else None, 9, addmode, _p(e1), _p(e2), alpha, None, _st())
        torch.cuda.synchronize()
        return buf, out.view(B, Nc, T)

    buf, out = launch(a, w)
    assert_written_inside_only(buf, n)
    R, x1, x2, absb = pair_reference(a[..., :Kc], w[..., :Kc], lambda X, Y: ref_conv(X, Y, k, dil, causal, tr))
    bD = c1(k * Kc) * absb + (gamma() * n_mma + 2.0 ** -23) * R.abs()
    m = torch.from_numpy(DM.mask(seed, 9, p, (B, Nc, T))).double().cuda()
    want, bound = conv_epilogue(R, bD, m, bias, epi == "bias_relu", addmode, e1, e2, alpha)
    r = ratio(out, want, bound)
    d = discriminator(out.double() - want, x1, x2) if p == 0 else float("nan")
    print("conv %s %s (%d tiles, %d K-iterations): error/bound %.3g, discriminator %.3g" % (
        case, cfg, tiles, n_iters, r, d))
    assert r <= 1, r
    assert p > 0 or d <= 1, d
    if nanpad:
        assert Kc % 8, "a pad-column rerun needs pad columns"
        buf2, out2 = launch(poison_pads(a, Kc), poison_pads(w, Kc))
        assert torch.equal(buf.view(torch.int32), buf2.view(torch.int32)), "a pad column was read"


GATED_CASES = [
    # (B, C, T, k, dilation, causal, mode, residual, speaker bias, saved outputs: "a", "s", "as" or "" = both NULL)
    (16, 512, 800, 3, 1, False, 0, True, False, "as"),         # 896 tiles
    (4, 256, 203, 5, 2, True, 0, False, True, "as"),
    (3, 128, 37, 3, 3, False, 1, False, False, "as"),
    (2, 256, 1, 8, 16, False, 1, False, True, ""),
    (4, 384, 128, 1, 1, False, 0, True, True, "a"),
    (2, 128, 129, 3, 1, True, 1, False, False, "s"),
    (2, 128, 50, 8, 16, False, 0, True, False, "as"),          # halo > T, taps wholly outside [0, T)
]


def gated_epilogue(D, bD, bias, spk, res, C, mode, residual):
    """fp64 gated epilogue and bounds, propagated as in tests/test_gpu_tc1.py test_gated_single_pass."""
    bd = bias.double()[None, :, None]
    sp = spk.double() if spk is not None else torch.zeros_like(D[:, :C])
    a = D[:, :C] + sp + bd[:, :C]
    ba = bD[:, :C] + 2 * U * (D[:, :C].abs() + sp.abs() + bd[:, :C].abs())
    b = D[:, C:] + bd[:, C:]
    bb = bD[:, C:] + 2 * U * (D[:, C:].abs() + bd[:, C:].abs())
    s = torch.sigmoid(b)
    bs = s * (1 - s) * bb + 4 * U
    r = res.double()
    if mode == 0:
        y = a * s
        by = s.abs() * ba + a.abs() * bs + U * y.abs()
        if residual:
            by = (by + U * (y.abs() + r.abs())) * 0.7072 + U * ((y + r) * 0.7071).abs()
            y = (y + r) * 0.7071067811865476
    else:
        y = s * a + (1 - s) * r
        by = s * ba + (a - r).abs() * bs + 4 * U * ((s * a).abs() + ((1 - s) * r).abs())
    return a, ba, s, bs, y, by


@pytest.mark.parametrize("case", GATED_CASES, ids=lambda c: "B%d_C%d_T%d_k%d_d%d%s_%s%s%s_save%s" % (
    c[0], c[1], c[2], c[3], c[4], "_causal" if c[5] else "", "glu" if c[6] == 0 else "highway",
    "_res" if c[7] else "", "_spk" if c[8] else "", c[9] or "none"))
def test_gated_pairs(case):
    B, C, T, k, dil, causal, mode, residual, has_spk, save = case
    cfg, n_iters, n_mma, tiles = gated_config(B, C, T, k)
    g = torch.Generator(device="cuda").manual_seed(C + 3 * T + 17 * k)
    X = torch.randn(B, T, C, device="cuda", generator=g)
    W = torch.randn(k, 2 * C, C, device="cuda", generator=g) * (k * C) ** -0.5
    bias = torch.randn(2 * C, device="cuda", generator=g) * 0.1
    res = torch.randn(B, C, T, device="cuda", generator=g)
    spk = torch.randn(B, C, T, device="cuda", generator=g) * 0.3 if has_spk else None
    x, w = pair_planes(X, True), pair_planes(W, True)
    n = B * C * T
    (ybuf, y), (abuf, sa), (sbuf, ss) = guarded(n), guarded(n), guarded(n)
    _call("dv3_tc_convblock_fwd", _p(x), _p(w), 2, _p(bias), _p(spk), _p(res), _p(y), _p(sa) if "a" in save else None,
          _p(ss) if "s" in save else None, B, C, T, k, dil, int(causal), mode, int(residual), None, _st())
    torch.cuda.synchronize()
    assert_written_inside_only(ybuf, n)
    for buf, name in ((abuf, "a"), (sbuf, "s")):
        if name in save:
            assert_written_inside_only(buf, n)
        else:
            assert bool((buf.view(torch.int32) == SENT32).all()), "NULL save_%s written" % name
    R, x1, x2, absb = pair_reference(x, w, lambda X_, W_: ref_conv(X_, W_, k, dil, causal, False))
    bD = c1(k * C) * absb + (gamma() * n_mma + 2.0 ** -23) * R.abs()
    a_ref, ba, s_ref, bs, y_ref, by = gated_epilogue(R, bD, bias, spk, res, C, mode, residual)
    y, sa, ss = y.view(B, C, T), sa.view(B, C, T), ss.view(B, C, T)
    ry = ratio(y, y_ref, by)
    ra = ratio(sa, a_ref, ba) if "a" in save else 0.0
    rs = ratio(ss, s_ref, bs) if "s" in save else 0.0
    d = discriminator(sa.double() - a_ref, x1[:, :C], x2[:, :C]) if "a" in save else float("nan")
    print("gated %s %s (%d tiles, %d K-iterations): error/bound y %.3g a %.3g s %.3g, discriminator %.3g" % (
        case, cfg, tiles, n_iters, ry, ra, rs, d))
    assert ry <= 1 and ra <= 1 and rs <= 1, (ry, ra, rs)
    assert "a" not in save or d <= 1, d


WGRAD_CASES = [
    # (B, Mw, Nw, T, k, dilation, causal, msplit form, NaN pad rerun)
    (16, 256, 128, 200, 3, 1, False, False, False),   # nsplit > 1
    (2, 80, 513, 37, 1, 1, False, False, False),      # T % 32 != 0, Mw / Nw tails
    (3, 513, 16, 20, 5, 2, True, False, True),        # T < 32, dilated causal
    (4, 128, 256, 50, 8, 16, False, False, False),    # k = 8: taps wholly outside [0, T) -> zero slots
    (16, 256, 128, 100, 1, 1, False, True, False),    # msplit = 2: the ConvTranspose weight layout
    (1, 256, 256, 256, 1, 1, False, False, False),    # nsplit = 1
]


def ref_wgrad(DY, X, k, dil, causal):
    """fp64 DY (B,T,M), X (B,T,N) -> (M, N, k) = sum_{b,t} DY[b,t,m] X[b,t+off_j,n], zero outside [0, T)."""
    T = X.shape[1]
    padl = (k - 1) * dil if causal else (k - 1) // 2 * dil
    D = torch.zeros(DY.shape[2], X.shape[2], k, dtype=torch.float64, device=DY.device)
    for j in range(k):
        off = j * dil - padl
        sh = torch.zeros_like(X)
        lo, hi = max(0, -off), min(T, T - off)
        if hi > lo:
            sh[:, lo:hi] = X[:, lo + off:hi + off]
        D[:, :, j] = torch.einsum("btm,btn->mn", DY, sh)
    return D


def run_wgrad(dy, x, B, Mw, Nw, T, k, dil, causal, convt, gap=37):
    """Launch into NaN-sentinel slots split_stride = numel + gap apart -> (buffer, slots [nsplit][numel], nsplit, idx)
    with idx mapping (m, n, j) to the element of a slot."""
    from deepvoice3_pytorch_b200._lib import lib
    nsplit = lib.raw("dv3_tc_wgrad_nsplit")(B, Mw, Nw, T, k)
    numel, stride = Mw * Nw * k, Mw * Nw * k + gap
    buf, parts = guarded(nsplit * stride)
    if convt:       # m = (j, co) with Cout = Mw / 2 -> element at (m % Cout) * 2 + m // Cout + n * Mw
        ms, s_m, s_mh, s_n, s_j = Mw // 2, 2, 1, Mw, 0
    else:
        ms, s_m, s_mh, s_n, s_j = Mw, Nw, 0, 1, Mw * Nw
    _call("dv3_tc_wgrad_mn", _p(dy), _p(x), _p(parts), stride, B, Mw, Nw, T, k, dil, int(causal), ms, s_m, s_mh, s_n,
          s_j, _st())
    torch.cuda.synchronize()
    m = torch.arange(Mw, device="cuda")[:, None, None]
    n = torch.arange(Nw, device="cuda")[None, :, None]
    j = torch.arange(k, device="cuda")[None, None, :]
    idx = ((m % ms) * s_m + (m // ms) * s_mh + n * s_n + j * s_j).flatten()
    return buf, parts.view(nsplit, stride), nsplit, idx


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "B%d_M%d_N%d_T%d_k%d%s%s" % (
    c[0], c[1], c[2], c[3], c[4], "_msplit2" if c[7] else "", "_nanpad" if c[8] else ""))
def test_wgrad_pairs(case):
    B, Mw, Nw, T, k, dil, causal, convt, nanpad = case
    g = torch.Generator(device="cuda").manual_seed(Mw + 3 * Nw + T)
    DY = torch.randn(B, T, Mw, device="cuda", generator=g) * 1e-3
    X = torch.randn(B, T, Nw, device="cuda", generator=g)
    dy, x = pair_planes(DY, False), pair_planes(X, False)
    buf, parts, nsplit, idx = run_wgrad(dy, x, B, Mw, Nw, T, k, dil, causal, convt)
    numel = Mw * Nw * k
    bits = buf.view(torch.int32)
    assert bool((bits[:GUARD] == SENT32).all()) and bool((bits[GUARD + nsplit * parts.shape[1]:] == SENT32).all())
    assert bool((parts[:, numel:].view(torch.int32) == SENT32).all()), "write into the gap between slots"
    assert bool(torch.isfinite(parts[:, :numel]).all()), "slot element left unwritten"
    bps, kb_n = -(-B // nsplit), -(-T // 32)
    total = torch.zeros(Mw, Nw, k, dtype=torch.float64, device="cuda")
    R, X1, X2, worst = 0.0, 0.0, 0.0, 0.0
    for s in range(nsplit):
        b0, b1 = s * bps, min(B, (s + 1) * bps)
        Rs, x1, x2, absb = pair_reference(dy[:, b0:b1, :, :Mw], x[:, b0:b1, :, :Nw],
                                          lambda P, Q: ref_wgrad(P, Q, k, dil, causal))
        got = parts[s, :numel][idx].view(Mw, Nw, k)
        n_mma = 2 * (b1 - b0) * kb_n
        bound = c1((b1 - b0) * T) * absb + (gamma() * n_mma + 2.0 ** -23) * Rs.abs()
        worst = max(worst, ratio(got, Rs, bound))
        total += got.double()
        R, X1, X2 = R + Rs, X1 + x1, X2 + x2
    d = discriminator(total - R, X1, X2)
    print("wgrad %s (nsplit %d): error/bound %.3g, discriminator %.3g" % (case, nsplit, worst, d))
    assert worst <= 1 and d <= 1, (worst, d)
    if nanpad:
        assert Mw % 8 or Nw % 8, "a pad-column rerun needs pad columns"
        buf2, _, _, _ = run_wgrad(poison_pads(dy, Mw), poison_pads(x, Nw), B, Mw, Nw, T, k, dil, causal, convt)
        assert torch.equal(buf.view(torch.int32), buf2.view(torch.int32)), "a pad column was read"


def test_case_lists_walk_several_tiles_per_cta():
    """Persistent scheduling with the device's own SM count: the 128-column conv and the gated kernel have a case of
    more than two tiles per CTA; the 64-column configurations (at most 198 tiles: the launcher takes them only below 100
    128-column tiles) have a case where CTAs walk a second tile.  In each, a tile's K-iterations are not a multiple of
    the ring depth where the configuration allows it (a gated tile has k * C / 32 with C % 128 == 0)."""
    n = sms()
    seen = {}
    for c in CONV_CASES:
        cfg, it, _, tiles = conv_config(*c[:4], c[4])
        if it % STAGES[cfg]:
            seen[cfg] = max(seen.get(cfg, 0), tiles)
    for c in GATED_CASES:
        cfg, _, _, tiles = gated_config(*c[:4])
        seen[cfg] = max(seen.get(cfg, 0), tiles)
    assert seen[(1, 128, 32)] > 2 * n and seen[(2, 64, 32)] > 2 * n, seen
    assert seen[(1, 64, 64)] > n and seen[(1, 64, 32)] > n, seen


# ---- 4. truncation compensation ---------------------------------------------------------------------------------------
def _bias(out, R):
    return float(((out.double() - R) * R).sum() / (R * R).sum())


def trunc_biases():
    """<out - R, R> / <R, R> and n_mma of a forward conv, a data gradient and a weight gradient with long contractions
    (also run in a subprocess under DV3_TC_GAMMA=0)."""
    res = {}
    B, K, N, T, k = 4, 512, 512, 800, 5
    g = torch.Generator(device="cuda").manual_seed(99)
    for tr in (0, 1):
        A = torch.randn(B, T, K, device="cuda", generator=g)
        W = torch.randn(k, N, K, device="cuda", generator=g) * (k * K) ** -0.5
        a, w = pair_planes(A, not tr), pair_planes(W, not tr)
        out = torch.empty(B, N, T, device="cuda")
        _call("dv3_tc_conv", _p(a), _p(w), 2, _p(out), B, K, N, T, k, 1, 0, tr, None, 0, 0.0, None, 0, 0, None, None,
              0.0, None, _st())
        torch.cuda.synchronize()
        R = pair_reference(a, w, lambda X, Y: ref_conv(X, Y, k, 1, False, bool(tr)))[0]
        res["dgrad" if tr else "conv"] = (_bias(out, R), conv_config(B, K, N, T, k)[2])
    B, M, N, T = 2, 256, 256, 4096
    dy = pair_planes(torch.randn(B, T, M, device="cuda", generator=g), False)
    x = pair_planes(torch.randn(B, T, N, device="cuda", generator=g), False)
    _, parts, nsplit, idx = run_wgrad(dy, x, B, M, N, T, 1, 1, False, False)
    got = parts[:, :M * N].double().sum(0)[idx].view(M, N, 1)
    R = pair_reference(dy, x, lambda P, Q: ref_wgrad(P, Q, 1, 1, False))[0]
    res["wgrad"] = (_bias(got, R), 2 * -(-B // nsplit) * -(-T // 32))
    return res


def test_truncation_compensation():
    if os.environ.get("DV3_TC_GAMMA") is not None:
        pytest.skip("measures the default calibration of the compensation")
    here = trunc_biases()
    env = dict(os.environ, DV3_TC_GAMMA="0")
    tests = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; from test_gpu_tc_pairs import trunc_biases; "
            "print('BIASES ' + json.dumps(trunc_biases()))" % (tests, os.path.dirname(tests)))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    proc = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-2000:]
    off = json.loads([ln for ln in proc.stdout.splitlines() if ln.startswith("BIASES ")][-1][7:])
    for name, (b, n_mma) in here.items():
        b0 = off[name][0]
        print("truncation %s (n_mma %d): bias %+.3g compensated, %+.3g with DV3_TC_GAMMA=0; gamma0 n_mma %.3g" % (
            name, n_mma, b, b0, GAMMA0 * n_mma))
        assert abs(b) <= 0.25 * GAMMA0 * n_mma, (name, b)
        assert abs(b0) > 0.5 * GAMMA0 * n_mma, (name, b0)
