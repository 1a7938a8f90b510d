"""GPU: the fused epilogues of the tensor-core conv kernel against the same epilogue computed in torch.

Each case launches its GEMM twice on the same operand planes: once with the epilogue under test and once as a plain
dv3_tc_conv with no epilogue math (addmode 0, no bias, no dropout, no ReLU), whose output is the raw accumulator
tile.  A gated forward's raw GEMM is the conv with 2C output channels over the same (B,T,C) input and [k][2C][C]
weight planes: columns [0, C) are its a half, [C, 2C) its b half.  The epilogue is recomputed from the raw output:
  * bit for bit where the kernel only adds and masks: the gated a = acc (+ speaker) + bias, the conv's bias-only,
    ReLU-only and plain outputs;
  * within a few float32 ulp of a float64 evaluation where it multiplies into a sum (the compiler contracts those into
    FMAs: the conv's dropout scale, addends and alpha) or calls expf (the gate's sigmoid, and y).
Every output lies between canary guard bands that must be untouched.  All cases are launched on one stream and
checked once, after one synchronise.

The cases walk the store paths of the epilogue: TMA bulk stores clipped at T and at the channel count (T = 72, 200,
1000; the 80-channel mel projection and a 513-channel output; an input padded from 20 to 24 channels), and the
per-thread stores taken when the output rows cannot be TMA rows (T = 1 and T = 102, not multiples of 4, and an
output 4 bytes off 16-byte alignment); both gate modes, residual and speaker bias on and off, saved a / s on and off,
dropout, addmodes 0 / 1 / 2, ReLU, data gradients; unit counts from one CTA to several per SM, two planes and one.
"""
import numpy as np
import pytest
import torch

from oracle import dropout_mask

pytestmark = pytest.mark.gpu

GUARD = 1024                                  # floats of canary on each side of an output
CANARY = -3.0e38                              # no epilogue writes this
EPS = 2.0 ** -23

# (B, C, T, k, dilation, causal, mode, residual, speaker bias, saved outputs, npl)
GATED = [
    (1, 128, 1, 3, 1, True, 0, True, False, "as", 2),       # one unit, per-thread stores (T % 4 != 0)
    (2, 256, 72, 3, 2, False, 1, False, True, "as", 2),     # highway gate, speaker bias, T tail inside a box
    (4, 128, 200, 3, 1, True, 0, False, False, "", 2),      # plain GLU, nothing saved
    (8, 256, 1000, 3, 1, False, 0, True, True, "a", 2),     # 256 units
    (2, 128, 102, 3, 1, False, 1, False, False, "as", 2),   # per-thread stores over several units
    (3, 128, 1000, 3, 3, True, 1, False, False, "s", 1),    # single plane
    (16, 128, 200, 3, 1, False, 0, True, True, "as", 1),
]
# (B, Kc, Nc, T, k, dilation, causal, transpose_taps, bias, relu, p_drop, addmode, npl, misaligned output)
CONV = [
    (1, 80, 80, 1, 1, 1, False, False, True, True, 0.0, 0, 2, False),      # one unit, T = 1
    (4, 20, 80, 72, 1, 1, False, False, True, True, 0.0, 0, 2, False),     # input padded 20 -> 24 channels
    (16, 256, 80, 200, 1, 1, False, False, True, False, 0.0, 0, 2, False),  # mel projection, 64-wide tiles
    (8, 256, 513, 1000, 1, 1, False, False, False, False, 0.3, 0, 2, False),  # 513 channels, dropout, 320 units
    (4, 512, 256, 200, 3, 1, True, True, False, False, 0.3, 1, 2, False),   # data gradient, dropout, addmode 1
    (6, 256, 256, 1000, 3, 2, False, True, False, False, 0.0, 2, 2, False),  # data gradient, addmode 2
    (2, 128, 128, 200, 1, 1, False, False, True, False, 0.0, 0, 2, True),   # unaligned output: per-thread stores
    (2, 128, 256, 72, 1, 1, False, False, False, True, 0.0, 0, 1, False),   # single plane, ReLU only
    (3, 96, 128, 1000, 1, 1, False, True, True, False, 0.3, 2, 1, False),   # single plane, everything
    (2, 256, 128, 102, 3, 1, True, True, False, False, 0.0, 1, 1, False),   # T % 4 != 0, data gradient
]


def _lib():
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    return ops, lib


class Guarded:
    """A (B, C, T) fp32 output between canary bands; `offset` floats past a 16-byte boundary."""

    def __init__(self, shape, offset=0):
        n = int(np.prod(shape))
        self.n, self.offset = n, offset
        self.buf = torch.full((2 * GUARD + n + offset,), CANARY, device="cuda")
        self.t = self.buf[GUARD + offset:GUARD + offset + n].view(shape)
        self.t.fill_(float("nan"))

    def guards_intact(self):
        b = self.buf.cpu().numpy()
        return bool((b[:GUARD + self.offset] == CANARY).all() and (b[GUARD + self.offset + self.n:] == CANARY).all())


def _planes(g, shape, npl, dtype, scale=1.0):
    hi = (torch.randn(*shape, generator=g) * scale).to(dtype)
    lo = (torch.randn(*shape, generator=g) * scale * 2.0 ** -11).to(dtype)
    return torch.stack([hi, lo][:npl]).cuda()


def _ulp_close(got, want, mag, ulps):
    """|got - want| <= ulps * eps32 * mag elementwise (want, mag float64)."""
    got = got.double()
    return bool(torch.isfinite(got).all()) and bool(((got - want).abs() <= ulps * EPS * mag + 1e-30).all())


def _launch_gated(case, idx, st):
    ops, lib = _lib()
    B, C, T, k, dil, causal, mode, residual, has_spk, saved, npl = case
    g = torch.Generator().manual_seed(500 + idx)
    xd = _planes(g, (B, T, C), npl, torch.float16)
    w = _planes(g, (k, 2 * C, C), npl, torch.float16, scale=(1.0 / (k * C)) ** 0.5)
    bias = (torch.randn(2 * C, generator=g) * 0.1).cuda()
    spk = (torch.randn(B, C, T, generator=g) * 0.1).cuda() if has_spk else None
    res = torch.randn(B, C, T, generator=g).cuda() if (mode or residual) else None
    outs = {n: Guarded((B, C, T)) for n in "yas" if n == "y" or n in saved}
    raw = Guarded((B, 2 * C, T))
    lib.call("dv3_tc_convblock_fwd", ops._p(xd), ops._p(w), npl, ops._p(bias), ops._p(spk), ops._p(res),
             ops._p(outs["y"].t), ops._p(outs["a"].t if "a" in outs else None),
             ops._p(outs["s"].t if "s" in outs else None), B, C, T, k, dil, int(causal), mode, int(residual), None, st)
    lib.call("dv3_tc_conv", ops._p(xd), ops._p(w), npl, ops._p(raw.t), B, C, 2 * C, T, k, dil, int(causal), 0,
             None, 0, 0.0, None, 0, 0, None, None, 0.0, None, st)
    return dict(case=case, bias=bias, spk=spk, res=res, outs=outs, raw=raw)


def _check_gated(r):
    B, C, T, k, dil, causal, mode, residual, has_spk, saved, npl = r["case"]
    raw, bias = r["raw"].t, r["bias"]
    va = raw[:, :C]
    if r["spk"] is not None:
        va = va + r["spk"]
    a = va + bias[:C, None]                                          # float32, as the kernel adds
    xb = (raw[:, C:] + bias[C:, None]).double()
    s = 1.0 / (1.0 + torch.exp(-xb))
    ad = a.double()
    rr = r["res"].double() if r["res"] is not None else torch.zeros_like(ad)
    if mode == 0:
        y = ad * s
        mag = y.abs()
        if residual:
            y = (y + rr) * 0.70710678118654752
            mag = (mag + rr.abs()) * 0.71
    else:
        y = s * ad + (1.0 - s) * rr
        mag = (s * ad).abs() + rr.abs()               # an ulp of s is an ulp of rr in (1 - s) * rr
    errs = []
    if not _ulp_close(r["outs"]["y"].t, y, mag, 8):
        errs.append("y")
    if "a" in r["outs"] and not torch.equal(r["outs"]["a"].t, a):
        errs.append("a")
    if "s" in r["outs"] and not _ulp_close(r["outs"]["s"].t, s, s, 4):
        errs.append("s")
    errs += ["guard %s" % n for n, o in list(r["outs"].items()) + [("raw", r["raw"])] if not o.guards_intact()]
    return errs


def _launch_conv(case, idx, st):
    ops, lib = _lib()
    B, Kc, Nc, T, k, dil, causal, tt, has_bias, relu, p, addmode, npl, misaligned = case
    g = torch.Generator().manual_seed(700 + idx)
    dt = torch.bfloat16 if tt else torch.float16
    kp = (Kc + 7) // 8 * 8
    a = _planes(g, (B, T, kp), npl, dt)
    w = _planes(g, (k, Nc, kp), npl, dt, scale=(1.0 / (k * Kc)) ** 0.5)
    bias = (torch.randn(Nc, generator=g) * 0.1).cuda() if has_bias else None
    e1 = torch.randn(B, Nc, T, generator=g).cuda() if addmode else None
    e2 = torch.rand(B, Nc, T, generator=g).cuda() if addmode == 2 else None
    alpha = 0.70710678 if addmode == 1 else 0.0
    seed = torch.tensor([0x1234_5678_9ABC + idx], dtype=torch.int64, device="cuda")
    salt = 11 + idx
    out = Guarded((B, Nc, T), offset=1 if misaligned else 0)
    raw = Guarded((B, Nc, T))
    lib.call("dv3_tc_conv", ops._p(a), ops._p(w), npl, ops._p(out.t), B, Kc, Nc, T, k, dil, int(causal), int(tt),
             ops._p(bias), int(relu), p, ops._p(seed) if p > 0 else None, salt, addmode, ops._p(e1), ops._p(e2),
             alpha, None, st)
    lib.call("dv3_tc_conv", ops._p(a), ops._p(w), npl, ops._p(raw.t), B, Kc, Nc, T, k, dil, int(causal), int(tt),
             None, 0, 0.0, None, 0, 0, None, None, 0.0, None, st)
    return dict(case=case, bias=bias, e1=e1, e2=e2, alpha=alpha, seed=seed, salt=salt, out=out, raw=raw)


def _check_conv(r):
    B, Kc, Nc, T, k, dil, causal, tt, has_bias, relu, p, addmode, npl, misaligned = r["case"]
    raw, out = r["raw"].t, r["out"].t
    errs = [n for n, o in (("out", r["out"]), ("raw", r["raw"])) if not o.guards_intact()]
    if p == 0 and addmode == 0:                                      # adds and masks only: bit for bit
        want = raw + r["bias"][:, None] if r["bias"] is not None else raw
        if relu:
            want = torch.clamp_min(want, 0.0)
        return errs + ([] if torch.equal(out, want) else ["out (bit for bit)"])
    m = torch.from_numpy(dropout_mask.mask(r["seed"].cpu(), r["salt"], p, (B, Nc, T))).cuda().double()
    terms = [raw.double() * m]
    if r["bias"] is not None:
        terms.append(r["bias"].double()[:, None].expand(B, Nc, T))
    if addmode == 1:
        terms.append(r["alpha"] * r["e1"].double())
    elif addmode == 2:
        terms.append(r["e1"].double() * (1.0 - r["e2"].double()))
    want = sum(terms)
    mag = sum(t.abs() for t in terms)
    if relu:
        want = torch.clamp_min(want, 0.0)
    return errs + ([] if _ulp_close(out, want, mag, 4) else ["out"])


def test_epilogues_match_torch_on_the_raw_gemm():
    ops, lib = _lib()
    st = ops._stream()
    launched = [("gated", c, _launch_gated(c, i, st)) for i, c in enumerate(GATED)]
    launched += [("conv", c, _launch_conv(c, i, st)) for i, c in enumerate(CONV)]
    torch.cuda.synchronize()
    ops.check_index_errors()
    bad = {}
    for kind, case, r in launched:
        errs = _check_gated(r) if kind == "gated" else _check_conv(r)
        if errs:
            bad["%s %s" % (kind, case)] = errs
    assert not bad, bad
