"""GPU: shape sweep of the tensor-core attention kernels (csrc/tc_attn.cu: dv3_tc_attn_fwd / dv3_tc_attn_bwd) and of
the exact-fp32 fallback they hand unsupported shapes to, against an fp64 attention core with elementwise error bounds
derived from the kernels' arithmetic (no dropout here; tests/test_gpu_dropout.py covers the mask).

Error model (every bound is elementwise, computed by the same fp64 contraction on absolute values):
  * GEMM with contraction depth K: each fp32 operand is split in-kernel into bf16 hi = rn(x), lo = rn(x - hi), so
    |x - hi - lo| <= 2^-16 |x|; the products hi*hi + hi*lo + lo*hi drop lo*lo (<= 2^-16 |a||b|) and the two residuals
    (2 x 2^-16 |a||b|).  The fp32 tensor-core accumulation aligns the 16 products of one MMA to the largest exponent
    and truncates: less than 2^-23 of the running magnitude per term, i.e. <= K 2^-22 sum|a||b| with a factor 2 for
    the per-MMA alignment.  Hence |C - C_exact| <= c(K) (|A|.|B|), c(K) = 3 2^-16 (1 + 2^-7) + K 2^-22 + 2^-23.
    The exact-fp32 fallback (dv3_bgemm) reads full fp32 operands and forms each output as one serial fmaf chain:
    c(K) = gamma(K) = K 2^-24 / (1 - K 2^-24), 7-10x tighter at K = 128-256.
  * Softmax: a score error dS moves p_s by p_s (dS_s - sum_r p_r dS_r); the fp32 exp (<= 2 ulp), the argument s - max
    (2^-24 |s - max|), the row sum ((Ts - 1) 2^-24) and the reciprocal and product (2^-24 each) add relative errors.
  * The backward is checked against the fp64 backward of the kernel's own fp32 probabilities (the saved tensor it
    reads), so forward and backward bounds do not compound.
The largest observed error-to-bound ratio of every tensor is printed (run with -s); all must be <= 1.
"""
import math
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24


def c_gemm(K):
    return 3 * 2.0 ** -16 * (1 + 2.0 ** -7) + K * 2.0 ** -22 + 2.0 ** -23


def _scale(Ts):
    return Ts * (1.0 / Ts) ** 0.5                         # deepvoice3.py:170-171


def ref_forward(q, k, v, mask, drop=None, c=c_gemm):
    """fp64 q (B,E,Td), k, v (B,E,Ts), mask (B,Ts) bool or None, drop (B,Td,Ts) dropout mask or None ->
    (probs, out, bound(probs), bound(out)); c(K) the GEMMs' error coefficient (gamma(K) on the exact-fp32 path)."""
    B, E, Td = q.shape
    Ts = k.shape[2]
    S = torch.einsum("bet,bes->bts", q, k)
    bS = c(E) * torch.einsum("bet,bes->bts", q.abs(), k.abs())
    if mask is not None:
        S = S.masked_fill(mask[:, None, :], -math.inf)
        bS = bS.masked_fill(mask[:, None, :], 0.0)
    P = torch.softmax(S, dim=-1)
    mx = S.max(dim=-1, keepdim=True).values
    e = 2 * 2.0 ** -23 + U24 * (S - mx).abs().nan_to_num(posinf=0.0)      # exp argument + expf ulps
    if mask is not None:
        e = e.masked_fill(mask[:, None, :], 0.0)
    rel = bS + (P * bS).sum(-1, keepdim=True) + e + (P * e).sum(-1, keepdim=True) + (Ts + 2) * U24
    bP = P * rel * (1 + float(bS.max()))                  # (1 + max dS) bounds the second-order remainder
    sc = _scale(Ts)
    Pd, bPd = (P, bP) if drop is None else (P * drop, (bP + U24 * P) * drop)   # + the rounding of p * 1/(1-p)
    out = sc * torch.einsum("bes,bts->bet", v, Pd)
    bout = sc * (torch.einsum("bes,bts->bet", v.abs(), bPd) + c(Ts) * torch.einsum("bes,bts->bet", v.abs(), Pd)) \
        + 2.0 ** -22 * out.abs()
    return P, out, bP, bout


def ref_backward(q, k, v, P, dout, dprobs, c=c_gemm):
    """fp64 backward of the core given the probabilities P the kernel saved (fp32 values) -> {name: (value, bound)}."""
    B, E, Td = q.shape
    Ts = k.shape[2]
    sc = _scale(Ts)
    dPd = sc * torch.einsum("bet,bes->bts", dout, v)
    b_g = c(E) * sc * torch.einsum("bet,bes->bts", dout.abs(), v.abs()) + 2.0 ** -23 * dPd.abs()
    g = dPd if dprobs is None else dPd + dprobs
    b_g = b_g + U24 * g.abs()
    dot = (g * P).sum(-1, keepdim=True)
    b_dot = (b_g * P).sum(-1, keepdim=True) + Ts * U24 * (g.abs() * P).sum(-1, keepdim=True)
    dS = P * (g - dot)
    b_dS = P * (b_g + b_dot) + 2.0 ** -23 * P * (g.abs() + dot.abs())
    dq = torch.einsum("bes,bts->bet", k, dS)
    dk = torch.einsum("bet,bts->bes", q, dS)
    dv = sc * torch.einsum("bet,bts->bes", dout, P)
    adS = dS.abs() + b_dS
    b_dq = torch.einsum("bes,bts->bet", k.abs(), b_dS) + c(Ts) * torch.einsum("bes,bts->bet", k.abs(), adS) \
        + U24 * dq.abs()
    b_dk = torch.einsum("bet,bts->bes", q.abs(), b_dS) + c(Td) * torch.einsum("bet,bts->bes", q.abs(), adS) \
        + U24 * dk.abs()
    b_dv = c(Td) * sc * torch.einsum("bet,bts->bes", dout.abs(), P) + 2.0 ** -22 * dv.abs()
    return {"dq": (dq, b_dq), "dk": (dk, b_dk), "dv": (dv, b_dv)}


def bound_ratio(got, want, bound):
    """max |got - want| / bound (0 where both the error and the bound are 0)."""
    err = (got.double() - want).abs()
    return float((err / bound.clamp_min(1e-300)).max())


def inputs(B, E, Td, Ts, seed, lengths=None):
    """q, k with entries of std 1.2 E^-1/4 (scores of std ~1.4: a softmax that is neither flat nor one-hot),
    v ~ N(0, 1); mask from per-utterance key lengths."""
    gen = torch.Generator().manual_seed(seed)
    s = 1.2 * E ** -0.25
    q = (s * torch.randn(B, E, Td, generator=gen)).cuda()
    k = (s * torch.randn(B, E, Ts, generator=gen)).cuda()
    v = torch.randn(B, E, Ts, generator=gen).cuda()
    dout = torch.randn(B, E, Td, generator=gen).cuda()
    dprobs = torch.randn(B, Td, Ts, generator=gen).cuda()
    mask = None
    if lengths is not None:
        mask = (torch.arange(Ts)[None, :] >= torch.as_tensor(lengths)[:, None]).cuda()
    return q, k, v, dout, dprobs, mask


def mask_lengths(B, Ts, rot):
    """Per-utterance key lengths: 1, Ts and the values around the 32- and 64-key boundaries that fit."""
    pool = [n for n in (1, Ts, 31, 32, 33, 63, 64, 65, 97, Ts - 1) if 1 <= n <= Ts]
    return [pool[(rot + b) % len(pool)] for b in range(B)]


def check_forward(P_dev, out_dev, P, out, bP, bout, mask, what):
    Ts = P.shape[-1]
    rP, rout = bound_ratio(P_dev, P, bP), bound_ratio(out_dev, out, bout)
    if mask is not None:
        assert bool((P_dev.masked_select(mask[:, None, :].expand_as(P_dev)) == 0).all()), what + ": masked key p != 0"
    row_err = float((P_dev.double().sum(-1) - 1).abs().max())
    assert row_err <= (Ts + 2) * 2.0 ** -23, "%s: row sum off by %.3e" % (what, row_err)
    assert rP <= 1 and rout <= 1, "%s: probs %.3f out %.3f x bound" % (what, rP, rout)
    return {"probs": rP, "out": rout}


def check_backward(got, ref, what):
    r = {n: bound_ratio(got[n], *ref[n]) for n in ("dq", "dk", "dv")}
    assert max(r.values()) <= 1, "%s: error / bound %s" % (what, r)
    return r


def _tc_call(q, k, v, mask, dout, dprobs):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    B, E, Td = q.shape
    Ts = k.shape[2]
    sc = _scale(Ts)
    mask_u8 = None if mask is None else mask.to(torch.uint8).contiguous()
    probs = torch.empty(B, Td, Ts, device="cuda")
    out = torch.empty(B, E, Td, device="cuda")
    lib.call("dv3_tc_attn_fwd", ops._p(q), ops._p(k), ops._p(v), ops._p(mask_u8), ops._p(probs), ops._p(out), B, E, Td,
             Ts, sc, 0.0, None, 0, ops._stream())
    ds = torch.empty(B, Td, Ts, device="cuda")
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    lib.call("dv3_tc_attn_bwd", ops._p(dout), ops._p(q), ops._p(k), ops._p(v), ops._p(probs), ops._p(dprobs),
             ops._p(ds), ops._p(dq), ops._p(dk), ops._p(dv), B, E, Td, Ts, sc, 0.0, None, 0, ops._stream())
    torch.cuda.synchronize()
    return probs, out, {"dq": dq, "dk": dk, "dv": dv}


def _sweep():
    """Seeded subset of E x Ts x Td x B that takes every value of every axis, plus the two benchmark shapes."""
    Es, Tss, Tds, Bs = [16, 112, 128, 144, 256], [1, 7, 31, 32, 33, 63, 64, 65, 100, 127, 128], \
        [1, 5, 127, 128, 129, 200, 257], [1, 3, 16]
    rnd = random.Random(2024)
    for ax in (Es, Tds, Bs):
        rnd.shuffle(ax)
    cases = [(Bs[i % 3], Es[i % 5], Tds[i % 7], Ts) for i, Ts in enumerate(Tss)]
    return cases + [(16, 256, 200, 128), (16, 128, 200, 128)]


@pytest.mark.parametrize("case", list(enumerate(_sweep())), ids=lambda c: "B%d-E%d-Td%d-Ts%d" % c[1])
def test_tc_attention_vs_fp64(case):
    from deepvoice3_pytorch_b200._lib import lib
    i, (B, E, Td, Ts) = case
    assert lib.raw("dv3_tc_attn_supported")(B, E, Td, Ts)
    masked = i % 2 == 0 or Td == 200
    q, k, v, dout, dprobs, mask = inputs(B, E, Td, Ts, 100 + i, mask_lengths(B, Ts, i) if masked else None)
    P, out, bP, bout = ref_forward(q.double(), k.double(), v.double(), mask)
    ratios = {}
    for use_dp in (False, True):
        dp = dprobs if use_dp else None
        probs, out_dev, grads = _tc_call(q, k, v, mask, dout, dp)
        what = "tc B=%d E=%d Td=%d Ts=%d mask=%s dprobs=%s" % (B, E, Td, Ts, masked, use_dp)
        ratios.update(check_forward(probs, out_dev, P, out, bP, bout, mask, what))
        ref = ref_backward(q.double(), k.double(), v.double(), probs.double(), dout.double(),
                           None if dp is None else dp.double())
        for n, r in check_backward(grads, ref, what).items():
            ratios[n + ("+dprobs" if use_dp else "")] = r
    print("max error/bound %s: %s" % (what, " ".join("%s %.3g" % kv for kv in sorted(ratios.items()))))


@pytest.mark.parametrize("B,E,Td,Ts", [(3, 40, 129, 65), (2, 272, 31, 33), (3, 128, 200, 129), (16, 256, 200, 200),
                                       (1, 16, 5, 257), (2, 64, 37, 144), (3, 128, 64, 160), (2, 96, 100, 192),
                                       (16, 256, 200, 128)])
def test_attention_fallback_vs_fp64(B, E, Td, Ts, monkeypatch):
    """E % 16 != 0, E > 256 and Ts > 128 are refused by the tensor-core kernels; ops.attention_core runs them on the
    exact-fp32 bgemm + softmax kernels, held to the same bounds with the exact-fp32 GEMM coefficient gamma(K) in place
    of c_gemm(K) (tests/test_gpu_fp32_attention.py pins the two kernels one by one).  A shape the tensor-core kernels
    accept (the benchmark's) runs under conv_math = "fp32".  The launches are recorded: bgemm and softmax ran, no
    tensor-core attention kernel did."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    from test_gpu_fp32_conv import gamma
    if lib.raw("dv3_tc_attn_supported")(B, E, Td, Ts):
        monkeypatch.setattr(ops, "conv_math", "fp32")
    called = []
    real = lib.call

    def spy(name, *args):
        called.append(name)
        return real(name, *args)
    monkeypatch.setattr(lib, "call", spy)
    q, k, v, dout, dprobs, mask = inputs(B, E, Td, Ts, B + E + Td + Ts, mask_lengths(B, Ts, Td))
    qg, kg, vg = [t.clone().requires_grad_(True) for t in (q, k, v)]
    out_dev, probs = ops.attention_core(qg, kg, vg, mask, 0.0, False)
    what = "fallback B=%d E=%d Td=%d Ts=%d" % (B, E, Td, Ts)
    P, out, bP, bout = ref_forward(q.double(), k.double(), v.double(), mask, c=gamma)
    ratios = check_forward(probs.detach(), out_dev.detach(), P, out, bP, bout, mask, what)
    ((out_dev * dout).sum() + (probs * dprobs).sum()).backward()
    ref = ref_backward(q.double(), k.double(), v.double(), probs.detach().double(), dout.double(), dprobs.double(),
                       c=gamma)
    ratios.update(check_backward({"dq": qg.grad, "dk": kg.grad, "dv": vg.grad}, ref, what))
    assert {"dv3_bgemm", "dv3_softmax_fwd", "dv3_softmax_bwd"} <= set(called), called
    assert not [n for n in called if n.startswith("dv3_tc_attn")], called
    print("max error/bound %s: %s" % (what, " ".join("%s %.3g" % kv for kv in sorted(ratios.items()))))
