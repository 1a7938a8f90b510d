"""GPU: the persistent tensor-core weight gradient (tc_wgrad_mn_kernel, DESIGN.md section 2.2) where its schedule
matters: CTAs that walk three or more work units, a short last split (B not a multiple of the utterances per split),
T not a multiple of 32, k = 1 and k = 3 at dilation 27, the ConvTranspose layout, one and two operand planes, and the
same launch twice bit for bit.

Every slot s of the nsplit slots (dv3_tc_wgrad_nsplit) is checked against fp64 over exactly its own utterances
[s * bps, min(B, (s + 1) * bps)), with the bound of tests/test_gpu_tc_pairs.py test_wgrad_pairs (n_mma = 2 per 32-row
time chunk of the slot); two-plane launches also pass the cross-term discriminator on the slot sum.  Slots sit in a
sentinel-filled buffer a gap apart: nothing outside them is written and every element inside is."""
import pytest
import torch

from test_gpu_tc1 import _call, _p, _st, c1, ratio
from test_gpu_tc_pairs import (GUARD, SENT32, discriminator, gamma, guarded, pair_planes, pair_reference,
                               ref_wgrad, sms)

pytestmark = pytest.mark.gpu

CASES = [
    # (B, Mw, Nw, T, k, dilation, causal, ConvTranspose layout, npl)
    (16, 1024, 512, 800, 3, 1, False, False, 2),     # the (16, 512, 800) ConvBlock: three units per CTA
    (16, 1024, 512, 800, 3, 1, False, False, 1),
    (16, 1024, 512, 128, 3, 27, False, False, 2),    # the encoder shape at dilation 27
    (37, 512, 256, 64, 3, 27, True, False, 2),       # B prime: a short last split
    (37, 512, 256, 64, 3, 27, True, False, 1),
    (13, 1024, 512, 100, 3, 27, False, False, 2),    # T % 32 != 0
    (77, 1024, 512, 40, 1, 27, False, False, 2),     # k = 1, short last split, T % 32 != 0
    (77, 1024, 512, 40, 1, 1, False, True, 2),       # the ConvTranspose layout
    (77, 1024, 512, 40, 1, 1, False, True, 1),
]


def cta0_units(B, Mw, Nw, k, nsplit):
    units = -(-Mw // 128) * -(-Nw // 128) * k * nsplit
    return -(-units // min(units, sms()))


def launch(dy, x, npl, B, Mw, Nw, T, k, dil, causal, convt, gap=37):
    """-> (sentinel buffer, slots [nsplit][numel + gap], nsplit, idx mapping (m, n, j) to a slot element)."""
    from deepvoice3_pytorch_b200._lib import lib
    nsplit = lib.raw("dv3_tc_wgrad_nsplit")(B, Mw, Nw, T, k)
    numel, stride = Mw * Nw * k, Mw * Nw * k + gap
    buf, parts = guarded(nsplit * stride)
    if convt:       # m = (j, co) with Cout = Mw / 2 -> element at (m % Cout) * 2 + m // Cout + n * Mw
        ms, s_m, s_mh, s_n, s_j = Mw // 2, 2, 1, Mw, 0
    else:
        ms, s_m, s_mh, s_n, s_j = Mw, Nw, 0, 1, Mw * Nw
    _call("dv3_tc_wgrad_mn_npl", _p(dy), _p(x), npl, _p(parts), stride, B, Mw, Nw, T, k, dil, int(causal), ms, s_m,
          s_mh, s_n, s_j, _st())
    torch.cuda.synchronize()
    m = torch.arange(Mw, device="cuda")[:, None, None]
    n = torch.arange(Nw, device="cuda")[None, :, None]
    j = torch.arange(k, device="cuda")[None, None, :]
    idx = ((m % ms) * s_m + (m // ms) * s_mh + n * s_n + j * s_j).flatten()
    return buf, parts.view(nsplit, stride), nsplit, idx


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_M%d_N%d_T%d_k%d_d%d%s%s_npl%d" % (
    c[0], c[1], c[2], c[3], c[4], c[5], "_causal" if c[6] else "", "_convT" if c[7] else "", c[8]))
def test_wgrad_persistent(case):
    B, Mw, Nw, T, k, dil, causal, convt, npl = case
    g = torch.Generator(device="cuda").manual_seed(Mw + 3 * Nw + T + B)
    DY = torch.randn(B, T, Mw, device="cuda", generator=g) * 1e-3
    X = torch.randn(B, T, Nw, device="cuda", generator=g)
    dy, x = pair_planes(DY, False), pair_planes(X, False)
    if npl == 1:
        dy, x = dy[:1].contiguous(), x[:1].contiguous()
    buf, parts, nsplit, idx = launch(dy, x, npl, B, Mw, Nw, T, k, dil, causal, convt)
    numel = Mw * Nw * k
    bits = buf.view(torch.int32)
    assert bool((bits[:GUARD] == SENT32).all()) and bool((bits[GUARD + nsplit * parts.shape[1]:] == SENT32).all())
    assert bool((parts[:, numel:].view(torch.int32) == SENT32).all()), "write into the gap between slots"
    assert bool(torch.isfinite(parts[:, :numel]).all()), "slot element left unwritten"
    bps, kb_n = -(-B // nsplit), -(-T // 32)
    worst, R, X1, X2, total = 0.0, 0.0, 0.0, 0.0, 0.0
    for s in range(nsplit):
        b0, b1 = s * bps, min(B, (s + 1) * bps)
        got = parts[s, :numel][idx].view(Mw, Nw, k)
        fn = lambda P, Q: ref_wgrad(P, Q, k, dil, causal)  # noqa: E731
        if npl == 2:
            Rs, x1, x2, absb = pair_reference(dy[:, b0:b1, :, :Mw], x[:, b0:b1, :, :Nw], fn)
            X1, X2 = X1 + x1, X2 + x2
        else:
            P, Q = dy[0, b0:b1, :, :Mw].double(), x[0, b0:b1, :, :Nw].double()
            Rs, absb = fn(P, Q), fn(P.abs(), Q.abs())
        n_mma = 2 * (b1 - b0) * kb_n
        bound = c1((b1 - b0) * T) * absb + (gamma() * n_mma + 2.0 ** -23) * Rs.abs()
        worst = max(worst, ratio(got, Rs, bound))
        total, R = total + got.double(), R + Rs
    d = discriminator(total - R, X1, X2) if npl == 2 else float("nan")
    print("wgrad %s: nsplit %d, %d units on CTA 0, last split %d of %d utterances; error/bound %.3g, discriminator "
          "%.3g" % (case, nsplit, cta0_units(B, Mw, Nw, k, nsplit), B - (nsplit - 1) * bps, bps, worst, d))
    assert worst <= 1, worst
    assert npl == 1 or d <= 1, d
    buf2, _, _, _ = launch(dy, x, npl, B, Mw, Nw, T, k, dil, causal, convt)
    assert torch.equal(buf.view(torch.int32), buf2.view(torch.int32)), "two launches differ"


def test_cases_cover_the_schedule():
    """With the device's SM count: a case per plane count where CTA 0 walks three or more units, and cases with a
    short last split at k = 3 and in the ConvTranspose layout."""
    from deepvoice3_pytorch_b200._lib import lib
    many, short = set(), set()
    for B, Mw, Nw, T, k, dil, causal, convt, npl in CASES:
        ns = lib.raw("dv3_tc_wgrad_nsplit")(B, Mw, Nw, T, k)
        if cta0_units(B, Mw, Nw, k, ns) >= 3:
            many.add(npl)
        if B % -(-B // ns):
            short.add("convT" if convt else "k%d" % k)
    assert many == {1, 2}, many
    assert {"k3", "convT"} <= short, short
