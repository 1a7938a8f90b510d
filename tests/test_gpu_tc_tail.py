"""GPU: the last unit of every CTA of the tensor-core GEMMs, whose epilogue the two consumer warpgroups share with the
epilogue warpgroup (DESIGN.md section 2.2), and the L2 prefetch of the epilogue inputs.

The unit counts sit around the device's SM count (SMs - 1, SMs, SMs + 1, 2 SMs - 1, or the nearest even counts for
the gated forward, whose tiles come in channel pairs), so that the last units of CTAs with one unit and of CTAs with
two are both hit.  The epilogues are checked as in tests/test_gpu_tc_epilogue.py against the same epilogue applied
in torch to the raw GEMM, every output between canary bands; since the raw GEMM runs through the same last-unit path,
it is checked too, against float64 (a misplaced slice of the tile is an O(1) error there).  The cases walk gated GLU
and highway with and without residual and speaker bias, data-gradient addmodes 0 / 1 / 2 with dropout and ReLU, both
plane counts, ragged T (72, 200), channel tails (80, 513), the per-thread stores (T % 4 != 0, a misaligned output),
and the weight gradient's tap-major and ConvTranspose partials with Mw / Nw tails against float64."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_tc_epilogue import _check_conv, _check_gated, _launch_conv, _launch_gated, _planes
from test_gpu_tc_wgrad import test_wgrad_persistent as _check_wgrad

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gated_cases(S):
    # (B, C, T, k, dilation, causal, mode, residual, speaker bias, saved outputs, npl); C = 128, T <= 128: 2 B units
    return [
        ((S - 2) // 2, 128, 72, 3, 1, True, 0, True, False, "as", 2),
        (S // 2, 128, 128, 3, 2, False, 1, False, True, "as", 2),
        ((S + 2) // 2, 128, 100, 3, 1, False, 0, False, True, "a", 1),
        (S - 1, 128, 128, 3, 1, False, 0, True, True, "s", 2),
        (S // 2, 128, 102, 3, 1, False, 1, False, False, "as", 2),     # per-thread stores and residual fill
    ]


def _conv_cases(S):
    # (B, Kc, Nc, T, k, dilation, causal, transpose_taps, bias, relu, p_drop, addmode, npl, misaligned output)
    return [
        # 128-wide tiles, one per utterance (B >= 100): B units
        (S - 1, 128, 128, 72, 1, 1, False, False, True, True, 0.0, 0, 2, False),
        (S, 128, 128, 128, 1, 1, False, True, False, False, 0.3, 1, 2, False),
        (S + 1, 128, 128, 100, 1, 1, False, True, True, False, 0.3, 2, 1, False),
        (2 * S - 1, 128, 128, 64, 1, 1, False, True, False, True, 0.0, 2, 2, False),
        # 64-wide data gradients at the step's one-wave shapes and one past them
        (16, 512, 256, 200, 3, 1, True, True, False, False, 0.05, 1, 2, False),
        (16, 1024, 512, 128, 3, 3, False, True, False, False, 0.0, 2, 2, False),
        (17, 1024, 512, 128, 3, 1, False, True, False, True, 0.05, 2, 1, False),
        # channel tails, per-thread stores
        (16, 256, 80, 200, 1, 1, False, False, True, False, 0.0, 0, 2, False),
        (8, 256, 513, 72, 1, 1, False, False, False, False, 0.3, 0, 2, False),
        (S - 1, 128, 128, 102, 1, 1, False, True, False, False, 0.0, 1, 2, False),
        (S, 128, 128, 72, 1, 1, False, False, True, False, 0.0, 0, 2, True),
    ]


WGRAD = [
    # (B, Mw, Nw, T, k, dilation, causal, ConvTranspose layout, npl)
    (16, 1024, 512, 128, 3, 1, False, False, 2),     # the encoder shape: 96 units, one per CTA
    (16, 512, 256, 200, 3, 1, True, False, 2),       # the decoder shape
    (16, 512, 256, 200, 3, 1, True, False, 1),
    (11, 200, 72, 96, 3, 1, False, False, 2),        # Mw / Nw tails
    (40, 328, 264, 72, 1, 1, False, True, 2),        # ConvTranspose layout with tails
    (40, 328, 264, 72, 1, 1, False, True, 1),
]


def _raw_ref(r, kind, idx):
    """float64 GEMM of the planes the raw launch of case idx consumed, (B, N, T): the launchers' own draws, replayed
    from their seeds."""
    if kind == "gated":
        B, C, T, k, dil, causal = r["case"][:6]
        npl, tt, Kc = r["case"][10], False, C
        g = torch.Generator().manual_seed(500 + idx)
        a = _planes(g, (B, T, C), npl, torch.float16)
        w = _planes(g, (k, 2 * C, C), npl, torch.float16, scale=(1.0 / (k * C)) ** 0.5)
    else:
        B, Kc, Nc, T, k, dil, causal, tt = r["case"][:8]
        npl, kp = r["case"][12], (Kc + 7) // 8 * 8
        g = torch.Generator().manual_seed(700 + idx)
        dt = torch.bfloat16 if tt else torch.float16
        a = _planes(g, (B, T, kp), npl, dt)
        w = _planes(g, (k, Nc, kp), npl, dt, scale=(1.0 / (k * Kc)) ** 0.5)
    val = lambda pl: pl[0].double() + (pl[1].double() * 2.0 ** -11 if pl.shape[0] == 2 else 0.0)  # noqa: E731
    x = val(a)[..., :Kc].transpose(1, 2)                              # (B, Kc, T)
    wt = val(w)[..., :Kc].permute(1, 2, 0)                            # (N, Kc, k)
    padl = (k - 1) * dil if causal else (k - 1) // 2 * dil
    if tt:                                                            # offsets padl - j d: taps reversed
        wt, pad = wt.flip(2), ((k - 1) * dil - padl, padl)
    else:
        pad = (padl, (k - 1) * dil - padl)
    xp = F.pad(x, pad)
    return F.conv1d(xp, wt, dilation=dil), F.conv1d(xp.abs(), wt.abs(), dilation=dil)


def _raw_ok(r, kind, idx):
    want, mag = _raw_ref(r, kind, idx)
    got = r["raw"].t.double()
    return bool(torch.isfinite(got).all()) and bool(((got - want).abs() <= 1e-4 * mag + 1e-30).all())


def test_last_unit_epilogues_match_torch():
    from deepvoice3_pytorch_b200 import ops
    st = ops._stream()
    S = _sms()
    launched = [("gated", 40 + i, _launch_gated(c, 40 + i, st)) for i, c in enumerate(_gated_cases(S))]
    launched += [("conv", 40 + i, _launch_conv(c, 40 + i, st)) for i, c in enumerate(_conv_cases(S))]
    torch.cuda.synchronize()
    ops.check_index_errors()
    bad = {}
    for kind, idx, r in launched:
        errs = _check_gated(r) if kind == "gated" else _check_conv(r)
        if not _raw_ok(r, kind, idx):
            errs.append("raw GEMM against float64")
        if errs:
            bad["%s %s" % (kind, r["case"])] = errs
    assert not bad, bad


def test_cases_cover_the_unit_counts():
    """The conv cases give SMs - 1, SMs, SMs + 1 and 2 SMs - 1 units; the gated ones fewer, as many and more units
    than SMs."""
    S = _sms()
    conv = {B * -(-T // 128) for B, Kc, Nc, T, k, *_ in _conv_cases(S) if Nc == 128 and B >= 100}
    assert {S - 1, S, S + 1, 2 * S - 1} <= conv, conv
    gated = {2 * B * -(-T // 128) for B, C, T, *_ in _gated_cases(S)}
    assert min(gated) < S and S in gated and max(gated) > S, gated


@pytest.mark.parametrize("case", WGRAD, ids=lambda c: "B%d_M%d_N%d_T%d_k%d%s_npl%d" % (
    c[0], c[1], c[2], c[3], c[4], "_convT" if c[7] else "", c[8]))
def test_last_unit_wgrad_partials(case):
    _check_wgrad(case)
