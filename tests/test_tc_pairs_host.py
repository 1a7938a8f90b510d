"""CPU-only checks of what tests/test_gpu_tc_pairs.py trusts: the fp64 conv oracle ref_conv against torch's own float64
conv1d / conv_transpose1d, the torch restatement of common.cuh split_pair on hand-picked values, and the launcher's
configuration rule, so that the GPU case list reaches every two-plane instantiation of the tensor-core GEMMs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_tc1 import ref_conv
from test_gpu_tc_pairs import (CONV_CASES, GATED_CASES, STAGES, WGRAD_CASES, conv_config, gated_config, ref_wgrad,
                               split_pair)

TAPS = [
    # (k, dilation, causal)
    (1, 1, False), (3, 1, False), (3, 2, True), (5, 3, False), (8, 16, False), (8, 16, True), (4, 2, False),
]


@pytest.mark.parametrize("taps", TAPS, ids=lambda c: "k%d_d%d%s" % (c[0], c[1], "_causal" if c[2] else ""))
def test_ref_conv_equals_conv1d_and_its_transpose(taps):
    k, dil, causal = taps
    B, K, N, T = 2, 5, 3, 50
    g = torch.Generator().manual_seed(k * 10 + dil)
    A = torch.randn(B, T, K, dtype=torch.float64, generator=g)
    W = torch.randn(k, N, K, dtype=torch.float64, generator=g)
    padl = (k - 1) * dil if causal else (k - 1) // 2 * dil
    x = F.pad(A.transpose(1, 2), (padl, (k - 1) * dil - padl))
    want = F.conv1d(x, W.permute(1, 2, 0), dilation=dil)                     # weight (N, K, k)
    torch.testing.assert_close(ref_conv(A, W, k, dil, causal, False), want, rtol=1e-12, atol=1e-12)
    # data gradient: ref_conv with transposed taps is the input gradient of the forward conv whose weight is
    # W[j, n, kc] read as (out = kc, in = n): the adjoint of conv1d, conv_transpose1d, cropped to the padded window
    full = F.conv_transpose1d(A.transpose(1, 2), W.permute(2, 1, 0), dilation=dil)   # weight (in = K, out = N, k)
    torch.testing.assert_close(ref_conv(A, W, k, dil, causal, True), full[:, :, padl:padl + T], rtol=1e-12,
                               atol=1e-12)


def test_ref_wgrad_is_the_weight_gradient_of_conv1d():
    B, M, N, T = 2, 4, 3, 40
    for k, dil, causal in TAPS:
        g = torch.Generator().manual_seed(k + dil)
        DY = torch.randn(B, T, M, dtype=torch.float64, generator=g)
        X = torch.randn(B, T, N, dtype=torch.float64, generator=g)
        w = torch.zeros(M, N, k, dtype=torch.float64, requires_grad=True)
        padl = (k - 1) * dil if causal else (k - 1) // 2 * dil
        y = F.conv1d(F.pad(X.transpose(1, 2), (padl, (k - 1) * dil - padl)), w, dilation=dil)
        (y * DY.transpose(1, 2)).sum().backward()
        torch.testing.assert_close(ref_wgrad(DY, X, k, dil, causal), w.grad, rtol=1e-12, atol=1e-12)


def _check(x, f16, hi, lo):
    p = split_pair(torch.tensor([x], dtype=torch.float32), f16).float()
    got = (float(p[0, 0]), float(p[1, 0]))
    assert got == (hi, lo), (x, got, (hi, lo))
    assert all(np.signbit(g) == np.signbit(w) for g, w in zip(got, (hi, lo))), (x, got)


def test_split_pair_fp16_hand_picked():
    e = 2.0 ** -10                                                   # fp16 spacing on [1, 2)
    _check(1 + e / 2, True, 1.0, 1.0)                                # tie -> even (down); lo = 2^-11 * 2^11
    _check(1 + 3 * e / 2, True, 1 + 2 * e, -1.0)                     # tie -> even (up)
    _check(65504.0, True, 65504.0, 0.0)
    _check(-65504.0, True, -65504.0, 0.0)
    _check(65500.0, True, 65504.0, -8192.0)                          # below the top: rounds up to it
    for past in (65519.0, 65520.0, 7e4, 1e6, 3e38):                  # clamped: the fp16 pair stays finite
        _check(past, True, 65504.0, 0.0)
        _check(-past, True, -65504.0, 0.0)
    _check(1.5 * 2.0 ** -24, True, 2.0 ** -23, -(2.0 ** -14))       # subnormal tie -> even; lo at the normal minimum
    _check(2.0 ** -25, True, 0.0, 2.0 ** -14)                        # tie with zero -> +0
    _check(-0.0, True, -0.0, 0.0)
    # against numpy's float16 rounding (round to nearest even, subnormals included) over a spread of magnitudes
    g = np.random.default_rng(0)
    x = (g.standard_normal(4096) * 10.0 ** g.uniform(-8, 5, 4096)).astype(np.float32)
    c = np.clip(x, -65504, 65504)
    hi = c.astype(np.float16)
    lo = ((c - hi.astype(np.float32)) * np.float32(2048)).astype(np.float16)
    p = split_pair(torch.from_numpy(x), True)
    assert np.array_equal(p[0].numpy().view(np.int16), hi.view(np.int16))
    assert np.array_equal(p[1].numpy().view(np.int16), lo.view(np.int16))


def test_split_pair_bf16_hand_picked():
    e = 2.0 ** -7                                                    # bf16 spacing on [1, 2)
    _check(1 + e / 2, False, 1.0, 8.0)                               # tie -> even (down): lo = 2^-8 * 2^11
    _check(1 + 3 * e / 2, False, 1 + 2 * e, -8.0)                    # tie -> even (up)
    _check(65520.0, False, 65536.0, -32768.0)                        # no clamp in the bf16 pair
    _check(1e6, False, 999424.0, 576.0 * 2048)
    for exact in (1.5, -3.0 * 2.0 ** 50, 2.0 ** -100, 1.0 + e, -(2.0 ** 127) * 1.5):   # bf16 values: lo = +0 exactly
        _check(exact, False, exact, 0.0)
    _check(-0.0, False, -0.0, 0.0)


def _tap_outside(k, dil, causal, T):
    padl = (k - 1) * dil if causal else (k - 1) // 2 * dil
    return any(abs(j * dil - padl) >= T for j in range(k))


def _ids_reached():
    cfgs = {}
    for c in CONV_CASES:
        cfg, it, _, tiles = conv_config(*c[:4], c[4])
        cfgs.setdefault(cfg, []).append((tiles, it % STAGES[cfg] != 0, c))
    for c in GATED_CASES:
        cfg, it, _, tiles = gated_config(*c[:4])
        cfgs.setdefault(cfg, []).append((tiles, it % STAGES[cfg] != 0, c))
    return cfgs


def test_case_list_reaches_every_two_plane_configuration():
    cfgs = _ids_reached()
    assert set(cfgs) == {(2, 64, 32), (1, 128, 32), (1, 64, 64), (1, 64, 32)}, set(cfgs)
    assert WGRAD_CASES                                                # tc_wgrad_mn_kernel<2>
    sms = 132                                                         # H100 SXM; the GPU test uses the device's count
    # 128-column conv: more than two waves with a tile's K-iterations not a multiple of the ring depth
    assert any(t > 2 * sms and odd for t, odd, _ in cfgs[(1, 128, 32)])
    # gated: more than two waves (its K-iterations, k * C / 32 with C % 128 == 0, always fill whole rings)
    assert any(t > 2 * sms for t, _, _ in cfgs[(2, 64, 32)])
    # 64-column convs: the launcher picks them only below 100 128-column tiles, so at most 198 tiles; the case list
    # has CTAs walking a second tile, at a ring phase that is not a multiple of the depth
    for cfg in ((1, 64, 64), (1, 64, 32)):
        assert any(t > sms and odd for t, odd, _ in cfgs[cfg]), cfg
    narrow = [conv_config(B, 64, N, T, 1) for B in range(1, 100) for N in range(65, 1100, 7)
              for T in range(1, 1500, 97)]
    assert max(tiles for cfg, _, _, tiles in narrow if cfg[1] == 64) < 200


def test_case_list_covers_the_axes():
    """fp16 and bf16 operands, ragged T, N and K tails, taps, and every epilogue, on each conv configuration."""
    cfgs = _ids_reached()
    for cfg in ((1, 128, 32), (1, 64, 64), (1, 64, 32)):
        cases = [c for _, _, c in cfgs[cfg]]
        assert {c[7] for c in cases} == {False, True}, cfg
        assert {1, 37, 128, 129, 203} <= {c[3] for c in cases}, cfg
        assert {1, 3, 5, 8} <= {c[4] for c in cases}, cfg
        assert {"none", "bias_relu", "drop", "add1", "add2"} <= {c[8] for c in cases}, cfg
        assert any(c[5] > 1 for c in cases) and any(c[6] for c in cases), cfg
        assert any(_tap_outside(c[4], c[5], c[6], c[3]) for c in cases), cfg
        if cfg != (1, 64, 64):                                                # Kc % 64 == 0 there
            assert {8, 16, 80, 513} <= {c[1] for c in cases}, cfg
            assert any(c[9] for c in cases), cfg                              # NaN pad-column rerun
    assert {16, 80, 513} <= {c[2] for _, _, c in cfgs[(1, 128, 32)]}
    assert 513 in {c[2] for cfg in ((1, 64, 64), (1, 64, 32)) for _, _, c in cfgs[cfg]}
    g = [c for _, _, c in cfgs[(2, 64, 32)]]
    assert {(c[6], c[7]) for c in g} >= {(0, True), (0, False), (1, False)} and any(c[8] for c in g)
    assert {c[9] for c in g} >= {"", "a", "s", "as"}
    w = WGRAD_CASES
    assert any(c[3] % 32 and c[3] > 32 for c in w) and any(c[3] < 32 for c in w)
    assert any(_tap_outside(c[4], c[5], c[6], c[3]) for c in w)
    assert {16, 80, 513} <= {c[1] for c in w} | {c[2] for c in w} and any(c[7] for c in w) and any(c[8] for c in w)
