"""GPU: the ring depths of tc_ring.cuh, walked by every tensor-core GEMM configuration.

Each case's K-iterations per work unit are not a multiple of its configuration's ring depth, and its unit count
exceeds the SM count, so a persistent CTA starts its second unit (and every later one) at a ring phase that is not
zero and wraps the barrier parity mid-unit.  The checks are those of the existing kernel tests, called with these
cases: tests/test_gpu_tc_pairs.py for the two-plane GEMMs (fp64 value of the three products the kernel issues,
the cross-term discriminator, sentinel-guarded write extent) and tests/test_gpu_tc1.py for the single-plane ones.

The T = 1000 cases at B = 16 have short contractions (k = 1, or one 64-channel block per tap) next to the full
epilogue (residual, speaker bias, saved a / s for the gated forward; dropout, addends for the conv), so the
epilogue warpgroup is still storing one unit when the consumers hand off the next.
"""
import pytest

import test_gpu_tc1 as tc1
import test_gpu_tc_pairs as pairs

pytestmark = pytest.mark.gpu

# (NBOX, BR, BK, NPL) -> ring depth, as tc_ring.cuh ConvRing / WgCfg state it
CONV_STAGES = {(2, 64, 32, 2): 4, (1, 128, 32, 2): 4, (1, 64, 64, 2): 4, (1, 64, 32, 2): 6,
               (2, 64, 64, 1): 4, (1, 128, 64, 1): 4, (1, 128, 32, 1): 6, (1, 64, 64, 1): 6, (1, 64, 32, 1): 6}
WGRAD_STAGES = {2: 5, 1: 6}

# two planes: (B, Kc, Nc, T, k, dilation, causal, transpose_taps, epilogue, NaN pad rerun) of test_conv_pairs
PAIR_CONV_CASES = [
    (16, 160, 512, 1000, 1, 1, False, False, "drop", False),    # <1,128,32>: 5 K-iterations, 512 tiles
    (16, 544, 256, 1000, 1, 1, False, True, "add2", False),     # <1,128,32>: data gradient, 17 K-iterations
    (6, 384, 256, 1000, 1, 1, False, False, "add1", False),     # <1,64,64>: 6 K-iterations, 192 tiles
    (6, 84, 256, 1000, 3, 1, True, True, "bias_relu", True),    # <1,64,32>: 9 K-iterations, 192 tiles
]
# (B, C, T, k, dilation, causal, mode, residual, speaker bias, saved outputs) of test_gated_pairs
PAIR_GATED_CASES = [
    (16, 512, 1000, 3, 1, False, 0, True, True, "as"),          # 48 K-iterations, 1024 tiles
    (16, 128, 1000, 3, 2, True, 1, False, True, "as"),          # 12 K-iterations, 256 tiles
]
# one plane: (B, Kc, Nc, T, k, dilation, causal, transpose, p_drop) of test_conv_single_pass
TC1_CONV_CASES = [
    (16, 320, 512, 1000, 1, 1, False, False, 0.0),              # <1,128,64,1>: 5 K-iterations
    (16, 80, 512, 1000, 1, 1, False, True, 0.3),                # <1,128,32,1>: 3 K-iterations, dropout
    (6, 448, 256, 1000, 1, 1, False, False, 0.0),               # <1,64,64,1>: 7 K-iterations
    (6, 80, 256, 1000, 3, 1, True, True, 0.0),                  # <1,64,32,1>: 9 K-iterations
]
# (B, C, T, k, dilation, causal, mode, residual, speaker bias) of test_gated_single_pass
TC1_GATED_CASES = [
    (16, 384, 1000, 3, 1, False, 0, True, True),                # <2,64,64,1>: 18 K-iterations
]
# (B, Mw, Nw, T, k, dilation, causal, msplit form[, NaN pad rerun]) of test_wgrad_pairs / test_wgrad_single_pass
WGRAD_CASES = [
    (16, 1024, 512, 1000, 3, 1, False, False),             # the (16, 512, 1000) ConvBlock's, 96 units per split
    (12, 256, 128, 72, 3, 2, True, False),                 # ragged T, dilated causal
]


def conv_config(B, Kc, Nc, T, k, npl):
    """(NBOX, BR, BK, NPL), K-iterations per tile and tile count of dv3_tc_conv."""
    t_tiles = -(-T // 128)
    narrow = Nc > 64 and (k == 1 or Nc % 64 == 0) and t_tiles * -(-Nc // 128) * B < 100
    bk = 64 if (narrow or npl == 1) and Kc % 64 == 0 else 32
    br = 64 if narrow else 128
    return (1, br, bk, npl), k * -(-Kc // bk), t_tiles * -(-Nc // br) * B


def gated_config(B, C, T, k, npl):
    bk = 32 if npl == 2 else 64
    return (2, 64, bk, npl), k * C // bk, -(-T // 128) * (C // 64) * B


def wgrad_units(B, Mw, Nw, T, k):
    """K-iterations of the longest unit and the unit count of dv3_tc_wgrad_mn."""
    from deepvoice3_pytorch_b200._lib import lib
    ns = lib.raw("dv3_tc_wgrad_nsplit")(B, Mw, Nw, T, k)
    return -(-B // ns) * -(-T // 32), -(-Mw // 128) * -(-Nw // 128) * k * ns


def test_cases_cover_every_ring_off_phase():
    """Every conv configuration and both weight-gradient rings have a case with more units than SMs whose
    K-iterations per unit are not a multiple of the ring depth.  The two-plane gated forward cannot: its k * C / 32
    K-iterations (C % 128 == 0) are a multiple of its 4-deep ring, so it has multi-unit cases only."""
    n = pairs.sms()
    seen = set()
    for cases, npl in ((PAIR_CONV_CASES, 2), (TC1_CONV_CASES, 1)):
        for c in cases:
            cfg, it, tiles = conv_config(*c[:5], npl)
            if it % CONV_STAGES[cfg] and tiles > n:
                seen.add(cfg)
    for cases, npl in ((PAIR_GATED_CASES, 2), (TC1_GATED_CASES, 1)):
        for c in cases:
            cfg, it, tiles = gated_config(*c[:4], npl)
            if (it % CONV_STAGES[cfg] or cfg == (2, 64, 32, 2)) and tiles > n:
                seen.add(cfg)
    assert seen == set(CONV_STAGES), set(CONV_STAGES) - seen
    for npl, depth in WGRAD_STAGES.items():
        assert any(it % depth and units > n for it, units in (wgrad_units(*c[:5]) for c in WGRAD_CASES)), npl


def _ids(c):
    return "_".join(str(int(v)) if isinstance(v, bool) else str(v) for v in c)


@pytest.mark.parametrize("case", PAIR_CONV_CASES, ids=_ids)
def test_conv_pairs_ring(case):
    pairs.test_conv_pairs(case)


@pytest.mark.parametrize("case", PAIR_GATED_CASES, ids=_ids)
def test_gated_pairs_ring(case):
    pairs.test_gated_pairs(case)


@pytest.mark.parametrize("case", WGRAD_CASES, ids=_ids)
def test_wgrad_pairs_ring(case):
    pairs.test_wgrad_pairs(case + (False,))


@pytest.mark.parametrize("case", TC1_CONV_CASES, ids=_ids)
def test_conv_single_pass_ring(case):
    tc1.test_conv_single_pass(case)


@pytest.mark.parametrize("case", TC1_GATED_CASES, ids=_ids)
def test_gated_single_pass_ring(case):
    tc1.test_gated_single_pass(case)


@pytest.mark.parametrize("case", WGRAD_CASES, ids=_ids)
def test_wgrad_single_pass_ring(case):
    tc1.test_wgrad_single_pass(case)

