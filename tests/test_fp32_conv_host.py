"""CPU-only: the exact-fp32 conv entry points (csrc/conv.cu) refuse problems past 32-bit indexing before they launch.

The kernels gather with int arithmetic ((b * Cin + ci) * T + tt) and index the dropout hash with uint32, so a tensor of
2^31 elements or more must fail with a message instead of overflowing silently.  Every call here passes NULL pointers at
a refused size: the refusal has to come before any launch.  (No call uses a size the guards accept: with NULL pointers
that would launch a kernel on them.  Every launch of tests/test_gpu_fp32_conv.py shows that ordinary sizes pass.)
"""
import pytest

LIMIT = 2 ** 31

# (B, C_small, C_large, T): B * C_large * T elements in the largest tensor, exactly 2^31 or past it
SIZES = [(2, 1, 2 ** 15, 2 ** 15), (1, 3, 2 ** 16, 2 ** 15 + 1), (2 ** 15, 16, 2 ** 16, 1)]


@pytest.fixture(scope="module", autouse=True)
def built_library():
    from deepvoice3_pytorch_b200 import _build
    _build.build()


def _calls(B, Cs, Cl, T):
    """(entry point, arguments) for each conv launcher, the large channel count on either side of the GEMM."""
    fwd = lambda Cin, Cout: ("dv3_conv1d_fwd", (None, None, None, None, B, Cin, Cout, T, 1, 1, 0, 0, None))
    dgrad = lambda M, Cin: ("dv3_conv1d_dgrad", (None, None, None, B, M, Cin, T, 1, 1, 0, 0.0, None, 0, 0, None, None,
                                                 0.0, None))
    wgrad = lambda M, Cin: ("dv3_conv1d_wgrad", (None, None, None, 0, B, M, Cin, T, 1, 1, 0, 0.0, None, 0, M, Cin, 0,
                                                 1, 0, None))
    block = ("dv3_convblock_fwd", (None, None, None, None, None, None, None, B, Cl, T, 1, 1, 0, 0, 1, 0.0, None, 0,
                                   None))
    return [fwd(Cs, Cl), fwd(Cl, Cs), dgrad(Cs, Cl), dgrad(Cl, Cs), wgrad(Cs, Cl), wgrad(Cl, Cs), block]


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "B%d_C%d_T%d" % (s[0], s[2], s[3]))
def test_conv_launchers_refuse_32bit_overflow(size):
    from deepvoice3_pytorch_b200._lib import Dv3Error, lib
    B, Cs, Cl, T = size
    n = B * Cl * T
    assert n >= LIMIT and B * T < LIMIT
    for name, args in _calls(B, Cs, Cl, T):
        with pytest.raises(Dv3Error, match=r"%s: tensor of %d elements too large for 32-bit indexing"
                           % (name[4:], n)):
            lib.call(name, *args)
