"""CPU-only checks of the single-pass mode's host side: ops.conv_math accepts "tc1" (and still refuses an unknown
value), the one-plane entry points resolve with argtypes derived from include/dv3b200.h, and a TrainStep refuses to
step under another mode than the one it was built in."""
import ctypes

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module", autouse=True)
def built_library():
    from deepvoice3_pytorch_b200 import _build
    _build.build()


def test_conv_math_modes(monkeypatch):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import Dv3Error
    for mode, tc, npl in (("tc", True, 2), ("bf16x3", True, 2), ("tc1", True, 1), ("fp32", False, None)):
        monkeypatch.setattr(ops, "conv_math", mode)
        assert ops._tc_selected() is tc
        if tc:
            assert ops._npl() == npl
    monkeypatch.setattr(ops, "conv_math", "tf32")
    with pytest.raises(Dv3Error, match="unknown conv_math"):
        ops._tc_selected()


def test_single_plane_entry_points_resolve_from_the_header():
    from deepvoice3_pytorch_b200._lib import lib, parse_header
    decls = parse_header()
    want = {"dv3_tc_gate_bwd_split_npl": ("npl", "tlen", "tmult"), "dv3_tc_grad_split_npl": ("npl", "tlen", "tmult"),
            "dv3_tc_wgrad_mn_npl": ("npl",), "dv3_tc_weightnorm_fwd_batched_npl": ("npl",)}
    lib.load()
    for name, args in want.items():
        assert name in decls, name
        _, params = decls[name]
        names = [n for _, n in params]
        assert all(a in names for a in args), (name, names)
        assert params[names.index("npl")][0] is ctypes.c_int
        fn = lib.raw(name)
        assert fn.argtypes == [t for t, _ in params] and fn.restype is ctypes.c_int
    # the pair-only entry points keep their signatures
    assert "npl" not in [n for _, n in decls["dv3_tc_wgrad_mn"][1]]
    assert "npl" not in [n for _, n in decls["dv3_tc_gate_bwd_split"][1]]


def test_train_step_refuses_a_mode_switch(monkeypatch):
    from deepvoice3_pytorch_b200 import builder, ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    kw = dict(n_vocab=149, embed_dim=32, mel_dim=80, linear_dim=129, r=1, downsample_step=4, kernel_size=3,
              encoder_channels=32, decoder_channels=32, converter_channels=32, max_positions=64)
    monkeypatch.setattr(ops, "conv_math", "tc1")
    step = TrainStep(builder.deepvoice3(**kw), weight_bank=True)
    assert step.math == "tc1" and step.bank.npl == 1
    monkeypatch.setattr(ops, "conv_math", "tc")
    with pytest.raises(ValueError, match="conv_math"):
        step.step({})
    monkeypatch.setattr(ops, "conv_math", "fp32")
    with pytest.raises(ValueError, match="conv_math"):
        step.step({})
