"""Weight-norm entry points, bit for bit.  Every packed layout must equal w = v * scale, recomputed in torch from the
kernel's own ``scale`` output: as is in fp32 (dv3_weightnorm_fwd), or split into the 16-bit operand pairs of the
tensor-core path (dv3_tc_weightnorm_fwd, dv3_tc_weightnorm_convt_fwd, dv3_tc_weightnorm_fwd_batched).  The per-layer
and the batched backward share one row body and no atomics, so they must agree exactly.  Pad columns are not compared.
The checks pin outputs, not a build: they pass against any library of the same ABI (DV3_LIB)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CONV_SHAPES = [(129, 80, 1), (256, 16, 3), (45, 70, 5), (1024, 512, 3)]      # v (Cout, Cin, k)
CONVT_SHAPES = [(80, 129), (256, 256)]                                         # v (Cin, Cout, 2)


def _ops():
    from deepvoice3_pytorch_b200 import ops
    return ops


def _params(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    v = torch.randn(*shape, generator=gen)
    g = torch.rand(shape[0], generator=gen) * 4 + 0.1
    g[0] = 1.0e5                       # a row past the fp16 range: exercises the clamp of the fp16 pair
    return v.cuda(), g.view(-1, 1, 1).cuda()


def _same_bits(a, b):
    as_int = {4: torch.int32, 2: torch.int16}[a.element_size()]
    return a.shape == b.shape and torch.equal(a.contiguous().view(as_int), b.contiguous().view(as_int))


def _norm_outputs(v_rows, g, inv, scale):
    """inv = 1/||v|| to fp32 rounding; scale = g * inv bit for bit."""
    want = 1.0 / v_rows.double().norm(dim=1)
    np.testing.assert_allclose(inv.double().cpu().numpy(), want.cpu().numpy(), rtol=1e-5)
    assert _same_bits(scale, g.flatten() * inv)


def _pair(w, f16):
    """The (hi, lo) split of common.cuh split_pair: [2, *w.shape]."""
    if f16:
        c = w.clamp(-65504.0, 65504.0)
        hi = c.half()
        return torch.stack([hi, ((c - hi.float()) * 2048.0).half()])
    hi = w.bfloat16()
    return torch.stack([hi, ((w - hi.float()) * 2048.0).bfloat16()])


@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_fp32_weightnorm_layouts_are_v_times_scale(shape):
    ops = _ops()
    Cout, Cin, k = shape
    v, g = _params(shape, 10 + k)
    w_f = torch.empty(k, Cin, Cout, device="cuda")
    w_b = torch.empty(k, Cout, Cin, device="cuda")
    inv, scale = torch.empty(Cout, device="cuda"), torch.empty(Cout, device="cuda")
    ops.lib.call("dv3_weightnorm_fwd", ops._p(v), ops._p(g), ops._p(inv), ops._p(scale), ops._p(w_f), ops._p(w_b),
                 Cout, Cin, k, 1, Cout, Cin * Cout, Cin, 1, Cout * Cin, ops._stream())
    torch.cuda.synchronize()
    _norm_outputs(v.reshape(Cout, -1), g, inv, scale)
    w = v * scale[:, None, None]
    assert _same_bits(w_f, w.permute(2, 1, 0))
    assert _same_bits(w_b, w.permute(2, 0, 1))


@pytest.mark.parametrize("shape", CONVT_SHAPES)
def test_fp32_weightnorm_convt_layouts_are_v_times_scale(shape):
    """The ConvTranspose1d(k=2,s=2) layouts of ops._CONVT: w_f [ci][(j,co)], w_b [(j,co)][ci]."""
    ops = _ops()
    Cin, Cout = shape
    v, g = _params((Cin, Cout, 2), 20 + Cin)
    w_f = torch.empty(Cin, 2 * Cout, device="cuda")
    w_b = torch.empty(2 * Cout, Cin, device="cuda")
    inv, scale = torch.empty(Cin, device="cuda"), torch.empty(Cin, device="cuda")
    ops.lib.call("dv3_weightnorm_fwd", ops._p(v), ops._p(g), ops._p(inv), ops._p(scale), ops._p(w_f), ops._p(w_b),
                 Cin, Cout, 2, 2 * Cout, 1, Cout, 1, Cin, Cout * Cin, ops._stream())
    torch.cuda.synchronize()
    _norm_outputs(v.reshape(Cin, -1), g, inv, scale)
    w = v * scale[:, None, None]                                  # (ci, co, j)
    assert _same_bits(w_f, w.permute(0, 2, 1).reshape(Cin, 2 * Cout))
    assert _same_bits(w_b, w.permute(2, 1, 0).reshape(2 * Cout, Cin))


def _tc_conv_planes(v, g):
    ops = _ops()
    Cout, Cin, k = v.shape
    wfwd = torch.empty(2, k, Cout, ops._pad8(Cin), device="cuda", dtype=torch.float16)
    wbwd = torch.empty(2, k, Cin, ops._pad8(Cout), device="cuda", dtype=torch.bfloat16)
    inv, scale = torch.empty(Cout, device="cuda"), torch.empty(Cout, device="cuda")
    ops.lib.call("dv3_tc_weightnorm_fwd", ops._p(v), ops._p(g), ops._p(inv), ops._p(scale), ops._p(wfwd), 2,
                 ops._p(wbwd), Cout, Cin, k, ops._stream())
    torch.cuda.synchronize()
    return inv, scale, wfwd, wbwd


def _check_conv_planes(v, scale, wfwd, wbwd):
    Cout, Cin, k = v.shape
    w = v * scale[:, None, None]
    assert _same_bits(wfwd[..., :Cin], _pair(w.permute(2, 0, 1), True))      # [k][Cout][Cin] fp16 pair
    assert _same_bits(wbwd[..., :Cout], _pair(w.permute(2, 1, 0), False))    # [k][Cin][Cout] bf16 pair


@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_tc_weightnorm_planes_are_split_of_v_times_scale(shape):
    v, g = _params(shape, 30 + shape[2])
    inv, scale, wfwd, wbwd = _tc_conv_planes(v, g)
    _norm_outputs(v.reshape(shape[0], -1), g, inv, scale)
    _check_conv_planes(v, scale, wfwd, wbwd)


@pytest.mark.parametrize("shape", CONVT_SHAPES)
def test_tc_weightnorm_convt_planes_are_split_of_v_times_scale(shape):
    ops = _ops()
    Cin, Cout = shape
    v, g = _params((Cin, Cout, 2), 40 + Cin)
    wfwd = torch.empty(2, 2 * Cout, ops._pad8(Cin), device="cuda", dtype=torch.float16)
    wbwd = torch.empty(2, Cin, ops._pad8(2 * Cout), device="cuda", dtype=torch.bfloat16)
    inv, scale = torch.empty(Cin, device="cuda"), torch.empty(Cin, device="cuda")
    ops.lib.call("dv3_tc_weightnorm_convt_fwd", ops._p(v), ops._p(g), ops._p(inv), ops._p(scale), ops._p(wfwd), 2,
                 ops._p(wbwd), Cin, Cout, ops._stream())
    torch.cuda.synchronize()
    _norm_outputs(v.reshape(Cin, -1), g, inv, scale)
    w = v * scale[:, None, None]                                  # (ci, co, j)
    assert _same_bits(wfwd[..., :Cin], _pair(w.permute(2, 1, 0).reshape(2 * Cout, Cin), True))
    assert _same_bits(wbwd[..., :2 * Cout], _pair(w.permute(0, 2, 1).reshape(Cin, 2 * Cout), False))


def test_batched_weightnorm_planes_equal_per_layer_split():
    from deepvoice3_pytorch_b200.weight_bank import WeightBank, _Layer
    params = [_params(s, 50 + i) for i, s in enumerate(CONV_SHAPES[:3])]
    bank = WeightBank()
    for v, g in params:
        bank.layers[v.data_ptr()] = _Layer(v, g)
    bank.begin_step()
    torch.cuda.synchronize()
    for (v, g), L in zip(params, bank.layers.values()):
        _norm_outputs(v.reshape(v.shape[0], -1), g, L.inv, L.scale)
        _check_conv_planes(v, L.scale, L.wfwd, L.wbwd)
        inv, scale, wfwd, wbwd = _tc_conv_planes(v, g)              # the per-layer entry point: the same bits
        assert _same_bits(inv, L.inv) and _same_bits(scale, L.scale)
        assert _same_bits(wfwd[..., :v.shape[1]], L.wfwd[..., :v.shape[1]])
        assert _same_bits(wbwd[..., :v.shape[0]], L.wbwd[..., :v.shape[0]])


def _wn_bwd_reference(partials_tap, v, g, inv):
    """float64 dv, dg from tap-major partials [nsplit][k][Cout][Cin]."""
    dW = partials_tap.double().sum(0).permute(1, 2, 0)            # (Cout, Cin, k)
    v64, inv64 = v.double(), inv.double()
    sc = g.double().flatten() * inv64
    dot = (dW * v64).flatten(1).sum(1)
    dv = sc[:, None, None] * dW - (sc * dot * inv64 * inv64)[:, None, None] * v64
    return dv, (dot * inv64).view_as(g)


def test_weightnorm_bwd_per_layer_equals_batched():
    ops = _ops()
    from deepvoice3_pytorch_b200.weight_bank import _Layer, _upload
    nsplit, layers, ents, blocks = 3, [], [], 0
    for i, shape in enumerate(CONV_SHAPES[:3]):
        Cout, Cin, k = shape
        v, g = _params(shape, 60 + i)
        inv = _tc_conv_planes(v, g)[0]
        gen = torch.Generator().manual_seed(70 + i)
        partials = (torch.randn(nsplit, k, Cout, Cin, generator=gen) * 0.01).cuda()
        layers.append((v, g, inv, partials))
        L = _Layer(v, g)
        e = L.entry()
        part_b = partials.clone().view(nsplit, -1)                   # each call overwrites slot 0 of its own copy
        dv_b, dg_b = torch.empty_like(v), torch.empty_like(g)
        e.inv_norm = inv.data_ptr()
        e.partials, e.split_stride, e.nsplit = part_b.data_ptr(), part_b.shape[1], nsplit
        e.dv, e.dg, e.blk_bwd = dv_b.data_ptr(), dg_b.data_ptr(), blocks
        blocks += Cout
        ents.append((e, part_b, dv_b, dg_b))
    table = _upload([e for e, *_ in ents], "cuda")
    ops.lib.call("dv3_weightnorm_bwd_batched", ops._p(table), len(ents), blocks, 0, ops._stream())
    for (v, g, inv, partials), (_, _, dv_b, dg_b) in zip(layers, ents):
        Cout, Cin, k = v.shape
        dv_r, dg_r = _wn_bwd_reference(partials, v, g, inv)
        part_t = partials.clone().view(nsplit, -1)
        dv_t, dg_t = torch.empty_like(v), torch.empty_like(g)
        ops.lib.call("dv3_weightnorm_bwd", ops._p(part_t), part_t.shape[1], nsplit, 1, ops._p(v), ops._p(g),
                     ops._p(inv), ops._p(dv_t), ops._p(dg_t), Cout, Cin, k, 0, ops._stream())
        # v's own layout: the same reduction in another summation order -> fp32 rounding only
        part_v = partials.permute(0, 2, 3, 1).reshape(nsplit, -1).clone()     # a copy even where reshape is a view
        dv_v, dg_v = torch.empty_like(v), torch.empty_like(g)
        ops.lib.call("dv3_weightnorm_bwd", ops._p(part_v), part_v.shape[1], nsplit, 0, ops._p(v), ops._p(g),
                     ops._p(inv), ops._p(dv_v), ops._p(dg_v), Cout, Cin * k, 1, 0, ops._stream())
        torch.cuda.synchronize()
        assert _same_bits(dv_t, dv_b) and _same_bits(dg_t, dg_b)
        for got in (dv_t, dv_v):
            np.testing.assert_allclose(got.double().cpu().numpy(), dv_r.cpu().numpy(), rtol=1e-4,
                                       atol=1e-5 * float(dv_r.abs().max()))
        for got in (dg_t, dg_v):
            np.testing.assert_allclose(got.double().cpu().numpy(), dg_r.cpu().numpy(), rtol=1e-4,
                                       atol=1e-5 * float(dg_r.abs().max()))
