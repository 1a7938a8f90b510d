"""GPU: the deterministic training mode (ops.deterministic, DESIGN.md section 2.10).

Kernel level: every dv3_*_det entry point against an fp64 reference under an elementwise bound, twice for bit equality,
against its atomic twin within that twin's tolerance, and with non-zero accumulators on entry.  The inputs make the
summation order matter: magnitudes over eight decades, one id repeated, all padding, T off the 4- and 64-frame grids,
odd channel counts on the exact-fp32 kernels, a logical extent shorter than T.
Step level: two fresh runs of one seed agree bit for bit (losses, loss terms, gradients, parameters, Adam moments) for
the three topologies x conv_math x eager / graph; training from wav batches equals training from the .npy corpus.

Nothing here tries to show that the default mode is NOT reproducible: that would be a flaky test."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    from deepvoice3_pytorch_b200._lib import lib
    lib.call(name, *args)


def _raw(name):
    from deepvoice3_pytorch_b200._lib import lib
    return lib.raw(name)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _wide(shape, g, decades=8.0):
    """randn scaled by 10^u, u uniform over ``decades`` decades centred on 1: an order-sensitive sum."""
    return torch.randn(shape, device="cuda", generator=g) * \
        10.0 ** ((torch.rand(shape, device="cuda", generator=g) - 0.5) * decades)


def _within(got, want, bound, what):
    err = (got.double() - want).abs()
    worst = float((err / bound.clamp_min(1e-300)).max())
    print("%s: worst error / bound %.3g" % (what, worst))
    assert worst <= 1, (what, worst)


# ---- losses ---------------------------------------------------------------------------------------------------------
def _spec_ref(y_hat, y, lengths, TL, r, w, bw, pbin, pw):
    """fp64 (loss, L1 term, binary-divergence term, sum of |terms|) of csrc/loss.cu's spec loss."""
    B, T, D = y_hat.shape
    p, tg = y_hat.double()[:, :TL - r], y.double()[:, r:TL]
    t = torch.arange(TL - r, device="cuda")
    m = (t[None, :] + r < lengths[:, None]).double()[:, :, None]
    sm = float((lengths - r).clamp(0, TL - r).sum()) * D
    coef = w * m * (1.0 / sm if sm > 0 else 0.0) + (1 - w) / (B * (TL - r) * D)
    c1 = torch.ones(D, dtype=torch.float64, device="cuda")
    if pbin > 0 and pw > 0:
        c1 = (1 - pw) + (torch.arange(D, device="cuda") < pbin).double() * pw * D / pbin
    l1 = coef * c1 * (p - tg).abs()
    L = torch.log(p + 1e-8) - torch.log(1 - p + 1e-8)
    z = (-tg * L + torch.log1p(torch.exp(L))) if bw > 0 else torch.zeros_like(l1)
    e = (1 - bw) * l1 + bw * coef * z
    return float(e.sum()), float(l1.sum()), float((coef * z).sum()), float(e.abs().sum())


@pytest.mark.parametrize("case", [
    # (B, T, D, r, logical extent or None, w, bw, priority bin, priority weight)
    (16, 203, 513, 1, None, 0.5, 0.1, 120, 0.3),        # more elements than 132 * 8 blocks hold once
    (3, 77, 80, 4, 61, 0.5, 0.1, 0, 0.0),               # extent shorter than T, frame shift 4
    (2, 9, 5, 1, None, 0.0, 0.0, 0, 0.0),               # one block; no masked mean, no binary divergence
], ids=["lin", "mel_ext", "tiny"])
def test_spec_loss_det(case):
    B, T, D, r, TL, w, bw, pbin, pw = case
    g = _gen(B * T + D)
    y_hat = torch.rand(B, T, D, device="cuda", generator=g) * 0.98 + 0.01
    y = torch.rand(B, T, D, device="cuda", generator=g)
    lengths = torch.randint(r + 1, T + 1, (B,), device="cuda", generator=g)
    lengths[0] = T
    t_log = None if TL is None else torch.tensor([TL], dtype=torch.int64, device="cuda")
    scratch = torch.zeros(_raw("dv3_loss_det_scratch_floats")(), device="cuda")
    runs = []
    for _ in range(2):
        grad, loss, terms = torch.empty_like(y_hat), torch.full((1,), 3.0, device="cuda"), torch.full((2,), -1.0, device="cuda")
        _call("dv3_spec_loss_det", _p(y_hat), _p(y), _p(lengths), _p(t_log), _p(grad), _p(loss), _p(terms), _p(scratch),
              B, T, D, r, w, bw, pbin, pw, _st())
        runs.append((grad, loss, terms))
    plain = torch.zeros(1, device="cuda")            # terms = NULL: the plain / _ext form
    _call("dv3_spec_loss_det", _p(y_hat), _p(y), _p(lengths), _p(t_log), _p(torch.empty_like(y_hat)), _p(plain), None,
          _p(scratch), B, T, D, r, w, bw, pbin, pw, _st())
    a_grad, a_loss, a_terms = torch.empty_like(y_hat), torch.zeros(1, device="cuda"), torch.zeros(2, device="cuda")
    _call("dv3_spec_loss_terms", _p(y_hat), _p(y), _p(lengths), _p(t_log), _p(a_grad), _p(a_loss), _p(a_terms), B, T, D,
          r, w, bw, pbin, pw, _st())
    torch.cuda.synchronize()
    assert int(scratch[-1].view(torch.int32)) == 0                       # the ticket is left at zero
    for x, y2 in zip(runs[0], runs[1]):
        assert torch.equal(x, y2)
    grad, loss, terms = runs[0]
    assert torch.equal(grad, a_grad)                                     # the gradient is the atomic kernel's, bit for bit
    want, l1, bd, mag = _spec_ref(y_hat, y, lengths, T if TL is None else TL, r, w, bw, pbin, pw)
    n = B * T * D
    bound = (16 + np.log2(n)) * 8 * U * mag + 1e-12      # fp32 terms (log / exp: a few ulp each) + a tree of fp32 adds
    assert abs(float(loss) - 3.0 - want) <= bound + 3 * 2 * U, (float(loss) - 3.0, want, bound)
    assert abs(float(plain) - want) <= bound
    assert abs(float(terms[0]) + 1.0 - l1) <= bound + 2 * U and abs(float(terms[1]) + 1.0 - bd) <= bound + 2 * U
    np.testing.assert_allclose(float(plain), float(a_loss), rtol=1e-5)
    np.testing.assert_allclose((terms + 1.0).cpu().numpy(), a_terms.cpu().numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("ext", [None, (37, 19)], ids=["full", "ext"])
def test_aux_loss_det(ext):
    A, B, Td, Ts, sigma = 3, 5, 41, 23, 0.2
    g = _gen(7)
    done_hat = torch.rand(B, Td, device="cuda", generator=g) * 0.98 + 0.01
    done = (torch.rand(B, Td, device="cuda", generator=g) > 0.8).float()
    attn = torch.softmax(_wide((A, B, Td, Ts), g, 2.0), -1).contiguous()
    in_len = torch.randint(5, Ts + 1, (B,), device="cuda", generator=g)
    dec_len = torch.randint(5, Td + 1, (B,), device="cuda", generator=g)
    e = None if ext is None else torch.tensor(ext, dtype=torch.int64, device="cuda")
    scratch = torch.zeros(_raw("dv3_loss_det_scratch_floats")(), device="cuda")

    def run(name, *tail):
        d_done, d_attn = torch.empty_like(done_hat), torch.empty_like(attn)
        loss, terms = torch.full((1,), 0.5, device="cuda"), torch.zeros(2, device="cuda")
        _call(name, _p(done_hat), _p(done), _p(d_done), B * Td, _p(attn), _p(d_attn), _p(in_len), _p(dec_len), _p(e), A, B,
              Td, Ts, sigma, 1, _p(loss), _p(terms), *tail, _st())
        return d_done, d_attn, loss, terms
    r0, r1 = run("dv3_aux_loss_det", _p(scratch)), run("dv3_aux_loss_det", _p(scratch))
    ra = run("dv3_aux_loss_terms")
    torch.cuda.synchronize()
    for x, y in zip(r0, r1):
        assert torch.equal(x, y)
    assert torch.equal(r0[0], ra[0]) and torch.equal(r0[1], ra[1])
    TdL, TsL = (Td, Ts) if ext is None else ext
    p, t = done_hat.double()[:, :TdL], done.double()[:, :TdL]
    bce = -(t * torch.log(p) + (1 - t) * torch.log(1 - p)) / (B * TdL)
    n_i = torch.arange(Ts, device="cuda").double()[None, None, :]
    t_i = torch.arange(Td, device="cuda").double()[None, :, None]
    N, Tl = in_len.double()[:, None, None], dec_len.double()[:, None, None]
    W = 1 - torch.exp(-(n_i / N - t_i / Tl) ** 2 / (2 * sigma * sigma))
    W = W * ((n_i < N) & (t_i < Tl) & (n_i < TsL) & (t_i < TdL))
    ga = attn.double() * W[None] / (A * B * TdL * TsL)
    bound = 64 * U * float(bce.sum() + ga.sum())
    assert abs(float(r0[3][0]) - float(bce.sum())) <= bound and abs(float(r0[3][1]) - float(ga.sum())) <= bound
    assert abs(float(r0[2]) - 0.5 - float(bce.sum() + ga.sum())) <= bound + U
    np.testing.assert_allclose(r0[3].cpu().numpy(), ra[3].cpu().numpy(), rtol=1e-5)


# ---- bias gradients -------------------------------------------------------------------------------------------------
def _bias_scratch(B, nch, T, tiled):
    n = _raw("dv3_bias_det_scratch_floats")(B, nch, T, tiled)
    return torch.full((n,), float("nan"), device="cuda"), n      # every partial the reduction reads must be written


@pytest.mark.parametrize("mode,residual", [(0, 1), (1, 0)], ids=["glu_res", "highway"])
def test_gate_bwd_det_fp32(mode, residual):
    B, C, T = 5, 513, 203
    g = _gen(3 + mode)
    dy, a, x = _wide((B, C, T), g), torch.randn(B, C, T, device="cuda", generator=g), torch.randn(B, C, T, device="cuda", generator=g)
    s = torch.rand(B, C, T, device="cuda", generator=g)
    init = torch.randn(2 * C, device="cuda", generator=g)
    scratch, n = _bias_scratch(B, 2 * C, T, 0)
    outs = []
    for _ in range(2):
        dab, db = torch.empty(B, 2 * C, T, device="cuda"), init.clone()
        _call("dv3_convblock_gate_bwd_det", _p(dy), _p(a), _p(s), _p(x), _p(dab), _p(db), _p(scratch), n, B, C, T, mode,
              residual, _st())
        outs.append((dab, db))
    dab_a, db_a = torch.empty(B, 2 * C, T, device="cuda"), init.clone()
    _call("dv3_convblock_gate_bwd", _p(dy), _p(a), _p(s), _p(x), _p(dab_a), _p(db_a), B, C, T, mode, residual, _st())
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][0], dab_a)
    gs = 0.70710678118654752 if (mode == 0 and residual) else 1.0
    gd = dy.double() * gs
    da = gd * s.double()
    dbv = gd * (a.double() if mode == 0 else a.double() - x.double()) * s.double() * (1 - s.double())
    terms = torch.cat([da, dbv], 1)
    want = init.double() + terms.sum((0, 2))
    bound = (B * T + 16) * U * terms.abs().sum((0, 2)) + 2 * U * init.double().abs()
    _within(outs[0][1], want, bound, "gate_bwd_det dbias")
    _within(db_a, want, bound, "gate_bwd (atomic) dbias")


@pytest.mark.parametrize("relu", [0, 1])
def test_bias_act_bwd_det_fp32(relu):
    B, C, T = 7, 513, 77
    g = _gen(11 + relu)
    dy, y = _wide((B, C, T), g), torch.randn(B, C, T, device="cuda", generator=g)
    init = torch.randn(C, device="cuda", generator=g)
    scratch, n = _bias_scratch(B, C, T, 0)
    outs = []
    for _ in range(2):
        dyr, db = torch.empty_like(dy), init.clone()
        _call("dv3_bias_act_bwd_det", _p(dy), _p(y), _p(dyr) if relu else None, _p(db), _p(scratch), n, B, C, T, relu,
              _st())
        outs.append((dyr, db))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][1], outs[1][1])
    terms = dy.double() * ((y > 0).double() if relu else 1.0)
    if relu:
        assert torch.equal(outs[0][0].double(), terms)
    want = init.double() + terms.sum((0, 2))
    bound = (B * T + 16) * U * terms.abs().sum((0, 2)) + 2 * U * init.double().abs()
    _within(outs[0][1], want, bound, "bias_act_bwd_det dbias")


def _mask_t(x, tlen):
    x = x.clone()
    x[:, :, tlen:] = 0
    return x


@pytest.mark.parametrize("npl", [1, 2])
@pytest.mark.parametrize("tlen", [None, 70])
def test_tc_splits_det(npl, tlen):
    """Gate split (GLU with residual, highway) and gradient split (ReLU or not): planes bit-identical to the atomic
    twin's, the bias gradient within the fp64 bound, added to what dbias held, frames past the extent left out."""
    B, T = 3, 101
    g = _gen(5 + npl)
    tl = None if tlen is None else torch.tensor([tlen], dtype=torch.int64, device="cuda")    # alive across the calls
    e = (_p(tl), 1)
    TL = T if tlen is None else tlen
    BF = torch.bfloat16
    for mode, residual in ((0, 1), (1, 0)):
        C = 128
        dy, a, x = _wide((B, C, T), g), torch.randn(B, C, T, device="cuda", generator=g), torch.randn(B, C, T, device="cuda", generator=g)
        s = torch.rand(B, C, T, device="cuda", generator=g)
        init = torch.randn(2 * C, device="cuda", generator=g)
        scratch, n = _bias_scratch(B, 2 * C, T, 1)
        outs = []
        for _ in range(2):
            pl, db = torch.zeros(npl, B, T, 2 * C, device="cuda", dtype=BF), init.clone()
            _call("dv3_tc_gate_bwd_split_det", _p(dy), _p(a), _p(s), _p(x), _p(pl), npl, _p(db), _p(scratch), n, B, C, T,
                  mode, residual, e[0], e[1], _st())
            outs.append((pl, db))
        pl_a, db_a = torch.zeros(npl, B, T, 2 * C, device="cuda", dtype=BF), init.clone()
        _call("dv3_tc_gate_bwd_split_npl", _p(dy), _p(a), _p(s), _p(x), _p(pl_a), npl, None, _p(db_a), B, C, T, mode,
              residual, e[0], e[1], _st())
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16))
        assert torch.equal(outs[0][1], outs[1][1])
        assert torch.equal(outs[0][0].view(torch.int16), pl_a.view(torch.int16))
        gd = dy.double() * (0.70710678118654752 if (mode == 0 and residual) else 1.0)
        da = gd * s.double()
        dbv = gd * (a.double() if mode == 0 else a.double() - x.double()) * s.double() * (1 - s.double())
        terms = _mask_t(torch.cat([da, dbv], 1), TL)
        want = init.double() + terms.sum((0, 2))
        bound = (B * T + 16) * U * terms.abs().sum((0, 2)) + 2 * U * init.double().abs()
        _within(outs[0][1], want, bound, "tc_gate_bwd_split_det dbias mode %d" % mode)
        _within(db_a, want, bound, "tc_gate_bwd_split (atomic) dbias mode %d" % mode)
    for relu in (0, 1):
        C = 136
        Cp = (C + 7) // 8 * 8
        dy, y = _wide((B, C, T), g), torch.randn(B, C, T, device="cuda", generator=g)
        init = torch.randn(C, device="cuda", generator=g)
        scratch, n = _bias_scratch(B, C, T, 1)
        outs = []
        for _ in range(2):
            pl, db = torch.zeros(npl, B, T, Cp, device="cuda", dtype=BF), init.clone()
            _call("dv3_tc_grad_split_det", _p(dy), _p(y), _p(pl), npl, _p(db), _p(scratch), n, B, C, T, relu, e[0], e[1],
                  _st())
            outs.append((pl, db))
        pl_a = torch.zeros(npl, B, T, Cp, device="cuda", dtype=BF)
        _call("dv3_tc_grad_split_npl", _p(dy), _p(y), _p(pl_a), npl, None, None, B, C, T, relu, e[0], e[1], _st())
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16))
        assert torch.equal(outs[0][1], outs[1][1])
        assert torch.equal(outs[0][0][..., :C].view(torch.int16), pl_a[..., :C].view(torch.int16))
        terms = _mask_t(dy.double() * ((y > 0).double() if relu else 1.0), TL)
        want = init.double() + terms.sum((0, 2))
        bound = (B * T + 16) * U * terms.abs().sum((0, 2)) + 2 * U * init.double().abs()
        _within(outs[0][1], want, bound, "tc_grad_split_det dbias relu %d" % relu)


def test_det_entry_points_refuse_a_short_scratch():
    from deepvoice3_pytorch_b200._lib import Dv3Error
    B, C, T = 2, 128, 64
    dy = torch.zeros(B, C, T, device="cuda")
    pl, db, scratch = torch.zeros(2, B, T, C, device="cuda", dtype=torch.bfloat16), torch.zeros(C, device="cuda"), torch.zeros(8, device="cuda")
    with pytest.raises(Dv3Error):
        _call("dv3_tc_grad_split_det", _p(dy), None, _p(pl), 2, _p(db), _p(scratch), 8, B, C, T, 0, None, 1, _st())
    with pytest.raises(Dv3Error):
        _call("dv3_bias_act_bwd_det", _p(dy), None, None, _p(db), _p(scratch), 8, B, C, T, 0, _st())


# ---- table gradients ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ids_kind", ["random", "one_id", "all_padding"])
@pytest.mark.parametrize("V,D,N", [(149, 256, 2048), (108, 16, 777), (64, 513, 300)])
def test_embedding_bwd_det(ids_kind, V, D, N):
    g = _gen(V + D)
    pad = 0
    if ids_kind == "random":
        ids = torch.randint(0, V, (N,), device="cuda", generator=g)
    else:
        ids = torch.full((N,), 7 if ids_kind == "one_id" else pad, dtype=torch.int64, device="cuda")
    dy = _wide((N, D), g)
    init = torch.randn(V, D, device="cuda", generator=g)
    outs = []
    for _ in range(2):
        dt = init.clone()
        _call("dv3_embedding_bwd_det", _p(ids), _p(dy), _p(dt), N, D, V, pad, _st())
        outs.append(dt)
    dt_a = init.clone()
    _call("dv3_embedding_bwd", _p(ids), _p(dy), _p(dt_a), N, D, V, pad, _st())
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    keep = (ids != pad)
    want = init.double().index_add(0, ids[keep], dy.double()[keep])
    mag = torch.zeros(V, D, dtype=torch.float64, device="cuda").index_add(0, ids[keep], dy.double().abs()[keep])
    bound = (N + 2) * U * mag + 2 * U * init.double().abs()
    _within(outs[0], want, bound, "embedding_bwd_det %s" % ids_kind)
    _within(dt_a, want, bound, "embedding_bwd (atomic) %s" % ids_kind)
    assert torch.equal(outs[0][pad], init[pad])
    if ids_kind == "all_padding":
        assert torch.equal(outs[0], init)


@pytest.mark.parametrize("nw", [1, "B"])
@pytest.mark.parametrize("pos_kind", ["ramp", "one_pos", "all_padding"])
def test_sinusoid_bwd_det(nw, pos_kind):
    B, T, D, P = 6, 67, 128, 512
    nw = B if nw == "B" else 1
    g = _gen(B + T + nw)
    if pos_kind == "ramp":          # positions 1..len, then padding 0
        lens = torch.randint(1, T + 1, (B,), device="cuda", generator=g)
        ar = torch.arange(1, T + 1, device="cuda")[None, :]
        pos = torch.where(ar <= lens[:, None], ar, torch.zeros_like(ar)).contiguous()
    else:
        pos = torch.full((B, T), 5 if pos_kind == "one_pos" else 0, dtype=torch.int64, device="cuda")
    table = torch.randn(P, D, device="cuda", generator=g) * 3
    w = torch.rand(nw, device="cuda", generator=g) + 0.5
    dy = _wide((B, T, D), g)
    init = torch.randn(P, D, device="cuda", generator=g)
    outs = []
    for _ in range(2):
        dt, dw = init.clone(), torch.zeros(nw, device="cuda")
        _call("dv3_sinusoid_bwd_det", _p(pos), _p(table), _p(w), nw, _p(dy), _p(dt), _p(dw), B, T, D, P, _st())
        outs.append((dt, dw))
    dt_a, dw_a = init.clone(), torch.zeros(nw, device="cuda")
    _call("dv3_sinusoid_bwd", _p(pos), _p(table), _p(w), nw, _p(dy), _p(dt_a), _p(dw_a), B, T, D, P, _st())
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][1], dw_a)                        # the rate gradient is the same kernel
    wb = (w if nw == B else w.expand(B))[:, None, None]
    a = (wb * table[pos]).double()                              # the fp32 product the kernels form
    odd = (torch.arange(D, device="cuda") % 2 == 1)
    deriv = torch.where(odd, -torch.sin(a), torch.cos(a))
    terms = dy.double() * deriv * wb.double() * (pos > 0).double()[:, :, None]
    flat = pos.flatten()
    want = init.double().index_add(0, flat, terms.view(B * T, D))
    mag = torch.zeros(P, D, dtype=torch.float64, device="cuda").index_add(0, flat, terms.abs().view(B * T, D))
    # sinf / cosf to ~2 ulp of 1 (not of the derivative): the term error is relative to |dy * w|
    slack = torch.zeros(P, D, dtype=torch.float64, device="cuda").index_add(
        0, flat, ((dy.double() * wb.double()).abs() * (pos > 0).double()[:, :, None]).view(B * T, D))
    bound = (B * T + 4) * U * mag + 8 * U * slack + 2 * U * init.double().abs()
    _within(outs[0][0], want, bound, "sinusoid_bwd_det %s" % pos_kind)
    _within(dt_a, want, bound, "sinusoid_bwd (atomic) %s" % pos_kind)
    assert torch.equal(outs[0][0][0], init[0])
    if pos_kind == "all_padding":
        assert torch.equal(outs[0][0], init)


# ---- the training step ----------------------------------------------------------------------------------------------
@pytest.fixture
def det_on(monkeypatch):
    from deepvoice3_pytorch_b200 import ops
    monkeypatch.setattr(ops, "deterministic", "1")


def _shapes(topo):
    from test_gpu_train_ragged import _batches
    a, _ = _batches(topo)
    b, _ = _batches(topo, text_lens=(31, 12, 20), frame_lens=(90, 40, 61), seed=1)
    c, _ = _batches(topo, text_lens=(8, 5, 7), frame_lens=(24, 30, 17), seed=2)
    return a, b, c


def _state(step):
    terms = {k: v.clone() for k, v in step.loss_terms().items()}
    return [step.arena.grad.clone(), step.arena.flat.clone(), step.opt.m.clone(), step.opt.v.clone()] + \
        [terms[k] for k in sorted(terms)]


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("math", ["tc", "tc1", "fp32"])
@pytest.mark.parametrize("topo", ["deepvoice3", "nyanko", "multispeaker"])
def test_two_runs_of_one_seed_are_bit_identical(topo, math, graph, det_on):
    """Shapes A, B, A, C, B with dropout 0.05: in graph mode A is the exact graph, B and C are buckets captured lazily
    and replayed out of capture order."""
    from test_gpu_train_ragged import _train
    a, b, c = _shapes(topo)
    seq = [a, b, a, c, b]
    l0, g0, n0, _, s0 = _train(topo, seq, math, dropout=0.05, graph=graph)
    st0 = _state(s0)
    l1, g1, n1, _, s1 = _train(topo, seq, math, dropout=0.05, graph=graph)
    st1 = _state(s1)
    assert s0.deterministic and s1.deterministic and (not graph or s0.graphs_captured == 3)
    assert np.all(np.isfinite(l0)) and float(g0.abs().max()) > 0
    assert l0.tolist() == l1.tolist(), (l0, l1)
    assert torch.equal(g0, g1) and n0 == n1
    for x, y in zip(st0, st1):
        assert torch.equal(x, y)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """-> {False: (in_dir, out_dir)}: the wav corpus of tests/test_gpu_wav_train.py, preprocessed without rescaling."""
    import os
    import test_gpu_wav_train as W
    from deepvoice3_pytorch_b200 import audio, preprocess
    root = str(tmp_path_factory.mktemp("wavcorpus_det"))
    in_dir, out_dir = os.path.join(root, "in"), os.path.join(root, "out")
    W._write_corpus(in_dir)
    os.makedirs(out_dir)
    old = audio.hparams.rescaling
    try:
        audio.hparams.rescaling = False
        preprocess.write_metadata(preprocess.build_from_path(in_dir, out_dir, batch_clips=8), out_dir)
    finally:
        audio.hparams.rescaling = old
    return {False: (in_dir, out_dir)}


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_training_on_wavs_equals_training_on_npy_bit_for_bit(corpus, graph, det_on):
    """The claim tests/test_gpu_wav_train.py could only report as an expected failure: the .npy path repeats itself,
    and the wav path gives the same losses and parameters."""
    import test_gpu_wav_train as W
    npy, wds = W._datasets(corpus, False, False)
    order = [list(range(0, 4)), list(range(4, 8)), list(range(8, 12)), list(range(0, 4))]
    pairs = [W._pair(npy, wds, idx, 1, 4) for idx in order]
    l0, p0 = W._train([w for w, _ in pairs], graph)
    l1, p1 = W._train([w for w, _ in pairs], graph)
    l2, p2 = W._train([g for _, g in pairs], graph)
    assert np.all(np.isfinite(l0))
    assert l0 == l1 and torch.equal(p0, p1)
    assert l2 == l0 and torch.equal(p2, p0)


@pytest.mark.parametrize("math", ["fp32", "tc"])
@pytest.mark.parametrize("topo", ["deepvoice3", "nyanko", "multispeaker"])
def test_deterministic_padded_step_equals_plain_eager_step(topo, math, monkeypatch):
    """Still correct: deterministic steps on a batch padded to a bucket against default-mode eager steps on the unpadded
    batch, within the tolerances of tests/test_gpu_train_ragged.py; gradients past the logical extents are exactly 0."""
    from deepvoice3_pytorch_b200 import ops
    from test_gpu_train_ragged import TOL, _batches, _excess, _train
    rtol, atol = TOL[math]
    plain, padded = _batches(topo)
    l_ref, g_ref, n_ref, p_ref, ref = _train(topo, [plain] * 4, math)
    assert not ref.deterministic
    monkeypatch.setattr(ops, "deterministic", "1")
    l_pad, g_pad, n_pad, p_pad, step = _train(topo, [padded] * 4, math)
    assert step.deterministic
    assert _excess(l_pad, l_ref, rtol, atol) <= 1, (l_pad, l_ref)
    assert _excess(n_pad, n_ref, rtol, atol) <= 1, (n_pad, n_ref)
    torch.testing.assert_close(g_pad, g_ref, rtol=rtol, atol=atol)
    torch.testing.assert_close(p_pad, p_ref, rtol=rtol, atol=atol)


def test_gradients_past_the_extent_are_exactly_zero(det_on):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import fused_training_loss
    from test_gpu_train_ragged import _batches, _build
    _, padded = _batches("deepvoice3")
    model = _build("deepvoice3", 0.0).cuda().train()
    ext = padded["extents"]
    from deepvoice3_pytorch_b200 import data
    with ops.extent_scope(ext, data.batch_extents(padded)):
        outs = model(padded["x"], padded["mel"], text_positions=padded["text_positions"],
                     frame_positions=padded["frame_positions"], input_lengths=padded["input_lengths_dev"])
        for o in outs:
            o.retain_grad()
        loss = fused_training_loss(outs, padded)
    loss.backward()
    e = [int(v) for v in ext.cpu()]
    mel_out, lin_out, attn, done_hat = outs
    assert float(mel_out.grad.abs().max()) > 0 and float(lin_out.grad.abs().max()) > 0
    assert float(mel_out.grad[:, e[ops.EXT_MEL]:].abs().max()) == 0
    assert float(lin_out.grad[:, e[ops.EXT_LIN]:].abs().max()) == 0
    assert float(attn.grad[:, :, e[ops.EXT_DEC]:].abs().max()) == 0
    assert float(attn.grad[..., e[ops.EXT_TEXT]:].abs().max()) == 0
    assert float(done_hat.grad.view(done_hat.shape[0], -1)[:, e[ops.EXT_DEC]:].abs().max()) == 0


# kernel launches of one captured step of the three test topologies on tests/test_gpu_train_ragged.py's first batch, in
# the default mode and conv_math "tc": the numbers of the commit before the deterministic mode existed
LAUNCHES_BEFORE = {"deepvoice3": 300, "nyanko": 364, "multispeaker": 561}


@pytest.mark.parametrize("topo", ["deepvoice3", "nyanko", "multispeaker"])
def test_off_means_off(topo, monkeypatch):
    """Default mode: no deterministic entry point is called, and a captured step launches what it launched before."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    from test_gpu_train_ragged import _batches, _train
    assert ops.is_deterministic() is False
    called = []
    real = lib.call

    def spy(name, *args):
        called.append(name)
        return real(name, *args)
    monkeypatch.setattr(lib, "call", spy)
    plain, _ = _batches(topo)
    _, _, _, _, step = _train(topo, [plain] * 2, "tc", dropout=0.05, graph=True)
    assert called and not [n for n in called if n.endswith("_det")]
    assert not step.deterministic and step._det_scratch is None
    print("launches per step, %s: %d" % (topo, step.launches_per_step))
    assert step.launches_per_step == LAUNCHES_BEFORE[topo]
    called.clear()
    monkeypatch.setattr(ops, "deterministic", "1")
    _, _, _, _, det = _train(topo, [plain] * 2, "tc", dropout=0.05, graph=True)
    assert {n for n in called if n.endswith("_det")} >= {"dv3_spec_loss_det", "dv3_aux_loss_det", "dv3_embedding_bwd_det",
                                                        "dv3_tc_gate_bwd_split_det"}
    atomic = {"dv3_spec_loss_terms", "dv3_aux_loss_terms", "dv3_embedding_bwd", "dv3_sinusoid_bwd", "dv3_bias_act_bwd",
              "dv3_convblock_gate_bwd", "dv3_tc_gate_bwd_split_npl", "dv3_tc_grad_split_npl"}
    assert not atomic & set(called), atomic & set(called)
    print("launches per deterministic step, %s: %d" % (topo, det.launches_per_step))


def _ddp_worker(rank, world, port, out):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DV3_DETERMINISTIC="1")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from deepvoice3_pytorch_b200 import ops
        from deepvoice3_pytorch_b200.train_step import TrainStep
        from test_gpu_train_ragged import _batches, _build
        ops.deterministic = "1"
        torch.manual_seed(0)
        ops.rng.manual_seed(77 + rank, torch.device("cuda"))
        step = TrainStep(_build("deepvoice3", 0.05).cuda().train())
        batch, _ = _batches("deepvoice3", seed=rank)
        for _ in range(3):
            step.step(batch)
        torch.cuda.synchronize()
        torch.save(step.arena.flat.cpu(), os.path.join(out, "rank%d.pt" % rank))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_agree_and_repeat(tmp_path):
    import os
    import torch.multiprocessing as mp
    runs = []
    for i in range(2):
        out = str(tmp_path / ("run%d" % i))
        os.makedirs(out)
        mp.spawn(_ddp_worker, args=(2, 29533 + i, out), nprocs=2, join=True)
        runs.append([torch.load(os.path.join(out, "rank%d.pt" % r)) for r in range(2)])
    assert torch.equal(runs[0][0], runs[0][1])
    assert torch.equal(runs[0][0], runs[1][0])
