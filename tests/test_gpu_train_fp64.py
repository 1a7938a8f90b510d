"""GPU: the training-step kernels after the model's outputs, elementwise against the fp64 references and derived
bounds of tests/train_bounds.py (its header gives the error model).  Calls the C ABI directly.

  * dv3_spec_loss_terms and dv3_spec_loss_det, terms on and off: one bound for all four forms, and one gradient, bit
    for bit.  Planted saturated predictions (0, 2^-149, k 2^-24, 1 - k 2^-24, 1), p == y and p = y +- 1 ulp, targets 0
    and 1; lengths full, <= r, > T, and all <= r (Sm = 0: the kernel takes the masked mean as 0 where the reference's
    is 0/0); t_log None, T, < T, r + 1, > T and <= r; every loss setting of a small batch.
  * dv3_aux_loss_terms and dv3_aux_loss_det: d_done on both sides of the 1e-12 clamp, d_attn with dec_len = 0 rows,
    extents past Td and of one text position, use_attn = 0 with d_attn set.
  * dv3_sumsq, dv3_adam_clip and every instantiation of dv3_adam_clip_opts: around the 1056-block grid cap, at the
    deepvoice3_ljspeech arena size, with zero, 1e-20 and 1e3 gradients, clip active, inactive and off; several steps
    teacher-forced; FlatAdam with two parts at different clocks (one launch per part, at an offset).
  * dv3_sinusoid_fwd on the presets' position tables and random ones, and the rate gradient of dv3_sinusoid_bwd[_det]
    with and without the table gradient, on sums that cancel.
Every output lives in a sentinel-guarded buffer; accumulated outputs start from non-zero values."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import train_bounds as TB
from test_gpu_tc_pairs import GUARD, SENT32, assert_written_inside_only, guarded

pytestmark = pytest.mark.gpu

WORST = {}


def _note(what, r):
    WORST[what] = max(WORST.get(what, 0.0), r)
    print("%s: worst error / bound %.3g" % (what, r))
    assert r <= 1.0, (what, r)


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


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _filled(a):
    """A sentinel-guarded fp32 buffer whose inside holds ``a`` (an accumulated or in-place output)."""
    a = np.asarray(a, np.float32).reshape(-1)
    buf, view = guarded(a.size)
    view.copy_(_dev(a))
    return buf, view


def _untouched(buf):
    return bool((buf.view(torch.int32) == SENT32).all())


def _np(t):
    return t.detach().double().cpu().numpy()


# ---- spectrogram loss -----------------------------------------------------------------------------------------------
def _spec_run(yh, y, ln, r, w, bw, pbin, pw, t_log, ref):
    B, T, D = yh.shape
    n = B * T * D
    d_yh, d_y, d_ln = _dev(yh), _dev(y), _dev(np.asarray(ln, np.int64))
    d_tl = None if t_log is None else _dev(np.asarray([t_log], np.int64))
    scratch = torch.zeros(_raw("dv3_loss_det_scratch_floats")(), device="cuda")
    grads = []
    for det in (False, True):
        for terms_on in (False, True):
            gbuf, grad = guarded(n)
            lbuf, loss = _filled([3.0])
            tbuf, terms = _filled([-1.0, 0.5])
            tp = _p(terms) if terms_on else None
            if det:
                _call("dv3_spec_loss_det", _p(d_yh), _p(d_y), _p(d_ln), _p(d_tl), _p(grad), _p(loss), tp, _p(scratch),
                      B, T, D, r, w, bw, pbin, pw, _st())
            else:
                _call("dv3_spec_loss_terms", _p(d_yh), _p(d_y), _p(d_ln), _p(d_tl), _p(grad), _p(loss), tp, B, T, D,
                      r, w, bw, pbin, pw, _st())
            torch.cuda.synchronize()
            form = "spec_loss%s%s" % ("_det" if det else "", " terms" if terms_on else "")
            assert_written_inside_only(gbuf, n)
            assert_written_inside_only(lbuf, 1)
            if terms_on:
                assert_written_inside_only(tbuf, 2)
            else:
                assert float(terms[0]) == -1.0 and float(terms[1]) == 0.5, form + ": terms written with terms NULL"
                assert _untouched(tbuf[:GUARD]) and _untouched(tbuf[GUARD + 2:])
            _note("spec grad", TB.ratio(_np(grad).reshape(B, T, D), ref["grad"], ref["grad_bound"]))
            lb = TB.scalar_bound(ref["h"], 3.0, ref["mag_loss"], ref["err_loss"])
            _note("spec loss", abs(float(loss[0]) - (3.0 + ref["loss"])) / lb)
            if terms_on:
                b1 = TB.scalar_bound(ref["h"], 1.0, ref["mag_l1"], ref["err_l1"])
                b2 = TB.scalar_bound(ref["h"], 0.5, ref["mag_bd"], ref["err_bd"])
                _note("spec terms", max(abs(float(terms[0]) - (ref["l1"] - 1.0)) / b1,
                                        abs(float(terms[1]) - (ref["bd"] + 0.5)) / b2))
            grads.append(grad.clone())
    assert int(scratch[-1].view(torch.int32)) == 0
    for g in grads[1:]:
        assert torch.equal(g.view(torch.int32), grads[0].view(torch.int32)), "the four forms differ in the gradient"


def _spec_case(B, T, D, r, kind, seed):
    yh, y0 = TB.planted_pairs(B, T, D, seed)
    return yh, TB.shift_targets(yh, y0, r), TB.lengths_for(kind, B, T, r, seed)


@pytest.mark.parametrize("case", TB.SPEC_SHAPES, ids=[c[0] for c in TB.SPEC_SHAPES])
def test_spec_loss_shapes(case):
    cid, B, T, D, r, kind, tl, w, bw, pbin, pw = case
    yh, y, ln = _spec_case(B, T, D, r, kind, B * T + D)
    ref = TB.spec_loss(yh, y, ln, r, w, bw, pbin, pw, t_log=tl)
    if kind == "all_masked":
        assert ref["grad"].any() == (w < 1)           # Sm = 0: only the plain mean is left
    _spec_run(yh, y, ln, r, w, bw, pbin, pw, tl, ref)


@pytest.mark.parametrize("t_log", TB.SPEC_TLOG, ids=[str(t) for t in TB.SPEC_TLOG])
def test_spec_loss_t_log(t_log):
    B, T, D, r = 5, 61, 80, 2
    yh, y, ln = _spec_case(B, T, D, r, "ragged", 7)
    ref = TB.spec_loss(yh, y, ln, r, 0.5, 0.1, 70, 0.5, t_log=t_log)
    _spec_run(yh, y, ln, r, 0.5, 0.1, 70, 0.5, t_log, ref)


def test_spec_loss_settings():
    B, T, D, r = TB.SETTING_SHAPE
    yh, y, ln = _spec_case(B, T, D, r, "ragged", 5)
    for w, bw, pbin, pw in TB.SETTINGS:
        ref = TB.spec_loss(yh, y, ln, r, w, bw, pbin, pw)
        _spec_run(yh, y, ln, r, w, bw, pbin, pw, None, ref)


# ---- auxiliary loss -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", TB.AUX_CASES, ids=[c[0] for c in TB.AUX_CASES])
def test_aux_loss(case):
    cid, A, B, Td, Ts, ext, use_attn = case
    dh, done, attn, il, dl = TB.aux_inputs(A, B, Td, Ts, Td + Ts)
    ref = TB.aux_loss(dh, done, attn, il, dl, TB.AUX_SIGMA, use_attn, ext)
    d_dh, d_done, d_attn, d_il, d_dl = _dev(dh), _dev(done), _dev(attn), _dev(il), _dev(dl)
    d_ext = None if ext is None else _dev(np.asarray(ext, np.int64))
    scratch = torch.zeros(_raw("dv3_loss_det_scratch_floats")(), device="cuda")
    nd, na = B * Td, attn.size
    outs = []
    for det in (False, True):
        for terms_on in (False, True):
            dbuf, dd = guarded(nd)
            abuf, da = guarded(na)
            lbuf, loss = _filled([0.5])
            tbuf, terms = _filled([0.25, -2.0])
            tail = (_p(scratch),) if det else ()
            _call("dv3_aux_loss_det" if det else "dv3_aux_loss_terms", _p(d_dh), _p(d_done), _p(dd), nd, _p(d_attn),
                  _p(da), _p(d_il), _p(d_dl), _p(d_ext), A, B, Td, Ts, TB.AUX_SIGMA, use_attn, _p(loss),
                  _p(terms) if terms_on else None, *tail, _st())
            torch.cuda.synchronize()
            assert_written_inside_only(dbuf, nd)
            assert_written_inside_only(abuf, na)
            assert_written_inside_only(lbuf, 1)
            _note("aux d_done", TB.ratio(_np(dd), ref["d_done"], ref["d_done_bound"]))
            _note("aux d_attn", TB.ratio(_np(da).reshape(attn.shape), ref["d_attn"], ref["d_attn_bound"]))
            lb = TB.scalar_bound(ref["h"], 0.5, ref["mag_bce"] + ref["mag_ga"], ref["err_bce"] + ref["err_ga"])
            _note("aux loss", abs(float(loss[0]) - (0.5 + ref["loss"])) / lb)
            if terms_on:
                b1 = TB.scalar_bound(ref["h"], 0.25, ref["mag_bce"], ref["err_bce"])
                b2 = TB.scalar_bound(ref["h"], 2.0, ref["mag_ga"], ref["err_ga"])
                _note("aux terms", max(abs(float(terms[0]) - (0.25 + ref["bce"])) / b1,
                                       abs(float(terms[1]) - (ref["ga"] - 2.0)) / b2))
            else:
                assert float(terms[0]) == 0.25 and float(terms[1]) == -2.0
            outs.append((dd.clone(), da.clone()))
    if not use_attn:
        assert float(outs[0][1].abs().max()) == 0.0
    for dd, da in outs[1:]:
        assert torch.equal(dd, outs[0][0]) and torch.equal(da, outs[0][1])


# ---- sumsq and clip + Adam ------------------------------------------------------------------------------------------
def _arena_size():
    """The parameter arena of the deepvoice3_ljspeech training step (bench.py's preset), counted on the CPU."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("_bench_presets", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    from deepvoice3_pytorch_b200 import builder
    bname, kw, _ = bench.PRESETS[TB.ARENA_PRESET]
    model = getattr(builder, bname)(**kw)
    return sum((p.numel() + 3) // 4 * 4 for p in model.get_trainable_parameters())


@pytest.fixture(scope="module")
def arena_n():
    return _arena_size()


def _sumsq(gview, n):
    obuf, out = guarded(1)
    scratch = torch.zeros(_raw("dv3_sumsq_scratch_floats")(), device="cuda")
    _call("dv3_sumsq", _p(gview), n, _p(out), _p(scratch), _st())
    torch.cuda.synchronize()
    assert_written_inside_only(obuf, 1)
    assert int(scratch[-1].view(torch.int32)) == 0
    return out


@pytest.mark.parametrize("n", TB.OPT_SIZES + ["arena"])
def test_sumsq(n, arena_n):
    n = arena_n if n == "arena" else n
    g = TB.optim_grads(n, n % 1000)
    gbuf, gv = _filled(g)
    out = _sumsq(gv, n)
    ref, b = TB.sumsq_bound(g)
    _note("sumsq", abs(float(out[0]) - ref) / b)
    for scale in (1e-20, 0.0):                                 # every square subnormal; all zero
        gs = (g / np.float32(1e3) * np.float32(scale)).astype(np.float32) if scale else np.zeros(n, np.float32)
        gv.copy_(_dev(gs))
        out = _sumsq(gv, n)
        ref, b = TB.sumsq_bound(gs)
        _note("sumsq", abs(float(out[0]) - ref) / b)
        if not scale:
            assert float(out[0]) == 0.0


def _adam(n, g, state, hyper, sumsq, max_norm, wd, plain=False):
    """One launch of dv3_adam_clip_opts (or dv3_adam_clip) on guarded copies of the state -> fp32 numpy outputs."""
    p, m, v, vmax = state
    bufs = [_filled(x) if x is not None else (None, None) for x in (g, p, m, v, vmax)]
    hbuf, hv = _filled(hyper)
    sbuf, sv = _filled([sumsq])
    (gb, gv), (pb, pv), (mb, mv), (vb, vv), (xb, xv) = bufs
    b1, b2 = TB.OPT_BETAS
    if plain:
        _call("dv3_adam_clip", _p(pv), _p(gv), _p(mv), _p(vv), n, _p(hv), _p(sv), b1, b2, TB.OPT_EPS, max_norm, _st())
    else:
        _call("dv3_adam_clip_opts", _p(pv), _p(gv), _p(mv), _p(vv), _p(xv), n, _p(hv), _p(sv), b1, b2, TB.OPT_EPS,
              max_norm, wd, _st())
    torch.cuda.synchronize()
    for buf in (gb, pb, mb, vb, xb, hbuf, sbuf):
        if buf is not None:
            assert_written_inside_only(buf, buf.numel() - 2 * GUARD)
    assert np.array_equal(gv.cpu().numpy(), np.asarray(g, np.float32))
    return [None if x is None else x.cpu().numpy() for x in (pv, mv, vv, xv)]


def _check_adam(out, ref, ams, what):
    for k, got in zip(("p", "m", "v"), out[:3]):
        _note("adam %s" % k, TB.ratio(got, ref[k], ref[k + "_b"]))
    if ams:
        _note("adam vmax", TB.ratio(out[3], ref["vmax"], ref["vmax_b"]))


def _kernel_sumsq(g):
    gbuf, gv = _filled(g)
    return np.float32(float(_sumsq(gv, g.size)[0]))


def test_adam_settings():
    """Every clip / grad_scale / weight decay / AMSGrad setting: the four dv3_adam_clip_opts instantiations, and the
    plain dv3_adam_clip where the setting is its own."""
    n = 1023
    for (cid, scale, max_norm), gs, wd, ams in TB.OPT_SETTINGS:
        g = TB.optim_grads(n, 11, scale)
        state = TB.optim_state(n, 11, ams)
        S = _kernel_sumsq(g)
        hyper = TB.hyper_for(1, gs=gs)
        ref = TB.adam_step(state[0], g, state[1], state[2], state[3], hyper, S, TB.OPT_BETAS[0], TB.OPT_BETAS[1],
                           TB.OPT_EPS, max_norm, wd)
        _check_adam(_adam(n, g, state, hyper, S, max_norm, wd), ref, ams, cid)
        if wd == 0.0 and not ams:
            _check_adam(_adam(n, g, state, hyper, S, max_norm, wd, plain=True), ref, False, cid)


@pytest.mark.parametrize("n", TB.OPT_SIZES + ["arena"])
def test_adam_sizes(n, arena_n):
    n = arena_n if n == "arena" else n
    for (cid, scale, max_norm), gs, wd, ams in ((TB.CLIPS[0], 0.5, 1e-2, True), (TB.CLIPS[2], 1.0, 0.0, False)):
        g = TB.optim_grads(n, n % 977, scale)
        state = TB.optim_state(n, n % 977, ams)
        S = _kernel_sumsq(g)
        hyper = TB.hyper_for(3, gs=gs)
        ref = TB.adam_step(state[0], g, state[1], state[2], state[3], hyper, S, TB.OPT_BETAS[0], TB.OPT_BETAS[1],
                           TB.OPT_EPS, max_norm, wd)
        _check_adam(_adam(n, g, state, hyper, S, max_norm, wd), ref, ams, cid)


def test_adam_steps_teacher_forced():
    """Five steps on one state: each step's reference starts from the kernel's own fp32 state and sumsq."""
    n, max_norm, wd = 4099, 0.1, 1e-2
    p, m, v, vmax = (_filled(x)[1] for x in TB.optim_state(n, 3, True))
    for t in range(1, 6):
        g = TB.optim_grads(n, 100 + t)
        gbuf, gv = _filled(g)
        obuf, out = guarded(1)
        scratch = torch.zeros(_raw("dv3_sumsq_scratch_floats")(), device="cuda")
        _call("dv3_sumsq", _p(gv), n, _p(out), _p(scratch), _st())
        hyper = TB.hyper_for(t, gs=0.5)
        hb, hvv = _filled(hyper)
        torch.cuda.synchronize()
        before = [x.cpu().numpy() for x in (p, m, v, vmax)]
        S = np.float32(float(out[0]))
        ref = TB.adam_step(before[0], g, before[1], before[2], before[3], hyper, S, TB.OPT_BETAS[0], TB.OPT_BETAS[1],
                           TB.OPT_EPS, max_norm, wd)
        _call("dv3_adam_clip_opts", _p(p), _p(gv), _p(m), _p(v), _p(vmax), n, _p(hvv), _p(out), TB.OPT_BETAS[0],
              TB.OPT_BETAS[1], TB.OPT_EPS, max_norm, wd, _st())
        torch.cuda.synchronize()
        _check_adam([x.cpu().numpy() for x in (p, m, v, vmax)], ref, True, "step %d" % t)


def test_flat_adam_split_parts_at_an_offset():
    """FlatAdam with two parts whose clocks differ: one launch per part, the second at an offset, each with its own
    bias corrections; elementwise against the fp64 step of each part."""
    from deepvoice3_pytorch_b200.train_step import FlatAdam, ParameterArena
    torch.manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(1001, device="cuda")), torch.nn.Parameter(torch.randn(4099, device="cuda"))]
    arena = ParameterArena(None, params=params)
    n = arena.numel
    cut = arena.offsets[1]
    opt = FlatAdam(arena, lr=5e-4, betas=TB.OPT_BETAS, eps=TB.OPT_EPS, clip_thresh=0.1, weight_decay=1e-2,
                   amsgrad=True, parts=[(0, cut), (cut, n)])
    opt.part_t = [3, 0]
    _, m, v, vmax = TB.optim_state(n, 9, True)
    opt.m.copy_(_dev(m)), opt.v.copy_(_dev(v)), opt.vmax.copy_(_dev(vmax))
    g = TB.optim_grads(n, 9)
    g[1001:cut] = 0.0                                          # the arena's alignment padding carries no gradient
    arena.grad.copy_(_dev(g))
    p = arena.flat.cpu().numpy()
    opt.set_hyper(5e-4, grad_scale=0.5)
    assert opt.split_update() and opt.part_t == [4, 1]
    opt.apply()
    torch.cuda.synchronize()
    S = np.float32(float(opt.sumsq[0]))
    ref_s, b_s = TB.sumsq_bound(g)
    _note("sumsq", abs(float(S) - ref_s) / b_s)
    hyper = opt.hyper.cpu().numpy()
    got = [x.cpu().numpy() for x in (arena.flat, opt.m, opt.v, opt.vmax)]
    for k, (lo, hi) in enumerate(opt.parts):
        sl = slice(lo, hi)
        ref = TB.adam_step(p[sl], g[sl], m[sl], v[sl], vmax[sl], hyper[4 * k:4 * k + 4], S, TB.OPT_BETAS[0],
                           TB.OPT_BETAS[1], TB.OPT_EPS, 0.1, 1e-2)
        _check_adam([x[sl] for x in got], ref, True, "part %d" % k)


# ---- sinusoidal position encoding -----------------------------------------------------------------------------------
def _tables():
    from deepvoice3_pytorch_b200.modules import position_encoding_init
    out = [(P, D, position_encoding_init(P, D, 1.0, sinusoidal=False).numpy()) for P, D in TB.SIN_TABLES]
    rng = np.random.RandomState(0)
    out += [(300, 96, (rng.randn(300, 96) * 3).astype(np.float32)), (64, 513, (rng.randn(64, 513) * 3).astype(np.float32))]
    return out


TABLES = [(P, D) for P, D in TB.SIN_TABLES] + [(300, 96), (64, 513)]


@pytest.mark.parametrize("ti", range(len(TABLES)), ids=["%dx%d" % t for t in TABLES])
def test_sinusoid_fwd(ti):
    P, D, table = _tables()[ti]
    B, T = 4, 97
    pos, _ = TB.dw_inputs(B, T, D, P, P + D, per_utt=False, cancel=False)
    d_pos, d_tab = _dev(pos), _dev(table)
    for w in ([TB.SIN_RATES[0]], [TB.SIN_RATES[1]], [TB.SIN_RATES[2]], list(np.linspace(0.9, 1.5, B))):
        w = np.asarray(w, np.float32)
        obuf, out = guarded(B * T * D)
        err = torch.zeros(1, dtype=torch.int32, device="cuda")
        _call("dv3_sinusoid_fwd", _p(d_pos), _p(d_tab), _p(_dev(w)), w.size, _p(out), B, T, D, P, _p(err), _st())
        torch.cuda.synchronize()
        assert int(err[0]) == 0
        assert_written_inside_only(obuf, B * T * D)
        ref, b = TB.sinusoid_fwd(pos, table, w)
        got = _np(out).reshape(B, T, D)
        assert np.all(got[pos == 0] == 0)
        _note("sinusoid fwd", TB.ratio(got, ref, b))


@pytest.mark.parametrize("ti", range(len(TABLES)), ids=["%dx%d" % t for t in TABLES])
@pytest.mark.parametrize("cancel", [False, True], ids=["random", "cancelling"])
def test_sinusoid_rate_gradient(ti, cancel):
    P, D, table = _tables()[ti]
    d_tab = _dev(table)
    for B, T, w in ((4, 97, [TB.SIN_RATES[2]]), (3, 64, [1.0, 1.29, 1.385])):
        w = np.asarray(w, np.float32)
        pos, dy = TB.dw_inputs(B, T, D, P, B + T + D, per_utt=w.size > 1, cancel=cancel)
        if cancel:
            dy = TB.cancelling_dy(pos, table, w, 2)
        d_pos, d_dy, d_w = _dev(pos), _dev(dy), _dev(w)
        dw0 = np.full(w.size, 0.25, np.float32)
        ref, b = TB.sinusoid_dw(pos, table, w, dy, dw0)
        init = np.random.RandomState(1).randn(P, D).astype(np.float32)
        terms, deriv = TB._dw_terms(pos, table, w, dy)
        wb = np.repeat(w, B) if w.size == 1 else w
        tt = np.asarray(dy, np.float64) * deriv * wb[:, None, None].astype(np.float64) * (pos > 0)[:, :, None]
        want, mag, slack = init.astype(np.float64), np.zeros((P, D)), np.zeros((P, D))
        np.add.at(want, pos.reshape(-1), tt.reshape(-1, D))
        np.add.at(mag, pos.reshape(-1), np.abs(tt).reshape(-1, D))
        np.add.at(slack, pos.reshape(-1), (np.abs(dy) * wb[:, None, None] * (pos > 0)[:, :, None]).reshape(-1, D))
        cnt = np.bincount(pos.reshape(-1), minlength=P)[:, None]
        # every add of a row's term rounds at the size of the running value, init included: (count + 4) u (|init| +
        # mag); sinf / cosf within 2 ulp of 1 relative to |dy w| (slack)
        tbound = (cnt + 4) * TB.U * (mag + np.abs(init)) + 8 * TB.U * slack + 2 * TB.U * np.abs(init)
        for name in ("dv3_sinusoid_bwd", "dv3_sinusoid_bwd_det"):
            for with_table in (False, True):
                wbuf, dw = _filled(dw0)
                tbuf, dt = _filled(init) if with_table else (None, None)
                _call(name, _p(d_pos), _p(d_tab), _p(d_w), w.size, _p(d_dy), _p(dt), _p(dw), B, T, D, P, _st())
                torch.cuda.synchronize()
                assert_written_inside_only(wbuf, w.size)
                _note("sinusoid dw", TB.ratio(_np(dw), ref, b))
                if with_table:
                    assert_written_inside_only(tbuf, P * D)
                    got = _np(dt).reshape(P, D)
                    assert np.array_equal(got[0], init[0])
                    _note("sinusoid dtable", TB.ratio(got, want, tbound))


def test_zz_report():
    """The largest error / bound ratio per output over the tests above (run with -s to see it)."""
    print("\nlargest error / bound, per output:")
    for k in sorted(WORST):
        print("  %-18s %.3g" % (k, WORST[k]))
