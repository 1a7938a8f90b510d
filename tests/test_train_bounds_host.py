"""CPU: the bounds of tests/train_bounds.py have teeth.  Each defect below is applied to the fp64 reference; on the
inputs the GPU tests use, the perturbed reference must leave the bound of the true one by more than a factor of two on
at least one element (or scalar), so a kernel within its bound cannot carry the defect.  Also the finding behind the
cancellation-free binary-divergence gradient in csrc/loss.cu: an fp32 emulation of the parent kernel's formula leaves
the new bound on saturated predictions."""
import numpy as np
import pytest

import train_bounds as TB

FACTOR = 2.0


def _report(what, factors):
    print("\n%s: defect / bound" % what)
    for k, v in sorted(factors.items(), key=lambda kv: kv[1]):
        print("  %-45s %10.3g" % (k, v))
    for k, v in factors.items():
        assert v > FACTOR, (k, v)


def _spec_case(B, T, D, r, kind, seed):
    yh, y0 = TB.planted_pairs(B, T, D, seed)
    return yh, TB.shift_targets(yh, y0, r), TB.lengths_for(kind, B, T, r, seed)


SPEC_DEFECTS = ["mask one frame late", "eps 1e-7", "eps term sign flipped", "priority gain without D/pbin",
                "plain mean over B T D", "frame shift on y_hat", "t_log ignored"]


def test_spec_loss_bounds_catch_defects():
    cases = []
    for cid, B, T, D, r, kind, tl, w, bw, pbin, pw in TB.SPEC_SHAPES:
        if cid in ("linear", "linear1025"):
            continue                                   # same arithmetic as "mel", at sizes the CPU need not repeat
        cases.append((_spec_case(B, T, D, r, kind, B * T + D), r, tl, w, bw, pbin, pw))
    B, T, D, r = 5, 61, 80, 2
    data = _spec_case(B, T, D, r, "ragged", 7)
    for tl in TB.SPEC_TLOG:
        cases.append((data, r, tl, 0.5, 0.1, 70, 0.5))
    factors = {}
    for defect in SPEC_DEFECTS:
        worst = 0.0
        for (yh, y, ln), r, tl, w, bw, pbin, pw in cases:
            ref = TB.spec_loss(yh, y, ln, r, w, bw, pbin, pw, t_log=tl)
            bad = TB.spec_loss(yh, y, ln, r, w, bw, pbin, pw, t_log=tl, defect=defect)
            worst = max(worst, TB.ratio(bad["grad"], ref["grad"], ref["grad_bound"]))
        factors[defect] = worst
    _report("spectrogram loss gradient", factors)


def test_spec_loss_eps_defect_needs_saturation():
    """eps 1e-7 for 1e-8 is visible only where p is saturated: on the unplanted values it stays inside the bound."""
    rng = np.random.RandomState(3)
    yh = rng.uniform(0.05, 0.95, (2, 30, 80)).astype(np.float32)
    y = rng.uniform(0.05, 0.95, (2, 30, 80)).astype(np.float32)
    ln = np.full(2, 30)
    ref = TB.spec_loss(yh, y, ln, 1, 0.5, 0.1, 0, 0.0)
    bad = TB.spec_loss(yh, y, ln, 1, 0.5, 0.1, 0, 0.0, defect="eps 1e-7")
    assert TB.ratio(bad["grad"], ref["grad"], ref["grad_bound"]) < 1.0


def test_parent_gradient_formula_leaves_the_bound_when_saturated():
    """The parent kernel's (sigmoid(L) - y) (1/(p+eps) + 1/(1-p+eps)), emulated in numpy fp32, against the exact
    derivative under the new bound: far outside it on saturated predictions and p == y pairs."""
    B, T, D, r = 16, 203, 80, 1
    yh, y0 = TB.planted_pairs(B, T, D, B * T + D)
    y = TB.shift_targets(yh, y0, r)
    old = TB.spec_loss_fp32_logit_grad(yh, y, r)
    exact = TB.spec_bd_exact_grad(yh, y, r)
    bound = TB.spec_bd_grad_bound(yh, y, r)
    p = yh[:, :T - r].astype(np.float64)
    sat = (p >= 1 - 64 * 2.0 ** -24) & (p < 1)
    r_sat = TB.ratio(old[sat], exact[sat], bound[sat])
    print("\nparent formula, p in [1 - 64 * 2^-24, 1): error / bound %.3g" % r_sat)
    assert r_sat > 100
    # the pairs of the table that motivated the change
    for p_, y_ in ((1 - 2.0 ** -24, 1.0), (1 - 2.0 ** -22, 1.0), (0.999, 0.999)):
        a = np.full((1, 2, 1), p_, np.float32)
        b = np.full((1, 2, 1), y_, np.float32)
        e = TB.spec_bd_exact_grad(a, b, 1)
        g = TB.spec_loss_fp32_logit_grad(a, b, 1)
        assert TB.ratio(g, e, TB.spec_bd_grad_bound(a, b, 1)) > 100, (p_, y_, float(g), float(e))


def test_new_gradient_formula_in_fp32_meets_the_bound():
    """The kernel's new formula, emulated in numpy fp32 (no fma), is inside the bound on the planted inputs."""
    B, T, D, r = 16, 203, 80, 1
    yh, y0 = TB.planted_pairs(B, T, D, B * T + D)
    y = TB.shift_targets(yh, y0, r)
    p, tg = yh[:, :T - r], y[:, r:]
    e = np.float32(TB.EPS_LOSS)
    one = np.float32(1)
    q = (((p - tg) + e * (one - np.float32(2) * tg)) / ((p + e) * (one - p + e))).astype(np.float32)
    rr = TB.ratio(q, TB.spec_bd_exact_grad(yh, y, r), TB.spec_bd_grad_bound(yh, y, r))
    print("\nnew formula in numpy fp32: error / bound %.3g" % rr)
    assert rr <= 1.0


AUX_DEFECTS = ["guided attention with batch maxima", "BCE clamp 1e-6", "d_done mean over n_done"]


def test_aux_loss_bounds_catch_defects():
    factors = {d: 0.0 for d in AUX_DEFECTS}
    for cid, A, B, Td, Ts, ext, use_attn in TB.AUX_CASES:
        dh, done, attn, il, dl = TB.aux_inputs(A, B, Td, Ts, Td + Ts)
        ref = TB.aux_loss(dh, done, attn, il, dl, TB.AUX_SIGMA, use_attn, ext)
        for d in AUX_DEFECTS:
            bad = TB.aux_loss(dh, done, attn, il, dl, TB.AUX_SIGMA, use_attn, ext, defect=d)
            factors[d] = max(factors[d], TB.ratio(bad["d_done"], ref["d_done"], ref["d_done_bound"]),
                             TB.ratio(bad["d_attn"], ref["d_attn"], ref["d_attn_bound"]))
    _report("auxiliary loss gradients", factors)


OPT_DEFECTS = ["bias correction 2 not square-rooted", "weight decay before clipping",
               "AMSGrad max against the previous v", "clip without +1e-6"]


def test_adam_bounds_catch_defects():
    n = 1023
    factors = {d: 0.0 for d in OPT_DEFECTS}
    for (cid, scale, max_norm), gs, wd, ams in TB.OPT_SETTINGS:
        g = TB.optim_grads(n, 11, scale)
        p, m, v, vmax = TB.optim_state(n, 11, ams)
        S = np.float32(np.dot(g.astype(np.float64), g))
        hyper = TB.hyper_for(1, gs=gs)
        args = (p, g, m, v, vmax, hyper, S, TB.OPT_BETAS[0], TB.OPT_BETAS[1], TB.OPT_EPS, max_norm, wd)
        ref = TB.adam_step(*args)
        for d in OPT_DEFECTS:
            bad = TB.adam_step(*args, defect=d)
            r = max(TB.ratio(bad[k], ref[k], ref[k + "_b"]) for k in ("p", "m", "v"))
            if ams:
                r = max(r, TB.ratio(bad["vmax"], ref["vmax"], ref["vmax_b"]))
            factors[d] = max(factors[d], r)
    for nn in TB.OPT_SIZES:
        if nn % 4:
            g = TB.optim_grads(nn, nn)
            ref, b = TB.sumsq_bound(g)
            bad, _ = TB.sumsq_bound(g, defect="sumsq drops the n % 4 tail")
            factors["sumsq drops the n % 4 tail"] = max(factors.get("sumsq drops the n % 4 tail", 0.0),
                                                        abs(bad - ref) / b)
    _report("clip + Adam and sumsq", factors)


def test_sumsq_bound_holds_for_an_fp32_sum():
    g = TB.optim_grads(100003, 5)
    ref, b = TB.sumsq_bound(g)
    s = np.add.reduce(g.astype(np.float32) ** 2, dtype=np.float32)
    assert abs(float(s) - ref) <= b


def _tables():
    from deepvoice3_pytorch_b200.modules import position_encoding_init
    out = [(P, D, position_encoding_init(P, D, 1.0, sinusoidal=False).numpy()) for P, D in TB.SIN_TABLES]
    rng = np.random.RandomState(0)
    out += [(300, 96, (rng.randn(300, 96) * 3).astype(np.float32))]
    return out


def test_sinusoid_bounds_catch_defects():
    factors = {"product in fp64": 0.0, "sin and cos swapped": 0.0}
    for P, D, table in _tables():
        B, T = 4, 97
        pos, _ = TB.dw_inputs(B, T, D, P, P + D, per_utt=False, cancel=False)
        for w in ([TB.SIN_RATES[1]], [TB.SIN_RATES[2]], list(np.linspace(0.9, 1.5, B))):
            w = np.asarray(w, np.float32)
            ref, b = TB.sinusoid_fwd(pos, table, w)
            for d in factors:
                bad, _ = TB.sinusoid_fwd(pos, table, w, defect=d)
                factors[d] = max(factors[d], TB.ratio(bad, ref, b))
    _report("sinusoid forward", factors)


def test_rate_gradient_bound_catches_fp32_accumulation():
    from deepvoice3_pytorch_b200.modules import position_encoding_init
    P, D = 512, 256
    table = position_encoding_init(P, D, 1.0, sinusoidal=False).numpy()
    worst = 0.0
    for B, T, w in ((4, 97, np.asarray([TB.SIN_RATES[2]], np.float32)),
                    (3, 64, np.asarray([1.0, 1.29, 1.385], np.float32))):
        pos, _ = TB.dw_inputs(B, T, D, P, 1, per_utt=w.size > 1, cancel=True)
        dy = TB.cancelling_dy(pos, table, w, 2)
        dw0 = np.full(w.size, 0.25)
        ref, b = TB.sinusoid_dw(pos, table, w, dy, dw0)
        terms, _ = TB._dw_terms(pos, table, w, dy)
        mag = np.abs(terms).reshape(w.size, -1).sum(1)
        assert np.all(np.abs(ref - dw0) <= 1e-3 * mag)                     # the sum cancels
        bad = TB.sinusoid_dw_fp32(pos, table, w, dy, dw0)
        worst = max(worst, TB.ratio(bad, ref, b))
    _report("rate gradient", {"dw accumulated in fp32": worst})
