"""TEST INFRASTRUCTURE ONLY.  fp64 references and elementwise error bounds for the kernels between the model outputs
and the parameter update: the spectrogram and auxiliary losses with their gradients (csrc/loss.cu), the squared
gradient norm and the clip + Adam update (csrc/optim.cu), and the sinusoidal position encoding with its rate gradient
(csrc/elementwise.cu).  The input builders at the end are shared by the CPU test of the bounds and the GPU tests.

Error model.  u = 2^-24.  The operands are the kernel's exact fp32 inputs; the constants are the fp32 values the kernel
receives (eps = fl(1e-8), the 1e-12 clamp, beta1, beta2, the Adam eps, the four hyper floats).  A rounded operation
contributes u of its result; with fma contraction (nvcc's default) a rounding disappears, which the bounds allow.  The
build is not fast-math (_build.py), so the CUDA C++ Programming Guide's accuracy figures apply: logf, log1pf 1 ulp;
expf, sinf, cosf, rsqrtf 2 ulp; sqrtf and / correctly rounded; double exp 1 ulp.  One ulp of a value is at most 2u of
it (ULP below).  Every bound is first order and scaled by SECOND_ORDER.

Reductions.  A sum whose terms pass through at most h roundings on their way to the result is within
gamma(h) = h u / (1 - h u) of the sum of the magnitudes added; h counts the serial run of one thread, the warp and
block trees, and the chain of atomic adds (or of the fixed-order tail).  The scalars are checked as
|got - (init + ref)| <= gamma(h) (|init| + sum |term|) + sum err(term).

Spectrogram loss (spec_loss_body), per pair (b, t < TL - r) with p = y_hat[b,t], y = y[b,t+r], d = p - y:
    coef = w m inv_sm + (1-w) inv_n          inv_sm: double 1/(Sm D) rounded; inv_n: three fp32 roundings;  <= 6u
    c1   = (1-pw) + [i < pbin] pw D / pbin                                                                <= 3u
    A    = c1 (1-bw) sign(d)                                                                               <= 5u
    Q    = (d + eps (1-2y)) / ((p+eps)(1-p+eps)):  the numerator within 3u (|d| + eps |1-2y|) = 3u N, the
           denominator 4u, the quotient u
    grad = coef (A + bw Q):  |err| <= 20u coef (|A| + bw N / den)
  Past TL - r the gradient is exactly 0.  Sm = sum_b clamp(len_b - r, 0, TL - r) D; when Sm = 0 the kernel's masked
  mean is 0 (coef = (1-w) inv_n) while the reference's is 0/0 = NaN: the reference here follows the kernel.
  z = -(y log(p+eps) + (1-y) log(1-p+eps)) + log1p(2eps): the rounded arguments cost u absolute per logarithm, logf
  2u of its result, the products and sums u each:  |err z| <= 4u (|y| + |1-y|) + 8u Z,  Z = y |log(p+eps)| +
  |1-y| |log(1-p+eps)| + log1p(2eps).  The loss term coef (c1 (1-bw) |d| + bw z) then errs by at most
  coef (10u c1 (1-bw) |d| + bw (err z + 10u Z)); the L1 term coef c1 |d| by 12u of itself.
Auxiliary loss (aux_loss_body):
    d_done = inv_nd (p - t) / max((1-p) p, 1e-12f):  6u relative (max is monotone and 1-Lipschitz, so the clamp
             branch needs no emulation).  Steps past ext[0] are exactly 0.
    d_attn = inv_na (float)W, W = 1 - exp(-q^2 / 2 sigma^2) formed in double: 4u relative, plus the absolute error of
             1 - exp(.) in double (4 2^-53, relative to W only where W is tiny).  Exactly 0 past in_len, dec_len, ext
             and everywhere when use_attn = 0.
    BCE term inv_nd (t max(log p, -100) + (1-t) max(log(1-p), -100)): 6u of itself plus 2u inv_nd (the rounded 1-p).
sumsq: h = 4 ceil(n4 / (blocks 256)) + 1 (fmaf run + tail) + 8 (warp and block trees) + ceil(blocks / 256) + 8 (the
  fixed-order tail over the partials); squares below the normal range lose 2^-150 per rounding:
  |err| <= gamma(h) sum g^2 + n 2^-150.
clip + Adam (adam_clip_kernel), one step from the kernel's fp32 state and its fp32 sumsq input:
    coef = gscale min(1, max_norm / (sqrt(S) gscale + 1e-6f)):  5u
    g'   = g coef + wd p:  8u (|g coef| + |wd p|) = 8u G
    m'   = b1 m + (1-b1) g':  3u (b1 |m| + (1-b1) G) + (1-b1) err g'
    v'   = b2 v + (1-b2) g'^2:  4u (b2 v + (1-b2) G^2) + 2 (1-b2) G err g',  plus 2^-147 below the normal range
    vmax' = max(vmax, v') (exact selection)
    p'   = p - (lr / bc1) m' / (sqrt(v'') rsqrt(bc2) + eps):  step 1u, rsqrtf 4u, sqrtf u plus the propagated
           err v'' / sqrt(v''), product and sum u each, quotient and difference u.
  Several steps are checked one at a time from the kernel's own state (teacher forcing), so the bound does not grow.
sinusoid forward: trig(fl(w table)) within 2 ulp (4u of the result) plus 2^-148; position 0 gives exactly 0.
rate gradient dw: each term fl(dy trig(a)) tv is exact in double after the fp32 product (u) and trig (4u); the double
  sum adds gamma_53(n); the float conversion and the += add u each:
  |err| <= (5u + gamma_53(n)) sum |dy trig(a) tv| + u (|S| + |dw0 + S|) + 2^-148.
"""
import numpy as np

U = 2.0 ** -24
U64 = 2.0 ** -53
ULP = 2.0 * U
SECOND_ORDER = 1.0 + 2.0 ** -10
F32 = np.float32
EPS_LOSS = float(F32(1e-8))
CLAMP_DONE = float(F32(1e-12))
CLIP_EPS = float(F32(1e-6))
LOSS_MAX_BLOCKS = 132 * 8
AUX_BLOCKS = 132 * 2
SUMSQ_MAX_BLOCKS = 132 * 8


def gamma(h, u=U):
    return h * u / (1.0 - h * u)


def ratio(got, ref, bound):
    """Largest |got - ref| / bound; exact agreement scores 0 even where the bound is 0; NaN scores inf."""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nan_to_num(r, nan=np.inf, posinf=np.inf).max()) if r.size else 0.0


def f32(x):
    return float(F32(x))


# ---- spectrogram loss ---------------------------------------------------------------------------------------------
def spec_chain(B, T, D):
    """Roundings a term passes through in the atomic form (the longer of the two): the grid-stride run, the block tree
    and one atomic per block, plus the initial value."""
    total = B * T * D
    blocks = min(LOSS_MAX_BLOCKS, -(-total // 256))
    return -(-total // (blocks * 256)) + 8 + blocks + 1


def spec_loss(y_hat, y, lengths, r, w, bw, pbin, pw, t_log=None, eps=EPS_LOSS, defect=None):
    """fp64 reference and bounds of dv3_spec_loss_terms / dv3_spec_loss_det.  y_hat, y (B, T, D) fp32; lengths (B,)
    int; t_log None or an int.  defect: one of the names in tests/test_train_bounds_host.py (the reference with that mistake).
    -> dict(grad, grad_bound, loss, l1, bd, mag_loss, err_loss, mag_l1, err_l1, mag_bd, err_bd, h)."""
    B, T, D = y_hat.shape
    w, bw, pw = f32(w), f32(bw), f32(pw)
    TL = T if t_log is None or defect == "t_log ignored" else int(min(T, max(r + 1, t_log)))
    n_pair = TL - r
    yh = np.asarray(y_hat, np.float64)
    yy = np.asarray(y, np.float64)
    if defect == "frame shift on y_hat":
        p, tg = yh[:, r:TL], yy[:, :n_pair]
    else:
        p, tg = yh[:, :n_pair], yy[:, r:TL]
    lengths = np.asarray(lengths, np.int64)
    t = np.arange(n_pair)
    late = defect == "mask one frame late"
    m = ((t[None, :] + r <= lengths[:, None]) if late else (t[None, :] + r < lengths[:, None])).astype(np.float64)
    sm = float(np.clip(lengths - r + (1 if late else 0), 0, n_pair).sum()) * D
    inv_sm = 1.0 / sm if sm > 0 else 0.0
    inv_n = 1.0 / (B * (T if defect == "plain mean over B T D" else n_pair) * D)
    coef = (w * m * inv_sm + (1 - w) * inv_n)[:, :, None]
    if pbin > 0 and pw > 0:
        gain = pw if defect == "priority gain without D/pbin" else pw * D / pbin
        c1 = (1 - pw) + (np.arange(D) < pbin) * gain
    else:
        c1 = np.ones(D)
    d = p - tg
    A = c1 * (1 - bw) * np.sign(d)
    sgn = -1.0 if defect == "eps term sign flipped" else 1.0
    e_ = 1e-7 if defect == "eps 1e-7" else eps
    den = (p + e_) * (1 - p + e_)
    N = np.abs(d) + e_ * np.abs(1 - 2 * tg)
    Q = (d + sgn * e_ * (1 - 2 * tg)) / den
    g = np.zeros_like(yh)
    g[:, :n_pair] = coef * (A + bw * Q)
    gb = np.zeros_like(yh)
    gb[:, :n_pair] = SECOND_ORDER * 20 * U * coef * (np.abs(A) + bw * N / den) + 2.0 ** -149
    with np.errstate(divide="ignore", invalid="ignore"):
        la, lc = np.log(p + e_), np.log(1 - p + e_)
        ya = np.where(tg == 0, 0.0, tg * la)
        yc = np.where(tg == 1, 0.0, (1 - tg) * lc)
    z = -(ya + yc) + np.log1p(2 * e_)
    Z = np.abs(ya) + np.abs(yc) + np.log1p(2 * e_)
    err_z = 4 * U * (np.abs(tg) + np.abs(1 - tg)) + 8 * U * Z
    l1 = coef * c1 * np.abs(d)
    bd = coef * z if bw > 0 else np.zeros_like(l1)
    e = coef * (c1 * (1 - bw) * np.abs(d)) + (bw * coef * z if bw > 0 else 0.0)
    err_e = coef * (10 * U * c1 * (1 - bw) * np.abs(d) + (bw * (err_z + 10 * U * Z) if bw > 0 else 0.0))
    err_bd = coef * (err_z + 10 * U * Z) if bw > 0 else np.zeros_like(l1)
    return dict(grad=g, grad_bound=gb, loss=float(e.sum()), l1=float(l1.sum()), bd=float(bd.sum()),
                mag_loss=float(np.abs(e).sum()), err_loss=float(err_e.sum()), mag_l1=float(l1.sum()),
                err_l1=float(12 * U * l1.sum()), mag_bd=float(np.abs(bd).sum()), err_bd=float(err_bd.sum()),
                h=spec_chain(B, T, D))


def scalar_bound(h, init, mag, err):
    return SECOND_ORDER * (gamma(h) * (abs(init) + mag + err) + err) + 2.0 ** -140


def spec_loss_fp32_logit_grad(y_hat, y, r, eps=EPS_LOSS):
    """numpy-fp32 emulation of the binary-divergence gradient as the parent kernel formed it,
    (u/(1+u) - y) (1/(p+eps) + 1/(1-p+eps)) with u = exp(log(p+eps) - log(1-p+eps)), over the pairs; (B, T-r, D)."""
    T = y_hat.shape[1]
    p, tg = y_hat[:, :T - r].astype(F32), y[:, r:].astype(F32)
    e = F32(eps)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        L = np.log(p + e) - np.log(F32(1) - p + e)
        u = np.exp(L)
        return ((u / (F32(1) + u) - tg) * (F32(1) / (p + e) + F32(1) / (F32(1) - p + e))).astype(F32)


def spec_bd_exact_grad(y_hat, y, r, eps=EPS_LOSS):
    T = y_hat.shape[1]
    p, tg = np.asarray(y_hat[:, :T - r], np.float64), np.asarray(y[:, r:], np.float64)
    return (p - tg + eps * (1 - 2 * tg)) / ((p + eps) * (1 - p + eps))


def spec_bd_grad_bound(y_hat, y, r, eps=EPS_LOSS):
    """The gradient bound of the binary-divergence part alone (bw = 1, coef = 1)."""
    T = y_hat.shape[1]
    p, tg = np.asarray(y_hat[:, :T - r], np.float64), np.asarray(y[:, r:], np.float64)
    return SECOND_ORDER * 20 * U * (np.abs(p - tg) + eps * np.abs(1 - 2 * tg)) / ((p + eps) * (1 - p + eps))


# ---- auxiliary loss -----------------------------------------------------------------------------------------------
def aux_loss(done_hat, done, attn, in_len, dec_len, sigma, use_attn, ext=None, defect=None):
    """fp64 reference and bounds of dv3_aux_loss_terms / dv3_aux_loss_det.  done_hat, done (B, Td) (or flat with
    ext None); attn (A, B, Td, Ts).  -> dict(d_done, d_done_bound, d_attn, d_attn_bound, loss, bce, ga, mag_*, err_*, h)."""
    A, B, Td, Ts = attn.shape
    p = np.asarray(done_hat, np.float64).reshape(-1)
    t = np.asarray(done, np.float64).reshape(-1)
    n_done = p.size
    TdL = Td if ext is None else int(min(Td, max(1, ext[0])))
    TsL = Ts if ext is None else int(min(Ts, max(1, ext[1])))
    keep = np.ones(n_done, bool) if ext is None else (np.arange(n_done) % Td) < TdL
    nd = n_done if ext is None or defect == "d_done mean over n_done" else B * TdL
    inv_nd = 1.0 / nd
    clamp = 1e-6 if defect == "BCE clamp 1e-6" else CLAMP_DONE
    dd = np.where(keep, inv_nd * (p - t) / np.maximum((1 - p) * p, clamp), 0.0)
    ddb = np.where(keep, SECOND_ORDER * 6 * U * np.abs(dd), 0.0) + 2.0 ** -149
    with np.errstate(divide="ignore"):
        lp, lq = np.maximum(np.log(p), -100.0), np.maximum(np.log(1 - p), -100.0)
    bce_t = np.where(keep, -inv_nd * (t * lp + (1 - t) * lq), 0.0)
    err_bce = np.where(keep, 6 * U * np.abs(bce_t) + 2 * U * inv_nd, 0.0)
    out = dict(d_done=dd, d_done_bound=ddb, bce=float(bce_t.sum()), mag_bce=float(np.abs(bce_t).sum()),
               err_bce=float(err_bce.sum()))
    blocks_stride = AUX_BLOCKS * 256
    h = -(-n_done // blocks_stride) + 8 + AUX_BLOCKS + 1
    if use_attn:
        inv_na = 1.0 / (A * B * TdL * TsL)
        n = np.arange(Ts, dtype=np.float64)[None, None, :]
        tt = np.arange(Td, dtype=np.float64)[None, :, None]
        il, dl = np.asarray(in_len, np.float64), np.asarray(dec_len, np.float64)
        if defect == "guided attention with batch maxima":
            il, dl = np.full_like(il, il.max()), np.full_like(dl, dl.max())
        N, Tl = il[:, None, None], dl[:, None, None]
        inside = (n < N) & (tt < Tl) & (n < TsL) & (tt < TdL)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = np.where(inside, n / np.where(N > 0, N, 1) - tt / np.where(Tl > 0, Tl, 1), 0.0)
        s = float(F32(sigma))
        W = np.where(inside, -np.expm1(-q * q / (2 * s * s)), 0.0)
        da = np.broadcast_to(inv_na * W[None], attn.shape)
        dab = np.where(np.broadcast_to(inside[None], attn.shape),
                       SECOND_ORDER * (4 * U * da + inv_na * 4 * U64), 0.0) + 2.0 ** -149
        ga_t = np.asarray(attn, np.float64) * da
        out.update(d_attn=da, d_attn_bound=dab, ga=float(ga_t.sum()), mag_ga=float(np.abs(ga_t).sum()),
                   err_ga=float((4 * U * np.abs(ga_t) + np.abs(attn) * inv_na * 4 * U64).sum()))
        h += -(-attn.size // blocks_stride)
    else:
        out.update(d_attn=np.zeros(attn.shape), d_attn_bound=np.full(attn.shape, 2.0 ** -149), ga=0.0, mag_ga=0.0,
                   err_ga=0.0)
    out["loss"] = out["bce"] + out["ga"]
    out["h"] = h
    return out


# ---- sumsq and clip + Adam ----------------------------------------------------------------------------------------
def sumsq_bound(g, defect=None):
    """(ref, bound) of dv3_sumsq on fp32 g."""
    g = np.asarray(g, np.float64)
    n = g.size
    if defect == "sumsq drops the n % 4 tail":
        g = g[:n // 4 * 4]
    n4 = n >> 2
    blocks = max(1, min(SUMSQ_MAX_BLOCKS, (n4 + 255) // 256))
    h = 4 * -(-n4 // (blocks * 256)) + 1 + 8 + -(-blocks // 256) + 8
    ref = float(np.dot(g, g))
    return ref, SECOND_ORDER * gamma(h) * ref + n * 2.0 ** -150 + 2.0 ** -149


def adam_step(p, g, m, v, vmax, hyper, sumsq, beta1, beta2, eps, max_norm, wd, defect=None):
    """One clip + Adam step in fp64 from the kernel's fp32 state (vmax None: no AMSGrad).
    -> dict(p, m, v, vmax, and their bounds p_b, m_b, v_b, vmax_b)."""
    p, g, m, v = (np.asarray(x, np.float64) for x in (p, g, m, v))
    lr, bc1, bc2, gs = (float(x) for x in np.asarray(hyper, np.float32)[:4])
    b1, b2, eps, max_norm, wd = f32(beta1), f32(beta2), f32(eps), f32(max_norm), f32(wd)
    S = float(np.float32(sumsq))
    coef = gs
    if max_norm > 0:
        c = max_norm / (np.sqrt(S) * gs + (0.0 if defect == "clip without +1e-6" else CLIP_EPS))
        coef *= min(c, 1.0)
    if defect == "weight decay before clipping":
        gi = (g * gs + wd * p) * (coef / gs)
    else:
        gi = g * coef + wd * p
    G = np.abs(g * coef) + np.abs(wd * p)
    eg = 8 * U * G
    m1 = b1 * m + (1 - b1) * gi
    v1 = b2 * v + (1 - b2) * gi * gi
    em = 3 * U * (b1 * np.abs(m) + (1 - b1) * G) + (1 - b1) * eg
    ev = 4 * U * (b2 * v + (1 - b2) * G * G) + 2 * (1 - b2) * G * eg + 2.0 ** -147
    if vmax is not None:
        vm0 = np.asarray(vmax, np.float64)
        vd = np.maximum(vm0, v if defect == "AMSGrad max against the previous v" else v1)
    else:
        vd = v1
    rs2 = 1.0 / (bc2 if defect == "bias correction 2 not square-rooted" else np.sqrt(bc2))
    step = lr / bc1
    sq = np.sqrt(vd)
    Dn = sq * rs2 + eps
    with np.errstate(divide="ignore", invalid="ignore"):
        dS = np.minimum(np.where(vd > 0, ev / np.where(vd > 0, sq, 1.0), np.inf), np.sqrt(ev))
    eD = rs2 * (dS + 6 * U * sq) + U * Dn
    p1 = p - step * m1 / Dn
    ep = step / Dn * (em + np.abs(m1) * (3 * U + eD / Dn)) + U * np.abs(p1)
    out = dict(p=p1, m=m1, v=v1, p_b=SECOND_ORDER * ep + 2.0 ** -149, m_b=SECOND_ORDER * em + 2.0 ** -149,
               v_b=SECOND_ORDER * ev)
    if vmax is not None:
        out.update(vmax=vd, vmax_b=SECOND_ORDER * ev)
    return out


# ---- sinusoidal position encoding ---------------------------------------------------------------------------------
def sinusoid_fwd(pos, table, w, defect=None):
    """(ref (B, T, D), bound) of dv3_sinusoid_fwd: trig of the fp32 product fl(w table[pos])."""
    pos = np.asarray(pos)
    B, T = pos.shape
    D = table.shape[1]
    wb = np.asarray(w, np.float32)
    wb = (wb if wb.size == B else np.repeat(wb, B))[:, None, None]
    row = np.asarray(table, np.float32)[pos]
    a = wb.astype(np.float64) * row.astype(np.float64) if defect == "product in fp64" else \
        (wb * row).astype(np.float64)
    odd = (np.arange(D) % 2 == 1)
    if defect == "sin and cos swapped":
        odd = ~odd
    y = np.where(odd, np.cos(a), np.sin(a))
    y = np.where((pos > 0)[:, :, None], y, 0.0)
    return y, np.where((pos > 0)[:, :, None], SECOND_ORDER * 2 * ULP * np.abs(y) + 2.0 ** -148, 0.0)


def _dw_terms(pos, table, w, dy):
    pos = np.asarray(pos)
    B, T = pos.shape
    D = table.shape[1]
    wb = np.asarray(w, np.float32)
    wb = (wb if wb.size == B else np.repeat(wb, B))[:, None, None]
    tv = np.asarray(table, np.float32)[pos]
    a = (wb * tv).astype(np.float64)
    odd = (np.arange(D) % 2 == 1)
    deriv = np.where(odd, -np.sin(a), np.cos(a))
    live = (pos > 0)[:, :, None]
    return np.where(live, np.asarray(dy, np.float64) * deriv * tv, 0.0), deriv


def sinusoid_dw(pos, table, w, dy, dw0):
    """(ref (nw,), bound) of the rate gradient of dv3_sinusoid_bwd[_det], added to dw0."""
    terms, _ = _dw_terms(pos, table, w, dy)
    nw = np.asarray(w).size
    S = terms.reshape(nw, -1).sum(1)
    mag = np.abs(terms).reshape(nw, -1).sum(1)
    n = terms.size // nw
    dw0 = np.asarray(dw0, np.float64)
    ref = dw0 + S
    return ref, SECOND_ORDER * ((5 * U + gamma(n + 16, U64)) * mag + U * (np.abs(S) + np.abs(ref))) + 2.0 ** -148


def sinusoid_dw_fp32(pos, table, w, dy, dw0):
    """The rate gradient accumulated in fp32 in sinusoid_dw_kernel's order: thread j of 256 adds the terms q = j,
    j + 256, ... of its rate's rows in turn, then the xor-shuffle tree of each warp and the 8 warp sums in order."""
    pos = np.asarray(pos)
    B, T = pos.shape
    D = table.shape[1]
    nw = np.asarray(w).size
    wb = np.asarray(w, np.float32)
    wb = (wb if wb.size == B else np.repeat(wb, B))[:, None, None]
    tv = np.asarray(table, np.float32)[pos]
    a = wb * tv
    odd = (np.arange(D) % 2 == 1)
    deriv = np.where(odd, -np.sin(a.astype(np.float64)), np.cos(a.astype(np.float64))).astype(np.float32)
    terms = np.where((pos > 0)[:, :, None], (np.asarray(dy, np.float32) * deriv) * tv, np.float32(0)).astype(np.float32)
    out = np.empty(nw)
    per = terms.reshape(nw, -1)
    for k in range(nw):
        x = per[k]
        n = x.size
        pad = np.zeros(-(-n // 256) * 256, np.float32)
        pad[:n] = x
        lanes = pad.reshape(-1, 256)
        acc = np.zeros(256, np.float32)
        for row in lanes:
            acc = (acc + row).astype(np.float32)
        acc = acc.reshape(8, 32)
        o = 16
        while o:
            acc = (acc + acc[:, np.arange(32) ^ o]).astype(np.float32)
            o >>= 1
        t = np.float32(0)
        for j in range(8):
            t = np.float32(t + acc[j, 0])
        out[k] = float(np.float32(np.float32(dw0[k]) + t))
    return out


# ---- input builders (shared by the CPU and GPU tests) -------------------------------------------------------------
def planted_pairs(B, T, D, seed, frac=0.5):
    """(y_hat, y) fp32 (B, T, D): uniform values, with a fraction ``frac`` of the elements replaced by planted
    predictions p in {0, 2^-149, k 2^-24, 1 - k 2^-24, 1} (k <= 64) and targets in {0, 1, p, p +- 1 ulp}."""
    rng = np.random.RandomState(seed)
    yh = rng.uniform(0, 1, (B, T, D)).astype(np.float32)
    y = rng.uniform(0, 1, (B, T, D)).astype(np.float32)
    k = rng.randint(1, 65, (B, T, D)).astype(np.float64)
    special = np.stack([np.zeros_like(k), np.full_like(k, 2.0 ** -149), k * 2.0 ** -24, 1 - k * 2.0 ** -24,
                        np.ones_like(k), yh.astype(np.float64)]).astype(np.float32)
    sel = rng.randint(0, special.shape[0], (B, T, D))
    ph = np.take_along_axis(special, sel[None], 0)[0]
    plant = rng.uniform(0, 1, (B, T, D)) < frac
    yh = np.where(plant, ph, yh).astype(np.float32)
    # targets planted against y_hat[b, t] at y[b, t]; shift_targets moves them to the frame the kernel pairs
    tsel = rng.randint(0, 6, (B, T, D))
    up = np.nextafter(yh, np.float32(2)).astype(np.float32)
    dn = np.nextafter(yh, np.float32(-1)).astype(np.float32)
    tgt = np.stack([np.zeros_like(yh), np.ones_like(yh), yh, np.clip(up, 0, 1), np.clip(dn, 0, 1), y])
    ty = np.take_along_axis(tgt, tsel[None], 0)[0]
    tplant = rng.uniform(0, 1, (B, T, D)) < frac
    return yh, np.where(tplant, ty, y).astype(np.float32)


def shift_targets(y_hat, y, r):
    """Move the targets planted against y_hat[b, t] to y[b, t + r], where the kernel pairs them."""
    out = y.copy()
    if r > 0:
        out[:, r:] = y[:, :-r]
    return out


def lengths_for(kind, B, T, r, seed):
    rng = np.random.RandomState(seed)
    if kind == "full":
        return np.full(B, T, np.int64)
    if kind == "ragged":        # full, <= r (a fully masked row), > T, random
        ln = rng.randint(r + 1, T + 1, B).astype(np.int64)
        ln[0] = T
        if B > 1:
            ln[1] = r
        if B > 2:
            ln[2] = T + 5
        return ln
    if kind == "all_masked":    # every row <= r: Sm = 0
        return rng.randint(0, r + 1, B).astype(np.int64)
    raise ValueError(kind)


def optim_grads(n, seed, scale=1.0):
    """fp32 gradients: randn * scale with exact zeros, 1e-20 (squares below the normal range) and 1e3 planted, and the
    last element (the n % 4 tail) planted at 1e3."""
    rng = np.random.RandomState(seed)
    g = (rng.randn(n) * scale).astype(np.float32)
    sel = rng.randint(0, 8, n)
    g[sel == 0] = 0.0
    g[sel == 1] = 1e-20 * np.sign(rng.randn(int((sel == 1).sum())))
    g[sel == 2] = 1e3 * scale
    g[-1] = 1e3 * scale
    return g


def optim_state(n, seed, ams):
    rng = np.random.RandomState(seed + 1)
    p = rng.randn(n).astype(np.float32)
    m = (0.01 * rng.randn(n)).astype(np.float32)
    v = (1e-4 * rng.rand(n) ** 2).astype(np.float32)
    v[::5] = 0.0
    vmax = (v * rng.uniform(0.5, 2.0, n)).astype(np.float32) if ams else None
    return p, m, v, vmax


def dw_inputs(B, T, D, P, seed, per_utt, cancel):
    """(pos, dy) for the rate gradient.  pos: 1..len (wrapping below P) then padding 0, one row at P - 1.  cancel: per column, the first
    row of each rate's rows carries +X, the last -X, and the rows between small terms of one sign, so the sum is about
    1e-4 of the sum of magnitudes and an fp32 accumulation in the kernel's order loses the small terms."""
    rng = np.random.RandomState(seed)
    ar = (np.arange(T)[None] % (P - 1)) + 1
    if cancel:
        pos = np.tile(ar, (B, 1)).astype(np.int64)
    else:
        lens = rng.randint(1, T + 1, B)
        pos = np.where(np.arange(1, T + 1)[None] <= lens[:, None], ar, 0).astype(np.int64)
    pos[0, 0] = P - 1
    dy = rng.randn(B, T, D).astype(np.float32)
    return pos, dy


def cancelling_dy(pos, table, w, seed):
    """dy for the cancelling rate-gradient case (see dw_inputs)."""
    pos = np.asarray(pos)
    B, T = pos.shape
    D = table.shape[1]
    nw = np.asarray(w).size
    rng = np.random.RandomState(seed)
    _, deriv = _dw_terms(pos, table, w, np.ones((B, T, D), np.float32))
    gfac = deriv * np.asarray(table, np.float64)[pos]
    ok = np.abs(gfac) >= 1e-3                                              # terms of columns with tiny factors: 0
    safe = np.where(ok, gfac, 1.0)
    dy = np.where(ok, rng.uniform(0.5, 1.0, (B, T, D)) * 2.0 ** -25 / safe, 0.0)   # one sign, < ulp(1) / 2
    rows = (B * T) // nw
    flat = dy.reshape(nw, rows, D)
    g2, ok2 = safe.reshape(nw, rows, D), ok.reshape(nw, rows, D)
    ends = ok2[:, 0] & ok2[:, -1]
    flat[:, 0] = np.where(ends, 1.0 / g2[:, 0], 0.0)                       # +1 at the first row
    flat[:, -1] = np.where(ends, -1.0 / g2[:, -1], 0.0)                    # about -1 at the last
    return flat.reshape(B, T, D).astype(np.float32)


# ---- the cases of the GPU tests -----------------------------------------------------------------------------------
# spectrogram loss: (id, B, T, D, r, lengths kind, t_log, w, bw, pbin, pw)
SPEC_SHAPES = [
    ("mel", 16, 203, 80, 1, "ragged", None, 0.5, 0.1, 70, 0.5),          # loops the 1056-block grid
    ("linear", 16, 812, 513, 1, "ragged", None, 0.5, 0.1, 139, 0.5),
    ("linear1025", 2, 97, 1025, 1, "full", None, 0.5, 0.1, 0, 0.0),
    ("one", 1, 2, 1, 1, "full", None, 0.5, 0.1, 0, 0.0),
    ("r4_T9", 3, 9, 37, 4, "ragged", None, 0.5, 1.0, 0, 0.0),
    ("odd", 3, 37, 83, 1, "ragged", None, 1.0, 0.5, 1, 1.0),             # B T D = 9213, not a multiple of 256
    ("all_masked", 4, 29, 80, 2, "all_masked", None, 0.5, 0.1, 0, 0.0),  # Sm = 0
    ("all_masked_w1", 4, 29, 80, 2, "all_masked", None, 1.0, 0.1, 0, 0.0),
]
# t_log of a (5, 61, 80), r = 2 batch: None, T, < T, r + 1, > T, <= r (clamped to r + 1)
SPEC_TLOG = [None, 61, 40, 3, 75, 1]
SETTING_SHAPE = (3, 41, 80, 1)
SETTINGS = [(w, bw, pbin, pw) for w in (0.0, 0.5, 1.0) for bw in (0.0, 0.1, 1.0) for pbin in (0, 1, 70, 80)
            for pw in (0.0, 0.5, 1.0)]

# auxiliary loss: (id, A, B, Td, Ts, ext, use_attn)
AUX_CASES = [("full", 3, 5, 41, 23, None, 1), ("ext", 3, 5, 41, 23, (37, 19), 1),
             ("ext_past_Td", 2, 4, 33, 17, (50, 1), 1), ("no_attn", 3, 5, 41, 23, None, 0)]
AUX_SIGMA = 0.2


def aux_inputs(A, B, Td, Ts, seed):
    """done_hat with 0, 1 and 1 - 2^-24 planted (and 1e-13: the clamp branch away from the ends), done in {0, 1},
    softmax attention rows with exact zeros, in_len / dec_len with a dec_len = 0 row."""
    rng = np.random.RandomState(seed)
    dh = rng.uniform(0.01, 0.99, (B, Td)).astype(np.float32)
    sel = rng.randint(0, 8, (B, Td))
    for k, val in enumerate((0.0, 1.0, 1 - 2.0 ** -24, 1e-13)):
        dh[sel == k] = val
    done = (rng.uniform(0, 1, (B, Td)) > 0.6).astype(np.float32)
    s = rng.randn(A, B, Td, Ts) * 3
    s[rng.uniform(0, 1, s.shape) < 0.2] = -np.inf
    s[..., 0] = np.maximum(s[..., 0], 0.0)
    e = np.exp(s - s.max(-1, keepdims=True))
    attn = (e / e.sum(-1, keepdims=True)).astype(np.float32)
    in_len = rng.randint(3, Ts + 1, B).astype(np.int64)
    dec_len = rng.randint(3, Td + 1, B).astype(np.int64)
    in_len[0], dec_len[0] = Ts, Td
    dec_len[-1] = 0
    return dh, done, attn, in_len, dec_len


# optimizer: n of the size sweep; the grid cap of dv3_sumsq is 1056 blocks x 256 threads x 4 = 1 081 344 elements
OPT_SIZES = [1, 3, 4, 5, 1023, 1081343, 1081345]
ARENA_PRESET = "deepvoice3_ljspeech"
OPT_BETAS, OPT_EPS, OPT_LR = (0.5, 0.9), 1e-6, 5e-4
# (id, gradient scale, max_norm): clip active, inactive, off, and active at a norm where its +1e-6 matters
CLIPS = [("active", 1.0, 0.1), ("inactive", 1.0, 1e9), ("off", 1.0, 0.0), ("active_small", 1e-6, 1e-6)]
OPT_SETTINGS = [(c, gs, wd, ams) for c in CLIPS for gs in (1.0, 0.5, 0.125) for wd in (0.0, 1e-6, 1e-2)
                for ams in (False, True)]


def hyper_for(t, lr=OPT_LR, gs=1.0, betas=OPT_BETAS):
    """FlatAdam.set_hyper's four floats at step t."""
    return np.array([lr, 1 - betas[0] ** t, 1 - betas[1] ** t, gs], np.float32)


# sinusoid: (max_positions, width, rates) of the presets' position tables; rates 1.0 / 1.29 / 1.385 are the query and
# key position rates of the presets and builders
SIN_TABLES = [(512, 256), (512, 128), (1024, 256)]
SIN_RATES = (1.0, 1.29, 1.385)
