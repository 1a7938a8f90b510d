"""GPU: the decoder step kernels of csrc/incremental.cu, called through the C ABI, against fp64 references computed with
plain torch ops -- the precision contract of the step (DESIGN.md section 6).

Error model (u = 2^-24; every bound is elementwise, first order, computed from the same fp64 contractions on absolute
values):
  * Conv step.  An output is one lane-wise fmaf chain of n = k 4 ceil(Cin/128) terms (vec4) or k ceil(Cin/32) terms
    (scalar), a 5-level warp_sum and the bias: |a - a_exact| <= (n + 7) u (|W|.|X| + |bias|), where |X| = |x| + |add|,
    plus one rounding u |W|.|X| for x + add (the ring holds that fp32 sum).  The bound is carried to first order
    through sigmoidf_ (expf <= 2 ulp, then an add and a divide: s (1 - s) da + 6 u s), the GLU / highway products,
    the speaker add and each (y + res) sqrt(1/2) (the sum, the fp32 constant and the product round once each).
    y2 is checked against the kernel's own y (sigmoid within 6 u s; y + yadd and the plain copy bit for bit), so the
    bounds do not compound.
  * Attention step.  Scores: a sequential fmaf chain over E, (E + 1) u |q|.|K|.  Softmax: the error terms of
    tests/test_gpu_attention.ref_forward with that chain bound in place of c_gemm.  Context: a sequential chain over
    Ts with the kernel's probabilities, (Ts + 1) u |P|.|V|, plus the probability errors and 2^-22 |ctx| for the
    scale and the product.
Guards: a conv reference that reads one tap's history one step stale, and a slot reference that runs every row at
row 0's step, each miss the bound by at least 10x -- the bound tells a wrong ring slot or a wrong row step from rounding.
Besides values: strided, padded layouts inside sentinel-filled buffers (inputs padded with NaN, so a stray read
poisons the result; outputs with a sentinel, so a stray write is seen after every step), the ring contents, the cursor
slots, the alignment row and its zero tail, and bit-exact checks of the context scale and of the control kernels.
Every test prints its largest error/bound ratio (run with -s); all must be <= 1.
"""
import ctypes
import math
import random

import numpy as np
import pytest
import torch

from test_gpu_tc1 import _call, _p, _st, ratio

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SQH = math.sqrt(0.5)
NAN = float("nan")
SENT = -1234.5          # output sentinel
SENT_I = -7             # cursor sentinel
MAX_E_TS = 48 * 1024 // 4 - 9      # the attention step's shared memory: 9 floats of scratch, q and the scores


# ---- fp64 references (device-agnostic: tests/test_inc_kernels_host.py runs them on the CPU) -------------------------
def chain_len(k, Cin, vec4):
    """fmaf terms per lane of one conv-step output."""
    return k * 4 * -(-Cin // 128) if vec4 else k * -(-Cin // 32)


def taps(X, W, k, d, stale=None):
    """X (B, T, Cin), W (Cout, k, Cin) -> (B, T, Cout): sum_j X[:, t - (k-1-j) d] . W[:, j], zero before t = 0.
    stale = j reads tap j one step older (the guard)."""
    B, T, _ = X.shape
    out = X.new_zeros(B, T, W.shape[0])
    for j in range(k):
        back = (k - 1 - j) * d + (1 if j == stale else 0)
        if back < T:
            out[:, back:] += X[:, :T - back] @ W[:, j].T
    return out


def ref_conv_step(x, W, bias, k, d, mode=0, act=0, add=None, spk=None, res1=None, res2=None, vec4=True, stale=None):
    """The output of every step t of a conv step program in fp64, with its bound: x, add (B, T, Cin) the inputs of
    steps 0..T-1, W (Cout, k, Cin), bias (Cout,), spk (B, C), res1 / res2 (B, T, C) -> y, by (B, T, C)."""
    Cin = W.shape[2]
    n = chain_len(k, Cin, vec4)
    X, Xa = x.double(), x.double().abs()
    if add is not None:
        X, Xa = X + add.double(), Xa + add.double().abs()
    Wd, bd = W.double(), bias.double()
    pre = taps(X, Wd, k, d, stale) + bd
    bpre = (n + 8) * U * (taps(Xa, Wd.abs(), k, d) + bd.abs())
    if mode == 0:
        y, by = pre, bpre
        if act == 1:
            y = y.clamp_min(0)
        elif act == 2:
            y = torch.sigmoid(pre)
            by = y * (1 - y) * bpre + 6 * U * y
    else:
        C = W.shape[0] // 2
        a, ba = pre[..., :C], bpre[..., :C]
        s = torch.sigmoid(pre[..., C:])
        bs = s * (1 - s) * bpre[..., C:] + 6 * U * s
        if mode == 1:
            if spk is not None:
                a = a + spk.double()[:, None]
                ba = ba + U * a.abs()
            y = a * s
            by = s * ba + a.abs() * bs + U * y.abs()
        else:
            xin = x.double()[..., :C]                   # gated blocks: Cin == C, the input without add
            y = s * a + (1 - s) * xin
            by = s * ba + (a - xin).abs() * bs + 4 * U * ((s * a).abs() + ((1 - s) * xin).abs())
    for r in (res1, res2):
        if r is not None:
            z = y + r.double()
            by = (by + U * z.abs()) * SQH + 2 * U * SQH * z.abs()
            y = z * SQH
    return y, by


def window(la, wb, wa, n):
    """unmasked keys [lo, hi) of a row with n keys and cursor la (reference deepvoice3.py:150-156)."""
    lo = la - wb if la - wb > 0 else 0
    hi = la + wa if la + wa < n else n
    return lo, hi


def ref_attn_step(q, K, V, lens, lo, hi):
    """fp64 attention step: q (B, E), K (B, E, Ts), V (B, Ts, E); row b attends to keys s < lens[b] in [lo[b], hi[b])
    -> P (B, Ts), bP, ctx (B, E) = P.V * lens Ts*sqrt(1/Ts), bctx."""
    B, E, Ts = K.shape
    dev = K.device
    n = torch.as_tensor(lens, dtype=torch.float64, device=dev)[:, None]
    s = torch.arange(Ts, device=dev)[None]
    lo_, hi_ = (torch.as_tensor(v, device=dev)[:, None] for v in (lo, hi))
    keep = (s < n) & (s >= lo_) & (s < hi_)
    Kd = torch.where((s < n)[:, None, :], K.double(), 0.0)
    Vd = torch.where((s < n)[:, :, None], V.double(), 0.0)
    qd = q.double()
    S = torch.einsum("be,bes->bs", qd, Kd).masked_fill(~keep, -math.inf)
    bS = ((E + 1) * U * torch.einsum("be,bes->bs", qd.abs(), Kd.abs())).masked_fill(~keep, 0.0)
    P = torch.softmax(S, dim=-1)
    mx = S.max(dim=-1, keepdim=True).values
    e = (2 * 2.0 ** -23 + U * (S - mx).abs()).masked_fill(~keep, 0.0)
    rel = bS + (P * bS).sum(-1, keepdim=True) + e + (P * e).sum(-1, keepdim=True) + (n + 2) * U
    bP = P * rel * (1 + bS.max(dim=-1, keepdim=True).values)
    sc = n * torch.sqrt(1.0 / n)
    ctx = sc * torch.einsum("bs,bse->be", P, Vd)
    bctx = sc * (torch.einsum("bs,bse->be", bP, Vd.abs()) + (n + 1) * U * torch.einsum("bs,bse->be", P, Vd.abs())) \
        + 2.0 ** -22 * ctx.abs()
    return P, bP, ctx, bctx


def stop_rule(done, t, stop, min_steps, max_steps):
    """dv3_inc_stop_rows restated per row: done[b][t[b]] of step t[b], n = t[b] + 1 steps ran -> new stop values."""
    out = list(stop)
    for b in range(len(t)):
        if out[b] != 0:
            continue
        n = t[b] + 1
        if (done[b][t[b]] > 0.5 and n > min_steps) or n > max_steps:
            out[b] = n
    return out


def context_scale(n):
    """the reference's context scale, deepvoice3.py:170-171: a double scalar applied to an fp32 tensor."""
    return np.float32(n * math.sqrt(1.0 / n))


# ---- cases ----------------------------------------------------------------------------------------------------------
# (B, Cin, Cout, k, dilation, mode, act, vec4, options); gated modes have Cout = 2 Cin.  options: add, spk, res1, res2,
# y2 (plain copy), y2s (y2_mode 1), y2a (y2_mode 2), shift (the rows start one float off 16-byte alignment)
CONV_CASES = [
    (1, 16, 24, 1, 1, 0, 0, 1, ()),
    (2, 256, 80, 3, 27, 0, 2, 1, ("add",)),
    (3, 81, 40, 5, 1, 0, 1, 0, ()),
    (4, 200, 64, 2, 9, 0, 0, 1, ("add", "y2s")),
    (5, 81, 162, 3, 3, 1, 0, 0, ("spk", "res1")),
    (9, 512, 1024, 5, 9, 1, 0, 1, ("res1", "res2", "y2a")),
    (2, 128, 256, 3, 1, 2, 0, 0, ("shift",)),
    (1, 64, 128, 2, 1, 1, 0, 1, ("res1", "y2")),
    (3, 256, 512, 3, 27, 2, 0, 1, ()),
    (9, 16, 1, 1, 1, 0, 2, 1, ()),
]

# (B, Cin, Cout, k, dilation, mode, vec4): GLU slots carry a speaker addend and a residual
SLOT_CASES = [
    (1, 16, 16, 3, 1, 0, 1),
    (2, 81, 40, 2, 3, 0, 0),
    (5, 64, 128, 3, 4, 1, 1),
    (9, 128, 256, 5, 2, 2, 1),
]

# (variant, B, E, Ts, text_len or None, window (backward, ahead) or None, cursor(s) read, step(s), align_scale or None)
ATTN_CASES = [
    ("plain", 3, 16, 1, None, None, None, 0, 1.0),
    ("plain", 2, 128, 257, None, (1, 3), 100, 5, 2.0),
    ("plain", 3, 300, 600, None, (40, 200), 0, 2, 1.0),
    ("plain", 2, 256, 255, None, (1, 3), 254, 7, 1.0),
    ("plain", 2, 256, 31, None, None, None, 3, None),
    ("plain", 1, MAX_E_TS - 600, 600, None, (1, 3), 300, 1, 1.0),            # 48 KB of shared memory exactly
    ("rows", 5, 256, 256, [256, 1, 31, 200, 2], (1, 3), [0, 0, 30, 199, 1], 4, 1.0),
    ("rows", 4, 16, 31, [31, 1, 2, 17], None, None, 1, 2.0),
    ("rows", 3, 128, 600, [600, 257, 255], (100, 300), [599, 10, 128], 6, 1.0),
    ("rows", 2, 256, MAX_E_TS - 256, [MAX_E_TS - 256, 5000], (2000, 8000), [6000, 4999], 0, 1.0),
    ("slots", 6, 300, 257, [257, 1, 256, 31, 2, 100], (1, 3), [5, 0, 255, 30, 1, 50], [0, 1, 2, 3, 10, 11], 1.0),
    ("slots", 3, 16, 2, [2, 1, 2], None, None, [4, 7, 0], 2.0),
]


def conv_id(c):
    return "B%d_Cin%d_Cout%d_k%d_d%d_m%d_a%d_v%d%s" % (c[:8] + ("".join("_" + o for o in c[8]),))


def attn_id(c):
    return "%s_B%d_E%d_Ts%d%s" % (c[0], c[1], c[2], c[3], "_win%d-%d" % c[5] if c[5] else "")


# ---- device helpers -------------------------------------------------------------------------------------------------
class Rows:
    """(B, T, C) rows inside a flat fill-valued fp32 buffer: row (b, t) starts at off + b*ld + t*ts, with ts > C and
    ld > T*ts (padding between rows and between steps), 16-byte aligned unless align is False or shift is set.
    operand: a number per operand of one launch, which widens ts, ld and off by 4 floats each, so that operands of the
    same width never share a stride or an offset (a kernel that indexes one operand with another's strides fails)."""

    def __init__(self, B, T, C, fill=NAN, align=True, shift=0, operand=0):
        ts, off = C + 3, 1
        if align:
            ts, off = -(-ts // 4) * 4, 4
        ts, off = ts + 4 * operand, off + 4 * operand
        ld = T * ts + (8 if align else 5) + 4 * operand
        assert ts > C and ld > T * ts
        self.ts, self.ld, self.off = ts, ld, off + shift
        self.buf = torch.full((self.off + B * ld + 8,), fill, device="cuda")
        ar = lambda n: torch.arange(n, device="cuda")          # noqa: E731
        self.idx = self.off + ar(B)[:, None, None] * ld + ar(T)[None, :, None] * ts + ar(C)
        assert self.off + (B - 1) * ld + (T - 1) * ts + C <= self.buf.numel()

    @property
    def ptr(self):
        return self.buf.data_ptr() + 4 * self.off

    def get(self):
        return self.buf[self.idx]

    def put(self, v):
        self.buf[self.idx] = v.to(self.buf.dtype)


def _distinct(*rows):
    """no two operands of a launch share a row stride, a step stride or a start offset"""
    rows = [r for r in rows if r is not None]
    for attr in ("ld", "ts", "off"):
        vals = [getattr(r, attr) for r in rows]
        assert len(set(vals)) == len(vals), (attr, vals)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _lib_error():
    from deepvoice3_pytorch_b200._lib import Dv3Error
    return Dv3Error


def _step_struct(x, W, bias, B, k, d, mode, act, vec4, add=None, ring=None, spk=None, res1=None, res2=None, y=None,
                 y2=None, y2_mode=0, yadd=None, t_ptr=None):
    from deepvoice3_pytorch_b200.incremental import Dv3IncStep
    s = Dv3IncStep()
    s.x, s.x_ld, s.x_t = x.ptr, x.ld, x.ts
    if add is not None:
        s.add, s.add_ld, s.add_t = add.ptr, add.ld, add.ts
    if ring is not None:
        s.ring = ring.data_ptr()
    s.w, s.bias = W.data_ptr(), bias.data_ptr()
    if spk is not None:
        s.spk, s.spk_ld = spk.ptr, spk.ld
    if res1 is not None:
        s.res1, s.res1_ld, s.res1_t = res1.ptr, res1.ld, res1.ts
    if res2 is not None:
        s.res2, s.res2_ld, s.res2_t = res2.ptr, res2.ld, res2.ts
    s.y, s.y_ld, s.y_t = y.ptr, y.ld, y.ts
    if y2 is not None:
        s.y2, s.y2_ld, s.y2_t, s.y2_mode = y2.ptr, y2.ld, y2.ts, y2_mode
    if yadd is not None:
        s.yadd, s.yadd_ld, s.yadd_t = yadd.ptr, yadd.ld, yadd.ts
    s.t_ptr = t_ptr.data_ptr()
    s.B, s.Cin, s.Cout, s.k, s.dilation, s.mode, s.act, s.vec4 = B, W.shape[2], W.shape[0], k, d, mode, act, vec4
    return s


def _ring_expect(Xf, tt, L):
    """ring (B, L, Cin) after row b computed step tt[b]: slot s holds the input of the latest step t' <= tt[b] with
    t' = s mod L, or zeros."""
    B = Xf.shape[0]
    s = torch.arange(L, device=Xf.device)[None]
    tt = torch.as_tensor(tt, device=Xf.device)[:, None]
    src = tt - torch.remainder(tt - s, L)
    rows = torch.arange(B, device=Xf.device)[:, None]
    got = Xf[rows, src.clamp_min(0)]
    return torch.where((src >= 0)[..., None], got, torch.zeros_like(got))


# ---- conv step ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CONV_CASES, ids=conv_id)
def test_conv_step_vs_fp64(case):
    B, Cin, Cout, k, d, mode, act, vec4, opts = case
    C = Cout // 2 if mode else Cout
    L = (k - 1) * d + 1
    T = 2 * L + 3 if k > 1 else 6
    g = torch.Generator(device="cuda").manual_seed(sum(case[:8]))
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)     # noqa: E731
    shift = int("shift" in opts)
    x = Rows(B, T, Cin, align=bool(vec4) or shift, shift=shift)
    x.put(rn(B, T, Cin))
    opt = {}
    for i, (name, shape, sc) in enumerate((("add", (B, T, Cin), 1.0), ("spk", (B, 1, C), 0.3),
                                           ("res1", (B, T, C), 1.0), ("res2", (B, T, C), 1.0))):
        if name in opts:
            opt[name] = Rows(*shape, align=bool(vec4), operand=1 + i)
            opt[name].put(sc * rn(*shape))
    W = (rn(Cout, k, Cin) * (k * Cin) ** -0.5).contiguous()
    bias = 0.1 * rn(Cout)
    y = Rows(B, T, C, fill=SENT, operand=5)
    y2 = Rows(B, T, C, fill=SENT, operand=6) if {"y2", "y2s", "y2a"} & set(opts) else None
    y2_mode = 1 if "y2s" in opts else 2 if "y2a" in opts else 0
    yadd = None
    if y2_mode == 2:
        yadd = Rows(B, T, C, operand=7)
        yadd.put(rn(B, T, C))
    _distinct(x, y, y2, yadd, *opt.values())
    ring = torch.zeros(B, L, Cin, device="cuda") if k > 1 else None
    tc = torch.zeros(1, dtype=torch.int32, device="cuda")
    s = _step_struct(x, W, bias, B, k, d, mode, act, vec4, add=opt.get("add"), ring=ring, spk=opt.get("spk"),
                     res1=opt.get("res1"), res2=opt.get("res2"), y=y, y2=y2, y2_mode=y2_mode, yadd=yadd, t_ptr=tc)
    xs = x.get()
    Xf = xs + opt["add"].get() if "add" in opts else xs               # what the kernel files into the ring
    snap = y.buf.clone()
    snap2 = y2.buf.clone() if y2 is not None else None
    for t in range(T):
        _call("dv3_inc_conv_step", ctypes.byref(s), _st())
        _call("dv3_inc_advance", _p(tc), _st())
        cur = y.idx[:, t]
        snap[cur] = y.buf[cur]
        assert _same(y.buf, snap), "step %d: y written outside (b, %d, c < C)" % (t, t)
        if y2 is not None:
            cur2 = y2.idx[:, t]
            snap2[cur2] = y2.buf[cur2]
            assert _same(y2.buf, snap2), "step %d: y2 written outside (b, %d, c < C)" % (t, t)
        if ring is not None:
            assert _same(ring, _ring_expect(Xf, [t] * B, L)), "step %d: ring is not the last L inputs" % t
    assert int(tc) == T
    sp = opt["spk"].get()[:, 0] if "spk" in opts else None
    refs = dict(add=opt["add"].get() if "add" in opts else None, spk=sp,
                res1=opt["res1"].get() if "res1" in opts else None, res2=opt["res2"].get() if "res2" in opts else None)
    want, bound = ref_conv_step(xs, W, bias, k, d, mode, act, vec4=bool(vec4), **refs)
    got = y.get()
    r = ratio(got, want, bound)
    msg = "conv %s: error/bound %.3g" % (conv_id(case), r)
    guard = None
    if k > 1:
        stale, _ = ref_conv_step(xs, W, bias, k, d, mode, act, vec4=bool(vec4), stale=0, **refs)
        guard = ratio(got[:, L - 1:], stale[:, L - 1:], bound[:, L - 1:])
        msg += ", stale-tap guard %.3g" % guard
    if y2 is not None:
        g2 = y2.get()
        if y2_mode == 1:
            sg = torch.sigmoid(got.double())
            r2 = ratio(g2, sg, 6 * U * sg + 1e-38)
            msg += ", y2 = sigmoid(y) %.3g" % r2
            assert r2 <= 1, msg
        elif y2_mode == 2:
            assert _same(g2, got + yadd.get()), "y2 != fp32(y + yadd)"
        else:
            assert _same(g2, got), "y2 != y"
    print(msg)
    assert r <= 1, msg
    assert guard is None or guard >= 10, msg


@pytest.mark.parametrize("case", SLOT_CASES, ids=lambda c: "B%d_Cin%d_Cout%d_k%d_d%d_m%d_v%d" % c)
def test_conv_step_slots_vs_fp64(case):
    """Rows at their own steps: staggered starts, random holds (stop != 0: the row recomputes its step and keeps its
    counter) and refills (dv3_inc_refill zeroes the row's ring and counter; the row starts a new input sequence).
    Every row's output is the fp64 reference of its own sequence at its own step."""
    B, Cin, Cout, k, d, mode, vec4 = case
    C = Cout // 2 if mode else Cout
    L = (k - 1) * d + 1
    R = 3 * L + 12                                       # rounds; no row runs more steps than that
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Cin)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)     # noqa: E731
    rnd = random.Random(B + Cin)
    x = Rows(B, R, Cin, align=bool(vec4))
    W = (rn(Cout, k, Cin) * (k * Cin) ** -0.5).contiguous()
    bias = 0.1 * rn(Cout)
    spk = res1 = None
    if mode == 1:
        spk, res1 = Rows(B, 1, C, operand=1), Rows(B, R, C, operand=2)
        spk.put(0.3 * rn(B, 1, C))
    y = Rows(B, R, C, fill=SENT, operand=3)
    _distinct(x, spk, res1, y)
    ring = torch.zeros(B, L, Cin, device="cuda")
    t = torch.zeros(B, dtype=torch.int32, device="cuda")
    stop = torch.zeros(B, dtype=torch.int32, device="cuda")
    s = _step_struct(x, W, bias, B, k, d, mode, 0, vec4, ring=ring, spk=spk, res1=res1, y=y, t_ptr=t)
    want = torch.zeros(B, R, C, dtype=torch.float64, device="cuda")
    bound = torch.zeros_like(want)

    def new_sequence(rows):
        for b in rows:
            xb = rn(1, R, Cin)
            x.buf[x.idx[b]] = xb[0]
            kw = {}
            if mode == 1:
                rb = rn(1, R, C)
                res1.buf[res1.idx[b]] = rb[0]
                kw = dict(spk=spk.get()[b:b + 1, 0], res1=rb)
            want[b], bound[b] = (v[0] for v in ref_conv_step(xb, W, bias, k, d, mode, vec4=bool(vec4), **kw))

    from deepvoice3_pytorch_b200.incremental import Dv3IncRefill
    table = (Dv3IncRefill * 2)()
    table[0].dst, table[0].row_bytes, table[0].dst_row_stride = ring.data_ptr(), L * Cin * 4, L * Cin * 4
    table[1].dst, table[1].row_bytes, table[1].dst_row_stride = t.data_ptr(), 4, 4
    table_dev = torch.frombuffer(bytearray(table), dtype=torch.uint8).cuda()
    refill_at = {L + 2: [B - 1, 0][:B], 2 * L + 5: [1, B - 2][:max(1, B - 1)] if B > 2 else [0]}

    new_sequence(range(B))
    th = [0] * B
    prev, prev_t = None, None
    worst, guard, moved = 0.0, math.inf, 0
    rows = torch.arange(B, device="cuda")
    for r in range(R):
        held = [1 if r < b or rnd.random() < 0.25 else 0 for b in range(B)]
        stop.copy_(torch.tensor(held, dtype=torch.int32))
        snap = y.buf.clone()
        _call("dv3_inc_conv_step_slots", ctypes.byref(s), _st())
        tt = torch.tensor(th, device="cuda")
        cur = y.idx[rows, tt]
        snap[cur] = y.buf[cur]
        assert _same(y.buf, snap), "round %d: y written outside each row's (b, t[b], c < C)" % r
        got = y.buf[cur]
        assert _same(ring, _ring_expect(x.get(), th, L)), "round %d: a ring row is not its last L inputs" % r
        if prev is not None:
            same = [b for b in range(B) if th[b] == prev_t[b]]
            assert _same(got[same], prev[same]), "round %d: a held row did not rewrite the same bits" % r
        worst = max(worst, ratio(got, want[rows, tt], bound[rows, tt]))
        other = [b for b in range(B) if th[b] != th[0]]
        if other:
            t0 = torch.full((len(other),), th[0], device="cuda")
            o = torch.tensor(other, device="cuda")
            guard = min(guard, ratio(got[o], want[o, t0], bound[o, t0]))
            moved += 1
        prev, prev_t = got.clone(), list(th)
        _call("dv3_inc_advance_rows", _p(t), _p(stop), B, _st())
        th = [v + (1 - h) for v, h in zip(th, held)]
        assert t.tolist() == th, "round %d: counters %s, expected %s" % (r, t.tolist(), th)
        if r in refill_at:
            lst = refill_at[r]
            slots = torch.tensor(lst, dtype=torch.int32, device="cuda")
            _call("dv3_inc_refill", _p(table_dev), 2, _p(slots), len(lst), _st())
            new_sequence(lst)
            for b in lst:
                th[b] = 0
                prev_t[b] = -1
            assert t.tolist() == th and not bool(ring[lst].any()), "refill did not zero the counter and ring row"
    print("conv slots %s: error/bound %.3g, row-0-step guard %.3g (%d rounds with rows apart)"
          % (case, worst, guard, moved))
    assert worst <= 1
    assert B == 1 or (moved > 0 and guard >= 10), guard                # one row: nothing to confuse


# ---- attention step -------------------------------------------------------------------------------------------------
def _attn_buffers(variant, B, E, Ts, lens, window_, cursors, steps, align_scale, seed):
    from deepvoice3_pytorch_b200.incremental import Dv3IncAttn
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = 1.2 * E ** -0.25
    q = Rows(B, 1, E, align=False)
    q.put(sd * torch.randn(B, 1, E, device="cuda", generator=g))
    K = sd * torch.randn(B, E, Ts, device="cuda", generator=g)
    V = torch.randn(B, Ts, E, device="cuda", generator=g)
    n = lens if lens is not None else [Ts] * B
    for b in range(B):                    # past a row's text: NaN (never read)
        K[b, :, n[b]:] = NAN
        V[b, n[b]:] = NAN
        if variant == "slots" and n[b] == 1:      # an idle slot attends one zero key
            K[b, :, 0] = 0.0
            V[b, 0] = 0.0
    ts = list(steps) if isinstance(steps, (list, tuple)) else [steps] * B
    ctx = Rows(B, 1, E, fill=SENT, align=False, operand=1)
    align = Rows(B, max(ts) + 2, Ts, fill=SENT, align=False, operand=2) if align_scale else None
    _distinct(q, ctx)
    per_row = variant != "plain"
    la = torch.full((2 * B if per_row else 2,), SENT_I, dtype=torch.int32, device="cuda")
    if window_ is not None:
        for b in range(B if per_row else 1):
            la[(ts[b] & 1) * B + b if per_row else ts[0] & 1] = cursors[b] if per_row else cursors
    tc = torch.tensor(ts if variant == "slots" else ts[:1], dtype=torch.int32, device="cuda")
    text_len = torch.tensor(n, dtype=torch.int32, device="cuda")
    a = Dv3IncAttn()
    a.q, a.q_ld = q.ptr, q.ld
    a.keys, a.values = K.data_ptr(), V.data_ptr()
    a.ctx, a.ctx_ld = ctx.ptr, ctx.ld
    if align is not None:
        a.align, a.align_ld, a.align_t, a.align_scale = align.ptr, align.ld, align.ts, align_scale
    if window_ is not None:
        a.last_attended = la.data_ptr()
        a.window_backward, a.window_ahead = window_
    a.t_ptr = tc.data_ptr()
    a.B, a.E, a.Ts = B, E, Ts
    return dict(a=a, q=q, K=K, V=V, ctx=ctx, align=align, la=la, tc=tc, text_len=text_len, n=n, ts=ts)


def _attn_launch(variant, bufs):
    name = {"plain": "dv3_inc_attn_step", "rows": "dv3_inc_attn_step_rows", "slots": "dv3_inc_attn_step_slots"}
    extra = () if variant == "plain" else (_p(bufs["text_len"]),)
    _call(name[variant], ctypes.byref(bufs["a"]), *extra, _st())


@pytest.mark.parametrize("case", ATTN_CASES, ids=attn_id)
def test_attn_step_vs_fp64(case):
    variant, B, E, Ts, lens, win, cursors, steps, align_scale = case
    # the cursor is the first argmax of the kernel's probabilities, read back exactly from the alignment row
    assert win is None or align_scale, "a windowed case needs an alignment row to check the cursor against"
    assert align_scale is None or math.frexp(align_scale)[0] == 0.5, "align_scale must be a power of two"
    bf = _attn_buffers(*case, seed=B * 7 + E + Ts)
    ctx, align, la = bf["ctx"], bf["align"], bf["la"]
    ctx0, al0, la0 = ctx.buf.clone(), align.buf.clone() if align else None, la.clone()
    _attn_launch(variant, bf)
    torch.cuda.synchronize()
    n, ts, per_row = bf["n"], bf["ts"], variant != "plain"
    lo, hi = [0] * B, list(n)
    if win is not None:
        for b in range(B):
            lo[b], hi[b] = window(cursors[b] if per_row else cursors, win[0], win[1], n[b])
    P, bP, want, bctx = ref_attn_step(bf["q"].get()[:, 0], bf["K"], bf["V"], n, lo, hi)
    rows = torch.arange(B, device="cuda")
    Pk = None                                          # the kernel's probabilities (B, Ts)
    ctx0[ctx.idx[:, 0]] = ctx.buf[ctx.idx[:, 0]]
    assert _same(ctx.buf, ctx0), "ctx written outside (b, e < E)"
    rc = ratio(ctx.get()[:, 0], want, bctx)
    msg = "attn %s: ctx error/bound %.3g" % (attn_id(case), rc)
    if align is not None:
        cur = align.idx[rows, torch.tensor(ts, device="cuda")]                 # (B, Ts)
        al0[cur] = align.buf[cur]
        assert _same(align.buf, al0), "alignment written outside (b, t[b], s < Ts)"
        Pk = align.buf[cur] / align_scale                                      # a power of two: exact
        valid = torch.arange(Ts, device="cuda")[None] < torch.tensor(n, device="cuda")[:, None]
        assert bool((Pk[~valid] == 0).all()), "alignment columns [text_len, Ts) are not zero"
        rp = ratio(torch.where(valid, Pk, 0.0), P, bP)
        msg += ", probs %.3g" % rp
        assert rp <= 1, msg
    if win is not None:
        Pc = Pk.cpu()
        for b in range(B if per_row else 1):
            rd = (ts[b] & 1) * B + b if per_row else ts[0] & 1
            wr = ((ts[b] + 1) & 1) * B + b if per_row else (ts[0] + 1) & 1
            la0[wr] = int(torch.argmax(Pc[b, :n[b]]))
            assert int(la[rd]) == (cursors[b] if per_row else cursors), "the read cursor slot changed"
        assert torch.equal(la, la0), "cursors %s, expected %s" % (la.tolist(), la0.tolist())
    else:
        assert torch.equal(la, la0)
    print(msg)
    assert rc <= 1, msg


def test_attn_step_context_scale_bit_exact():
    """A one-key window (backward 0, ahead 1, cursor at text_len[b] - 1) makes the probability exactly 1, so row b's
    context is fp32(V[b, text_len[b] - 1] * float(Ts*sqrt(1/Ts))) with Ts = text_len[b] = b + 1, for b < 1024."""
    B, E, Ts = 1024, 16, 1024
    lens = list(range(1, B + 1))
    bf = _attn_buffers("rows", B, E, Ts, lens, (0, 1), [n - 1 for n in lens], 0, None, seed=5)
    _attn_launch("rows", bf)
    torch.cuda.synchronize()
    sc = torch.tensor([context_scale(n) for n in lens], device="cuda")
    want = bf["V"][torch.arange(B, device="cuda"), torch.tensor(lens, device="cuda") - 1] * sc[:, None]
    got = bf["ctx"].get()[:, 0]
    bad = (_bits(got) != _bits(want)).any(1).nonzero().flatten().tolist()
    print("context scale: %d of %d text lengths differ from float(Ts*sqrt(1/Ts)) %s" % (len(bad), B, bad[:8]))
    assert not bad
    assert bf["la"][B:].tolist() == [n - 1 for n in lens]


def test_attn_step_refuses_more_than_48kb():
    """E + Ts one float past the limit: every variant refuses before launching; no output changes."""
    B, E, Ts = 2, MAX_E_TS + 1 - 12000, 12000
    for variant in ("plain", "rows", "slots"):
        bf = _attn_buffers(variant, B, E, Ts, [Ts, 7] if variant != "plain" else None, (1, 3), [3, 2] if
                           variant != "plain" else 3, [1, 2] if variant == "slots" else 1, 1.0, seed=9)
        c0, a0, l0 = bf["ctx"].buf.clone(), bf["align"].buf.clone(), bf["la"].clone()
        with pytest.raises(_lib_error(), match="exceed the %d that fit in 48 KB" % MAX_E_TS):
            _attn_launch(variant, bf)
        torch.cuda.synchronize()
        assert _same(bf["ctx"].buf, c0) and _same(bf["align"].buf, a0) and torch.equal(bf["la"], l0)


# ---- control kernels ------------------------------------------------------------------------------------------------
def test_stop_rows_vs_rule():
    B, min_steps, max_steps, ld = 1024, 10, 50, 64
    rnd = random.Random(3)
    half_up = float(np.nextafter(np.float32(0.5), np.float32(1)))
    half_dn = float(np.nextafter(np.float32(0.5), np.float32(0)))
    ns = [min_steps, min_steps + 1, max_steps, max_steps + 1, max_steps + 2, 1, 30]
    dv = [0.5, half_up, half_dn, 0.0, 1.0]
    t = [rnd.choice(ns) - 1 for _ in range(B)]
    stop0 = [rnd.choice([0, 0, 0, -1, 9]) for _ in range(B)]
    done = np.empty((B, ld), dtype=np.float32)
    for b in range(B):
        v = dv[(b + b // 7) % len(dv)]
        done[b] = 0.0 if v > 0.5 else 1.0           # every other column says the opposite
        done[b, t[b]] = v
    want = stop_rule(done.astype(np.float64), t, stop0, min_steps, max_steps)
    assert len(set(want)) > 3 and any(w == 0 for w in want)
    d_dev = torch.from_numpy(done).cuda()
    t_dev = torch.tensor(t, dtype=torch.int32, device="cuda")
    stop = torch.tensor(stop0, dtype=torch.int32, device="cuda")
    _call("dv3_inc_stop_rows", _p(d_dev), ld, _p(t_dev), _p(stop), B, min_steps, max_steps, _st())
    assert stop.tolist() == want
    assert t_dev.tolist() == t
    _call("dv3_inc_stop_rows", _p(d_dev), ld, _p(t_dev), _p(stop), B, min_steps, max_steps, _st())
    assert stop.tolist() == want                     # written once


@pytest.mark.parametrize("B", [3, 1024])
def test_advance_rows_and_advance(B):
    rnd = random.Random(B)
    t0 = [rnd.randrange(0, 500) for _ in range(B)]
    st = [rnd.choice([0, 0, 3, -1]) for _ in range(B)]
    t = torch.tensor(t0, dtype=torch.int32, device="cuda")
    stop = torch.tensor(st, dtype=torch.int32, device="cuda")
    _call("dv3_inc_advance_rows", _p(t), _p(stop), B, _st())
    assert t.tolist() == [v + (s == 0) for v, s in zip(t0, st)] and stop.tolist() == st
    _call("dv3_inc_advance_rows", _p(t), None, B, _st())
    assert t.tolist() == [v + (s == 0) + 1 for v, s in zip(t0, st)]
    c = torch.tensor([41, 99], dtype=torch.int32, device="cuda")
    _call("dv3_inc_advance", _p(c), _st())
    _call("dv3_inc_advance", _p(c), _st())
    assert c.tolist() == [43, 99]


def test_refill():
    """Entries with different row sizes and strides (src stride != dst stride), a zeroing entry, a row longer than the
    16-block grid stride, an unordered non-contiguous slot list; rows not listed and the padding keep their bits."""
    from deepvoice3_pytorch_b200.incremental import Dv3IncRefill
    g = torch.Generator(device="cuda").manual_seed(8)
    S, slots = 6, [4, 1, 3]
    long_w = 16 * 256 * 3 + 7
    # (row words, dst stride words, src stride words or None)
    spec = [(long_w, long_w + 5, long_w + 2), (10, 13, None), (1, 1, 2), (33, 40, 33)]
    rint = lambda n: torch.randint(-2 ** 31, 2 ** 31 - 1, (n,), generator=g, device="cuda", dtype=torch.int32)  # noqa
    dst = [rint(S * ds + 3) for _, ds, _ in spec]
    src = [rint(len(slots) * ss + 3) if ss else None for _, _, ss in spec]
    table = (Dv3IncRefill * len(spec))()
    for e, (w, ds, ss), d, s in zip(table, spec, dst, src):
        e.dst, e.row_bytes, e.dst_row_stride = d.data_ptr(), 4 * w, 4 * ds
        if s is not None:
            e.src, e.src_row_stride = s.data_ptr(), 4 * ss
    table_dev = torch.frombuffer(bytearray(table), dtype=torch.uint8).cuda()
    before = [d.clone() for d in dst]
    sl = torch.tensor(slots, dtype=torch.int32, device="cuda")
    _call("dv3_inc_refill", _p(table_dev), len(spec), _p(sl), 0, _st())
    torch.cuda.synchronize()
    assert all(torch.equal(d, b) for d, b in zip(dst, before)), "n_slots = 0 changed something"
    _call("dv3_inc_refill", _p(table_dev), len(spec), _p(sl), len(slots), _st())
    for (w, ds, ss), d, b, s in zip(spec, dst, before, src):
        want = b.clone()
        for i, row in enumerate(slots):
            want[row * ds:row * ds + w] = s[i * ss:i * ss + w] if s is not None else 0
        assert torch.equal(d, want), "entry (%d words, stride %d): wrong rows" % (w, ds)
