"""CPU checks of the fp64 references and case lists of tests/test_gpu_inc_kernels.py: the conv-step reference against
the oracle's ring-buffer convolution (oracle/dv3_incremental.IncConv and its gate stacks, pinned to the reference's
golden vectors) and against a causal dilated conv1d on whole sequences; the attention-step reference against a dense
masked softmax; the stop-rule restatement against incremental._stop_step; the guards' discrimination on the
references alone; and the case lists reaching every instantiation of the step kernels."""
import math
import random

import numpy as np
import torch
import torch.nn.functional as F

import test_gpu_inc_kernels as K
from oracle import dv3_incremental as OI
from oracle import dv3_oracle as O


def _wn(Cout, Cin, k, g):
    v = torch.randn(Cout, Cin, k, generator=g, dtype=torch.float64)
    return v, torch.rand(Cout, 1, 1, generator=g, dtype=torch.float64) + 0.5


def _sd(prefix, Cout, Cin, k, g):
    v, gg = _wn(Cout, Cin, k, g)
    return {prefix + ".weight_v": v, prefix + ".weight_g": gg,
            prefix + ".bias": 0.1 * torch.randn(Cout, generator=g, dtype=torch.float64)}


def _steps(fn, x):
    return torch.cat([fn(x[:, t:t + 1]) for t in range(x.size(1))], dim=1)


def test_conv_reference_matches_oracle_ring_buffer():
    g = torch.Generator().manual_seed(0)
    B, T = 3, 40
    for Cin, Cout, k, d, act in ((5, 7, 1, 1, 0), (6, 4, 3, 4, 1), (9, 3, 5, 2, 2), (4, 6, 2, 9, 0)):
        sd = _sd("c", Cout, Cin, k, g)
        x = torch.randn(B, T, Cin, generator=g, dtype=torch.float64)
        want = _steps(OI.IncConv(sd, "c", k, d).step, x)
        want = want.clamp_min(0) if act == 1 else torch.sigmoid(want) if act == 2 else want
        W = O._w(sd, "c").permute(0, 2, 1)
        y, by = K.ref_conv_step(x, W, sd["c.bias"], k, d, 0, act)
        torch.testing.assert_close(y, want, rtol=1e-12, atol=1e-12)
        assert bool((by > 0).all())
    # GLU (speaker addend, residual) and highway through the oracle's gate stacks
    C, k, d = 6, 3, 2
    for kind in ("glu", "hw"):
        sd = _sd("s.0.conv", 2 * C, C, k, g)
        spk_embed = torch.randn(B, 5, generator=g, dtype=torch.float64)
        layer = ("glu", 0, C, k, d, True, True) if kind == "glu" else ("hw", 0, C, k, d, True)
        kw = {}
        if kind == "glu":
            sd.update(_sd("s.0.speaker_proj", C, 5, 1, g))
            for n in ("weight_v", "weight_g"):
                sd["s.0.speaker_proj." + n] = sd["s.0.speaker_proj." + n][..., 0]
            soft = F.softsign(O.linear(sd, "s.0.speaker_proj", spk_embed))
            kw = dict(spk=soft)
        x = torch.randn(B, T, C, generator=g, dtype=torch.float64)
        want = _steps(OI.make_stack(sd, "s", [layer], spk_embed if kind == "glu" else None)[0], x)
        W = O._w(sd, "s.0.conv").permute(0, 2, 1)
        if kind == "glu":
            kw["res1"] = x
        y, _ = K.ref_conv_step(x, W, sd["s.0.conv.bias"], k, d, 1 if kind == "glu" else 2, **kw)
        torch.testing.assert_close(y, want, rtol=1e-12, atol=1e-12)


def test_conv_reference_matches_causal_conv1d():
    g = torch.Generator().manual_seed(1)
    for B, Cin, Cout, k, d, T in ((2, 8, 5, 3, 27, 120), (1, 16, 3, 5, 1, 17), (3, 4, 4, 2, 9, 30)):
        x = torch.randn(B, T, Cin, generator=g, dtype=torch.float64)
        add = torch.randn(B, T, Cin, generator=g, dtype=torch.float64)
        W = torch.randn(Cout, k, Cin, generator=g, dtype=torch.float64)
        bias = torch.randn(Cout, generator=g, dtype=torch.float64)
        xin = F.pad((x + add).transpose(1, 2), ((k - 1) * d, 0))
        want = F.conv1d(xin, W.permute(0, 2, 1), bias, dilation=d).transpose(1, 2)
        y, _ = K.ref_conv_step(x, W, bias, k, d, add=add)
        torch.testing.assert_close(y, want, rtol=1e-12, atol=1e-12)
        # the stale-tap guard reference is the same conv with tap 0 one step further back
        W2 = W.clone()
        W2[:, 1:] = 0
        want0 = F.conv1d(F.pad((x + add).transpose(1, 2), ((k - 1) * d + 1, 0))[..., :-1], W2.permute(0, 2, 1),
                         dilation=d).transpose(1, 2)
        st, _ = K.ref_conv_step(x, W, torch.zeros_like(bias), k, d, add=add, stale=0)
        rest, _ = K.ref_conv_step(x, W2 - W, torch.zeros_like(bias), k, d, add=add)
        torch.testing.assert_close(st, want0 - rest, rtol=1e-12, atol=1e-12)


def test_stale_tap_guard_discriminates():
    """On the references alone: for every GPU conv case with a ring, the fp32-rounded true reference is within the
    bound and the stale-tap reference misses it by >= 10x on the steps where tap 0 sees data."""
    for case in K.CONV_CASES:
        B, Cin, Cout, k, d, mode, act, vec4, opts = case
        if k == 1:
            continue
        C = Cout // 2 if mode else Cout
        L = (k - 1) * d + 1
        T = 2 * L + 3
        g = torch.Generator().manual_seed(sum(case[:8]))
        x = torch.randn(B, T, Cin, generator=g)
        W = torch.randn(Cout, k, Cin, generator=g) * (k * Cin) ** -0.5
        bias = 0.1 * torch.randn(Cout, generator=g)
        kw = {n: torch.randn(B, T, C, generator=g) for n in ("res1", "res2") if n in opts}
        y, by = K.ref_conv_step(x, W, bias, k, d, mode, act, vec4=bool(vec4), **kw)
        st, _ = K.ref_conv_step(x, W, bias, k, d, mode, act, vec4=bool(vec4), stale=0, **kw)
        assert K.ratio(y.float(), y, by) <= 1, case
        assert K.ratio(y[:, L - 1:].float(), st[:, L - 1:], by[:, L - 1:]) >= 10, case


def test_chain_length():
    assert K.chain_len(3, 200, True) == 3 * 4 * 2 and K.chain_len(3, 200, False) == 3 * 7
    assert K.chain_len(1, 16, True) == 4 and K.chain_len(5, 81, False) == 15


def test_attention_reference_matches_dense_masked_softmax():
    g = torch.Generator().manual_seed(2)
    B, E, Ts = 4, 7, 40
    q = torch.randn(B, E, generator=g, dtype=torch.float64)
    Kt = torch.randn(B, E, Ts, generator=g, dtype=torch.float64)
    V = torch.randn(B, Ts, E, generator=g, dtype=torch.float64)
    lens = [40, 1, 17, 2]
    cases = [(None, None), ((1, 3), [0, 0, 16, 1]), ((1, 3), [39, 0, 8, 0]), ((5, 30), [20, 0, 3, 1]),
             ((0, 1), [n - 1 for n in lens])]
    for win, las in cases:
        lo, hi = [0] * B, list(lens)
        if win is not None:
            lo, hi = zip(*(K.window(la, win[0], win[1], n) for la, n in zip(las, lens)))
        P, bP, ctx, bctx = K.ref_attn_step(q, Kt, V, lens, lo, hi)
        for b in range(B):
            n = lens[b]
            s = Kt[b, :, :n].T @ q[b]
            mask = torch.zeros(n, dtype=torch.bool)
            if win is not None:                                 # reference deepvoice3.py:150-156, literally
                backward = las[b] - win[0]
                if backward > 0:
                    mask[:backward] = True
                ahead = las[b] + win[1]
                if ahead < n:
                    mask[ahead:] = True
            p = torch.softmax(s.masked_fill(mask, -math.inf), 0)
            torch.testing.assert_close(P[b, :n], p, rtol=1e-12, atol=1e-15)
            assert bool((P[b, n:] == 0).all() and (bP[b, n:] == 0).all() and (bP[b, :n][mask] == 0).all())
            torch.testing.assert_close(ctx[b], (p @ V[b, :n]) * (n * math.sqrt(1.0 / n)), rtol=1e-12, atol=1e-12)
            assert bool((bctx[b] > 0).all())
    # the window is clipped at both ends
    assert K.window(0, 1, 3, 40) == (0, 3) and K.window(39, 1, 3, 40) == (38, 40) and K.window(5, 1, 3, 40) == (4, 8)


def test_context_scale_is_the_references_fp32_value():
    """float(Ts*sqrt(1/Ts)) as the reference applies it (a double scalar times an fp32 tensor) -- and it is not always
    the scale an fp32 evaluation gives, which is why the step kernel must round the double value once."""
    x = torch.ones(1, dtype=torch.float32)
    differ = 0
    for n in range(1, 300):
        assert float(x * (n * math.sqrt(1.0 / n))) == float(K.context_scale(n))
        f = np.float32(n)
        differ += np.float32(f * np.sqrt(np.float32(1.0) / f)) != K.context_scale(n)
    assert differ > 0


def test_stop_rule_matches_stop_step():
    from deepvoice3_pytorch_b200.incremental import _stop_step
    rnd = random.Random(4)
    vals = [0.5, float(np.nextafter(np.float32(0.5), np.float32(1))), 0.0, 1.0, 0.7]
    for trial in range(300):
        min_steps, max_steps = rnd.randrange(0, 8), rnd.randrange(5, 20)
        n = max_steps + 3
        done = [[rnd.choice(vals) for _ in range(n)]]
        stop = [0]
        for t in range(n):                                      # one row stepping: the rule after every step
            stop = K.stop_rule(done, [t], stop, min_steps, max_steps)
        want = _stop_step(torch.tensor(done, dtype=torch.float32), min_steps, max_steps)
        assert stop[0] == (want or 0), (done, min_steps, max_steps, stop, want)
    assert K.stop_rule([[0.0]], [0], [-1], 0, 0) == [-1] and K.stop_rule([[0.0]], [0], [0], 0, 0) == [1]


def test_case_lists_reach_every_instantiation():
    def bt(B):
        return 1 if B == 1 else 2 if B == 2 else 4
    conv = K.CONV_CASES
    assert {bt(c[0]) for c in conv} == {1, 2, 4} and {bt(c[0]) for c in K.SLOT_CASES} == {1, 2, 4}
    assert any(c[0] % 4 for c in conv if bt(c[0]) == 4) and any(c[0] % 4 for c in K.SLOT_CASES if bt(c[0]) == 4)
    assert {c[0] for c in conv} >= {1, 2, 3, 4, 5, 9}
    v4 = [c for c in conv if c[7]]
    assert {c[1] for c in v4} >= {16, 256, 512} and any(c[1] > 128 and c[1] % 128 for c in v4)
    sc = [c for c in conv if not c[7]]
    assert any(c[1] % 4 and c[5] == 0 for c in sc) and any(c[1] % 4 and c[5] for c in sc)
    assert any(c[1] % 4 == 0 and "shift" in c[8] for c in sc)
    assert {c[6] for c in K.SLOT_CASES} == {0, 1}
    assert {c[3] for c in conv} >= {1, 2, 3, 5} and {c[4] for c in conv if c[3] > 1} >= {1, 3, 9, 27}
    assert {c[6] for c in conv if c[5] == 0} == {0, 1, 2}
    glu = [c for c in conv if c[5] == 1]
    assert any("spk" in c[8] for c in glu) and any("spk" not in c[8] for c in glu)
    assert any(c[5] == 2 for c in conv) and {c[5] for c in K.SLOT_CASES} == {0, 1, 2}
    assert {c[3] for c in K.SLOT_CASES} - {1}, "the slot cases need a ring"
    assert any("res1" in c[8] and "res2" not in c[8] for c in conv) and any("res2" in c[8] for c in conv)
    for o in ("add", "y2", "y2s", "y2a"):
        assert any(o in c[8] for c in conv), o
    att = K.ATTN_CASES
    assert {c[0] for c in att} == {"plain", "rows", "slots"}
    assert {c[2] for c in att} >= {16, 128, 256, 300}
    assert {c[3] for c in att} >= {1, 2, 31, 255, 256, 257, 600}
    assert any(c[2] + c[3] == K.MAX_E_TS for c in att) and K.MAX_E_TS == 12279
    for v in ("plain", "rows", "slots"):
        assert any(c[0] == v and c[5] is None for c in att) and any(c[0] == v and c[5] for c in att), v
    clipped_lo = clipped_hi = interior = False
    for v, B, E, Ts, lens, win, las, steps, _ in att:
        if win is None:
            continue
        for b in range(B if v != "plain" else 1):
            n = lens[b] if lens else Ts
            la = las[b] if v != "plain" else las
            lo, hi = K.window(la, win[0], win[1], n)
            clipped_lo |= lo == 0 and la - win[0] <= 0
            clipped_hi |= hi == n and la + win[1] >= n
            interior |= 0 < lo and hi < n
    assert clipped_lo and clipped_hi and interior
    assert any(c[0] == "plain" and c[5] == (1, 3) for c in att) and any(c[5] and c[5][1] > 3 for c in att)
    assert any(c[0] != "plain" and 1 in c[4] for c in att)
    assert all(c[8] for c in att if c[5]), "windowed cases check the cursor against their alignment row"
    assert any(c[0] == "slots" and len({t & 1 for t in c[7]}) == 2 for c in att)
