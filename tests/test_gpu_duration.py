"""GPU: duration-guided synthesis (DESIGN.md section 2.22) -- the guided attention step against fp64, guided decoding
against the free run it restates, guided tts_batch / tts_stream / evaluate_attention, the parent's launch sequences
without durations, the duration loss against fp64, the predictor against fp64 autograd, its training step, and
learning on a synthetic corpus.

Loss bound (u = 2^-24): the kernels form every term and sum in fp64 and round once, so the loss is within u |loss| (+ a
few fp64 ulps) of the exact value, and each gradient entry within u |g| of its fp64 value; 2u is the bound used."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import duration_oracle as DO
from test_gpu_inc_kernels import _attn_buffers, _same, ratio, ref_attn_step, window
from test_gpu_synthesis import PRESETS, _conv_math, _model, _sequences
from test_gpu_tc1 import _call, _p, _st

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


@pytest.fixture
def math_mode():
    from deepvoice3_pytorch_b200 import ops
    old = ops.conv_math, ops.deterministic

    def set_(m, det=None):
        ops.conv_math = m
        if det is not None:
            ops.deterministic = det
    yield set_
    ops.conv_math, ops.deterministic = old


# ---- the guided attention step ------------------------------------------------------------------------------------------
# (variant, B, E, Ts, text_len, window, path centres, steps): centres at the clamped edges, past them, text_len = 1
PATH_CASES = [
    ("rows", 5, 256, 256, [256, 1, 31, 200, 2], (1, 3), [0, 0, 30, 199, 1], 4),
    ("rows", 4, 128, 600, [600, 257, 255, 3], (100, 300), [599, 10, 128, 2], 6),
    ("rows", 3, 16, 40, [40, 1, 40], (0, 1), [39, 0, 0], 0),
    ("slots", 6, 300, 257, [257, 1, 256, 31, 2, 100], (1, 3), [5, 0, 255, 30, 1, 50], [0, 1, 2, 3, 10, 11]),
    ("slots", 3, 64, 9, [9, 1, 9], (4, 4), [8, 0, 4], [7, 0, 3]),
]


@pytest.mark.parametrize("case", PATH_CASES, ids=lambda c: "%s_B%d_Ts%d" % (c[0], c[1], c[3]))
def test_path_attn_step_vs_fp64(case):
    variant, B, E, Ts, lens, win, centres, steps = case
    bf = _attn_buffers(variant, B, E, Ts, lens, win, centres, steps, 1.0, seed=B * 11 + Ts)
    bf["la"].fill_(-7)                                 # a sentinel the guided step must neither read nor write
    la0 = bf["la"].clone()
    ts = bf["ts"]
    T = max(ts) + 3
    path = torch.full((B, T + 5), -99, dtype=torch.int32, device="cuda")   # sentinel: any other step is wrong
    for b in range(B):
        path[b, ts[b]] = centres[b]
    ctx, align = bf["ctx"], bf["align"]
    name = "dv3_inc_attn_step_slots_path" if variant == "slots" else "dv3_inc_attn_step_path"
    _call(name, ctypes.byref(bf["a"]), _p(bf["text_len"]), _p(path), path.stride(0), _st())
    torch.cuda.synchronize()
    lo, hi = zip(*[window(centres[b], win[0], win[1], lens[b]) for b in range(B)])
    P, bP, want, bctx = ref_attn_step(bf["q"].get()[:, 0], bf["K"], bf["V"], lens, list(lo), list(hi))
    rc = ratio(ctx.get()[:, 0], want, bctx)
    cur = align.idx[torch.arange(B, device="cuda"), torch.tensor(ts, device="cuda")]
    Pk = align.buf[cur]
    valid = torch.arange(Ts, device="cuda")[None] < torch.tensor(lens, device="cuda")[:, None]
    assert bool((Pk[~valid] == 0).all())
    rp = ratio(torch.where(valid, Pk, 0.0), P, bP)
    assert torch.equal(bf["la"], la0)
    print("path %s: ctx error/bound %.3g, probs %.3g" % (variant, rc, rp))
    assert rc <= 1 and rp <= 1
    # the same launch through the ROWS / SLOTS step with the centres as cursors gives the same bits
    bf2 = _attn_buffers(variant, B, E, Ts, lens, win, centres, steps, 1.0, seed=B * 11 + Ts)
    _call("dv3_inc_attn_step_slots" if variant == "slots" else "dv3_inc_attn_step_rows", ctypes.byref(bf2["a"]),
          _p(bf2["text_len"]), _st())
    torch.cuda.synchronize()
    assert _same(ctx.buf, bf2["ctx"].buf) and _same(align.buf, bf2["align"].buf)


def test_stop_rows_total():
    t = torch.tensor([0, 4, 9, 2, 5, 0], dtype=torch.int32, device="cuda")
    stop = torch.tensor([0, 0, 0, 3, -1, 0], dtype=torch.int32, device="cuda")
    total = torch.tensor([1, 6, 10, 3, 6, 2], dtype=torch.int32, device="cuda")
    _call("dv3_inc_stop_rows_total", _p(t), _p(stop), _p(total), 6, _st())
    assert stop.tolist() == [1, 0, 10, 3, -1, 0]
    assert t.tolist() == [0, 4, 9, 2, 5, 0]


# ---- guided decoding ------------------------------------------------------------------------------------------------------
def _encode(model, seqs):
    from deepvoice3_pytorch_b200 import ops
    lens = [s.size for s in seqs]
    L = max(lens)
    text, tpos = np.zeros((len(seqs), L), np.int64), np.zeros((len(seqs), L), np.int64)
    for b, s in enumerate(seqs):
        text[b, :s.size], tpos[b, :s.size] = s, np.arange(1, s.size + 1)
    text, tpos = torch.from_numpy(text).cuda(), torch.from_numpy(tpos).cuda()
    tl = torch.tensor(lens).cuda()
    ops.rng.begin_forward(False, text.device)
    try:
        with torch.no_grad(), ops.length_scope(tl, L):
            keys, values = model.seq2seq.encoder(text)
    finally:
        ops.rng.end_forward()
    return keys, values, tpos, lens


def test_guided_decode_on_the_free_runs_cursor_path_reproduces_it_bit_for_bit():
    """nyanko: one attention layer with the monotonic window.  The free run's cursor of row b at step t is 0 at t = 0,
    then the first argmax of its alignment row t - 1; guided along that path, the decode is the free run."""
    from deepvoice3_pytorch_b200 import incremental
    model = _model("nyanko_ljspeech", max_steps=80, min_steps=5)
    assert model.seq2seq.decoder.force_monotonic_attention
    seqs = _sequences([30, 7, 19, 1, 44], seed=5)
    with _conv_math("fp32"):
        keys, values, tpos, lens = _encode(model, seqs)
        dec = model.seq2seq.decoder
        out, al, done, st, steps = incremental.decode_ragged(dec, (keys, values), tpos, lens)
        N = al.size(1)
        a = al.cpu().numpy()
        path = np.zeros((len(seqs), N), np.int64)
        for b, n in enumerate(lens):
            path[b, 1:] = a[b, :N - 1, :n].argmax(-1)
        g_out, g_al, g_done, g_st, g_steps = incremental._decode(dec, (keys, values), tpos, None, None, None, None,
                                                                  text_lengths=lens, guide=(path, steps))
    assert g_steps == steps
    for b, n in enumerate(steps):
        assert _same(g_out[b, :n], out[b, :n]) and _same(g_al[b, :n], al[b, :n])
        assert _same(g_done[b, :n], done[b, :n]) and _same(g_st[b, :n], st[b, :n])


def test_guided_rows_run_exactly_their_totals():
    from deepvoice3_pytorch_b200 import incremental
    model = _model("deepvoice3_ljspeech", max_steps=30)
    seqs = _sequences([12, 3, 25], seed=6)
    rng = np.random.RandomState(0)
    durs = [rng.randint(1, 6, s.size) for s in seqs]
    with _conv_math("fp32"):
        keys, values, tpos, lens = _encode(model, seqs)
        out, al, done, st, steps = incremental.decode_ragged(model.seq2seq.decoder, (keys, values), tpos, lens,
                                                             durations=durs)
    totals = [int(d.sum()) for d in durs]
    assert steps == totals and out.size(1) == max(totals) and done.shape == (3, max(totals))
    # the alignment mass sits inside each step's window around the prescribed token
    path, _ = incremental.path_table([np.asarray(d) for d in durs])
    a = al.cpu().numpy()
    att = model.seq2seq.decoder.attention[0] if isinstance(model.seq2seq.decoder.attention, torch.nn.ModuleList) \
        else model.seq2seq.decoder.attention
    for b, n in enumerate(totals):
        for t in range(n):
            lo, hi = window(int(path[b, t]), att.window_backward, att.window_ahead, lens[b])
            row = a[b, t, :lens[b]]
            assert row[:lo].sum() == 0 and row[hi:].sum() == 0


def _guided(model, seqs, seed):
    rng = np.random.RandomState(seed)
    return [rng.randint(1, 4, s.size).astype(np.int64) for s in seqs]


def _same_items(x, y):
    return all(a.shape == b.shape and np.array_equal(a, b) for a, b in zip(x, y))


def test_guided_tts_batch_rows_alone_shuffled_and_rerun():
    from deepvoice3_pytorch_b200 import synthesis
    model = _model("deepvoice3_ljspeech", max_steps=40)
    seqs = _sequences([20, 5, 33, 12], seed=8)
    durs = _guided(model, seqs, 1)
    with _conv_math("fp32"):
        got = synthesis.tts_batch(model, seqs, batch_size=4, durations=durs)
        again = synthesis.tts_batch(model, seqs, batch_size=4, durations=durs)
        perm = [2, 0, 3, 1]
        shuf = synthesis.tts_batch(model, [seqs[i] for i in perm], batch_size=4, durations=[durs[i] for i in perm])
        for k in range(len(seqs)):
            alone = synthesis.tts_batch(model, [seqs[k]], durations=[durs[k]])[0]
            assert _same_items(got[k], alone), k
            assert _same_items(got[k], again[k]) and _same_items(got[k], shuf[perm.index(k)])
            assert got[k][1].shape == (int(durs[k].sum()), seqs[k].size)
        slow = synthesis.tts_batch(model, seqs, batch_size=4, durations=durs, speed=0.5)
    assert [s[1].shape[0] for s in slow] == [int(np.rint(d.sum() / 0.5)) for d in durs]


@pytest.mark.parametrize("preset", PRESETS)
def test_guided_tts_stream_equals_guided_tts_batch(preset):
    from deepvoice3_pytorch_b200 import synthesis
    model = _model(preset, max_steps=40)
    seqs = _sequences([14, 3, 22, 9, 17, 5], seed=9)
    durs = _guided(model, seqs, 2)
    spk = [3, 17, 0, 54, 101, 7] if model.n_speakers > 1 else None
    with _conv_math("fp32"):
        want = synthesis.tts_batch(model, seqs, speaker_ids=spk, batch_size=4, durations=durs)
        for slots in (1, 4, 16):
            got = dict(synthesis.tts_stream(model, seqs, speaker_ids=spk, slots=slots, post_batch=3, durations=durs))
            assert sorted(got) == list(range(len(seqs)))
            for k in range(len(seqs)):
                assert _same_items(got[k], want[k]), (slots, k)


def test_guided_evaluate_attention():
    from deepvoice3_pytorch_b200.alignment import evaluate_attention
    model = _model("deepvoice3_ljspeech", max_steps=20)
    seqs = _sequences([9, 4, 15], seed=10)
    durs = [np.full(s.size, 7, np.int64) for s in seqs]        # totals past max_decoder_steps + 1
    with _conv_math("fp32"):
        ev = evaluate_attention(model, seqs, durations=durs)
        ev2 = evaluate_attention(model, seqs, durations=durs, speed=2.0)
    assert ev["steps"].tolist() == [int(d.sum()) for d in durs] and ev["stop_failures"] == 0
    assert ev2["steps"].tolist() == [int(np.rint(d.sum() / 2.0)) for d in durs] and ev2["stop_failures"] == 0


CALLS_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "incremental",
                            "calls_without_durations.json")


def record_calls():
    """The lib.call sequences of decode, decode_ragged, tts_batch and tts_stream without durations on a fixed
    deepvoice3_ljspeech model in fp32: [entry point, its integer and float arguments] per call.  Pointers are left out
    (ctypes pointers, and integers of 2^40 or more: device and host addresses), so the lists depend only on the
    launches.  Uses only what the package had before guided decoding, so the parent commit records the same way."""
    from deepvoice3_pytorch_b200 import incremental, synthesis
    from deepvoice3_pytorch_b200._lib import lib
    model = _model("deepvoice3_ljspeech", max_steps=30)
    seqs = _sequences([11, 4, 17], seed=12)
    calls, real = [], lib.call

    def rec(name, *a):
        calls.append([name] + [x for x in a if isinstance(x, (int, float)) and not isinstance(x, bool)
                               and abs(x) < 2 ** 40])
        return real(name, *a)
    out = {}
    lib.call = rec
    try:
        with _conv_math("fp32"):
            keys, values, tpos, lens = _encode(model, seqs)
            runs = [("decode", lambda: incremental.decode(model.seq2seq.decoder, (keys[:1, :lens[0]],
                                                                                   values[:1, :lens[0]]),
                                                          tpos[:1, :lens[0]])),
                    ("decode_ragged", lambda: incremental.decode_ragged(model.seq2seq.decoder, (keys, values), tpos,
                                                                        lens)),
                    ("tts_batch", lambda: synthesis.tts_batch(model, seqs, batch_size=4)),
                    ("tts_stream", lambda: list(synthesis.tts_stream(model, seqs, slots=2)))]
            for name, fn in runs:
                calls[:] = []
                fn()
                out[name] = list(calls)
    finally:
        lib.call = real
    return out


def test_launch_sequences_without_durations_are_the_parents():
    """Without durations, decode / decode_ragged / tts_batch / tts_stream make exactly the calls the parent commit
    made (recorded with ``record_calls`` there, tests/golden/incremental/calls_without_durations.json)."""
    with open(CALLS_GOLDEN) as f:
        want = json.load(f)
    got = json.loads(json.dumps(record_calls()))
    for name in ("decode", "decode_ragged", "tts_batch", "tts_stream"):
        assert len(want[name]) > 0
        assert got[name] == want[name], name


# ---- the loss ---------------------------------------------------------------------------------------------------------------
def _loss_inputs(B, L, seed):
    rng = np.random.RandomState(seed)
    lens = rng.randint(1, L + 1, B)
    lens[0] = L
    y = (rng.randn(B, L) * 2).astype(np.float32)
    d = rng.randint(1, 60, (B, L)).astype(np.int32)
    return y, d, lens.astype(np.int32)


def _row_losses(y, d, lens):
    B, L = y.shape
    row = torch.empty(B, dtype=torch.float64, device="cuda")
    loss = torch.empty((), device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    _call("dv3_duration_loss_fwd", _p(y), y.stride(0), _p(d), d.stride(0), _p(lens), B, L, _p(row), _p(loss), _p(err),
          _st())
    return row, loss, err


@pytest.mark.parametrize("B,L", [(1, 1), (16, 200), (5, 1024), (300, 37)])
def test_loss_and_gradient_against_fp64(B, L):
    from deepvoice3_pytorch_b200.duration import duration_loss
    y, d, lens = _loss_inputs(B, L, B + L)
    want, gw = DO.loss(y.astype(np.float64), d, lens)
    yt = torch.from_numpy(y).cuda().requires_grad_()
    loss = duration_loss(yt, d, lens)
    loss.backward()
    assert abs(loss.item() - want) <= 2 * U * abs(want)
    g = yt.grad.double().cpu().numpy()
    assert (np.abs(g - gw) <= 2 * U * np.abs(gw)).all()
    mask = np.arange(L)[None] >= lens[:, None]
    assert (g[mask] == 0).all()


def test_loss_rows_do_not_depend_on_the_batch_and_bad_rows_set_the_flag():
    y, d, lens = _loss_inputs(9, 50, 3)
    yd, dd, ld = (torch.from_numpy(x).cuda() for x in (y, d, lens))
    row, _, err = _row_losses(yd, dd, ld)
    assert int(err) == 0
    for b in range(9):                                         # alone, padded wider and strided
        wide_y = torch.full((1, 80), float("nan"), device="cuda")
        wide_y[0, :50] = yd[b]
        wide_d = torch.zeros(1, 80, dtype=torch.int32, device="cuda")
        wide_d[0, :50] = dd[b]
        r1, _, _ = _row_losses(yd[b:b + 1], dd[b:b + 1], ld[b:b + 1])
        r2, _, _ = _row_losses(wide_y, wide_d, ld[b:b + 1])
        assert _same(r1.view(torch.float32), row[b:b + 1].view(torch.float32))
        assert _same(r2.view(torch.float32), row[b:b + 1].view(torch.float32))
    perm = torch.randperm(9, generator=torch.Generator().manual_seed(0)).cuda()
    rp, _, _ = _row_losses(yd[perm].contiguous(), dd[perm].contiguous(), ld[perm].contiguous())
    assert _same(rp.view(torch.float32), row[perm].view(torch.float32))
    bad_d = dd.clone()
    bad_d[2, 0] = 0
    bad_l = ld.clone()
    bad_l[4] = 51
    r3, _, e3 = _row_losses(yd, bad_d, bad_l)
    assert int(e3) == 1 and float(r3[2]) == 0 and float(r3[4]) == 0
    keep = [b for b in range(9) if b not in (2, 4)]
    assert _same(r3[keep].view(torch.float32), row[keep].view(torch.float32))


# ---- the predictor ----------------------------------------------------------------------------------------------------------
def _w(m):
    v, g = m.weight_v.double(), m.weight_g.double()
    return v * (g / torch.norm_except_dim(v, 2, 0))


def _ref_forward(pred, values, lens, spk):
    """The predictor in fp64 torch: weight-normed convs, GLU blocks with the speaker addend, rows masked per block."""
    B, L, _ = values.shape
    mask = (torch.arange(L, device=values.device)[None] < lens[:, None])[:, None].double()
    x = F.relu(F.conv1d(values.double().transpose(1, 2), _w(pred.proj[0]), pred.proj[0].bias.double()))
    for f in pred.blocks:
        x = x * mask
        c = f.conv
        h = F.conv1d(x, _w(c), c.bias.double(), padding=c.padding[0], dilation=c.dilation[0])
        a, b = h.chunk(2, 1)
        if spk is not None:
            sp = f.speaker_proj
            a = a + F.softsign(spk.double() @ _w(sp).reshape(sp.out_features, -1).T + sp.bias.double())[:, :, None]
        x = (a * torch.sigmoid(b) + x) * 0.5 ** 0.5
    o = pred.out[0]
    return F.conv1d(x, _w(o), o.bias.double()).reshape(B, L)


def _predictor(E, C, n_speakers=1, seed=0):
    from deepvoice3_pytorch_b200.duration import DurationPredictor
    torch.manual_seed(seed)
    return DurationPredictor(E, channels=C, n_blocks=2, n_speakers=n_speakers, speaker_embed_dim=16).cuda()


@pytest.mark.parametrize("mode,n_speakers,tol", [("fp32", 1, 1e-4), ("fp32", 4, 1e-4), ("tc", 1, 5e-3)])
def test_predictor_against_fp64_autograd(math_mode, mode, n_speakers, tol):
    from deepvoice3_pytorch_b200.duration import duration_loss
    math_mode(mode)
    B, L, E, C = 6, 40, 64, 128
    pred = _predictor(E, C, n_speakers)
    g = torch.Generator(device="cuda").manual_seed(1)
    values = torch.randn(B, L, E, device="cuda", generator=g)
    lens = torch.tensor([40, 3, 17, 40, 1, 29], device="cuda")
    spk = torch.randn(B, 16, device="cuda", generator=g) if n_speakers > 1 else None
    d = torch.randint(1, 9, (B, L), device="cuda", generator=g).to(torch.int32)
    y = pred(values, lens, spk)
    loss = duration_loss(y, d, lens.to(torch.int32))
    loss.backward()
    params = [p for p in pred.parameters()]
    got_g = [p.grad.double().clone() for p in params]
    pred64 = pred
    for p in params:
        p.grad = None
    y64 = _ref_forward(pred64, values, lens, spk)
    mask = torch.arange(L, device="cuda")[None] < lens[:, None]
    l64 = (((y64 - torch.log(d.double())) ** 2 * mask).sum(1) / lens.double()).mean()
    want_g = torch.autograd.grad(l64, params)
    ey = ((y.double() - y64).abs() * mask).max() / (y64.abs() * mask).max()
    print("predictor %s: y rel error %.3g" % (mode, ey))
    assert ey <= tol
    assert abs(loss.item() - l64.item()) <= tol * abs(l64.item())
    for p, a, b in zip(params, got_g, want_g):
        e = (a - b).abs().max() / b.abs().max().clamp_min(1e-30)
        assert e <= 10 * tol, (tuple(p.shape), float(e))


def _synthetic(B, L, E, V, emb, rng):
    ids = rng.randint(0, V, (B, L))
    lens = rng.randint(L // 4, L + 1, B).astype(np.int32)
    values = emb[ids]
    for b in range(B):
        values[b, lens[b]:] = 0
    d = (1 + ids % 4).astype(np.int32)
    return {"values": torch.from_numpy(values.astype(np.float32)).cuda(), "durations": torch.from_numpy(d).cuda(),
            "token_lengths": torch.from_numpy(lens).cuda()}


def _run(steps, use_graph, batches, seed=3):
    from deepvoice3_pytorch_b200.duration import DurationPredictorStep
    st = DurationPredictorStep(_predictor(32, 128, seed=seed), lr=3e-3, use_graph=use_graph)
    losses = [st.step(b).clone() for b in batches[:steps]]
    torch.cuda.synchronize()
    return st, torch.stack(losses).cpu(), st.arena.flat.clone().cpu()


def _batches(n, seed=0):
    rng = np.random.RandomState(seed)
    emb = np.random.RandomState(99).randn(12, 32)
    return [_synthetic(8, 24, 32, 12, emb, rng) for _ in range(n)]


@pytest.mark.parametrize("use_graph", [False, True])
def test_step_is_deterministic(math_mode, use_graph):
    math_mode("tc", "1")
    bs = _batches(4)
    _, la, pa = _run(4, use_graph, bs)
    _, lb, pb = _run(4, use_graph, bs)
    assert torch.equal(la, lb) and torch.equal(pa, pb)


def test_step_graph_equals_eager_and_checkpoints_resume(math_mode):
    from deepvoice3_pytorch_b200.duration import DurationPredictorStep
    math_mode("tc1", "1")
    bs = _batches(6)
    _, le, pe = _run(4, False, bs)
    st_g, lg, pg = _run(4, True, bs)
    assert st_g.launches_per_step is not None and st_g.launches_per_step > 5
    np.testing.assert_allclose(lg.numpy(), le.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pg.numpy(), pe.numpy(), rtol=1e-4, atol=1e-6)
    st, _, _ = _run(3, True, bs)
    ckpt = st.state_dict()
    tail = [st.step(b).clone() for b in bs[3:]]
    straight = st.arena.flat.clone().cpu()
    res = DurationPredictorStep(_predictor(32, 128, seed=8), lr=3e-3, use_graph=True)
    res.load_state_dict(ckpt)
    l2 = [res.step(b).clone() for b in bs[3:]]
    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(tail, l2))
    assert torch.equal(res.arena.flat.cpu(), straight) and res.global_step == 6


def test_predictor_learns_durations_of_token_ids(math_mode):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.duration import DurationPredictorStep
    math_mode("tc")
    rng = np.random.RandomState(5)
    emb = np.random.RandomState(99).randn(12, 32)
    train = [_synthetic(16, 32, 32, 12, emb, rng) for _ in range(20)]
    pred = _predictor(32, 128, seed=4)
    st = DurationPredictorStep(pred, lr=3e-3, use_graph=True)
    first = float(st.step(train[0]))
    for k in range(1, 400):
        last = st.step(train[k % len(train)])
    ops.check_index_errors()
    held = _synthetic(32, 32, 32, 12, emb, np.random.RandomState(77))
    pred.eval()
    lens = held["token_lengths"].to(torch.int64)
    with torch.no_grad(), ops.length_scope(lens, 32):
        y = pred(held["values"], lens).double().cpu().numpy()
    d = np.maximum(1, np.rint(np.exp(y)))
    want = held["durations"].cpu().numpy()
    m = np.arange(32)[None] < lens.cpu().numpy()[:, None]
    acc = float((d == want)[m].mean())
    print("duration predictor: loss %.4f -> %.4f, held-out exact %.4f" % (first, float(last), acc))
    assert acc >= 0.95


@pytest.mark.parametrize("preset", ["deepvoice3_ljspeech", "deepvoice3_vctk"])
def test_duration_batch_and_predict_durations(math_mode, preset):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.alignment import teacher_forced_steps
    from deepvoice3_pytorch_b200.duration import (DurationPredictor, DurationPredictorStep, duration_batch,
                                                  predict_durations)
    from deepvoice3_pytorch_b200.train_step import to_device
    from test_gpu_models import preset_kwargs
    math_mode("fp32")
    model = _model(preset, max_steps=60)
    _, kw = preset_kwargs(preset)
    r, ds = kw["r"], kw["downsample_step"]
    seqs = _sequences([37, 5, 20, 12], seed=11)
    spk = [3, 17, 0, 54] if model.n_speakers > 1 else None
    rng = np.random.RandomState(12)
    items = []
    for k, s in enumerate(seqs):
        n = int(rng.randint(120, 400))
        item = (s, rng.rand(n, model.mel_dim).astype(np.float32), rng.rand(n, model.linear_dim).astype(np.float32))
        items.append(item + ((spk[k],) if spk else ()))
    batch = to_device(data.collate(items, r=r, downsample_step=ds), "cuda")
    out = duration_batch(model, batch, 64)
    steps = teacher_forced_steps(batch["target_lengths"].cpu().numpy(), r, ds)
    dur = out["durations"].cpu().numpy()
    assert out["values"].shape[:2] == (4, 64) and dur.shape == (4, 64)
    for b, s in enumerate(seqs):
        assert dur[b, :s.size].sum() == steps[b] and dur[b, :s.size].min() >= 1 and (dur[b, s.size:] == 0).all()
    assert ("speaker_embed" in out) == (spk is not None)
    E = out["values"].size(2)
    torch.manual_seed(2)
    pred = DurationPredictor(E, channels=128, n_blocks=1, n_speakers=model.n_speakers, speaker_embed_dim=16).cuda()
    st = DurationPredictorStep(pred, use_graph=True)
    st.step(out)
    st.step(out)
    got = predict_durations(pred, model, seqs, speaker_ids=spk, batch_size=3)
    for k, s in enumerate(seqs):
        alone = predict_durations(pred, model, [s], speaker_ids=None if spk is None else [spk[k]])[0]
        assert got[k].shape == s.shape and got[k].min() >= 1 and np.array_equal(got[k], alone)
