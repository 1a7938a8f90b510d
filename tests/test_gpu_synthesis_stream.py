"""GPU: continuous-batching synthesis (synthesis.tts_stream, incremental.decode_stream) against synthesizing each
sequence alone with tts_batch, and the slot kernels (dv3_inc_conv_step_slots, dv3_inc_attn_step_slots,
dv3_inc_stop_rows, dv3_inc_advance_rows, dv3_inc_refill) against the shared-counter step and a fresh program.

In exact-fp32 mode each slot runs its utterance at its own step with the arithmetic of the one-utterance path, and a
refilled slot starts from the zeros of a fresh program, so the comparison is bit for bit."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from test_gpu_models import preset_kwargs

PRESETS = ["deepvoice3_ljspeech", "nyanko_ljspeech", "deepvoice3_vctk"]
CHOICES = [5, 37, 90, 128, 161]


def _model(preset, max_steps, min_steps=10, seed=7):
    from deepvoice3_pytorch_b200 import builder
    bname, kw = preset_kwargs(preset)
    torch.manual_seed(seed)
    model = getattr(builder, bname)(dropout=0.0, **kw).cuda().eval()
    dec = model.seq2seq.decoder
    dec.max_decoder_steps, dec.min_decoder_steps = max_steps, min_steps
    return model


def _sequences(lengths, seed=3):
    rng = np.random.RandomState(seed)
    return [rng.randint(2, 149, size=n).astype(np.int64) for n in lengths]


def _stop_steps_for(pre, bias, min_steps, max_steps):
    """Stop steps the reference rule gives rows of done pre-activations pre (B, max_steps + 1) with the bias added."""
    n = np.arange(1, pre.shape[1] + 1)
    stop = ((pre + bias > 0) & (n > min_steps)) | (n > max_steps)
    return stop.argmax(axis=1) + 1


@torch.no_grad()
def spread_done_bias(model, seqs, speaker_ids=None):
    """Set the done head's bias so that a random-weight model stops its utterances at spread-out steps.

    Assumption: a random model's done pre-activation a_i(t) = fc(x_t) - bias does not depend on the bias (the done flag
    is not fed back into the decoder).  One run with the bias at -30 (nobody stops) records a_i(t); of 512 candidate
    biases (quantiles of -a_i(t)) the one that gives the most distinct stop steps, with at least one utterance running
    to max_decoder_steps, is set.  -> the bias."""
    from deepvoice3_pytorch_b200 import incremental, ops
    dec = model.seq2seq.decoder
    dec.fc.bias.fill_(-30.0)
    lens = [s.size for s in seqs]
    L = max(lens)
    text = torch.zeros(len(seqs), L, dtype=torch.long)
    tpos = torch.zeros(len(seqs), L, dtype=torch.long)
    for b, s in enumerate(seqs):
        text[b, :s.size] = torch.from_numpy(s)
        tpos[b, :s.size] = torch.arange(1, s.size + 1)
    text, tpos, text_len = text.cuda(), tpos.cuda(), torch.tensor(lens).cuda()
    spk = None if speaker_ids is None else model._speaker_embedding(torch.tensor(speaker_ids).cuda())
    with ops.length_scope(text_len, L):
        keys, values = model.seq2seq.encoder(text, speaker_embed=spk)
    _, _, dones, _, _ = incremental.decode_ragged(dec, (keys, values), tpos, text_len, spk)
    d = dones.double().clamp(1e-300, 1 - 1e-16)
    pre = (torch.log(d / (1 - d)) + 30.0).cpu().numpy()
    lo, hi = dec.min_decoder_steps, dec.max_decoder_steps
    best, bias = -1, -30.0
    for b in np.unique(np.quantile(-pre[:, lo:], np.linspace(0, 1, 512))):
        b = float(np.float32(b)) - 1e-3                     # stay clear of a pre-activation the bias would tie
        steps = _stop_steps_for(pre, b, lo, hi)
        score = len(set(steps.tolist())) if (steps == hi + 1).any() else 0
        if score > best:
            best, bias = score, b
    dec.fc.bias.fill_(bias)
    return bias


def _alone(model, seq, speaker_id):
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    return tts_batch(model, [seq], speaker_ids=None if speaker_id is None else [speaker_id], batch_size=1)[0]


# distinct stop steps the calibrated bias gives at least: the random nyanko model's done pre-activation has one spike,
# at step 27 in every utterance alike, and carries no per-utterance signal after it, so its utterances stop there or at
# max_decoder_steps
DISTINCT = {"nyanko_ljspeech": 2}


def _stream_vs_alone(preset, n, slots, post_batch, seed):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.synthesis import tts_stream
    model = _model(preset, max_steps=60)
    rng = np.random.RandomState(seed)
    lengths = [CHOICES[i] for i in rng.randint(0, len(CHOICES), size=n)]
    seqs = _sequences(lengths, seed=seed)
    spk = [int(x) for x in rng.permutation(model.n_speakers)[:n]] if model.n_speakers > 1 else None
    old = ops.conv_math
    ops.conv_math = "fp32"
    try:
        spread_done_bias(model, seqs, spk)
        stats = {}
        got = list(tts_stream(model, seqs, speaker_ids=spk, slots=slots, post_batch=post_batch, stats=stats))
        want = [_alone(model, s, None if spk is None else spk[i]) for i, s in enumerate(seqs)]
    finally:
        ops.conv_math = old
    assert sorted(i for i, _ in got) == list(range(n))
    for i, g in got:
        w = want[i]
        assert g[1].shape == w[1].shape and g[1].shape[1] == lengths[i], (i, g[1].shape, w[1].shape)     # steps
        for name, a, b in zip(("waveform", "alignment", "spectrogram", "mel"), g, w):
            assert a.shape == b.shape and np.array_equal(a, b), "sequence %d (%d tokens): %s differs" % (
                i, lengths[i], name)
    steps = [w[1].shape[0] for w in want]
    assert stats["useful_steps"] == sum(steps)
    return steps, stats, model


@pytest.mark.gpu
@pytest.mark.parametrize("preset", PRESETS)
def test_tts_stream_equals_each_sequence_alone_bit_for_bit(preset):
    """11 sequences on 4 slots: slots are refilled while the others are mid-decode, the utterances stop at different
    steps (one at max_decoder_steps) and every result equals tts_batch on that sequence alone, bit for bit.  On vctk
    every sequence has its own speaker, so neighbouring slots hold different speakers."""
    steps, stats, model = _stream_vs_alone(preset, 11, slots=4, post_batch=3, seed=21)
    assert len(set(steps)) >= DISTINCT.get(preset, 3), "stop steps %s: the done bias did not spread them" % steps
    assert model.seq2seq.decoder.max_decoder_steps + 1 in steps, steps
    assert any(busy > 0 for _, _, busy in stats["refills"]), stats["refills"]


@pytest.mark.gpu
@pytest.mark.parametrize("n, slots", [(4, 1), (5, 16)])
def test_tts_stream_one_slot_and_more_slots_than_sequences(n, slots):
    steps, stats, _ = _stream_vs_alone("nyanko_ljspeech", n, slots=slots, post_batch=2, seed=n)
    if slots == 1:
        assert [len(loaded) for _, loaded, _ in stats["refills"]] == [1] * (n - 1)


@pytest.mark.gpu
def test_tts_stream_tensor_core_mode_within_tolerance():
    """Default (tensor-core) mode: encoder groups differ from tts_batch's chunks, so the GEMMs may take other kernels;
    compare at the tts_batch tolerance with a done bias that lets nobody stop early."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.synthesis import tts_batch, tts_stream
    assert ops.conv_math == "tc"
    model = _model("deepvoice3_ljspeech", max_steps=20)
    with torch.no_grad():
        model.seq2seq.decoder.fc.bias.fill_(-30.0)
    lengths = [37, 5, 161, 90, 128]
    seqs = _sequences(lengths, seed=11)
    want = tts_batch(model, seqs)
    got = dict(tts_stream(model, seqs, slots=2, post_batch=2))
    for i in range(len(seqs)):
        g, w = got[i], want[i]
        assert g[1].shape == w[1].shape == (21, lengths[i])
        np.testing.assert_allclose(g[1], w[1], rtol=1e-3, atol=1e-4, err_msg="alignment %d" % i)
        np.testing.assert_allclose(g[3] / 100.0, w[3] / 100.0, rtol=1e-3, atol=1e-4, err_msg="mel %d" % i)
        np.testing.assert_allclose(g[2] / 100.0, w[2] / 100.0, rtol=1e-3, atol=1e-4, err_msg="linear %d" % i)


@torch.no_grad()
def _programs(preset, slots, B=3, Tmax=24):
    """The ragged decoder program of B encoded sequences, built with the shared counter or (slots) per-row counters."""
    from deepvoice3_pytorch_b200 import incremental, ops
    model = _model(preset, max_steps=Tmax - 1)
    dec = model.seq2seq.decoder
    dec.fc.bias.fill_(-30.0)
    lengths = [37, 5, 90][:B]
    seqs = _sequences(lengths, seed=4)
    L = max(lengths)
    text = torch.zeros(B, L, dtype=torch.long)
    tpos = torch.zeros(B, L, dtype=torch.long)
    for b, s in enumerate(seqs):
        text[b, :s.size] = torch.from_numpy(s)
        tpos[b, :s.size] = torch.arange(1, s.size + 1)
    text, tpos, lens = text.cuda(), tpos.cuda(), torch.tensor(lengths).cuda()
    spk = model.embed_speakers(torch.tensor([5, 9, 1][:B]).cuda()) if model.n_speakers > 1 else None
    old = ops.conv_math
    ops.conv_math = "fp32"
    try:
        with ops.length_scope(lens, L):
            keys, values = model.seq2seq.encoder(text, speaker_embed=spk)
        kv, pos, addend = incremental._constants(dec, keys, values, tpos, spk, Tmax)
        prog = incremental.StepProgram(B, keys.device, slots=slots)

        def spk_of(f):
            s = addend(f)
            if s is None:
                return None
            prog.keep.append(s)
            return incremental._Rows(s, s.size(-1))
        frames = prog.buf(B, Tmax + 1, dec.in_dim * dec.r)
        text_len = lens.to(torch.int32)
        states, aligns, dones = incremental._build_program(dec, prog, Tmax, keys.size(-1), kv, pos, spk_of,
                                                           text_len, frames)
    finally:
        ops.conv_math = old
    if slots:
        prog.stop_rule(dones, dec.min_decoder_steps, dec.max_decoder_steps)
        prog.stop.zero_()                           # every row running from step 0
    return prog, frames, states, aligns, dones


@pytest.mark.gpu
@pytest.mark.parametrize("preset", PRESETS)
def test_slot_step_kernels_with_equal_counters_equal_the_shared_counter_step(preset):
    Tmax = 24
    shared = _programs(preset, False, Tmax=Tmax)
    per_row = _programs(preset, True, Tmax=Tmax)
    shared[0].run(Tmax, use_graph=False)
    per_row[0].run(Tmax, use_graph=True)
    for name, a, b in zip(("frames", "states", "aligns", "dones"), shared[1:], per_row[1:]):
        assert torch.equal(a, b), name
    assert [x.shape for x in shared[0].rings] == [x.shape for x in per_row[0].rings]
    for a, b in zip(shared[0].rings + shared[0].cursors, per_row[0].rings + per_row[0].cursors):
        assert torch.equal(a, b)
    # the last step n = Tmax > max_decoder_steps stops every row; a stopped row keeps its step
    assert per_row[0].stop.tolist() == [Tmax] * 3 and per_row[0].t.tolist() == [Tmax - 1] * 3
    per_row[0].run(2, use_graph=True)                  # held rows recompute their last step: the same bits
    for name, a, b in zip(("frames", "states", "aligns", "dones"), shared[1:], per_row[1:]):
        assert torch.equal(a, b), name


@pytest.mark.gpu
def test_stop_rule_on_the_device_is_the_reference_rule():
    from deepvoice3_pytorch_b200 import incremental
    from deepvoice3_pytorch_b200._lib import lib
    rng = np.random.RandomState(0)
    B, T, lo, hi = 6, 30, 5, 25
    done = torch.from_numpy(rng.rand(B, T).astype(np.float32) * 0.53).cuda()
    done[0, :] = 0.0
    done[1, 3] = 0.9                                        # before min_steps: ignored
    t = torch.zeros(B, dtype=torch.int32, device="cuda")
    stop = torch.zeros(B, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = ctypes.c_void_p
    for _ in range(T):
        lib.call("dv3_inc_stop_rows", P(done.data_ptr()), T, P(t.data_ptr()), P(stop.data_ptr()), B, lo, hi, st)
        lib.call("dv3_inc_advance_rows", P(t.data_ptr()), P(stop.data_ptr()), B, st)
    want = incremental._row_stop_steps(done.cpu(), lo, hi)
    assert stop.tolist() == want and want[0] == hi + 1
    assert t.tolist() == [n - 1 for n in want]


@pytest.mark.gpu
def test_refill_resets_slots_to_a_fresh_program_and_loads_staged_rows():
    from deepvoice3_pytorch_b200 import incremental
    from deepvoice3_pytorch_b200._lib import lib
    fresh = _programs("deepvoice3_vctk", True)
    prog, frames = _programs("deepvoice3_vctk", True)[:2]
    frames[:, 0] = 1.0
    prog.run(7, use_graph=False)
    prog.stop[1] = 5
    before = [x.clone() for x in prog.rings + prog.cursors + [prog.t, prog.stop, frames]]
    assert all(r.abs().sum() > 0 for r in prog.rings)
    staged = torch.tensor([[11, 12], [13, 14]], dtype=torch.int32, device="cuda")
    dst = torch.zeros(3, 2, dtype=torch.int32, device="cuda")
    entries = incremental._reset_entries(prog, frames) + [(dst, torch.zeros_like(dst), 8, 0)]
    src = entries[-1][1]
    src[:2] = staged
    table = incremental._refill_table(entries, frames.device)
    slots = torch.tensor([2, 1], dtype=torch.int32, device="cuda")        # staged row i -> slot slots[i]
    lib.call("dv3_inc_refill", ctypes.c_void_p(table.data_ptr()), len(entries), ctypes.c_void_p(slots.data_ptr()),
             2, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert dst.tolist() == [[0, 0], [13, 14], [11, 12]]
    B = prog.B
    after = prog.rings + prog.cursors + [prog.t, prog.stop, frames]
    ref = fresh[0].rings + fresh[0].cursors + [fresh[0].t, fresh[0].stop, fresh[1]]
    n_ring = len(prog.rings)
    for j, (old, new, zero) in enumerate(zip(before, after, ref)):
        if n_ring <= j < n_ring + len(prog.cursors):                     # cursors int[2][B]: row b is [b] and [B+b]
            old, new, zero = (x.view(2, B).transpose(0, 1) for x in (old, new, zero))
        if new.dim() == 3 and new is frames:
            old, new, zero = old[:, :1], new[:, :1], zero[:, :1]          # only the go frame is reset
        assert torch.equal(new[0], old[0]), "slot 0 was not refilled and must keep its state (entry %d)" % j
        for b in (1, 2):
            assert torch.equal(new[b], zero[b]), "slot %d entry %d differs from a fresh program" % (b, j)
    assert torch.equal(frames[:, 1:], before[-1][:, 1:])


def test_refill_struct_matches_the_c_header(tmp_path):
    """Dv3IncRefill is mirrored by hand in ctypes; compile the header with gcc and compare sizeof / every offset."""
    from deepvoice3_pytorch_b200.incremental import Dv3IncRefill
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dv3b200.h"', 'int main(void) {',
             'printf("sizeof %zu\\n", sizeof(Dv3IncRefill));']
    for fname, _ in Dv3IncRefill._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(Dv3IncRefill, %s));' % (fname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split("\n")
    seen = 0
    for line in filter(None, out):
        field, value = line.split()
        got = ctypes.sizeof(Dv3IncRefill) if field == "sizeof" else getattr(Dv3IncRefill, field).offset
        assert got == int(value), "Dv3IncRefill.%s: ctypes %d vs C %s" % (field, got, value)
        seen += 1
    assert seen == len(Dv3IncRefill._fields_) + 1
