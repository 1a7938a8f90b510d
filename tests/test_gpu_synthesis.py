"""GPU: batched synthesis (deepvoice3_pytorch_b200.synthesis.tts_batch) against synthesizing each sequence alone the
way reference synthesis.py:42-73 does (model(...) -> denormalise -> audio.inv_spectrogram).

In exact-fp32 mode every kernel on the path computes a row from its own data in a batch-independent order, so the
comparison is bit for bit: step count, alignment, mel, linear spectrogram and waveform."""
import contextlib

import numpy as np
import pytest
import torch

from test_gpu_models import preset_kwargs

pytestmark = pytest.mark.gpu

LENGTHS = [37, 5, 161, 90, 128]          # ragged, out of order; 161 is the padded maximum
PRESETS = ["deepvoice3_ljspeech", "nyanko_ljspeech", "deepvoice3_vctk"]


@contextlib.contextmanager
def _conv_math(mode):
    from deepvoice3_pytorch_b200 import ops
    old = ops.conv_math
    ops.conv_math = mode
    try:
        yield
    finally:
        ops.conv_math = old


def _model(preset, max_steps, min_steps=10, done_bias=None, seed=7):
    from deepvoice3_pytorch_b200 import builder
    bname, kw = preset_kwargs(preset)
    torch.manual_seed(seed)
    model = getattr(builder, bname)(dropout=0.0, **kw).cuda().eval()
    dec = model.seq2seq.decoder
    dec.max_decoder_steps, dec.min_decoder_steps = max_steps, min_steps
    if done_bias is not None:
        with torch.no_grad():
            dec.fc.bias.fill_(done_bias)
    return model


def _sequences(lengths, seed=3):
    rng = np.random.RandomState(seed)
    return [rng.randint(2, 149, size=n).astype(np.int64) for n in lengths]


def _tts_alone(model, seq, speaker_id=None):
    """reference synthesis.py:tts on token ids."""
    from deepvoice3_pytorch_b200 import audio
    sequence = torch.from_numpy(seq).unsqueeze(0).long().cuda()
    text_positions = torch.arange(1, sequence.size(-1) + 1).unsqueeze(0).long().cuda()
    speaker_ids = None if speaker_id is None else torch.LongTensor([speaker_id]).cuda()
    with torch.no_grad():
        mel_outputs, linear_outputs, alignments, done = model(sequence, text_positions=text_positions,
                                                              speaker_ids=speaker_ids)
    linear_output = linear_outputs[0].cpu().data.numpy()
    spectrogram = audio._denormalize(linear_output)
    alignment = alignments[0].cpu().data.numpy()
    mel = audio._denormalize(mel_outputs[0].cpu().data.numpy())
    waveform = audio.inv_spectrogram(linear_output.T)
    return waveform, alignment, spectrogram, mel


@pytest.mark.parametrize("preset", PRESETS)
def test_tts_batch_equals_each_sequence_alone_bit_for_bit(preset):
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    model = _model(preset, max_steps=40)
    seqs = _sequences(LENGTHS)
    spk = [3, 17, 0, 54, 101] if model.n_speakers > 1 else None
    with _conv_math("fp32"):
        got = tts_batch(model, seqs, speaker_ids=spk, batch_size=16)
        want = [_tts_alone(model, s, None if spk is None else spk[i]) for i, s in enumerate(seqs)]
    assert len(got) == len(seqs)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g[1].shape == w[1].shape == (w[1].shape[0], LENGTHS[i]), (i, g[1].shape, w[1].shape)   # steps
        for name, a, b in zip(("waveform", "alignment", "spectrogram", "mel"), g, w):
            assert a.shape == b.shape and np.array_equal(a, b), "row %d (%d tokens): %s differs" % (i, LENGTHS[i], name)


def test_tts_batch_chunks_keep_input_order():
    """Several chunks (batch_size 2 over 5 sequences): same results as one chunk, in input order."""
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    model = _model("nyanko_ljspeech", max_steps=24)
    seqs = _sequences(LENGTHS, seed=9)
    with _conv_math("fp32"):
        one = tts_batch(model, seqs, batch_size=16)
        many = tts_batch(model, seqs, batch_size=2)
    for a, b in zip(one, many):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


@pytest.mark.parametrize("preset", PRESETS)
def test_ragged_teacher_forced_decode_equals_single_rows(preset):
    from deepvoice3_pytorch_b200 import incremental
    model = _model(preset, max_steps=40)
    seqs = _sequences(LENGTHS, seed=5)
    B, L, N = len(seqs), max(LENGTHS), 30
    text = torch.zeros(B, L, dtype=torch.long)
    tpos = torch.zeros(B, L, dtype=torch.long)
    for b, s in enumerate(seqs):
        text[b, :s.size] = torch.from_numpy(s)
        tpos[b, :s.size] = torch.arange(1, s.size + 1)
    text, tpos = text.cuda(), tpos.cuda()
    lens = torch.tensor(LENGTHS).cuda()
    mel = torch.rand(B, N, 80, generator=torch.Generator().manual_seed(2)).cuda()
    enc_kw = {}
    spk = None
    if model.n_speakers > 1:
        spk = model.embed_speakers(torch.tensor([5, 9, 1, 77, 30]).cuda())
        enc_kw = dict(speaker_embed=spk)
    dec = model.seq2seq.decoder
    from deepvoice3_pytorch_b200 import ops
    with _conv_math("fp32"), torch.no_grad():
        with ops.length_scope(lens, L):
            keys, values = model.seq2seq.encoder(text, **enc_kw)
        out, al, dn, st, steps = incremental.decode_ragged(dec, (keys, values), tpos, lens, spk, test_inputs=mel)
        assert steps == [N] * B
        for b, n in enumerate(LENGTHS):
            kw1 = dict(speaker_embed=spk[b:b + 1]) if spk is not None else {}
            k1, v1 = model.seq2seq.encoder(text[b:b + 1, :n], **kw1)
            assert torch.equal(k1, keys[b:b + 1, :n]) and torch.equal(v1, values[b:b + 1, :n]), "encoder row %d" % b
            o1, a1, d1, s1 = incremental.decode(dec, (k1, v1), tpos[b:b + 1, :n],
                                                None if spk is None else spk[b:b + 1], test_inputs=mel[b:b + 1])
            assert torch.equal(out[b:b + 1], o1) and torch.equal(st[b:b + 1], s1), "row %d" % b
            assert torch.equal(al[b:b + 1, :, :n], a1) and not al[b, :, n:].any(), "alignment row %d" % b
            assert torch.equal(dn[b:b + 1], torch.cat(d1, dim=1).reshape(1, -1)), "done row %d" % b


def test_monotonic_cursors_diverge_per_row():
    """Two rows with the same text, teacher-forced with different frames: their attention cursors move apart.  Each
    row must still equal its own single-row decode (the reference's quirk -- every row follows row 0's cursor -- holds
    for decode, not for the ragged batch)."""
    from deepvoice3_pytorch_b200 import incremental
    model = _model("deepvoice3_ljspeech", max_steps=60)
    dec = model.seq2seq.decoder
    assert all(dec.force_monotonic_attention)
    n, N = 60, 48
    gen = torch.Generator().manual_seed(4)
    text = torch.randint(2, 149, (1, n), generator=gen).repeat(2, 1).cuda()
    tpos = torch.arange(1, n + 1)[None].repeat(2, 1).cuda()
    mel = torch.stack([torch.rand(N, 80, generator=gen), torch.rand(N, 80, generator=gen) * 0.1]).cuda()
    lens = torch.tensor([n, n]).cuda()
    with _conv_math("fp32"), torch.no_grad():
        keys, values = model.seq2seq.encoder(text)
        _, al, _, _, _ = incremental.decode_ragged(dec, (keys, values), tpos, lens, test_inputs=mel)
        cur = al.argmax(-1).cpu()
        assert (cur[0] != cur[1]).any(), "the two rows' cursors never diverged: the test does not test anything"
        for b in range(2):
            _, a1, _, _ = incremental.decode(dec, (keys[b:b + 1], values[b:b + 1]), tpos[b:b + 1],
                                             test_inputs=mel[b:b + 1])
            assert torch.equal(al[b:b + 1], a1), "row %d" % b
        # the quirky batch decode makes row 1 follow row 0's cursor, so it differs from row 1 alone
        _, aq, _, _ = incremental.decode(dec, (keys, values), tpos, test_inputs=mel)
        _, a1, _, _ = incremental.decode(dec, (keys[1:], values[1:]), tpos[1:], test_inputs=mel[1:])
        assert not torch.equal(aq[1:], a1)


def test_tts_batch_tensor_core_mode_within_tolerance():
    """Default (tensor-core) mode: the batch's GEMMs may take other kernels than a short single sentence's, so compare
    at the model-level tolerance; the done bias is forced negative so every row runs the same number of steps."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    assert ops.conv_math == "tc"
    model = _model("deepvoice3_ljspeech", max_steps=20, done_bias=-30.0)
    seqs = _sequences(LENGTHS, seed=11)
    got = tts_batch(model, seqs)
    for i, s in enumerate(seqs):
        w = _tts_alone(model, s)
        g = got[i]
        assert g[1].shape == w[1].shape == (21, LENGTHS[i])
        np.testing.assert_allclose(g[1], w[1], rtol=1e-3, atol=1e-4, err_msg="alignment %d" % i)
        np.testing.assert_allclose(g[3] / 100.0, w[3] / 100.0, rtol=1e-3, atol=1e-4, err_msg="mel %d" % i)
        np.testing.assert_allclose(g[2] / 100.0, w[2] / 100.0, rtol=1e-3, atol=1e-4, err_msg="linear %d" % i)


def test_inv_spectrogram_batch_is_bit_identical_alone_and_reproducible():
    from deepvoice3_pytorch_b200 import audio
    from oracle import audio_oracle as A
    clips = [A.synthetic_clip(20 + i, n=n) for i, n in enumerate([3000, 22050, 256 * 40, 9000])]
    specs = [audio.spectrogram(c) for c in clips]                         # (513, T_c), ragged T
    assert len({s.shape[1] for s in specs}) == len(specs)
    batch = audio.inv_spectrogram_batch(specs, n_iter=8)
    again = audio.inv_spectrogram_batch(specs, n_iter=8)
    for c, s in enumerate(specs):
        alone = audio.inv_spectrogram(s, n_iter=8)
        assert batch[c].shape == alone.shape == (audio.inv_num_samples(s.shape[1]),)
        assert np.array_equal(batch[c], alone), "clip %d" % c
        assert np.array_equal(batch[c], again[c]), "clip %d not reproducible" % c
    rev = audio.inv_spectrogram_batch(specs[::-1], n_iter=8)[::-1]      # other neighbours, other padding
    assert all(np.array_equal(a, b) for a, b in zip(rev, batch))


def test_mask_time_kernel():
    from deepvoice3_pytorch_b200 import ops
    x = torch.randn(3, 5, 16, device="cuda")
    keep = x.clone()
    lengths = torch.tensor([8, 3, 1], device="cuda")
    with torch.no_grad(), ops.length_scope(lengths, 8):
        y = ops.mask_time(x)                                             # T = 16 = 2 * 8: mult 2
    assert torch.equal(x, keep)                                          # never writes the caller's tensor
    want = x.clone()
    for b, n in enumerate([16, 6, 2]):
        want[b, :, n:] = 0
    assert torch.equal(y, want)
    with torch.no_grad(), ops.length_scope(lengths, 5):
        with pytest.raises(Exception, match="length scope"):
            ops.mask_time(x)                                             # 16 is not a multiple of 5
