"""Host-side checks of continuous-batching synthesis (no GPU): synthesis.tts_stream refuses what tts_batch refuses,
before the first item, and its bookkeeping yields every index exactly once, post-net groups included."""
import numpy as np
import pytest
import torch


def _model(**kw):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    base = dict(n_vocab=20, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4, padding_idx=0,
                encoder_channels=16, decoder_channels=16, converter_channels=16, max_positions=32, dropout=0.0)
    base.update(kw)
    return builder.deepvoice3(**base).eval()


@pytest.mark.parametrize("sequences, kw, err", [
    ([], {}, ValueError),
    ([np.array([1, 2]), np.array([], dtype=np.int64)], {}, ValueError),
    ([np.ones((2, 3), dtype=np.int64)], {}, ValueError),
    ([np.ones(32, dtype=np.int64)], {}, ValueError),                  # positions 1..32 need a 33-row table
    ([np.array([1.5, 2.0])], {}, ValueError),
    ([np.array([1, 2])], {"speaker_ids": [0]}, ValueError),           # single-speaker model
    ([np.array([1, 2])], {"slots": 0}, ValueError),
    ([np.array([1, 2])], {"post_batch": 0}, ValueError),
    ([np.array([1, 2])], {}, RuntimeError),                           # model on the CPU
])
def test_tts_stream_refusals(sequences, kw, err):
    from deepvoice3_pytorch_b200.synthesis import tts_stream
    with pytest.raises(err):
        tts_stream(_model(), sequences, **kw)                         # raised by the call, not by the first next()


def test_tts_stream_refuses_speaker_mismatch_and_training_mode():
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.synthesis import tts_stream
    torch.manual_seed(0)
    multi = builder.deepvoice3_multispeaker(n_vocab=20, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4,
                                            n_speakers=3, encoder_channels=16, decoder_channels=16,
                                            converter_channels=16, max_positions=32, dropout=0.0).eval()
    seqs = [np.array([1, 2, 3]), np.array([4, 5])]
    with pytest.raises(ValueError):
        tts_stream(multi, seqs, speaker_ids=[0])
    with pytest.raises(ValueError):
        tts_stream(multi, seqs)
    with pytest.raises(RuntimeError, match="eval mode"):
        tts_stream(_model().train(), seqs)


def test_decode_stream_refuses_bad_slots_and_training_mode():
    from deepvoice3_pytorch_b200 import incremental
    dec = _model().seq2seq.decoder
    with pytest.raises(ValueError, match="slots"):
        next(incremental.decode_stream(dec, 0, []))
    with pytest.raises(RuntimeError, match="eval mode"):
        next(incremental.decode_stream(dec.train(), 2, []))


@pytest.mark.parametrize("n, slots, post_batch", [(11, 4, 3), (3, 8, 16), (5, 1, 1), (7, 3, 7)])
def test_tts_stream_yields_every_index_once(monkeypatch, n, slots, post_batch):
    """The encoder, decoder and post-net stages replaced by host stand-ins: requests are pulled lazily, finish in a
    scrambled order, and each one comes out once, with its own data, whatever the group sizes."""
    from deepvoice3_pytorch_b200 import incremental, synthesis
    rng = np.random.RandomState(n * 100 + slots)
    seqs = [np.arange(1, 2 + rng.randint(1, 9)) for _ in range(n)]
    encoded, post_groups = [], []

    def encode(model, idx, group, speaker_ids, stage):
        assert len(idx) <= slots and [s.size for s in group] == [seqs[i].size for i in idx]
        encoded.extend(idx)
        return [(i, torch.full((s.size, 2), float(i)), torch.zeros(s.size, 2), torch.arange(1, s.size + 1), None)
                for i, s in zip(idx, group)]

    def decode_stream(decoder, S, requests, stats=None, stage_timer=None):
        assert S == slots
        live = []
        for r in requests:
            live.append(r)
            if len(live) == S or rng.rand() < 0.3:
                rng.shuffle(live)
                r0 = live.pop()
                yield _decoded(r0)
        rng.shuffle(live)
        for r0 in live:
            yield _decoded(r0)

    def _decoded(r):
        i, k = r[0], r[1]
        N = 2 + i % 3
        return i, torch.full((N, 4), float(i)), torch.zeros(N, k.size(0)), torch.zeros(N), torch.full((N, 3), i), N

    def postnet_vocode(model, outputs, states, steps, spk, stage):
        assert len(steps) <= post_batch and outputs.shape[0] == len(steps)
        post_groups.append(len(steps))
        return [(np.full(3, outputs[b, 0, 0].item()), None, None) for b in range(len(steps))]

    monkeypatch.setattr(synthesis, "_encode", encode)
    monkeypatch.setattr(incremental, "decode_stream", decode_stream)
    monkeypatch.setattr(synthesis, "_postnet_vocode", postnet_vocode)
    got = list(synthesis._stream(_model(), seqs, None, slots, post_batch, lambda name: None, None))
    assert sorted(i for i, _ in got) == list(range(n))
    assert all(res[0][0] == i and res[1].shape[1] == seqs[i].size for i, res in got)
    assert sorted(encoded) == list(range(n))
    assert sum(post_groups) == n and all(g == post_batch for g in post_groups[:-1])
