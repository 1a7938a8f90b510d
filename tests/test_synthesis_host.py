"""Host-side checks of batched synthesis (no GPU): the refusals of synthesis.tts_batch, the length scope's guards and
the per-row stop rule of the ragged decoder."""
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
    ([np.array([1, 2])], {"batch_size": 0}, ValueError),
    ([np.array([1, 2])], {}, RuntimeError),                           # model on the CPU
])
def test_tts_batch_refusals(sequences, kw, err):
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    with pytest.raises(err):
        tts_batch(_model(), sequences, **kw)


def test_tts_batch_refuses_speaker_mismatch_and_training_mode():
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    torch.manual_seed(0)
    multi = builder.deepvoice3_multispeaker(n_vocab=20, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4,
                                            n_speakers=3, encoder_channels=16, decoder_channels=16,
                                            converter_channels=16, max_positions=32, dropout=0.0).eval()
    seqs = [np.array([1, 2, 3]), np.array([4, 5])]
    with pytest.raises(ValueError):
        tts_batch(multi, seqs, speaker_ids=[0])
    with pytest.raises(ValueError):
        tts_batch(multi, seqs)
    with pytest.raises(RuntimeError, match="eval mode"):
        tts_batch(_model().train(), seqs)


def test_length_scope_is_inference_only_and_does_not_nest():
    from deepvoice3_pytorch_b200 import ops
    lengths = torch.tensor([3, 2])
    with pytest.raises(RuntimeError, match="no_grad"):
        with ops.length_scope(lengths, 4):
            pass
    assert ops._length_scope is None
    x = torch.randn(2, 3, 4)
    assert ops.mask_time(x) is x                 # no scope: untouched, no launch


def test_ragged_stop_rule_is_the_single_rule_per_row():
    from deepvoice3_pytorch_b200.incremental import _row_stop_steps, _stop_step
    rng = np.random.RandomState(0)
    for _ in range(50):
        done = torch.from_numpy(rng.rand(4, 30).astype(np.float32) * 0.6)
        got = _row_stop_steps(done, 5, 25)
        assert got == [_stop_step(done[b:b + 1], 5, 25) for b in range(4)]
    done = torch.zeros(3, 12)
    done[0, 7] = 1.0                                             # row 0 stops after step 8; the others run to n > 10
    assert _row_stop_steps(done, 5, 10) == [8, 11, 11]
    assert _row_stop_steps(done[:, :9], 5, 10) == [8, None, None]
