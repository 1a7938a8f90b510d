"""No GPU: the argument checks of TrainStep(speaker_encoder=...), the speaker_embed argument of the multi-speaker
model, and the cloning samples of data.CloningSampleDataset + collate_cloning."""
import os

import numpy as np
import pytest
import torch

KW = dict(n_vocab=40, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4, kernel_size=3,
          encoder_channels=16, decoder_channels=16, converter_channels=16, max_positions=64, n_speakers=5,
          speaker_embed_dim=8, speaker_embedding_weight_std=0.2)


def _model(**over):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    return builder.deepvoice3_multispeaker(**dict(KW, **over))


def _encoder(**over):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder
    torch.manual_seed(1)
    return SpeakerEncoder(**dict(dict(mel_dim=8, speaker_embed_dim=8, channels=16, heads=2), **over))


# ---- argument checks --------------------------------------------------------------------------------------------------
def test_check_speaker_encoder_accepts_a_matching_pair():
    from deepvoice3_pytorch_b200.train_step import check_speaker_encoder
    check_speaker_encoder(_model(), _encoder(), True, True, None)


@pytest.mark.parametrize("case", ["single_speaker", "embed_dim", "mel_dim", "seq2seq_only", "postnet_only", "adapt"])
def test_trainstep_refuses_before_building_anything(case):
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.train_step import TrainStep
    model, enc, kw = _model(), _encoder(), {}
    if case == "single_speaker":
        model = builder.deepvoice3(**{k: v for k, v in KW.items() if k not in ("n_speakers", "speaker_embed_dim",
                                                                                "speaker_embedding_weight_std")})
    elif case == "embed_dim":
        enc = _encoder(speaker_embed_dim=4)
    elif case == "mel_dim":
        enc = _encoder(mel_dim=6)
    elif case == "seq2seq_only":
        kw = dict(train_postnet=False)
    elif case == "postnet_only":
        kw = dict(train_seq2seq=False)
    else:
        kw = dict(adapt_speakers=[4])
    before = [p.data_ptr() for p in list(model.parameters()) + list(enc.parameters())]
    for train_model in (True, False):
        with pytest.raises(ValueError):
            TrainStep(model, speaker_encoder=enc, train_model=train_model, **kw)
    assert [p.data_ptr() for p in list(model.parameters()) + list(enc.parameters())] == before   # no arena built


def test_trainstep_refuses_a_world_size_above_one(monkeypatch):
    import torch.distributed as dist
    from deepvoice3_pytorch_b200.train_step import TrainStep
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda *a: 2)
    with pytest.raises(ValueError, match="single process"):
        TrainStep(_model(), speaker_encoder=_encoder())


def test_speaker_embed_argument_checks():
    m = _model()
    e = torch.zeros(2, 8)
    assert m._speaker_embedding(None, e) is e
    with pytest.raises(ValueError):
        m._speaker_embedding(torch.zeros(2, dtype=torch.int64), e)
    with pytest.raises(ValueError):
        m._speaker_embedding(None, torch.zeros(2, 7))
    with pytest.raises(ValueError):
        m._speaker_embedding(None, torch.zeros(2, 1, 8))


# ---- CloningSampleDataset -----------------------------------------------------------------------------------------
def _corpus(tmp_path, frames_by_speaker, M=4):
    """Utterance j of speaker s: frame t holds s * 100 + j + t / 1000 in every channel."""
    rows = []
    for spk, frames in frames_by_speaker.items():
        for j, T in enumerate(frames):
            name = "mel-%d-%d.npy" % (spk, j)
            np.save(tmp_path / name, np.full((T, M), spk * 100 + j, dtype=np.float32) +
                    np.arange(T, dtype=np.float32)[:, None] / 1000)
            lin = "lin-%d-%d.npy" % (spk, j)
            np.save(tmp_path / lin, np.full((T, 5), -spk, dtype=np.float32))
            rows.append("%s|%s|%d|text%d|%d" % (lin, name, T, j, spk))
    (tmp_path / "train.txt").write_text("\n".join(rows) + "\n")
    from deepvoice3_pytorch_b200.data import TrainTxtDataset
    return TrainTxtDataset(str(tmp_path), lambda s: [1 + len(s) % 3, 2, 3][:1 + len(s) % 3])


FRAMES = {0: [20, 30, 12, 25, 40], 1: [40, 16, 9], 2: [15, 15, 15, 15, 15, 15]}


def test_draws_come_from_other_eligible_utterances_of_the_speaker(tmp_path):
    from deepvoice3_pytorch_b200.data import CloningSampleDataset
    ds = _corpus(tmp_path, FRAMES)
    cs = CloningSampleDataset(ds, N=3, T_crop=15, seed=4)
    assert len(cs) == len(ds)
    for epoch in range(4):
        cs.set_epoch(epoch)
        for i in range(len(ds)):
            item = cs[i]
            base = ds[i]
            assert len(item) == 5
            assert np.array_equal(item[0], base[0]) and np.array_equal(item[1], base[1]) and item[3] == base[3]
            crops = item[4]
            assert crops.shape == (3, 15, 4) and crops.dtype == np.float32
            items, offsets = cs.draws(i)
            spk = int(ds.rows[i][4])
            for k, (j, o) in enumerate(zip(items.tolist(), offsets.tolist())):
                assert j != i                                   # never the row's own utterance
                assert int(ds.rows[j][4]) == spk and ds.frame_lengths[j] >= 15
                assert 0 <= o <= ds.frame_lengths[j] - 15
                full = np.load(os.path.join(str(tmp_path), ds.rows[j][1]))
                assert np.array_equal(crops[k], full[o:o + 15])


def test_without_replacement_when_possible_with_replacement_otherwise(tmp_path):
    from deepvoice3_pytorch_b200.data import CloningSampleDataset
    ds = _corpus(tmp_path, FRAMES)
    cs = CloningSampleDataset(ds, N=3, T_crop=15, seed=0)
    spk = [int(r[4]) for r in ds.rows]
    repeated = False
    for epoch in range(20):
        cs.set_epoch(epoch)
        for i in range(len(ds)):
            items = cs.draws(i)[0].tolist()
            if spk[i] in (0, 2):            # >= 3 other eligible utterances: never a repeat
                assert len(set(items)) == 3, (i, items)
            else:                           # speaker 1: one other eligible utterance (40 frames) or two
                pool = [j for j in range(len(ds)) if spk[j] == 1 and j != i and ds.frame_lengths[j] >= 15]
                assert set(items) <= set(pool) and len(pool) < 3
                repeated |= len(set(items)) < 3
    assert repeated


def test_draws_depend_on_seed_epoch_and_index_only(tmp_path):
    from deepvoice3_pytorch_b200.data import CloningSampleDataset, collate_cloning
    ds = _corpus(tmp_path, FRAMES)
    a, b = CloningSampleDataset(ds, 2, 12, seed=3), CloningSampleDataset(ds, 2, 12, seed=3)
    a.set_epoch(2)
    b.set_epoch(2)
    order = list(range(len(ds)))
    want = {i: a.draws(i) for i in order}
    for i in reversed(order):                          # any order of access
        got = b.draws(i)
        assert np.array_equal(got[0], want[i][0]) and np.array_equal(got[1], want[i][1])
    b.set_epoch(3)
    assert any(not np.array_equal(b.draws(i)[1], want[i][1]) or not np.array_equal(b.draws(i)[0], want[i][0])
               for i in order)
    c = CloningSampleDataset(ds, 2, 12, seed=4)
    c.set_epoch(2)
    assert any(not np.array_equal(c.draws(i)[1], want[i][1]) for i in order)
    # whatever the batch composition and the number of DataLoader workers
    loaders = []
    for workers, bs in ((0, 2), (2, 3), (3, 1)):
        dl = torch.utils.data.DataLoader(a, batch_size=bs, shuffle=False, num_workers=workers,
                                         collate_fn=collate_cloning)
        loaders.append(torch.cat([batch["speaker_mels"] for batch in dl]))
    assert all(torch.equal(loaders[0], x) for x in loaders[1:])
    single = torch.from_numpy(np.stack([a[i][4] for i in order]))
    assert torch.equal(loaders[0], single)


def test_refuses_a_speaker_without_other_eligible_utterances(tmp_path):
    from deepvoice3_pytorch_b200.data import CloningSampleDataset, TrainTxtDataset
    ds = _corpus(tmp_path, {0: [20, 30], 7: [40, 10], 2: [20, 20]})
    with pytest.raises(ValueError, match="speaker 7"):
        CloningSampleDataset(ds, 2, 15)                 # speaker 7's only eligible utterance is the row itself
    CloningSampleDataset(ds, 2, 10)
    with pytest.raises(ValueError):
        CloningSampleDataset(TrainTxtDataset(str(tmp_path), lambda s: [1], speaker_id=0), 2, 10)
    with pytest.raises(ValueError):
        CloningSampleDataset(ds, 0, 10)


@pytest.mark.parametrize("r,ds_step", [(1, 4), (2, 4)])
def test_collate_cloning_equals_collate_plus_the_samples(tmp_path, r, ds_step):
    from deepvoice3_pytorch_b200.data import CloningSampleDataset, collate, collate_cloning
    ds = _corpus(tmp_path, FRAMES)
    cs = CloningSampleDataset(ds, 3, 15, seed=1)
    idx = [4, 0, 9, 6]
    items = [cs[i] for i in idx]
    got = collate_cloning(items, r, ds_step)
    want = collate([ds[i] for i in idx], r, ds_step)
    assert set(got) == set(want) | {"speaker_mels"}
    for k, v in want.items():
        if torch.is_tensor(v):
            assert torch.equal(got[k], v) and got[k].dtype == v.dtype, k
        else:
            assert np.array_equal(got[k], v), k
    assert got["speaker_mels"].shape == (4, 3, 15, 4) and got["speaker_mels"].dtype == torch.float32
    assert torch.equal(got["speaker_mels"], torch.from_numpy(np.stack([it[4] for it in items])))


def test_every_other_eligible_utterance_can_be_drawn_and_the_index_is_linear(tmp_path):
    """N = (eligible utterances of the speaker) - 1 without replacement draws exactly the others; the pools are one
    array per speaker (memory linear in the corpus, not in utterances x utterances per speaker)."""
    import types
    from deepvoice3_pytorch_b200.data import CloningSampleDataset
    ds = _corpus(tmp_path, FRAMES)
    cs = CloningSampleDataset(ds, N=5, T_crop=15, seed=2)
    for i in range(len(ds)):
        if int(ds.rows[i][4]) == 2:
            assert sorted(cs.draws(i)[0].tolist()) == [j for j in range(len(ds)) if int(ds.rows[j][4]) == 2 and j != i]
    rows = [("l", "m", "100", "t", str(i // 400)) for i in range(40000)]
    big = types.SimpleNamespace(multi_speaker=True, rows=rows, frame_lengths=[100] * len(rows))
    cs = CloningSampleDataset(big, N=8, T_crop=64)
    assert sum(a.size for a in cs._eligible.values()) == len(rows)
    items = cs.draws(12345)[0]
    assert len(set(items.tolist())) == 8 and 12345 not in items and all(j // 400 == 12345 // 400 for j in items)
