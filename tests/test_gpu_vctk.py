"""GPU: the VCTK corpus front-end.  The polyphase resampler against scipy's resample_poly in fp64 (rounded to fp32), the
trim-bounds kernel against the fp64 restatement (audio.trim_bounds_reference), and build_vctk_from_path against a
per-clip composition of those stages, through to one multi-speaker training step."""
import os

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

import vctk_fixtures as F

pytestmark = pytest.mark.gpu
RATES = [(48000, 22050), (44100, 22050), (16000, 22050), (24000, 22050)]


def _batch(clips, dtype):
    pitch = max(len(c) for c in clips) + 5                   # an odd pitch: no alignment assumed
    x = np.zeros((len(clips), pitch), dtype=dtype)
    for i, c in enumerate(clips):
        x[i, :len(c)] = c
    return torch.from_numpy(x).cuda()


def _pcm_clips(seed, lens):
    rng = np.random.RandomState(seed)
    return [(np.clip(F.clip(seed + i, n / 48000.0) * 1.5 + 0.01 * rng.randn(n), -1, 1) * 32767).astype(np.int16)
            for i, n in enumerate(lens)]


@pytest.mark.parametrize("sr_from,sr_to", RATES)
def test_resampler_against_scipy_fp64(sr_from, sr_to, monkeypatch):
    from deepvoice3_pytorch_b200 import audio
    monkeypatch.setattr(audio.hparams, "sample_rate", sr_to)
    lens = [1, 7, 1000, 48000, 100003, 33333]
    pcm = _pcm_clips(3, lens)
    f32 = [p.astype(np.float32) / 32768.0 for p in pcm]
    out16, olens = audio.resample_batch(_batch(pcm, np.int16), lens, sr_from)
    out32, _ = audio.resample_batch(_batch(f32, np.float32), lens, sr_from)
    again, _ = audio.resample_batch(_batch(pcm, np.int16), lens, sr_from)
    torch.cuda.synchronize()
    assert torch.equal(out16, out32) and torch.equal(out16, again)       # int16 == fp32 of the same samples; repeatable
    got = out16.cpu().numpy()
    up, down = audio.resample_ratio(sr_from)
    same = total = 0
    for i, x in enumerate(f32):
        want = resample_poly(x.astype(np.float64), up, down).astype(np.float32)
        assert olens[i] == len(want)
        g = got[i, :len(want)]
        assert np.all(np.abs(g.astype(np.float64) - want) <= np.spacing(np.abs(want))), (i, len(x))
        assert not got[i, len(want):].any()
        same += int(np.sum(g.view(np.int32) == want.view(np.int32)))
        total += len(want)
        alone, _ = audio.resample_batch(_batch([pcm[i]], np.int16), [lens[i]], sr_from)
        assert np.array_equal(alone.cpu().numpy()[0, :len(want)], g)   # a clip alone == its row of the ragged batch
    assert same >= 0.99 * total, (same, total)


def test_resampler_identity_and_input_checks():
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import Dv3Error
    pcm = _pcm_clips(5, [5000, 300])
    out, olens = audio.resample_batch(_batch(pcm, np.int16), [5000, 300], audio.hparams.sample_rate)
    assert olens == [5000, 300]
    assert np.array_equal(out.cpu().numpy()[1, :300], pcm[1].astype(np.float32) / 32768.0)
    wav = _batch(pcm, np.int16)
    with pytest.raises(Dv3Error):
        audio.resample_batch(wav.cpu(), [5000, 300], 48000)
    with pytest.raises(Dv3Error):
        audio.resample_batch(wav.to(torch.int32), [5000, 300], 48000)
    with pytest.raises(Dv3Error):
        audio.resample_batch(wav, [5000], 48000)
    with pytest.raises(Dv3Error):
        audio.trim_bounds_batch(wav, [5000, 300], 15, offsets=[10, 0])      # past the row
    with pytest.raises(Dv3Error):
        audio.trim_bounds_batch(wav, [5000, 300], [15])


def _trim_clips(seed):
    """fp32 clips at 22.05 kHz: quiet heads and tails of several lengths, segments shorter than one frame, a silent
    clip and an empty one."""
    rng = np.random.RandomState(seed)
    clips = [F.clip(seed + i, s, 22050).astype(np.float32) for i, s in enumerate([0.3, 1.0, 2.5, 0.05, 0.09, 4.0])]
    clips.append(np.zeros(3000, dtype=np.float32))
    clips.append((1e-3 * rng.randn(9000)).astype(np.float32))
    clips.append(np.zeros(0, dtype=np.float32))
    return clips


@pytest.mark.parametrize("top_db", [15, 25, 60])
@pytest.mark.parametrize("with_offsets", [False, True])
def test_trim_kernel_equals_fp64_oracle(top_db, with_offsets):
    from deepvoice3_pytorch_b200 import audio
    clips = _trim_clips(7)
    rng = np.random.RandomState(top_db)
    offs = [int(rng.randint(0, len(c) // 3 + 1)) if with_offsets else 0 for c in clips]
    lens = [len(c) - o - (int(rng.randint(0, len(c) // 4 + 1)) if with_offsets else 0) for c, o in zip(clips, offs)]
    wav = _batch([c if len(c) else np.zeros(1, np.float32) for c in clips], np.float32)
    pcm = _batch([(c * 32767).astype(np.int16) for c in clips], np.int16)
    got = audio.trim_bounds_batch(wav, lens, top_db, offs if with_offsets else None).cpu().numpy()
    got16 = audio.trim_bounds_batch(pcm, lens, [top_db] * len(clips), offs).cpu().numpy()
    for i, (c, o, n) in enumerate(zip(clips, offs, lens)):
        for g, y in ((got[i], c[o:o + n]), (got16[i], (c * 32767).astype(np.int16)[o:o + n] / 32768.0)):
            if n > 0:
                assert F.trim_margin(y, top_db) > 1e-6, (i, "a frame within 1e-6 dB of the threshold")
            assert tuple(int(v) for v in g) == audio.trim_bounds_reference(y, top_db), (i, o, n)
    assert tuple(got[-1]) == (0, 0) and tuple(got[-3]) == (0, lens[-3])


def _composition(in_dir, out_dir):
    """Per clip: GPU resampler alone -> numpy label cut -> fp64 trim oracle -> rescaling -> spectrograms_batch."""
    from deepvoice3_pytorch_b200 import audio, preprocess
    rows = []
    for idx, src, (text, spk) in preprocess.vctk_utterances(in_dir):
        pcm, sr, cut = preprocess._load_vctk(src)
        if sr != audio.hparams.sample_rate:
            out, olens = audio.resample_batch(_batch([pcm], pcm.dtype), [len(pcm)], sr)
            x = out.cpu().numpy()[0, :olens[0]]
        else:
            x = pcm.astype(np.float32) / 32768.0 if pcm.dtype == np.int16 else pcm
        off, n, top_db = F.cut_segment(x, cut)
        y = x[off:off + n]
        if n:
            assert F.trim_margin(y, top_db) > 1e-6, src
        s, e = audio.trim_bounds_reference(y, top_db)
        y = y[s:e]
        if not len(y):
            continue
        if audio.hparams.rescaling:
            y = y / np.abs(y).max() * audio.hparams.rescaling_max
        lin, mel = preprocess.spectrograms_batch([y])[0]
        np.save(os.path.join(out_dir, "vctk-spec-%05d.npy" % idx), lin, allow_pickle=False)
        np.save(os.path.join(out_dir, "vctk-mel-%05d.npy" % idx), mel, allow_pickle=False)
        rows.append(("vctk-spec-%05d.npy" % idx, "vctk-mel-%05d.npy" % idx, lin.shape[0], text, spk))
    return rows


@pytest.mark.parametrize("rescaling", [False, True])
def test_build_vctk_equals_per_clip_composition(tmp_path, rescaling, monkeypatch):
    from deepvoice3_pytorch_b200 import audio, preprocess
    monkeypatch.setattr(audio.hparams, "rescaling", rescaling)
    in_dir = str(tmp_path / "in")
    F.write_tree(in_dir)
    outs = {}
    for name, fn in (("want", lambda d: _composition(in_dir, d)),
                     ("b1", lambda d: preprocess.build_vctk_from_path(in_dir, d, batch_clips=1)),
                     ("b5", lambda d: preprocess.build_vctk_from_path(in_dir, d, num_workers=3, batch_clips=5))):
        d = str(tmp_path / name)
        os.makedirs(d)
        outs[name] = (d, fn(d))
    want_dir, want = outs["want"]
    assert len(want) == 8 and [r[4] for r in want] == [0, 0, 0, 1, 1, 2, 2, 2]
    for name in ("b1", "b5"):
        d, rows = outs[name]
        assert rows == want, name
        assert sorted(os.listdir(d)) == sorted(os.listdir(want_dir))
        for f in os.listdir(want_dir):
            assert open(os.path.join(d, f), "rb").read() == open(os.path.join(want_dir, f), "rb").read(), (name, f)


def test_vctk_output_trains_multispeaker_model(tmp_path):
    from deepvoice3_pytorch_b200 import builder, data, preprocess
    from deepvoice3_pytorch_b200.train_step import TrainStep, to_device
    in_dir, out_dir = str(tmp_path / "in"), str(tmp_path / "out")
    F.write_tree(in_dir)
    os.makedirs(out_dir)
    rows = preprocess.build_vctk_from_path(in_dir, out_dir, batch_clips=4)
    preprocess.write_metadata(rows, out_dir)
    ds = data.TrainTxtDataset(out_dir, lambda t: [ord(c) % 60 + 2 for c in t])
    assert ds.multi_speaker and len(ds) == len(rows)
    batch = to_device(data.collate([ds[i] for i in range(4)], r=1, downsample_step=4, pin=True), "cuda")
    torch.manual_seed(0)
    model = builder.deepvoice3_multispeaker(n_vocab=64, embed_dim=64, mel_dim=80, linear_dim=513, r=1,
                                            downsample_step=4, n_speakers=3, speaker_embed_dim=16, kernel_size=3,
                                            encoder_channels=128, decoder_channels=128, converter_channels=128,
                                            max_positions=512, dropout=0.0, use_memory_mask=True)
    loss = float(TrainStep(model.cuda().train(), use_graph=False).step(batch))
    assert np.isfinite(loss)
