"""GPU: training the multi-speaker preset straight from a VCTK tree.  The segment resampler
(audio.resample_segments, dv3_resample_segments_batched) against slices of the whole-clip resampler bit for bit, and
WavDataset.from_vctk -> collate_wav -> wav_batch_to_device against the preprocessed corpus
(build_vctk_from_path -> TrainTxtDataset -> collate -> to_device), key for key, bit for bit, through to identical
deterministic training."""
import os

import numpy as np
import pytest
import torch

import vctk_fixtures as F

pytestmark = pytest.mark.gpu


def tts(text):
    return [ord(c) % 60 + 2 for c in text]


def _rows(clips, dtype, pitch=None):
    pitch = pitch or max(1, max(len(c) for c in clips)) + 3                # an odd pitch: no alignment assumed
    x = np.zeros((len(clips), pitch), dtype=dtype)
    for i, c in enumerate(clips):
        x[i, :len(c)] = c
    return torch.from_numpy(x).cuda()


def _segments(rng, n_out):
    """Random segments of an n_out-sample output plus the edge cases: empty, one sample, touching either end, whole."""
    segs = [(0, 0), (n_out, 0), (0, 1), (n_out - 1, 1), (0, n_out), (0, n_out // 3), (n_out - n_out // 4, n_out // 4)]
    for _ in range(6):
        a = int(rng.randint(0, n_out))
        segs.append((a, int(rng.randint(0, n_out - a + 1))))
    return [(a, n) for a, n in segs if 0 <= a and n >= 0 and a + n <= n_out]


SOURCES = [48000, 44100, 16000, 22050]


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_segments_equal_slices_of_whole_clip_output(dtype):
    from deepvoice3_pytorch_b200 import audio, data
    rng = np.random.RandomState(11)
    lens = {48000: [1, 999, 48000, 30011], 44100: [7, 20000], 16000: [5000, 1], 22050: [4000, 17]}
    clips = {sr: [(np.clip(F.clip(sr + i, n / sr, sr), -1, 1) * 32767).astype(np.int16) for i, n in enumerate(ns)]
             for sr, ns in lens.items()}
    if dtype == np.float32:
        clips = {sr: [c.astype(np.float32) / 32768.0 for c in cs] for sr, cs in clips.items()}
    full = {}
    for sr, cs in clips.items():
        out, olens = audio.resample_batch(_rows(cs, dtype), [len(c) for c in cs], sr)
        full[sr] = (out.cpu().numpy(), olens)
    # one batch mixing every rate: each clip appears with several segments, with a full row and with its span only
    jobs = []
    for sr, cs in clips.items():
        for c, x, n_out in zip(cs, full[sr][0], full[sr][1]):
            for s0, n in _segments(rng, n_out):
                a, m = data.segment_span(len(c), s0, n, sr)
                jobs.append((sr, c, x, s0, n, 0, len(c)))
                jobs.append((sr, c, x, s0, n, a, m))
    order = rng.permutation(len(jobs))
    jobs = [jobs[i] for i in order]
    src = _rows([j[1][j[5]:j[5] + j[6]] for j in jobs], dtype)
    pitch_out = max(j[4] for j in jobs) + 5
    out = torch.full((len(jobs), pitch_out), float("nan"), device="cuda")
    for sr in SOURCES:
        seg = [[r, len(j[1]), j[5], j[6], j[3], j[4]] for r, j in enumerate(jobs) if j[0] == sr]
        audio.resample_segments(src, seg, sr, out)
    got = out.cpu().numpy()
    for r, (sr, c, x, s0, n, a, m) in enumerate(jobs):
        assert np.array_equal(got[r, :n].view(np.int32), x[s0:s0 + n].view(np.int32)), (sr, len(c), s0, n, a, m)
        assert not got[r, n:].any(), (sr, s0, n)
        if sr == 22050:                             # the identity: an exact copy of x / 32768
            want = c[s0:s0 + n].astype(np.float32) / (32768.0 if dtype == np.int16 else 1.0)
            assert np.array_equal(got[r, :n], want)
    # a clip alone == the same clip in the batch
    r = int(np.argmax([j[4] for j in jobs]))
    sr, c, x, s0, n, a, m = jobs[r]
    alone = torch.zeros(1, n + 1, device="cuda")
    audio.resample_segments(_rows([c[a:a + m]], dtype), [[0, len(c), a, m, s0, n]], sr, alone)
    assert np.array_equal(alone.cpu().numpy()[0, :n].view(np.int32), got[r, :n].view(np.int32))


def test_input_checks_raise_before_launch():
    from deepvoice3_pytorch_b200 import audio, data
    from deepvoice3_pytorch_b200._lib import Dv3Error, lib
    c = (F.clip(1, 0.5) * 32767).astype(np.int16)
    n_out = audio.resampled_length(len(c), *audio.resample_ratio(48000))
    a, m = data.segment_span(len(c), 1000, 2000, 48000)
    src = _rows([c[a:a + m]], np.int16)
    out = torch.zeros(1, 4096, device="cuda")
    ok = [0, len(c), a, m, 1000, 2000]
    audio.resample_segments(src, [ok], 48000, out)                 # first use: the filter bank upload
    torch.cuda.synchronize()
    bad = [
        [0, len(c), a, m, n_out - 100, 200],                           # segment past the clip's output
        [0, len(c), a, m, -1, 10],                                     # negative start
        [0, len(c), a, m, 0, 5000],                                    # longer than the output rows
        [0, len(c), a + 1, m - 1, 1000, 2000],                         # span misses the first input the segment reads
        [0, len(c), a, m - 1, 1000, 2000],                             # ... or the last
        [0, len(c), a, m + 10 ** 6, 1000, 2000],                       # span past the row
        [0, a + m - 1, a, m, 1000, 100],                               # span past the clip
        [1, len(c), a, m, 1000, 2000],                                 # no such row
    ]
    n0 = lib.raw("dv3_launch_count")()
    for seg in bad:
        with pytest.raises(Dv3Error):
            audio.resample_segments(src, [seg], 48000, out)
    with pytest.raises(Dv3Error):
        audio.resample_segments(src, [ok, ok], 48000, torch.zeros(2, 4096, device="cuda"))      # rows shared
    with pytest.raises(Dv3Error):
        audio.resample_segments(src.to(torch.int32), [ok], 48000, out)                          # wav dtype
    with pytest.raises(Dv3Error):
        audio.resample_segments(src, [ok], 48000, out.double())                                 # out dtype
    with pytest.raises(Dv3Error):
        audio.resample_segments(src, [ok], 48000, out, seg_dev=torch.tensor([ok], device="cuda"))   # int64 desc
    with pytest.raises(Dv3Error):
        audio.resample_segments(src.cpu(), [ok], 48000, out)
    with pytest.raises(Dv3Error):
        audio.resample_segments(src, [ok[:5]], 48000, out)
    assert lib.raw("dv3_launch_count")() == n0


# ---- the dataset against the preprocessed corpus ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """-> {rescaling: (in_dir, out_dir)}: the fixture tree preprocessed by build_vctk_from_path, rescaling off and on."""
    from deepvoice3_pytorch_b200 import audio, preprocess
    root = str(tmp_path_factory.mktemp("vctkwav"))
    in_dir = os.path.join(root, "in")
    F.write_tree(in_dir)
    out = {}
    old = audio.hparams.rescaling
    try:
        for rescaling in (False, True):
            audio.hparams.rescaling = rescaling
            out_dir = os.path.join(root, "out%d" % rescaling)
            os.makedirs(out_dir)
            preprocess.write_metadata(preprocess.build_vctk_from_path(in_dir, out_dir, batch_clips=3), out_dir)
            out[rescaling] = (in_dir, out_dir)
    finally:
        audio.hparams.rescaling = old
    return out


@pytest.fixture
def rescaling(request, monkeypatch):
    from deepvoice3_pytorch_b200 import audio
    monkeypatch.setattr(audio.hparams, "rescaling", request.param)
    return request.param


def _datasets(tree, rescaling):
    from deepvoice3_pytorch_b200 import data
    in_dir, out_dir = tree[rescaling]
    return data.TrainTxtDataset(out_dir, tts), data.WavDataset.from_vctk(in_dir, tts, batch_clips=4)


def _pair(npy, wds, idx, r, ds, pin=True):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    want = to_device(data.collate([npy[i] for i in idx], r, ds, pin=pin), "cuda")
    got = data.wav_batch_to_device(data.collate_wav([wds[i] for i in idx], r, ds, pin=pin), "cuda", r, ds)
    return want, got


def _assert_same(want, got, what):
    assert list(got) == list(want), what
    for k in want:
        if torch.is_tensor(want[k]):
            assert got[k].device == want[k].device and got[k].dtype == want[k].dtype, (what, k)
            assert torch.equal(got[k], want[k]), "%s: key %s differs" % (what, k)
        else:
            assert np.array_equal(got[k], want[k]), (what, k)


@pytest.mark.parametrize("rescaling", [False, True], indirect=True)
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("r,ds", [(1, 4), (4, 1), (2, 2)])
def test_wav_batch_equals_npy_batch(tree, rescaling, B, r, ds):
    npy, wds = _datasets(tree, rescaling)
    assert len(npy) == len(wds) == 8
    assert wds.frame_lengths == npy.frame_lengths
    assert [it[2] for it in wds.items] == [int(row[4]) for row in npy.rows]
    assert [it[1] for it in wds.items] == [row[3] for row in npy.rows]
    kinds = {(wds[i].sample_rate, wds[i].pcm.dtype.name) for i in range(len(wds))}
    assert kinds == {(48000, "int16"), (48000, "float32"), (22050, "int16")}
    for idx in ([[i] for i in range(len(wds))] if B == 1 else [list(range(8)), [7, 4, 0, 3, 5]]):
        want, got = _pair(npy, wds, idx, r, ds)
        torch.cuda.synchronize()
        _assert_same(want, got, "utterances %s" % idx)
        assert got["y"].abs().sum() > 0 and got["mel"].abs().sum() > 0


@pytest.mark.parametrize("r,ds", [(1, 4), (4, 1)])                 # pad_to_bucket needs T_lin = T_dec * r * ds
def test_bucket_padding_of_wav_batch(tree, r, ds):
    from deepvoice3_pytorch_b200 import data
    npy, wds = _datasets(tree, False)
    want, got = _pair(npy, wds, list(range(8)), r, ds)
    T_dec, T_text = data.batch_extents(want)[:2]
    T_text_b, T_dec_b = data.bucket_shape(T_text + 1, T_dec + 1)
    _assert_same(data.pad_to_bucket(want, T_text_b, T_dec_b, r, ds),
                 data.pad_to_bucket(got, T_text_b, T_dec_b, r, ds), "bucket")


def test_no_host_sync_and_graph_capture(tree, monkeypatch):
    from deepvoice3_pytorch_b200 import audio, data
    monkeypatch.setattr(audio.hparams, "rescaling", True)
    npy, wds = _datasets(tree, True)
    idx = list(range(8))
    host = data.collate_wav([wds[i] for i in idx], 1, 4, pin=True)
    data.wav_batch_to_device(host, "cuda", 1, 4)                 # first use: filter banks, tables, mel basis
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = data.wav_batch_to_device(host, "cuda", 1, 4)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want, _ = _pair(npy, wds, idx, 1, 4)
    _assert_same(want, got, "sync-free")
    # the device part, captured: inputs already on the device, the graph resamples and builds the targets again
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in host.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _device_part(host, dev)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y, mel = _device_part(host, dev)
    y.fill_(-1.0)
    mel.fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, want["y"]) and torch.equal(mel, want["mel"])


def _device_part(host, dev):
    """wav_batch_to_device's launches on inputs already on the device (dev), checked against the host batch's values:
    one segment launch per rate, then the targets."""
    from deepvoice3_pytorch_b200 import audio, data
    lens = host["wav_lengths"].tolist()
    out = torch.empty(len(lens), max(8, -(-max(lens) // 8) * 8), device="cuda")
    desc, rates = host["src_desc"].tolist(), host["src_rates"].tolist()
    for sr in sorted(set(rates)):
        rows = [i for i, x in enumerate(rates) if x == sr]
        audio.resample_segments(dev["wav"], [desc[i] for i in rows], sr, out,
                                seg_dev=dev["src_desc"][rows[0]:rows[-1] + 1])
    T_lin = data.max_target_length(host["target_lengths"].tolist(), 1, 4)
    return audio.stft_mel_targets(out, lens, T_lin, 1, 4, lengths_dev=dev["wav_lengths"])


def test_collate_refuses_mixed_items(tree):
    from deepvoice3_pytorch_b200 import data
    _, wds = _datasets(tree, False)
    it = wds[0]
    whole = (it.text_ids, np.zeros(3000, np.int16), data._num_frames(3000), 0)
    with pytest.raises(ValueError):
        data.collate_wav([it, whole])
    with pytest.raises(ValueError):
        data.collate_wav([whole, it])


# ---- training ----------------------------------------------------------------------------------------------------------
def _train(batches, graph):
    from bench import PRESETS
    from deepvoice3_pytorch_b200 import builder, ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    bname, kw, extra = PRESETS["deepvoice3_vctk"]
    torch.manual_seed(0)
    ops.rng.manual_seed(77, torch.device("cuda"))
    step = TrainStep(getattr(builder, bname)(**kw).cuda().train(), use_graph=graph, **extra)
    losses = [float(step.step(b)) for b in batches]
    torch.cuda.synchronize()
    return losses, step.arena.flat.clone()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_training_on_vctk_wavs_equals_training_on_npy(tree, graph, monkeypatch):
    """deepvoice3_vctk, deterministic mode, three batch shapes (graph mode captures buckets): identical losses and
    parameters from the wav source and from the npy source."""
    from deepvoice3_pytorch_b200 import ops
    monkeypatch.setattr(ops, "deterministic", "1")
    npy, wds = _datasets(tree, False)
    order = [[0, 1, 2, 3], [4, 5, 6, 7], [1, 6], [0, 1, 2, 3]]
    pairs = [_pair(npy, wds, idx, 1, 4) for idx in order]
    for w, g in pairs:
        _assert_same(w, g, "training batch")
    l0, p0 = _train([w for w, _ in pairs], graph)
    l1, p1 = _train([g for _, g in pairs], graph)
    assert np.all(np.isfinite(l0))
    assert l1 == l0 and torch.equal(p1, p0)
