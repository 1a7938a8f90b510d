"""GPU: training batches built from wav files (data.WavDataset -> collate_wav -> wav_batch_to_device, the targets by
audio.stft_mel_targets) equal, bit for bit and key for key, the batches of the preprocessed corpus
(preprocess.build_from_path -> TrainTxtDataset -> collate -> to_device), and train to the same parameters."""
import os

import numpy as np
import pytest
import torch

SR = 22050
SHORT, CROSS = 700, 15617            # shorter than one frame; 65 frames (crosses the 64-frame chunk of a CTA)
N_INT16 = 20


def tts(text):
    return [ord(c) % 60 + 2 for c in text]


def _write_corpus(root, seed=5):
    """LJSpeech layout: 20 int16 clips (the first two SHORT and CROSS samples long), one IEEE-float wav, one int16 wav
    at 16 kHz (resampled by audio.load_wav) and one utterance whose text is too short to be kept."""
    from scipy.io import wavfile
    rng = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, "wavs"), exist_ok=True)
    lines = []

    def text(i):
        return "utterance number %d says %s" % (i, "".join(rng.choice(list("abcdefgh "), rng.randint(0, 40))))

    for i in range(N_INT16 + 3):
        name = "LJ%03d" % i
        n = SHORT if i == 0 else CROSS if i == 1 else int(rng.randint(2000, 60000))
        t = np.arange(n) / SR
        x = 0.3 * np.sin(2 * np.pi * (200 + 40 * i) * t) + 0.05 * rng.randn(n)
        x *= 0.2 + 0.7 * rng.rand()                              # rescaling must change the bits
        if i == N_INT16:
            wavfile.write(os.path.join(root, "wavs", name + ".wav"), SR, x.astype(np.float32))
        elif i == N_INT16 + 1:
            wavfile.write(os.path.join(root, "wavs", name + ".wav"), 16000, (x * 32767).astype(np.int16))
        else:
            wavfile.write(os.path.join(root, "wavs", name + ".wav"), SR, (x * 32767).astype(np.int16))
        txt = "short" if i == N_INT16 + 2 else text(i)
        lines.append("%s|%s|%s\n" % (name, txt, txt))
    with open(os.path.join(root, "metadata.csv"), "w", encoding="utf-8") as f:
        f.writelines(lines)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """-> {rescaling: (in_dir, out_dir)}: one wav corpus preprocessed with rescaling off and on; each out_dir also has
    a 5-column train_ms/train.txt (speaker = row % 3)."""
    from deepvoice3_pytorch_b200 import audio, preprocess
    root = str(tmp_path_factory.mktemp("wavcorpus"))
    in_dir = os.path.join(root, "in")
    _write_corpus(in_dir)
    out = {}
    old = audio.hparams.rescaling
    try:
        for rescaling in (False, True):
            audio.hparams.rescaling = rescaling
            out_dir = os.path.join(root, "out%d" % rescaling)
            os.makedirs(os.path.join(out_dir, "ms"))
            rows = preprocess.build_from_path(in_dir, out_dir, batch_clips=8)
            preprocess.write_metadata(rows, out_dir)
            preprocess.write_metadata([tuple("../" + str(v) if j < 2 else v for j, v in enumerate(r)) + (i % 3,)
                                       for i, r in enumerate(rows)], os.path.join(out_dir, "ms"))
            out[rescaling] = (in_dir, out_dir)
    finally:
        audio.hparams.rescaling = old
    return out


@pytest.fixture
def rescaling(request):
    from deepvoice3_pytorch_b200 import audio
    old = audio.hparams.rescaling
    audio.hparams.rescaling = request.param
    yield request.param
    audio.hparams.rescaling = old


def _datasets(corpus, rescaling, multi):
    from deepvoice3_pytorch_b200 import data
    in_dir, out_dir = corpus[rescaling]
    wds = data.WavDataset.from_ljspeech(in_dir, tts)
    if not multi:
        return data.TrainTxtDataset(out_dir, tts), wds
    return (data.TrainTxtDataset(os.path.join(out_dir, "ms"), tts),
            data.WavDataset([it + (i % 3,) for i, it in enumerate(wds.items)], tts))


def _pair(npy, wds, idx, r, ds):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    want = to_device(data.collate([npy[i] for i in idx], r, ds, pin=True), "cuda")
    got = data.wav_batch_to_device(data.collate_wav([wds[i] for i in idx], r, ds, pin=True), "cuda", r, ds)
    return want, got


def _assert_same(want, got, what):
    assert list(got) == list(want), what
    for k in want:
        if torch.is_tensor(want[k]):
            assert got[k].device == want[k].device and got[k].dtype == want[k].dtype, (what, k)
            assert torch.equal(got[k], want[k]), "%s: key %s differs" % (what, k)
        else:
            assert np.array_equal(got[k], want[k]), (what, k)


BATCHES = {
    16: [list(range(N_INT16 - 16, N_INT16)), list(range(6, N_INT16 + 2))],   # int16 only; int16 + float + resampled
    1: [[0], [1], [N_INT16], [N_INT16 + 1], [7]],
}


@pytest.mark.gpu
@pytest.mark.parametrize("rescaling", [False, True], indirect=True)
@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("r,ds", [(1, 4), (4, 1), (2, 2)])
def test_wav_batch_equals_npy_batch(corpus, rescaling, multi, B, r, ds):
    npy, wds = _datasets(corpus, rescaling, multi)
    assert len(npy) == len(wds) == N_INT16 + 2
    assert [wds[i][2] for i in range(len(wds))] == npy.frame_lengths
    for idx in BATCHES[B]:
        want, got = _pair(npy, wds, idx, r, ds)
        torch.cuda.synchronize()
        _assert_same(want, got, "clips %s" % idx)
        assert got["y"].abs().sum() > 0 and got["mel"].abs().sum() > 0


@pytest.mark.gpu
def test_batch_dtypes_and_int16_staging(corpus):
    """The 16-clip batches cover both kernel inputs: all int16 files stay int16, a mix becomes float32."""
    from deepvoice3_pytorch_b200 import data
    _, wds = _datasets(corpus, False, False)
    assert data.collate_wav([wds[i] for i in BATCHES[16][0]])["wav"].dtype == torch.int16
    assert data.collate_wav([wds[i] for i in BATCHES[16][1]])["wav"].dtype == torch.float32
    assert wds[N_INT16][1].dtype == np.float32 and wds[N_INT16 + 1][1].dtype == np.float32


@pytest.mark.gpu
@pytest.mark.parametrize("r,ds", [(1, 4), (4, 1)])           # pad_to_bucket needs T_lin = T_dec * r * ds
def test_bucket_padding_of_wav_batch(corpus, r, ds):
    from deepvoice3_pytorch_b200 import data
    npy, wds = _datasets(corpus, False, False)
    want, got = _pair(npy, wds, BATCHES[16][1], r, ds)
    T_dec, T_text = data.batch_extents(want)[:2]
    _assert_same(data.pad_to_bucket(want, T_text + 9, T_dec + 3, r, ds),
                 data.pad_to_bucket(got, T_text + 9, T_dec + 3, r, ds), "bucket")


def _model():
    from deepvoice3_pytorch_b200 import builder
    return builder.deepvoice3(n_vocab=64, embed_dim=64, mel_dim=80, linear_dim=513, r=1, downsample_step=4,
                              kernel_size=3, encoder_channels=128, decoder_channels=128, converter_channels=128,
                              max_positions=512, dropout=0.0, use_memory_mask=True, key_projection=True,
                              value_projection=True)


def _train(batches, graph):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    torch.manual_seed(0)
    ops.rng.manual_seed(77, torch.device("cuda"))
    step = TrainStep(_model().cuda().train(), use_graph=graph)
    losses = [float(step.step(b)) for b in batches]
    torch.cuda.synchronize()
    return losses, step.arena.flat.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_training_on_wavs_equals_training_on_npy(corpus, graph):
    """Same seed, same batches: first the .npy path against itself (run-to-run bit reproducibility), then the wav
    path against it -- identical losses and parameters.  Graph mode: three batch shapes, so buckets are captured.

    The step is not bit-reproducible run to run today: the loss sums (loss.cu), bias gradients (conv.cu, tc_split.cu)
    and embedding gradients (elementwise.cu) are float atomicAdds across blocks.  While that holds the comparison
    cannot be exact, and the test reports it as an expected failure instead of comparing within a tolerance; the
    batches the two paths feed the step are compared bit for bit above."""
    npy, wds = _datasets(corpus, False, False)
    order = [list(range(0, 4)), list(range(4, 8)), list(range(8, 12)), list(range(0, 4))]
    pairs = [_pair(npy, wds, idx, 1, 4) for idx in order]
    for w, g in pairs:
        _assert_same(w, g, "training batch")
    l0, p0 = _train([w for w, _ in pairs], graph)
    l1, p1 = _train([w for w, _ in pairs], graph)
    assert np.all(np.isfinite(l0))
    if not (l0 == l1 and torch.equal(p0, p1)):
        pytest.xfail("the .npy path itself is not bit-reproducible run to run (losses %s vs %s)" % (l0, l1))
    l2, p2 = _train([g for _, g in pairs], graph)
    assert l2 == l0 and torch.equal(p2, p0)
    assert np.all(np.isfinite(l0))


@pytest.mark.gpu
def test_no_host_sync_and_graph_capture(corpus):
    from deepvoice3_pytorch_b200 import audio, data
    npy, wds = _datasets(corpus, True, False)
    host = data.collate_wav([wds[i] for i in BATCHES[16][0]], 1, 4, pin=True)
    data.wav_batch_to_device(host, "cuda", 1, 4)                 # first use: tables and filterbank upload
    torch.cuda.synchronize()
    old = audio.hparams.rescaling
    audio.hparams.rescaling = True
    try:
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = data.wav_batch_to_device(host, "cuda", 1, 4)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        want, _ = _pair(npy, wds, BATCHES[16][0], 1, 4)
        _assert_same(want, got, "sync-free")
        wav = host["wav"].cuda()
        lens = host["wav_lengths"].cuda()
        T_lin = want["y"].shape[1]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            audio.stft_mel_targets(wav, host["wav_lengths"], T_lin, 1, 4, lengths_dev=lens)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y, mel = audio.stft_mel_targets(wav, host["wav_lengths"], T_lin, 1, 4, lengths_dev=lens)
        y.fill_(-1.0)
        mel.fill_(-1.0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, want["y"]) and torch.equal(mel, want["mel"])
    finally:
        audio.hparams.rescaling = old


@pytest.mark.gpu
def test_input_checks_raise_before_launch():
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import Dv3Error
    wav = torch.zeros(2, 4096, dtype=torch.int16, device="cuda")
    lens = [4096, 3000]
    need = 1 + audio.num_frames(4096)
    with pytest.raises(Dv3Error):
        audio.stft_mel_targets(wav.to(torch.int32), lens, need, 1, 4)
    with pytest.raises(Dv3Error):
        audio.stft_mel_targets(wav.cpu(), lens, need, 1, 4)
    with pytest.raises(Dv3Error):
        audio.stft_mel_targets(wav, lens, need - 1, 1, 4)
    old = audio.hparams.hop_size
    audio.hparams.hop_size = 200
    try:
        with pytest.raises(Dv3Error):
            audio.stft_mel_targets(wav, lens, need, 1, 4)
    finally:
        audio.hparams.hop_size = old
    y, mel = audio.stft_mel_targets(wav, lens, need, 1, 4)           # one row more than the failing T_lin
    assert y.shape == (2, need, 513) and mel.shape[1] == -(-need // 4)
