"""CPU: the host side of VCTK preprocessing.  The resampler's filter bank with the kernel's polyphase indexing restated
in numpy against scipy's resample_poly; the fp64 trim restatement (the kernel's oracle) against a direct transcription
of its definition; HTS label parsing and the reference's start_at / end_at; the corpus walk, file names, rows and a
gloo world-2 sharded run, with the GPU stages replaced by host stand-ins."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp
from scipy.signal import resample_poly

import vctk_fixtures as F

RATES = [(48000, 22050), (44100, 22050), (16000, 22050), (24000, 22050), (22050, 16000)]


def polyphase(x, bank, pre_remove, up, down):
    """csrc/resample.cu's indexing: output m sums bank[j, p] * x[b - j] with t = (m + pre_remove) * down, p = t % up,
    b = t // up, x = 0 outside the clip."""
    from deepvoice3_pytorch_b200 import audio
    n = len(x)
    m = np.arange(audio.resampled_length(n, up, down))
    t = (m + pre_remove) * down
    p, b = t % up, t // up
    y = np.zeros(len(m))
    for j in range(bank.shape[0]):
        idx = b - j
        ok = (idx >= 0) & (idx < n)
        y += bank[j, p] * np.where(ok, x[np.clip(idx, 0, n - 1)], 0.0)
    return y


@pytest.mark.parametrize("sr_from,sr_to", RATES)
def test_filter_bank_matches_resample_poly(sr_from, sr_to):
    from deepvoice3_pytorch_b200 import audio
    up, down = audio.resample_ratio(sr_from, sr_to)
    bank, pre_remove = audio.resample_filter_bank(up, down)
    assert bank.shape[1] == up and bank.dtype == np.float64
    rng = np.random.RandomState(up + down)
    for n in (1, 7, 1000, 48000, 100003):
        x = rng.uniform(-1, 1, n)
        want = resample_poly(x, up, down)
        got = polyphase(x, bank, pre_remove, up, down)
        assert got.shape == want.shape
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def test_filter_bank_size_for_48k():
    from deepvoice3_pytorch_b200 import audio
    up, down = audio.resample_ratio(48000, 22050)
    bank, _ = audio.resample_filter_bank(up, down)
    assert (up, down) == (147, 320) and bank.shape == (46, 147) and bank.nbytes < 56 * 1024


def test_reflect_index_equals_numpy_pad():
    from deepvoice3_pytorch_b200 import audio
    for L in range(2, 3001):
        y = np.arange(L)
        assert np.array_equal(y[audio.reflect_index(np.arange(-1024, L + 1024), L)], np.pad(y, 1024, mode="reflect")), L


def _trim_direct(y, top_db):
    """The definition transcribed without the index map: np.pad(reflect), frames of 2048 every 512, power in dB."""
    y = np.asarray(y, dtype=np.float64)
    padded = np.pad(y, 1024, mode="reflect")
    mse = np.array([np.mean(padded[512 * f: 512 * f + 2048] ** 2) for f in range(len(y) // 512 + 1)])
    db = 10 * np.log10(np.maximum(1e-10, mse)) - 10 * np.log10(np.maximum(1e-10, mse.max()))
    nz = np.flatnonzero(db > -top_db)
    return (0, 0) if nz.size == 0 else (int(512 * nz[0]), int(min(len(y), 512 * (nz[-1] + 1))))


def test_trim_reference_hand_built_cases():
    from deepvoice3_pytorch_b200 import audio
    tone = np.sin(np.arange(20000) * 0.05)
    assert audio.trim_bounds_reference(np.zeros(0), 15) == (0, 0)
    assert audio.trim_bounds_reference(tone, 0) == (0, 0)                  # no frame lies above max - 0 dB
    assert audio.trim_bounds_reference(np.zeros(5000), 15) == (0, 5000)    # every frame equals the (zero) maximum
    head = tone.copy()
    head[:10000] = 0
    assert audio.trim_bounds_reference(head, 15) == (9216, 20000)          # frame 18 is the first to reach sample 10000
    tail = tone.copy()
    tail[10000:] = 0
    assert audio.trim_bounds_reference(tail, 15) == (0, 11264)             # frame 21, [9728, 11776), is the last
    assert audio.trim_bounds_reference(tone[:1500], 25) == (0, 1500)       # shorter than one frame


def test_trim_reference_equals_direct_definition():
    from deepvoice3_pytorch_b200 import audio
    for seed in range(6):
        y = F.clip(seed, 0.2 + 0.3 * seed, 22050)
        for L in (len(y), 700, 2047, 3000):
            for top_db in (15, 25, 60):
                assert audio.trim_bounds_reference(y[:L], top_db) == _trim_direct(y[:L], top_db), (seed, L, top_db)


def test_labels_and_cut(tmp_path):
    from deepvoice3_pytorch_b200 import preprocess
    p = tmp_path / "a.lab"
    p.write_text("0 2500000 pau\n2500000 6000000 h\n6000000 9500000 iy\n9500000 12000000 pau\n")
    labels = preprocess.load_labels(str(p))
    assert labels[1] == (2500000, 6000000, "h")
    assert preprocess.start_at(labels) == 2500000 and preprocess.end_at(labels) == 9500000
    assert preprocess.label_cut(str(p), 22050) == (int(2500000 * 1e-7 * 22050), int(9500000 * 1e-7 * 22050))
    assert preprocess.start_at([(0, 5, "a"), (5, 9, "pau")]) == 0 and preprocess.end_at([(0, 5, "a"), (5, 9, "b")]) == 9
    with pytest.raises(ValueError):                        # vctk.py:46 never looks at the first label
        preprocess.end_at([(0, 5, "a"), (5, 9, "pau")])
    q = tmp_path / "silent.lab"
    q.write_text("0 100 pau\n100 200 pau\n")
    with pytest.raises(ValueError, match="silent.lab"):
        preprocess.label_cut(str(q), 22050)


def host_resample_trim(clips):
    """Host stand-in of preprocess.resample_trim_batch: scipy fp64 resample_poly -> fp32, the label cut, the fp64 trim
    restatement."""
    from deepvoice3_pytorch_b200 import audio
    out = []
    for pcm, sr, cut in clips:
        x = pcm.astype(np.float32) / 32768.0 if pcm.dtype == np.int16 else pcm.astype(np.float32)
        if sr != audio.hparams.sample_rate:
            up, down = audio.resample_ratio(sr)
            x = resample_poly(x.astype(np.float64), up, down).astype(np.float32)
        off, n, top_db = F.cut_segment(x, cut)
        y = x[off:off + n]
        s, e = audio.trim_bounds_reference(y, top_db)
        out.append(y[s:e].copy())
    return out


def oracle_spectrograms(wavs):
    from oracle import audio_oracle as A
    return [A.process_utterance(w) for w in wavs]


def _stand_ins(preprocess):
    preprocess.resample_trim_batch = host_resample_trim
    preprocess.spectrograms_batch = oracle_spectrograms


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, in_dir, out_dir, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from deepvoice3_pytorch_b200 import preprocess
    _stand_ins(preprocess)
    ret[rank] = preprocess.build_vctk_from_path(in_dir, out_dir, num_workers=2, batch_clips=2)
    dist.barrier()
    dist.destroy_process_group()


def test_corpus_walk_and_sharded_run(tmp_path):
    from deepvoice3_pytorch_b200 import preprocess
    in_dir, out1, out2 = str(tmp_path / "in"), str(tmp_path / "one"), str(tmp_path / "two")
    F.write_tree(in_dir)
    os.makedirs(out1)
    os.makedirs(out2)
    items = preprocess.vctk_utterances(in_dir)
    stems = [os.path.basename(src[0])[:-4] for _, src, _ in items]
    assert stems == ["p225_001", "p225_002", "p225_003", "p226_001", "p226_002",
                     "p301_001", "p301_002", "p301_003", "p301_004"]          # p226_003 has no wav, p315 no txt
    assert [i for i, _, _ in items] == list(range(1, 10))
    assert [t[1] for _, _, t in items] == [0, 0, 0, 1, 1, 2, 2, 2, 2]
    assert [src[1] is not None for _, src, _ in items] == [True, False, True, False, False, False, True, True, False]
    assert items[4][2][0] == "Ça va, Zoë? naïve café." and items[0][2][0] == "Please call Stella."
    only = preprocess.vctk_utterances(in_dir, speakers=["p301", "225"])
    assert [t[1] for _, _, t in only] == [0, 0, 0, 0, 1, 1, 1]

    saved = preprocess.resample_trim_batch, preprocess.spectrograms_batch
    _stand_ins(preprocess)
    try:
        single = preprocess.build_vctk_from_path(in_dir, out1, batch_clips=4, rank=0, world=1)
    finally:
        preprocess.resample_trim_batch, preprocess.spectrograms_batch = saved
    # p301_002 (index 7): its label cut lies past the end of the audio -- no files, no row, index 7 stays unused
    assert [r[0] for r in single] == ["vctk-spec-%05d.npy" % i for i in (1, 2, 3, 4, 5, 6, 8, 9)]
    assert [r[1] for r in single] == ["vctk-mel-%05d.npy" % i for i in (1, 2, 3, 4, 5, 6, 8, 9)]
    assert [r[4] for r in single] == [0, 0, 0, 1, 1, 2, 2, 2]
    assert single[4][3] == "Ça va, Zoë? naïve café."
    assert not os.path.exists(os.path.join(out1, "vctk-spec-00007.npy"))

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), in_dir, out2, ret), nprocs=2, join=True)
    assert ret[0] == single and ret[1] == single
    for spec_name, mel_name, n_frames, _, _ in single:
        for name, width in ((spec_name, 513), (mel_name, 80)):
            a, b = np.load(os.path.join(out1, name)), np.load(os.path.join(out2, name))
            assert a.shape == (n_frames, width) and a.dtype == np.float32 and np.array_equal(a, b)
    preprocess.write_metadata(single, out1)
    from deepvoice3_pytorch_b200 import data
    ds = data.TrainTxtDataset(out1, lambda t: [ord(c) % 60 + 2 for c in t])
    assert ds.multi_speaker and len(ds) == 8 and ds[4][3] == 1
