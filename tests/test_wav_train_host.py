"""Host side of training from wav files (no GPU): collate_wav's shared keys, WavDataset's selection and header-derived
lengths, the Python frame count, the float32 rescale the kernel restates, and a ptxas guard of the new STFT
instantiations."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tts(text):
    return [ord(c) % 60 + 2 for c in text]


@pytest.mark.parametrize("r,ds", [(1, 4), (4, 1), (2, 2), (3, 2)])
@pytest.mark.parametrize("multi", [False, True])
def test_collate_wav_shares_collate_keys(r, ds, multi):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.audio import num_frames_host
    rng = np.random.RandomState(r * 10 + ds)
    wav_items, npy_items = [], []
    for i, n in enumerate([700, 15617, 4000, 33333, 1024]):
        ids = rng.randint(2, 60, rng.randint(5, 40)).astype(np.int32)
        pcm = rng.randint(-3000, 3000, n).astype(np.int16) if i != 2 else rng.rand(n).astype(np.float32)
        T = num_frames_host(n)
        w, p = (ids, pcm, T), (ids, np.zeros((T, 80), np.float32), np.zeros((T, 513), np.float32))
        wav_items.append(w + (i,) if multi else w)
        npy_items.append(p + (i,) if multi else p)
    want = data.collate(npy_items, r, ds)
    got = data.collate_wav(wav_items, r, ds, pin=False)
    assert [k for k in got if k not in ("wav", "wav_lengths")] == [k for k in want if k not in ("mel", "y")]
    for k in want:
        if k in ("mel", "y"):
            continue
        if torch.is_tensor(want[k]):
            assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
        else:
            assert np.array_equal(got[k], want[k]), k
    assert want["y"].shape[1] == data.max_target_length(got["target_lengths"].tolist(), r, ds)
    wav, lens = got["wav"], got["wav_lengths"]
    assert wav.dtype == torch.float32 and wav.shape[1] % 8 == 0 and lens.tolist() == [len(w[1]) for w in wav_items]
    for i, w in enumerate(wav_items):                         # int16 -> / 32768 exactly, zero padding
        x = w[1].astype(np.float32) / np.float32(32768.0) if w[1].dtype == np.int16 else w[1]
        assert np.array_equal(wav[i, :len(x)].numpy(), x) and not wav[i, len(x):].any()
    only16 = data.collate_wav([w for w in wav_items if w[1].dtype == np.int16], r, ds)
    assert only16["wav"].dtype == torch.int16


def test_collate_wav_rejects_wrong_frame_count():
    from deepvoice3_pytorch_b200 import data
    with pytest.raises(ValueError):
        data.collate_wav([(np.arange(5, dtype=np.int32), np.zeros(3000, np.int16), 7)])


def test_num_frames_host_equals_library():
    from deepvoice3_pytorch_b200 import audio
    for n in list(range(0, 3000)) + [15617, 65536, 220500, 10 ** 6 + 7]:
        assert audio.num_frames_host(n) == audio.num_frames(n), n


def _write_wavs(root):
    from scipy.io import wavfile
    rng = np.random.RandomState(3)
    os.makedirs(os.path.join(root, "wavs"))
    lines = []
    specs = [(22050, np.int16, 5000), (22050, np.float32, 7001), (16000, np.int16, 3333), (22050, np.int16, 11),
             (44100, np.int16, 9999), (22050, np.int16, 60000)]
    for i, (sr, dt, n) in enumerate(specs):
        x = rng.randint(-2000, 2000, n).astype(np.int16) if dt == np.int16 else (0.1 * rng.randn(n)).astype(dt)
        wavfile.write(os.path.join(root, "wavs", "U%d.wav" % i), sr, x)
        text = "x" * (10 if i == 3 else 25 + i)                  # utterance 3 falls under min_text
        lines.append("U%d|%s|%s\n" % (i, text, text))
    with open(os.path.join(root, "metadata.csv"), "w", encoding="utf-8") as f:
        f.writelines(lines)


def test_from_ljspeech_matches_build_from_path(tmp_path, monkeypatch):
    """Order, min_text filter, texts and frame counts of WavDataset.from_ljspeech == the rows build_from_path writes
    (its spectrogram batch replaced by zero arrays of the right shape, so this runs without a GPU)."""
    from deepvoice3_pytorch_b200 import audio, data, preprocess
    _write_wavs(str(tmp_path))
    monkeypatch.setattr(preprocess, "spectrograms_batch", lambda wavs: [
        (np.zeros((audio.num_frames_host(len(w)), 513), np.float32),
         np.zeros((audio.num_frames_host(len(w)), 80), np.float32)) for w in wavs])
    out = tmp_path / "out"
    out.mkdir()
    rows = preprocess.build_from_path(str(tmp_path), str(out), batch_clips=2)
    ds = data.WavDataset.from_ljspeech(str(tmp_path), tts)
    assert len(ds) == len(rows) == 5
    assert [it[1] for it in ds.items] == [r[3] for r in rows]
    assert ds.frame_lengths == [r[2] for r in rows]
    for i in range(len(ds)):
        ids, pcm, T = ds[i]
        assert T == audio.num_frames_host(len(pcm)) == ds.frame_lengths[i]
        assert np.array_equal(ids, np.asarray(tts(rows[i][3]), np.int32))


def test_header_lengths_equal_decoded_lengths(tmp_path):
    from deepvoice3_pytorch_b200 import audio, data
    _write_wavs(str(tmp_path))
    paths = sorted(os.path.join(tmp_path, "wavs", f) for f in os.listdir(os.path.join(tmp_path, "wavs")))
    ds = data.WavDataset([(p, "text", i % 2) for i, p in enumerate(paths)], tts)
    assert ds.multi_speaker
    for i, p in enumerate(paths):
        decoded = audio.load_wav(p)
        assert ds.frame_lengths[i] == audio.num_frames_host(len(decoded)), p
        ids, pcm, T, spk = ds[i]
        assert spk == i % 2 and len(pcm) == len(decoded)
        assert np.array_equal(pcm.astype(np.float32) / np.float32(32768.0) if pcm.dtype == np.int16 else pcm, decoded)
    kinds = [ds[i][1].dtype for i in range(len(paths))]
    assert kinds.count(np.int16) == 3                            # 16-bit mono at 22050 Hz stays int16
    one = data.WavDataset([(p, "t", i % 2) for i, p in enumerate(paths)], tts, speaker_id=1)
    assert len(one) == len(paths) // 2 and len(one[0]) == 3


def test_rescale_is_float32_divide_then_multiply(tmp_path):
    """preprocess._load's rescale == x / peak * float32(rescaling_max), each correctly rounded in float32: what the
    kernel computes with __fdiv_rn / __fmul_rn."""
    from scipy.io import wavfile
    from deepvoice3_pytorch_b200 import audio, preprocess
    rng = np.random.RandomState(1)
    x = rng.randint(-20000, 20000, 50000).astype(np.int16)
    p = str(tmp_path / "a.wav")
    wavfile.write(p, 22050, x)
    old = audio.hparams.rescaling
    audio.hparams.rescaling = True
    try:
        got = preprocess._load(p)
    finally:
        audio.hparams.rescaling = old
    f = x.astype(np.float32) / np.float32(32768.0)
    want = (f / np.abs(f).max()).astype(np.float32) * np.float32(audio.hparams.rescaling_max)
    assert got.dtype == np.float32 and np.array_equal(got, want)


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


def test_stft_kernels_no_spills_no_stack(tmp_path):
    """Every stft_mel_kernel instantiation (fp32 / int16 input, with and without the rescale) and the peak kernel:
    no spills, 0-byte stack frame."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "stft.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "stft.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    kernels, cur = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if ("stft_mel_kernel" in m.group(1) or "peak_abs_kernel" in m.group(1)) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            kernels[cur] = tuple(int(v) for v in m.groups())
            cur = None
    assert len([k for k in kernels if "stft_mel_kernel" in k]) == 4, kernels
    assert len([k for k in kernels if "peak_abs_kernel" in k]) == 2, kernels
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, "stack / spill bytes: %s" % bad
