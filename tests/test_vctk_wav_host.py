"""CPU: the host side of training from a VCTK tree (data.WavDataset.from_vctk).  The input-span rule against brute
force, the index and its cache keying, a gloo world-2 sharded index pass, collate_wav on segment items, the C ABI of
dv3_resample_segments_batched and a ptxas guard of the resampling kernel.  The GPU bounds pass
(preprocess.segment_bounds) is replaced by a host restatement."""
import ctypes
import os
import re
import shutil
import socket
import subprocess

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from scipy.signal import resample_poly

import vctk_fixtures as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tts(text):
    return [ord(c) % 60 + 2 for c in text]


def _brute_span(n_in, s0, n, up, down, ntaps, pre_remove):
    """Every input sample in [0, n_in) that outputs [s0, s0 + n) read, enumerated tap by tap."""
    reads = set()
    for m in range(s0, s0 + n):
        b = (m + pre_remove) * down // up
        reads.update(s for s in range(b - ntaps + 1, b + 1) if 0 <= s < n_in)
    return (min(reads), max(reads) + 1 - min(reads)) if reads else (0, 0)


@pytest.mark.parametrize("sr_from", [48000, 16000, 44100, 22050, 24000])
def test_input_span_equals_brute_force(sr_from):
    from deepvoice3_pytorch_b200 import audio
    up, down = audio.resample_ratio(sr_from, 22050)
    bank, pre_remove = audio.resample_filter_bank(up, down)
    ntaps = bank.shape[0]
    rng = np.random.RandomState(sr_from % 1000)
    cases = [(1, 0, 1), (5, 0, 0), (3000, 0, audio.resampled_length(3000, up, down))]
    for _ in range(60):
        n_in = int(rng.choice([1, 2, 50, 700, 5000]))
        n_out = audio.resampled_length(n_in, up, down)
        s0 = int(rng.randint(0, n_out + 1))
        cases.append((n_in, s0, int(rng.randint(0, min(n_out - s0, 400) + 1))))
        cases.append((n_in, max(0, n_out - 3), min(n_out, 3)))          # touching the end
    for n_in, s0, n in cases:
        got = audio.input_span(n_in, s0, n, up, down, ntaps, pre_remove)
        assert got == _brute_span(n_in, s0, n, up, down, ntaps, pre_remove), (n_in, s0, n)


def test_span_gives_the_segment_of_resample_poly():
    """Resampling only the span (zeros outside it) in fp64 reproduces the segment of the whole clip's output: the span
    covers everything the segment reads."""
    from deepvoice3_pytorch_b200 import data
    from test_vctk_host import polyphase
    from deepvoice3_pytorch_b200 import audio
    rng = np.random.RandomState(2)
    x = rng.uniform(-1, 1, 4801)
    for sr in (48000, 16000, 22050):
        up, down = audio.resample_ratio(sr)
        bank, pre_remove = audio.resample_filter_bank(up, down)
        whole = polyphase(x, bank, pre_remove, up, down)
        for s0, n in ((0, 1), (37, 500), (len(whole) - 200, 200), (0, len(whole))):
            a, m = data.segment_span(len(x), s0, n, sr)
            part = np.zeros_like(x)
            part[a:a + m] = x[a:a + m]
            assert np.array_equal(polyphase(part, bank, pre_remove, up, down)[s0:s0 + n], whole[s0:s0 + n])
    assert np.allclose(resample_poly(x, *audio.resample_ratio(48000)), polyphase(x, *_bank(48000)), atol=1e-12)


def _bank(sr):
    from deepvoice3_pytorch_b200 import audio
    up, down = audio.resample_ratio(sr)
    bank, pre_remove = audio.resample_filter_bank(up, down)
    return bank, pre_remove, up, down


def host_bounds(clips):
    """Host stand-in of preprocess.segment_bounds: scipy fp64 resample_poly -> fp32, the label cut, the fp64 trim."""
    from deepvoice3_pytorch_b200 import audio
    out = []
    for pcm, sr, cut in clips:
        x = pcm.astype(np.float32) / 32768.0 if pcm.dtype == np.int16 else pcm.astype(np.float32)
        if sr != audio.hparams.sample_rate:
            x = resample_poly(x.astype(np.float64), *audio.resample_ratio(sr)).astype(np.float32)
        off, n, top_db = F.cut_segment(x, cut)
        s, e = audio.trim_bounds_reference(x[off:off + n], top_db)
        out.append((off + s, e - s))
    return out


@pytest.fixture
def counted_bounds(monkeypatch):
    from deepvoice3_pytorch_b200 import preprocess
    calls = []

    def bounds(clips):
        calls.append(len(clips))
        return host_bounds(clips)
    monkeypatch.setattr(preprocess, "segment_bounds", bounds)
    return calls


def test_index_matches_build_rows(tmp_path, counted_bounds):
    """Order, texts, speaker ids, dropped utterance and frame counts == the rows build_vctk_from_path writes with the
    same bounds (its GPU stages replaced by host stand-ins); items carry their spans."""
    from deepvoice3_pytorch_b200 import audio, data, preprocess
    from test_vctk_host import host_resample_trim, oracle_spectrograms
    in_dir = str(tmp_path / "in")
    F.write_tree(in_dir)
    saved = preprocess.resample_trim_batch, preprocess.spectrograms_batch
    preprocess.resample_trim_batch, preprocess.spectrograms_batch = host_resample_trim, oracle_spectrograms
    try:
        out = tmp_path / "out"
        out.mkdir()
        rows = preprocess.build_vctk_from_path(in_dir, str(out), batch_clips=4)
    finally:
        preprocess.resample_trim_batch, preprocess.spectrograms_batch = saved
    ds = data.WavDataset.from_vctk(in_dir, tts, batch_clips=4)
    assert counted_bounds == [4, 4, 1]
    assert len(ds) == len(rows) == 8 and ds.frame_lengths == [r[2] for r in rows]
    assert [(it[1], it[2]) for it in ds.items] == [(r[3], r[4]) for r in rows]
    for i in range(len(ds)):
        it = ds[i]
        assert isinstance(it, data.SegmentItem) and it.speaker_id == rows[i][4]
        assert np.array_equal(it.text_ids, np.asarray(tts(rows[i][3]), np.int32))
        assert it.n_frames == audio.num_frames_host(it.seg_len) and it.seg_len > 0
        assert (it.in_start, len(it.pcm)) == data.segment_span(it.n_in, it.seg_start, it.seg_len, it.sample_rate)
        assert len(it.pcm) < it.n_in                                  # only the span travels
        sr, x = audio.decode_wav(ds.items[i][0])
        assert sr == it.sample_rate and len(x) == it.n_in
        got = it.pcm.astype(np.float32) / 32768.0 if it.pcm.dtype == np.int16 else it.pcm
        assert np.array_equal(got, x[it.in_start:it.in_start + len(it.pcm)])
    only = data.WavDataset.from_vctk(in_dir, tts, speakers=["p301"])
    assert [it[2] for it in only.items] == [0, 0, 0]


def test_index_cache_keying(tmp_path, counted_bounds, monkeypatch):
    from deepvoice3_pytorch_b200 import audio, data
    in_dir = str(tmp_path / "in")
    F.write_tree(in_dir)
    idx = str(tmp_path / "index.npz")
    first = data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert os.path.exists(idx) and len(counted_bounds) == 1

    def same(a, b):
        return a.items == b.items and a._segments == b._segments and a.frame_lengths == b.frame_lengths

    again = data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 1 and same(first, again)          # reused: no pass
    wav = os.path.join(in_dir, "wav48", "p225", "p225_002.wav")
    st = os.stat(wav)
    os.utime(wav, ns=(st.st_atime_ns, st.st_mtime_ns + 10 ** 9))
    data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 2                                   # touched wav: recomputed
    data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 2                                   # ... and the new cache reused
    lab = os.path.join(in_dir, "lab", "p301", "p301_003.lab")
    with open(lab, "a") as f:
        f.write("\n")
    data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 3                                   # label changed size
    monkeypatch.setattr(audio.hparams, "sample_rate", 16000)
    other = data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 4 and other.frame_lengths != first.frame_lengths
    monkeypatch.setattr(audio.hparams, "sample_rate", 22050)
    data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 5
    with open(idx, "wb") as f:                                        # unreadable cache: recomputed, not an error
        f.write(b"not an npz")
    assert same(data.WavDataset.from_vctk(in_dir, tts, index_path=idx), first) and len(counted_bounds) == 6
    with np.load(idx) as z:                                           # a cache whose key matches another tree
        key, index = str(z["key"]), z["index"].copy()
    index[:, 5] += 1
    with open(idx, "wb") as f:
        np.savez(f, key=np.array(key + "0"), index=index)
    data.WavDataset.from_vctk(in_dir, tts, index_path=idx)
    assert len(counted_bounds) == 7


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, in_dir, idx_path, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from deepvoice3_pytorch_b200 import data, preprocess
    seen = []

    def bounds(clips):
        seen.extend(len(c[0]) for c in clips)
        return host_bounds(clips)
    preprocess.segment_bounds = bounds
    ds = data.WavDataset.from_vctk(in_dir, tts, index_path=idx_path, batch_clips=2)
    ret[rank] = (ds.items, ds._segments, ds.frame_lengths, seen)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_index_equals_single_process(tmp_path, counted_bounds):
    from deepvoice3_pytorch_b200 import data
    in_dir = str(tmp_path / "in")
    F.write_tree(in_dir)
    single = data.WavDataset.from_vctk(in_dir, tts, batch_clips=3)
    mgr = mp.Manager()
    ret = mgr.dict()
    idx = str(tmp_path / "index.npz")
    mp.spawn(_worker, args=(2, _free_port(), in_dir, idx, ret), nprocs=2, join=True)
    for rank in (0, 1):
        items, segs, frames, _ = ret[rank]
        assert items == single.items and segs == single._segments and frames == single.frame_lengths
    assert len(ret[0][3]) + len(ret[1][3]) == 9 and len(ret[0][3]) == 5          # dealt round-robin
    cached = data.WavDataset.from_vctk(in_dir, tts, index_path=idx)                 # rank 0 wrote the cache
    assert len(counted_bounds) == 3 and cached._segments == single._segments


def test_collate_wav_on_segment_items(tmp_path, counted_bounds):
    from deepvoice3_pytorch_b200 import data
    in_dir = str(tmp_path / "in")
    F.write_tree(in_dir)
    ds = data.WavDataset.from_vctk(in_dir, tts)
    items = [ds[i] for i in (4, 0, 3, 7)]                              # native int16, int16, float32, int16
    for r, step in ((1, 4), (4, 1), (2, 2)):
        npy = [(it.text_ids, np.zeros((it.n_frames, 80), np.float32), np.zeros((it.n_frames, 513), np.float32),
                it.speaker_id) for it in items]
        want = data.collate(npy, r, step)
        got = data.collate_wav(items, r, step)
        extra = ("wav", "wav_lengths", "src_desc", "src_rates")
        assert [k for k in got if k not in extra] == [k for k in want if k not in ("mel", "y")]
        for k in want:
            if k in ("mel", "y"):
                continue
            if torch.is_tensor(want[k]):
                assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
            else:
                assert np.array_equal(got[k], want[k]), k
    assert got["wav_lengths"].tolist() == [it.seg_len for it in items]
    assert got["wav"].dtype == torch.float32                           # a float32 source: every row float32
    assert got["src_rates"].tolist() == [22050, 48000, 48000, 48000]
    assert got["src_desc"].tolist() == [[i, it.n_in, it.in_start, len(it.pcm), it.seg_start, it.seg_len]
                                        for i, it in sorted(enumerate(items), key=lambda p: (p[1].sample_rate, p[0]))]
    for i, it in enumerate(items):
        x = it.pcm.astype(np.float32) / np.float32(32768.0) if it.pcm.dtype == np.int16 else it.pcm
        assert np.array_equal(got["wav"][i, :len(x)].numpy(), x) and not got["wav"][i, len(x):].any()
    ints = data.collate_wav([ds[i] for i in (0, 1, 4)])
    assert ints["wav"].dtype == torch.int16
    whole = (items[0].text_ids, np.zeros(3000, np.int16), data._num_frames(3000), 0)
    with pytest.raises(ValueError):
        data.collate_wav([items[0], whole])
    with pytest.raises(ValueError):
        data.collate_wav([whole, items[0]])
    with pytest.raises(ValueError):
        data.collate_wav([items[0]._replace(n_frames=items[0].n_frames + 1)])


def test_segment_entry_point_matches_the_header():
    """Declared in include/dv3b200.h with the argument types audio.py passes, returning int, exported by the library;
    the whole-clip entry point keeps its signature."""
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import parse_header, LIB_PATH
    _build.build()
    decls = parse_header()
    P, I = ctypes.c_void_p, ctypes.c_int
    name = "dv3_resample_segments_batched"
    assert [t for t, _ in decls[name][1]] == [P, I, I, P, I, P, I, P, I, I, I, I, P]
    assert [a for _, a in decls[name][1]] == ["wav", "wav_int16", "pitch_in", "seg", "nclips", "out", "pitch_out",
                                              "bank", "up", "down", "ntaps", "pre_remove", "stream"]
    assert decls[name][0] is ctypes.c_int and hasattr(ctypes.CDLL(LIB_PATH), name)
    assert [t for t, _ in decls["dv3_resample_poly_batched"][1]] == [P, I, P, I, P, I, I, P, I, I, I, I, P]


def test_segment_entry_point_refuses_bad_arguments():
    """No descriptors, or a launch shape out of range, return an error before any CUDA call."""
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import lib, Dv3Error
    _build.build()
    fake = ctypes.c_void_p(16)
    with pytest.raises(Dv3Error, match="descriptors"):
        lib.call("dv3_resample_segments_batched", fake, 1, 64, None, 1, fake, 64, fake, 1, 1, 1, 0, None)
    with pytest.raises(Dv3Error, match="nclips"):
        lib.call("dv3_resample_segments_batched", fake, 1, 64, fake, 0, fake, 64, fake, 1, 1, 1, 0, None)
    with pytest.raises(Dv3Error, match="bad filter"):
        lib.call("dv3_resample_segments_batched", fake, 1, 64, fake, 1, fake, 64, fake, 0, 1, 1, 0, None)


def test_resample_kernel_no_spills_no_stack(tmp_path):
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c) and os.access(c, os.X_OK)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "resample.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "resample.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    found = re.findall(r"Compiling entry function '(\w*resample_poly_kernel\w*)'.*?(\d+) bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout + r.stderr, re.S)
    assert len(found) == 2, r.stdout + r.stderr                       # int16 and fp32 input
    assert all(f[1:] == ("0", "0", "0") for f in found), found
