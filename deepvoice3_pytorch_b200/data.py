"""Host side of the data path feeding ``TrainStep`` (SURVEY.md section 8f row 2): batching with the reference's
padding rules, and a distributed variant of its length-bucketed sampler.

* ``collate`` restates reference train.py:293-360 (``collate_fn``) plus the per-step slicing the train loop applies
  (mel[:, 0::downsample_step], train.py:639-640) and returns the dict ``TrainStep.step`` consumes (optionally in
  pinned memory so the H2D copies are asynchronous).
* ``TrainTxtDataset`` reads the on-disk format ``preprocess.py`` writes (``train.txt`` with one
  ``spec.npy|mel.npy|n_frames|text[|speaker_id]`` line per utterance, preprocess.py:27-30; the three reference data
  sources TextDataSource / MelSpecDataSource / LinearSpecDataSource + PyTorchDataset, train.py:96-257, in one class).
  The text frontend (string -> token ids) stays the caller's: pass the reference's ``frontend.text_to_sequence``.
* ``WavDataset`` + ``collate_wav`` + ``wav_batch_to_device`` train from the wav files instead: the loader moves
  waveforms (int16 where the files are), and the GPU computes each batch's targets in ``collate``'s layout, bit-identical
  to ``TrainTxtDataset`` + ``collate`` over what ``preprocess.build_from_path`` writes for the same corpus.
  ``WavDataset.from_vctk`` does the same for a VCTK tree at its recording rate: its items carry the part of each file
  that the label cut and the silence trim keep, and the GPU resamples just that part per batch
  (``audio.resample_segments``), bit-identical to what ``preprocess.build_vctk_from_path`` writes.
* ``CloningSampleDataset`` + ``collate_cloning`` add each row's cloning samples ("speaker_mels") for fine-tuning a
  speaker encoder through the training loss (``TrainStep(speaker_encoder=...)``).
* ``DistributedSimilarLengthSampler`` restates ``PartialyRandomizedSimilarTimeLengthSampler`` (train.py:195-239):
  sort by length, shuffle inside groups of ``batch_group_size``, permute whole mini-batches -- then deals the
  mini-batches round-robin to the ranks, so every rank sees disjoint batches of similar length (what the
  data-parallel step needs: one utterance batch per GPU, no collective on the data path).
"""
from collections import namedtuple

import numpy as np
import torch


def _pad(seq, max_len, constant_values=0):
    return np.pad(seq, (0, max_len - len(seq)), mode="constant", constant_values=constant_values)


def _pad_2d(x, max_len, b_pad=0):
    return np.pad(x, [(b_pad, max_len - len(x) - b_pad), (0, 0)], mode="constant", constant_values=0)


def collate(batch, r=1, downsample_step=4, pin=False):
    """batch: list of (text_ids int array, mel (T, num_mels) float32, linear (T, n_freq) float32[, speaker_id]).

    Padding rules of the reference: target length rounded up to a multiple of r and of downsample_step, plus r *
    downsample_step leading zero frames ("initial decoder state"); text / text positions zero-padded; frame positions
    1..T_dec; done = 0 for the first len//r//ds - 1 decoder steps, then 1."""
    max_target_len = max_target_length([len(b[1]) for b in batch], r, downsample_step)
    b_pad = r
    mel = torch.from_numpy(np.array([_pad_2d(b[1], max_target_len, b_pad=b_pad) for b in batch], dtype=np.float32))
    y = torch.from_numpy(np.array([_pad_2d(b[2], max_target_len, b_pad=b_pad) for b in batch], dtype=np.float32))
    if downsample_step > 1:
        mel = mel[:, 0::downsample_step, :].contiguous()          # train.py:639-640
    return _collate_common(batch, [len(b[1]) for b in batch], r, downsample_step, pin, {"mel": mel, "y": y})


def max_target_length(target_lengths, r=1, downsample_step=4):
    """collate's padded frame count of a batch: the longest target rounded up to a multiple of r and of
    downsample_step, plus the r * downsample_step leading zero frames."""
    max_target_len = max(target_lengths)
    if max_target_len % r != 0:
        max_target_len += r - max_target_len % r
    if max_target_len % downsample_step != 0:
        max_target_len += downsample_step - max_target_len % downsample_step
    return max_target_len + r * downsample_step


def _collate_common(batch, target_lengths, r, downsample_step, pin, spectrograms):
    """Every key of a collated batch but the spectrograms, with ``spectrograms`` ({"mel", "y"} for collate; the
    waveforms for collate_wav) placed after frame_positions.  batch items: (text ids, target, ...[, speaker_id])."""
    multi_speaker = len(batch[0]) == 4
    input_lengths = [len(x[0]) for x in batch]
    max_input_len = max(input_lengths)
    max_target_len = max_target_length(target_lengths, r, downsample_step)

    x = torch.from_numpy(np.array([_pad(np.asarray(b[0]), max_input_len) for b in batch], dtype=np.int64))
    text_positions = torch.from_numpy(np.array(
        [_pad(np.arange(1, len(b[0]) + 1), max_input_len) for b in batch], dtype=np.int64))
    T_dec = max_target_len // r // downsample_step
    frame_positions = torch.arange(1, T_dec + 1).long().unsqueeze(0).expand(len(batch), T_dec).clone()
    done = torch.from_numpy(np.array(
        [_pad(np.zeros(n // r // downsample_step - 1), T_dec, constant_values=1) for n in target_lengths],
        dtype=np.float32)).unsqueeze(-1)
    out = {"x": x, "text_positions": text_positions, "frame_positions": frame_positions, **spectrograms,
           "done": done, "target_lengths": torch.tensor(target_lengths, dtype=torch.int64),
           "input_lengths_dev": torch.tensor(input_lengths, dtype=torch.int64)}
    if multi_speaker:
        out["speaker_ids"] = torch.tensor([b[3] for b in batch], dtype=torch.int64)
    if pin:
        out = {k: v.pin_memory() for k, v in out.items()}
    out["input_lengths"] = np.asarray(input_lengths, dtype=np.int64)
    return out


SegmentItem = namedtuple("SegmentItem", "text_ids pcm n_frames speaker_id sample_rate n_in in_start seg_start seg_len")
SegmentItem.__doc__ = """A ``WavDataset.from_vctk`` item: pcm holds samples [in_start, in_start + len(pcm)) of a source clip of n_in
samples at sample_rate (int16, or float32 for other formats), the input span of resampled samples
[seg_start, seg_start + seg_len) at ``hparams.sample_rate`` -- the utterance's training segment, n_frames STFT frames."""


def _pcm_rows(clips):
    """[pcm (n,) int16 / float32] -> (B, pitch) zero-padded rows, pitch a multiple of 8 samples (16-byte rows for int16
    and fp32 alike); int16 when every clip is int16, else float32 (int16 / 32768 is exact)."""
    pitch = max(8, -(-max(len(w) for w in clips) // 8) * 8)
    int16 = all(w.dtype == np.int16 for w in clips)
    wav = np.zeros((len(clips), pitch), dtype=np.int16 if int16 else np.float32)
    for i, w in enumerate(clips):
        wav[i, :len(w)] = w if int16 or w.dtype != np.int16 else w.astype(np.float32) / np.float32(32768.0)
    return torch.from_numpy(wav)


def collate_wav(batch, r=1, downsample_step=4, pin=False):
    """batch: list of ``WavDataset`` items (text_ids, pcm (n,) int16 or float32, n_frames[, speaker_id]), or of
    ``SegmentItem`` (``WavDataset.from_vctk``); one batch never mixes the two (ValueError).

    Host-only (safe in DataLoader workers): every key of ``collate`` except "mel" and "y", computed by the same code,
    plus "wav" (B, pitch) -- the waveforms zero-padded to a pitch of a multiple of 8 samples, int16 when every clip is
    int16, else float32 (int16 / 32768 is exact) -- and "wav_lengths" (B) int32.  ``wav_batch_to_device`` computes the
    two spectrogram targets on the GPU.

    For ``SegmentItem`` batches "wav" holds each item's source span and "wav_lengths" its segment length; two more keys
    describe the sources: "src_desc" (B, 6) int32, one ``audio.SEG_FIELDS`` row per item with the item's batch index
    as its row, ordered by source rate, and "src_rates" (B) int32, the rate of each "src_desc" row."""
    kinds = {isinstance(b, SegmentItem) for b in batch}
    if len(kinds) > 1:
        raise ValueError("a batch mixes WavDataset.from_vctk segment items with whole-clip items")
    if kinds == {True}:
        return _collate_segments(batch, r, downsample_step, pin)
    lens = [len(b[1]) for b in batch]
    for b, n in zip(batch, lens):
        if b[2] != _num_frames(n):
            raise ValueError("item has %d samples but n_frames=%d (expected %d)" % (n, b[2], _num_frames(n)))
    spectrograms = {"wav": _pcm_rows([b[1] for b in batch]), "wav_lengths": torch.tensor(lens, dtype=torch.int32)}
    return _collate_common(batch, [b[2] for b in batch], r, downsample_step, pin, spectrograms)


def _collate_segments(batch, r, downsample_step, pin):
    for b in batch:
        if b.n_frames != _num_frames(b.seg_len):
            raise ValueError("segment has %d samples but n_frames=%d (expected %d)"
                             % (b.seg_len, b.n_frames, _num_frames(b.seg_len)))
    order = sorted(range(len(batch)), key=lambda i: (batch[i].sample_rate, i))     # one launch per source rate
    desc = [[i, batch[i].n_in, batch[i].in_start, len(batch[i].pcm), batch[i].seg_start, batch[i].seg_len]
            for i in order]
    spectrograms = {"wav": _pcm_rows([b.pcm for b in batch]),
                    "wav_lengths": torch.tensor([b.seg_len for b in batch], dtype=torch.int32),
                    "src_desc": torch.tensor(desc, dtype=torch.int32),
                    "src_rates": torch.tensor([batch[i].sample_rate for i in order], dtype=torch.int32)}
    return _collate_common([(b.text_ids, None, None, b.speaker_id) for b in batch], [b.n_frames for b in batch], r,
                           downsample_step, pin, spectrograms)


def wav_batch_to_device(batch, device, r=1, downsample_step=4):
    """A ``collate_wav`` batch -> the dict ``collate`` + ``train_step.to_device`` give for the same utterances after
    ``preprocess.build_from_path`` (``preprocess.build_vctk_from_path`` for ``WavDataset.from_vctk`` items), bit for
    bit: asynchronous H2D copies (pin the batch for them to overlap), for segment items one
    ``audio.resample_segments`` launch per source rate, then the targets in one launch on the current stream
    (``audio.stft_mel_targets``; the peak pass first when ``hparams.rescaling`` is on).  No host synchronisation."""
    from . import audio
    out = {}
    for k, v in batch.items():
        if k in ("wav", "wav_lengths", "src_desc", "src_rates"):
            continue
        out[k] = v.to(device, non_blocking=True) if torch.is_tensor(v) else v
    wav = batch["wav"].to(device, non_blocking=True)
    if "src_desc" in batch:
        wav = _resample_rows(wav, batch)
    lens_dev = batch["wav_lengths"].to(device, non_blocking=True)
    T_lin = max_target_length(batch["target_lengths"].tolist(), r, downsample_step)
    y, mel = audio.stft_mel_targets(wav, batch["wav_lengths"], T_lin, r, downsample_step, lengths_dev=lens_dev)
    order = ("x", "text_positions", "frame_positions")
    return {**{k: out[k] for k in order}, "mel": mel, "y": y, **{k: v for k, v in out.items() if k not in order}}


def _resample_rows(src, batch):
    """The segments of a ``SegmentItem`` batch at ``hparams.sample_rate`` from its source spans ``src`` (on the
    device): (B, pitch) fp32, pitch as ``collate_wav`` pads, one launch per rate."""
    from . import audio
    lens = batch["wav_lengths"].tolist()
    desc, rates = batch["src_desc"].tolist(), batch["src_rates"].tolist()
    if sorted(d[0] for d in desc) != list(range(len(lens))) or len(rates) != len(desc):
        raise ValueError("src_desc must give one row per item of the batch")
    out = torch.empty(len(lens), max(8, -(-max(lens) // 8) * 8), device=src.device)     # every row is written
    desc_dev = batch["src_desc"].to(src.device, non_blocking=True)
    g0 = 0
    while g0 < len(desc):
        g1 = g0 + 1
        while g1 < len(desc) and rates[g1] == rates[g0]:
            g1 += 1
        audio.resample_segments(src, desc[g0:g1], rates[g0], out, seg_dev=desc_dev[g0:g1])
        g0 = g1
    return out


def _num_frames(n_samples):
    from .audio import num_frames_host
    return num_frames_host(n_samples)


# Bucket grid of the CUDA-graph training step (train_step.TrainStep): a batch whose shape differs from the first one is
# padded up to the next multiple of BUCKET_TEXT text positions and BUCKET_DEC decoder steps, and one graph is captured
# per bucket.  Multiples of 4 keep the float4 paths of the operand-split and attention kernels on (T % 4 == 0); the
# tensor-core convs themselves take any T.  On the LJSpeech-like length model of bench_train_ragged.py (64 batches of
# 16, 53 distinct shapes) this grid adds 2 % padded frames to collate's own padding and needs 9 buckets.
BUCKET_TEXT, BUCKET_DEC = 16, 8


def bucket_shape(T_text, T_dec):
    """(text positions, decoder steps) of a batch -> the bucket it is padded to (rounded up to the grid)."""
    return -(-int(T_text) // BUCKET_TEXT) * BUCKET_TEXT, -(-int(T_dec) // BUCKET_DEC) * BUCKET_DEC


def batch_extents(batch):
    """Logical extents of a batch as ``collate`` returns it: (decoder steps, text positions, mel frames, linear
    frames), the slots ops.EXT_DEC, EXT_TEXT, EXT_MEL, EXT_LIN."""
    return (int(batch["done"].shape[1]), int(batch["x"].shape[1]), int(batch["mel"].shape[1]), int(batch["y"].shape[1]))


def pad_to_bucket(batch, T_text, T_dec, r=1, downsample_step=4, out=None):
    """Pad a batch as ``collate`` returns it (host or device tensors) to T_text text positions and T_dec decoder steps
    (T_dec*r mel frames, T_dec*r*downsample_step linear frames) and attach its logical extents.

    Text, text positions, mel, y and done are zero past the logical extent; frame positions are 1..T_dec_logical, then 0
    (so a bucket never indexes past the model's max_positions); per-row lengths and speaker ids are unchanged.
    ``extents`` is int64[4] (``batch_extents``) on the batch's device.  ``TrainStep`` runs such a batch with the loss,
    gradients and update of the unpadded one.  out: a dict of the same keys in the bucket shape to fill in place
    (``out["extents"]`` included) -- then nothing is allocated but the 32-byte staging of the extents."""
    ext = batch_extents(batch)
    T_dec_log, T_text_log = ext[0], ext[1]
    if ext[2] != T_dec_log * r or ext[3] != T_dec_log * r * downsample_step:
        raise ValueError("batch shapes %s do not fit r=%d downsample_step=%d" % (ext, r, downsample_step))
    if T_text < T_text_log or T_dec < T_dec_log:
        raise ValueError("bucket (T_text=%d, T_dec=%d) is smaller than the batch (%d, %d)" % (T_text, T_dec,
                                                                                            T_text_log, T_dec_log))
    if batch.get("extents") is not None:
        raise ValueError("batch is already padded to a bucket")
    sizes = {"x": T_text, "text_positions": T_text, "frame_positions": T_dec, "mel": T_dec * r,
             "y": T_dec * r * downsample_step, "done": T_dec}
    fill = out is not None
    out = {} if out is None else out
    for k, v in batch.items():
        if k == "extents":
            continue
        if k not in sizes or not torch.is_tensor(v):
            if not fill:
                out[k] = v.clone() if torch.is_tensor(v) else v
            elif torch.is_tensor(v):
                out[k].copy_(v, non_blocking=True)
            else:
                out[k] = v
            continue
        T = v.shape[1]
        if not fill:
            shape = (v.shape[0], sizes[k]) + tuple(v.shape[2:])
            out[k] = torch.empty(shape, dtype=v.dtype, device=v.device, pin_memory=v.is_pinned())
        out[k][:, :T].copy_(v, non_blocking=True)
        out[k][:, T:].zero_()
    dev = batch["x"].device
    host = torch.tensor(ext, dtype=torch.int64)
    if dev.type == "cuda" or batch["x"].is_pinned():
        host = host.pin_memory()
    if fill:
        out["extents"].copy_(host, non_blocking=True)
    else:
        out["extents"] = host.to(dev, non_blocking=True) if dev.type == "cuda" else host
    return out


class TrainTxtDataset(torch.utils.data.Dataset):
    """Items are what ``collate`` consumes: (token ids int32, mel (T, num_mels) float32, linear (T, n_freq) float32
    [, speaker_id]).  ``frame_lengths`` (column 3 of train.txt) feeds the length-bucketed sampler without touching
    the .npy files.  ``speaker_id`` filters a multi-speaker corpus down to one speaker (and then yields 3-tuples),
    like the reference data sources do (train.py:101-122, 169-177)."""

    def __init__(self, data_root, text_to_sequence, speaker_id=None, mmap=True):
        import os
        self.data_root, self.text_to_sequence, self.mmap = data_root, text_to_sequence, mmap
        with open(os.path.join(data_root, "train.txt"), "rb") as f:
            rows = [line.decode("utf-8").rstrip("\n").split("|") for line in f if line.strip()]
        if not rows:
            raise ValueError("empty train.txt under %s" % data_root)
        n = len(rows[0])
        if n not in (4, 5) or any(len(r) != n for r in rows):
            raise ValueError("train.txt lines must have 4 or 5 '|'-separated fields")
        self.multi_speaker = n == 5
        if self.multi_speaker and speaker_id is not None:
            rows = [r for r in rows if int(r[4]) == speaker_id]
            self.multi_speaker = False
        self.rows = rows
        self.frame_lengths = [int(r[2]) for r in rows]

    def __len__(self):
        return len(self.rows)

    def _load(self, name):
        import os
        return np.load(os.path.join(self.data_root, name), mmap_mode="r" if self.mmap else None)

    def __getitem__(self, idx):
        r = self.rows[idx]
        seq = np.asarray(self.text_to_sequence(r[3]), dtype=np.int32)
        item = (seq, np.asarray(self._load(r[1]), dtype=np.float32), np.asarray(self._load(r[0]), dtype=np.float32))
        return item + (int(r[4]),) if self.multi_speaker else item


def _wav_header(path):
    """-> (sample rate, samples, channels, dtype) of a wav file, reading only its header (memory map)."""
    from scipy.io import wavfile
    sr, x = wavfile.read(path, mmap=True)
    return int(sr), int(x.shape[0]), (1 if x.ndim == 1 else int(x.shape[1])), x.dtype


def _resampled_length(n, sr_from, sr_to):
    """Output length of ``audio.load_wav``'s resampling (scipy resample_poly): ceil(n * up / down)."""
    from math import gcd
    g = gcd(int(sr_from), int(sr_to))
    up, down = sr_to // g, sr_from // g
    return -(-n * up // down)


class WavDataset(torch.utils.data.Dataset):
    """Training straight from wav files: items are what ``collate_wav`` consumes, (token ids int32, pcm, n_frames
    [, speaker_id]); the spectrogram targets are computed per batch on the GPU (``wav_batch_to_device``), bit-identical
    to training on what ``preprocess.build_from_path`` writes for the same files.

    items: [(wav_path, text[, speaker_id])].  pcm is the file's int16 samples when it is 16-bit mono PCM at
    ``hparams.sample_rate`` (half the bytes of fp32 through the loader and over PCIe), otherwise ``audio.load_wav``'s
    float32 waveform.  ``frame_lengths`` comes from the wav headers alone (the resampled length where the rate
    differs), so ``DistributedSimilarLengthSampler`` runs without decoding any audio.  ``speaker_id`` keeps only that
    speaker's items (and then yields 3-tuples), like ``TrainTxtDataset``."""

    def __init__(self, items, text_to_sequence, speaker_id=None):
        from .audio import hparams
        items = [tuple(it) for it in items]
        if not items:
            raise ValueError("WavDataset needs at least one item")
        n = len(items[0])
        if n not in (2, 3) or any(len(it) != n for it in items):
            raise ValueError("items must all be (wav_path, text) or all (wav_path, text, speaker_id)")
        self.multi_speaker = n == 3
        if self.multi_speaker and speaker_id is not None:
            items = [it[:2] for it in items if int(it[2]) == speaker_id]
            self.multi_speaker = False
        self.items, self.text_to_sequence = items, text_to_sequence
        self.sample_rate = hparams.sample_rate
        self.frame_lengths, self._segments = [], None
        self._native = []                    # 16-bit mono at the training rate: returned as int16 without conversion
        for it in items:
            sr, n_samples, channels, dtype = _wav_header(it[0])
            if sr != self.sample_rate:
                n_samples = _resampled_length(n_samples, sr, self.sample_rate)
            self._native.append(sr == self.sample_rate and channels == 1 and dtype == np.int16)
            self.frame_lengths.append(_num_frames(n_samples))

    @classmethod
    def from_ljspeech(cls, in_dir, text_to_sequence):
        """The utterances ``preprocess.build_from_path(in_dir, ...)`` processes, in its order (metadata.csv, the
        ``hparams.min_text`` filter): item i is row i of the train.txt it writes."""
        import os
        from .audio import hparams
        items = []
        with open(os.path.join(in_dir, "metadata.csv"), encoding="utf-8") as f:
            for line in f:
                parts = line.strip().split("|")
                text = parts[2]
                if len(text) < hparams.min_text:
                    continue
                items.append((os.path.join(in_dir, "wavs", "%s.wav" % parts[0]), text))
        return cls(items, text_to_sequence)

    @classmethod
    def from_vctk(cls, in_dir, text_to_sequence, speakers=None, index_path=None, batch_clips=64):
        """The rows ``preprocess.build_vctk_from_path(in_dir, ..., speakers=speakers)`` writes, straight from the wav48
        files: item i is a ``SegmentItem`` of row i (same order, texts and speaker ids; an utterance whose trimmed
        segment is empty has no row).  Its segment comes from one indexing pass at construction that resamples
        whole clips, cuts them to the labels and trims them on the GPU (``preprocess.segment_bounds``, ``batch_clips``
        clips per set of launches); ``frame_lengths`` is train.txt's n_frames column.  Under an initialised
        ``torch.distributed`` the pass is dealt round-robin over the ranks and merged with one ``all_gather_object``.

        index_path: a ``.npz`` file that caches the index, keyed by every wav's and label's path, size and mtime, by
        ``hparams.sample_rate`` and by a format version.  It is used only when its key matches (otherwise the pass runs
        again) and written by rank 0 after a pass."""
        from .audio import hparams
        from . import preprocess
        utts = preprocess.vctk_utterances(in_dir, speakers)
        if not utts:
            raise ValueError("no VCTK utterances under %s" % in_dir)
        key = _vctk_index_key(utts, hparams.sample_rate)
        index = _read_vctk_index(index_path, key, [u[0] for u in utts]) if index_path else None
        if index is None:
            index, rank = _vctk_index(utts, batch_clips)
            if index_path and rank == 0:
                _write_vctk_index(index_path, key, index)
        ds = cls.__new__(cls)
        ds.text_to_sequence, ds.sample_rate, ds.multi_speaker = text_to_sequence, hparams.sample_rate, True
        ds.items, ds._segments, ds.frame_lengths = [], [], []
        for (_, (wav, _), (text, spk)), (sr, n_in, is16, s0, n) in zip(utts, index[:, 1:].tolist()):
            if n == 0:
                continue
            ds.items.append((wav, text, spk))
            ds._segments.append((sr, n_in, bool(is16), s0, n) + segment_span(n_in, s0, n, sr))
            ds.frame_lengths.append(_num_frames(n))
        return ds

    def __len__(self):
        return len(self.items)

    def __getitem__(self, idx):
        it = self.items[idx]
        if self._segments is not None:
            return self._segment_item(idx)
        if self._native[idx]:
            from scipy.io import wavfile
            pcm = np.array(wavfile.read(it[0], mmap=True)[1], dtype=np.int16)
        else:
            from .audio import load_wav
            pcm = load_wav(it[0])
        seq = np.asarray(self.text_to_sequence(it[1]), dtype=np.int32)
        item = (seq, pcm, self.frame_lengths[idx])
        return item + (int(it[2]),) if self.multi_speaker else item


    def _segment_item(self, idx):
        wav_path, text, spk = self.items[idx]
        sr, n_in, is16, s0, n, a, m = self._segments[idx]
        if is16:                                  # memory-mapped: only the pages of the span are read
            from scipy.io import wavfile
            pcm = np.array(wavfile.read(wav_path, mmap=True)[1][a:a + m], dtype=np.int16)
        else:
            from .audio import decode_wav
            pcm = np.ascontiguousarray(decode_wav(wav_path)[1][a:a + m], dtype=np.float32)
        seq = np.asarray(self.text_to_sequence(text), dtype=np.int32)
        return SegmentItem(seq, pcm, self.frame_lengths[idx], int(spk), sr, n_in, a, s0, n)


def segment_span(n_in, seg_start, seg_len, sr_from):
    """-> (start, length) of the input samples that resampling an n_in-sample clip from sr_from to
    ``hparams.sample_rate`` reads for output samples [seg_start, seg_start + seg_len) (``audio.input_span`` with the
    filter of that rate pair): what a ``SegmentItem`` carries."""
    from . import audio
    up, down = audio.resample_ratio(sr_from)
    ntaps, pre_remove = _host_bank(up, down)
    return audio.input_span(n_in, seg_start, seg_len, up, down, ntaps, pre_remove)


_host_banks = {}


def _host_bank(up, down):
    """(ntaps, pre_remove) of ``audio.resample_filter_bank(up, down)``, cached (the design runs firwin)."""
    if (up, down) not in _host_banks:
        from .audio import resample_filter_bank
        bank, pre_remove = resample_filter_bank(up, down)
        _host_banks[(up, down)] = (bank.shape[0], pre_remove)
    return _host_banks[(up, down)]


VCTK_INDEX_VERSION = 1


def _vctk_index_key(utts, sample_rate):
    """sha256 over the index format version, the target rate, and every wav's and label's absolute path, size and
    mtime, in walk order."""
    import hashlib
    import os
    h = hashlib.sha256(("dv3-vctk-index|%d|%d\n" % (VCTK_INDEX_VERSION, int(sample_rate))).encode())
    for idx, paths, _ in utts:
        for p in paths:
            if p is None:
                h.update(b"-\n")
                continue
            st = os.stat(p)
            h.update(("%d|%s|%d|%d\n" % (idx, os.path.abspath(p), st.st_size, st.st_mtime_ns)).encode("utf-8"))
    return h.hexdigest()


def _vctk_index(utts, batch_clips):
    """The indexing pass -> ((n, 6) int64 rows [file index, source rate, n_in, int16, seg_start, seg_len] in walk
    order, this process's rank)."""
    import torch.distributed as dist
    from . import preprocess
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    mine = utts[rank::world]
    rows = []
    for i in range(0, len(mine), batch_clips):
        batch = mine[i:i + batch_clips]
        clips = [preprocess._load_vctk(src) for _, src, _ in batch]
        for (idx, _, _), (pcm, sr, _), (s0, n) in zip(batch, clips, preprocess.segment_bounds(clips)):
            rows.append((idx, sr, len(pcm), int(pcm.dtype == np.int16), s0, n))
    if world > 1:
        parts = [None] * world
        dist.all_gather_object(parts, rows)
        rows = [r for part in parts for r in part]
    return np.array(sorted(rows), dtype=np.int64).reshape(-1, 6), rank


def _read_vctk_index(path, key, file_indices):
    """The cached index at path when it exists, is readable and its key and file indices match; else None."""
    import os
    if not os.path.exists(path):
        return None
    try:
        with np.load(path, allow_pickle=False) as z:
            if str(z["key"]) != key:
                return None
            index = np.asarray(z["index"], dtype=np.int64)
    except (OSError, ValueError, KeyError):
        return None
    if index.shape != (len(file_indices), 6) or index[:, 0].tolist() != list(file_indices):
        return None
    return index


def _write_vctk_index(path, key, index):
    import os
    tmp = "%s.%d.tmp" % (path, os.getpid())
    with open(tmp, "wb") as f:
        np.savez(f, key=np.array(key), index=index)
    os.replace(tmp, path)


class DistributedSimilarLengthSampler(torch.utils.data.Sampler):
    """Yields the dataset indices of this rank's mini-batches, batch after batch (use with
    ``DataLoader(batch_size=batch_size, sampler=..., collate_fn=...)`` and ``drop_last=True``)."""

    def __init__(self, lengths, batch_size=16, batch_group_size=None, permutate=True, rank=0, world_size=1, seed=0):
        lengths = torch.as_tensor(np.asarray(lengths), dtype=torch.int64)
        self.lengths, self.sorted_indices = torch.sort(lengths)
        self.batch_size = batch_size
        if batch_group_size is None:
            batch_group_size = min(batch_size * 32, len(self.lengths))
            if batch_group_size % batch_size != 0:
                batch_group_size -= batch_group_size % batch_size
        assert batch_group_size % batch_size == 0 and batch_group_size > 0
        self.batch_group_size = batch_group_size
        self.permutate = permutate
        self.rank, self.world_size, self.seed, self.epoch = rank, world_size, seed, 0
        n_batches = len(self.lengths) // batch_size
        self.batches_per_rank = n_batches // world_size

    def set_epoch(self, epoch):
        self.epoch = epoch

    def _global_order(self):
        rng = np.random.RandomState(self.seed + self.epoch)       # identical on every rank
        idx = self.sorted_indices.numpy().copy()
        g, e = self.batch_group_size, 0
        for i in range(len(idx) // g):
            s, e = i * g, (i + 1) * g
            rng.shuffle(idx[s:e])
        if self.permutate and e > 0:
            perm = rng.permutation(e // self.batch_size)
            idx[:e] = idx[:e].reshape(-1, self.batch_size)[perm].reshape(-1)
        if e < len(idx):
            rng.shuffle(idx[e:])
        return idx

    def __iter__(self):
        idx = self._global_order()
        n_batches = self.batches_per_rank * self.world_size
        batches = idx[:n_batches * self.batch_size].reshape(n_batches, self.batch_size)
        mine = batches[self.rank::self.world_size]
        return iter(mine.reshape(-1).tolist())

    def __len__(self):
        return self.batches_per_rank * self.batch_size


class CloningSampleDataset(torch.utils.data.Dataset):
    """A multi-speaker ``TrainTxtDataset`` whose items carry cloning samples, for fine-tuning a speaker encoder through
    the training loss (``TrainStep(speaker_encoder=...)``).  Item i is the dataset's item i plus, last, N crops
    (N, T_crop, num_mels) float32 of T_crop frames each, from other utterances of the same speaker that have at least
    T_crop frames: drawn without replacement when the speaker has at least N of them, with replacement otherwise; each
    crop at a uniform offset, read from the memory-mapped .npy file.  The draws are a function of (seed, epoch, i)
    alone, so a row's samples depend neither on the batch it lands in nor on the DataLoader's workers; ``set_epoch``
    moves to another epoch.  ValueError at construction for a speaker with fewer than two such utterances (one of its
    utterances would have no other to draw from)."""

    def __init__(self, dataset, N, T_crop, seed=0):
        if not getattr(dataset, "multi_speaker", False):
            raise ValueError("CloningSampleDataset needs a multi-speaker train.txt (5 columns)")
        if N < 1 or T_crop < 1:
            raise ValueError("N=%d, T_crop=%d must be >= 1" % (N, T_crop))
        self.dataset, self.N, self.T_crop, self.seed = dataset, int(N), int(T_crop), int(seed)
        self.frame_lengths = dataset.frame_lengths
        self._speaker = np.array([int(row[4]) for row in dataset.rows], dtype=np.int64)
        eligible = {}
        for i, (s, n) in enumerate(zip(self._speaker.tolist(), dataset.frame_lengths)):
            if n >= T_crop:
                eligible.setdefault(s, []).append(i)
        # one ascending array per speaker; item i's own utterance is skipped at draw time
        self._eligible = {s: np.array(idx, dtype=np.int64) for s, idx in eligible.items()}
        for s in sorted(set(self._speaker.tolist())):
            n = len(self._eligible.get(s, ()))
            if n < 2:       # none at all, or one that has no other to draw from
                raise ValueError("speaker %d has %d utterance(s) of >= %d frames: every utterance of the speaker needs "
                                 "another one to draw its cloning samples from" % (s, n, T_crop))
        self.epoch = 0

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __len__(self):
        return len(self.dataset)

    def draws(self, i):
        """-> (dataset indices (N,), crop offsets (N,)) of item i's cloning samples in the current epoch."""
        rng = np.random.default_rng([self.seed, self.epoch, int(i)])
        pool = self._eligible[int(self._speaker[i])]
        p = int(np.searchsorted(pool, i))
        own = bool(p < pool.size and pool[p] == i)
        m = pool.size - int(own)                # the pool without item i's own utterance
        k = rng.choice(m, self.N, replace=m < self.N)
        if own:
            k = k + (k >= p)                    # positions at or past the own one shift by one
        items = pool[k]
        offsets = np.array([rng.integers(0, self.dataset.frame_lengths[j] - self.T_crop + 1) for j in items],
                           dtype=np.int64)
        return items, offsets

    def __getitem__(self, i):
        import os
        items, offsets = self.draws(i)
        crops = None
        for k, (j, o) in enumerate(zip(items, offsets)):
            name = self.dataset.rows[j][1]
            mel = np.load(os.path.join(self.dataset.data_root, name), mmap_mode="r")
            if mel.shape[0] < o + self.T_crop:
                raise ValueError("%s has %d frames, train.txt says %d" % (name, mel.shape[0],
                                                                          self.dataset.frame_lengths[j]))
            if crops is None:
                crops = np.empty((self.N, self.T_crop, mel.shape[1]), dtype=np.float32)
            crops[k] = mel[o:o + self.T_crop]
        return tuple(self.dataset[i]) + (crops,)


def collate_cloning(batch, r=1, downsample_step=4, pin=False):
    """batch: ``CloningSampleDataset`` items -> ``collate`` of the items without their cloning samples, plus
    "speaker_mels" (B, N, T_crop, num_mels) float32, the samples stacked."""
    out = collate([b[:-1] for b in batch], r, downsample_step, pin)
    mels = torch.from_numpy(np.stack([b[-1] for b in batch]))
    out["speaker_mels"] = mels.pin_memory() if pin else mels
    return out


class SpeakerSampleBatches:
    """Training batches of the speaker encoder (speaker_encoder.SpeakerEncoderStep) over a multi-speaker
    ``TrainTxtDataset``: every batch holds B distinct speakers, each drawn from the speakers with at least N utterances
    of >= T_crop frames, and N such utterances of each, without replacement, each cropped to T_crop frames at a
    uniform offset.  Iterating yields {"mels": (B, N, T_crop, num_mels) float32, "speaker_ids": (B,) int64, "items":
    (B, N) dataset indices, "offsets": (B, N) crop offsets}, len(self) batches per epoch (every eligible speaker at
    most once), read from the .npy files (memory-mapped).  The draws are a function of (seed, epoch) alone;
    ``set_epoch`` moves to another epoch.  ValueError when fewer than B speakers qualify."""

    def __init__(self, dataset, B, N, T_crop, seed=0):
        if not getattr(dataset, "multi_speaker", False):
            raise ValueError("SpeakerSampleBatches needs a multi-speaker train.txt (5 columns)")
        if B < 1 or N < 1 or T_crop < 1:
            raise ValueError("B=%d, N=%d, T_crop=%d must be >= 1" % (B, N, T_crop))
        self.dataset, self.B, self.N, self.T_crop, self.seed = dataset, int(B), int(N), int(T_crop), int(seed)
        groups = {}
        for i, (row, n) in enumerate(zip(dataset.rows, dataset.frame_lengths)):
            if n >= T_crop:
                groups.setdefault(int(row[4]), []).append(i)
        self.groups = {s: idx for s, idx in sorted(groups.items()) if len(idx) >= N}
        self.speakers = sorted(self.groups)
        if len(self.speakers) < B:
            raise ValueError("%d speakers have >= %d utterances of >= %d frames; a batch needs %d"
                             % (len(self.speakers), N, T_crop, B))
        self.epoch = 0

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __len__(self):
        return len(self.speakers) // self.B

    def __iter__(self):
        rng = np.random.default_rng([self.seed, self.epoch])
        order = rng.permutation(len(self.speakers))
        for k in range(len(self)):
            spk = [self.speakers[j] for j in order[k * self.B:(k + 1) * self.B]]
            items = np.stack([rng.choice(self.groups[s], self.N, replace=False) for s in spk])
            offsets = np.zeros_like(items)
            mels = None
            for b in range(self.B):
                for j in range(self.N):
                    i = int(items[b, j])
                    mel = self.dataset._load(self.dataset.rows[i][1])
                    if mel.shape[0] < self.T_crop:
                        raise ValueError("%s has %d frames, train.txt says %d"
                                         % (self.dataset.rows[i][1], mel.shape[0], self.dataset.frame_lengths[i]))
                    o = int(rng.integers(0, mel.shape[0] - self.T_crop + 1))
                    offsets[b, j] = o
                    if mels is None:
                        mels = np.empty((self.B, self.N, self.T_crop, mel.shape[1]), dtype=np.float32)
                    mels[b, j] = mel[o:o + self.T_crop]
            yield {"mels": torch.from_numpy(mels), "speaker_ids": torch.tensor(spk, dtype=torch.int64),
                   "items": torch.from_numpy(items.astype(np.int64)), "offsets": torch.from_numpy(offsets)}


class RecognizerBatches:
    """Training batches of the token recognizer (recognition.TokenRecognizerStep) over any dataset whose items are
    (tokens, mel (T, num_mels), ...), such as ``TrainTxtDataset``: utterances with at most T_max frames and L_max
    tokens, drawn without replacement, each batch padded with zeros to the one shape (B, T_max) / (B, L_max) that the
    step's CUDA graph takes.  Iterating yields {"mels": (B, T_max, num_mels) float32, "mel_lengths": (B,) int32,
    "tokens": (B, L_max) int64, "token_lengths": (B,) int32, "items": (B,) dataset indices}, len(self) batches per
    epoch.  The draws are a function of (seed, epoch) alone; ``set_epoch`` moves to another epoch.  Lengths come from
    ``frame_lengths`` and the text column of a ``TrainTxtDataset`` without loading its mels, from the items otherwise.
    ValueError when fewer than B utterances qualify.

    The batches carry no length scope: in training, a row's last few frames see the padded neighbour activations of
    the deeper layers within the receptive field (DESIGN.md section 2.21)."""

    def __init__(self, dataset, B, T_max, L_max, seed=0):
        if B < 1 or T_max < 1 or L_max < 1:
            raise ValueError("B=%d, T_max=%d, L_max=%d must be >= 1" % (B, T_max, L_max))
        self.dataset, self.B, self.T_max, self.L_max, self.seed = dataset, int(B), int(T_max), int(L_max), int(seed)
        self.eligible = [i for i in range(len(dataset)) if self._frames(i) <= T_max and self._tokens(i) <= L_max]
        if len(self.eligible) < B:
            raise ValueError("%d utterances have <= %d frames and <= %d tokens; a batch needs %d"
                             % (len(self.eligible), T_max, L_max, B))
        self.epoch = 0

    def _frames(self, i):
        fl = getattr(self.dataset, "frame_lengths", None)
        return int(fl[i]) if fl is not None else int(np.asarray(self.dataset[i][1]).shape[0])

    def _tokens(self, i):
        ds = self.dataset
        if hasattr(ds, "rows") and hasattr(ds, "text_to_sequence"):
            return len(ds.text_to_sequence(ds.rows[i][3]))
        return int(np.asarray(ds[i][0]).size)

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __len__(self):
        return len(self.eligible) // self.B

    def __iter__(self):
        rng = np.random.default_rng([self.seed, self.epoch])
        order = rng.permutation(len(self.eligible))
        for k in range(len(self)):
            items = [self.eligible[j] for j in order[k * self.B:(k + 1) * self.B]]
            mels, toks = None, np.zeros((self.B, self.L_max), np.int64)
            ml, tl = np.zeros(self.B, np.int32), np.zeros(self.B, np.int32)
            for b, i in enumerate(items):
                item = self.dataset[i]
                tok, mel = np.asarray(item[0]), np.asarray(item[1], np.float32)
                if mel.ndim != 2 or mel.shape[0] > self.T_max or tok.size > self.L_max:
                    raise ValueError("item %d: mel %s and %d tokens, expected (<= %d, num_mels) and <= %d"
                                     % (i, mel.shape, tok.size, self.T_max, self.L_max))
                if mels is None:
                    mels = np.zeros((self.B, self.T_max, mel.shape[1]), np.float32)
                mels[b, :mel.shape[0]] = mel
                toks[b, :tok.size] = tok
                ml[b], tl[b] = mel.shape[0], tok.size
            yield {"mels": torch.from_numpy(mels), "mel_lengths": torch.from_numpy(ml), "tokens": torch.from_numpy(toks),
                   "token_lengths": torch.from_numpy(tl), "items": torch.tensor(items, dtype=torch.int64)}


class VocoderBatches:
    """Training batches of the neural vocoder (``vocoder.NeuralVocoderStep`` through ``vocoder.vocoder_batch``).
    source: a ``WavDataset`` or a list of 1-D float32 waveforms at ``hparams.sample_rate``.  Each batch draws B
    utterances with at least ``seg_frames`` frames without replacement, and for each a start frame uniform over the
    segments of seg_frames frames that fit it.  A ``WavDataset`` must hold whole utterances at ``hparams.sample_rate``
    (``WavDataset(items)`` / ``from_ljspeech``, whose items are resampled on load): the segment items of
    ``WavDataset.from_vctk`` carry raw input spans at the file's rate, which this class does not resample, and are
    refused.  Iterating yields {"pcm": (B, pitch) float32 (int16 PCM read as
    x / 32768), "lengths": (B,) int32, "starts": (B,) int32, "items": (B,) source indices}, len(self) batches per epoch.
    The draws are a function of (seed, epoch) alone; ``set_epoch`` moves to another epoch.  ValueError when
    seg_frames < 1, fewer than B utterances qualify or the source is a segmented WavDataset."""

    def __init__(self, source, B, seg_frames=32, seed=0):
        from .audio import num_frames_host
        if int(B) < 1 or int(seg_frames) < 1:
            raise ValueError("B=%r and seg_frames=%r must be >= 1" % (B, seg_frames))
        self.source, self.B, self.seg_frames, self.seed = source, int(B), int(seg_frames), int(seed)
        if isinstance(source, WavDataset):
            if source._segments is not None:
                raise ValueError("VocoderBatches takes whole utterances at the training rate; a segmented WavDataset "
                                 "(WavDataset.from_vctk) holds raw input spans at the file's rate")
            frames = [int(f) for f in source.frame_lengths]
        else:
            frames = [num_frames_host(np.asarray(w).reshape(-1).size) for w in source]
        self.frames = frames
        self.eligible = [i for i, f in enumerate(frames) if f >= self.seg_frames]
        if len(self.eligible) < self.B:
            raise ValueError("%d utterances have >= %d frames; a batch needs %d"
                             % (len(self.eligible), self.seg_frames, self.B))
        self.epoch = 0

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __len__(self):
        return len(self.eligible) // self.B

    def _pcm(self, i):
        if isinstance(self.source, WavDataset):
            x = np.asarray(self.source[i][1])
        else:
            x = np.asarray(self.source[i]).reshape(-1)
        if x.dtype == np.int16:
            return x.astype(np.float32) * np.float32(3.0517578125e-05)        # x / 32768, exactly
        return np.ascontiguousarray(x, dtype=np.float32)

    def __iter__(self):
        rng = np.random.default_rng([self.seed, self.epoch])
        order = rng.permutation(len(self.eligible))
        for k in range(len(self)):
            items = [self.eligible[j] for j in order[k * self.B:(k + 1) * self.B]]
            starts = np.array([rng.integers(0, self.frames[i] - self.seg_frames + 1) for i in items], np.int32)
            wavs = [self._pcm(i) for i in items]
            pcm = np.zeros((self.B, max(w.size for w in wavs)), np.float32)
            for b, w in enumerate(wavs):
                pcm[b, :w.size] = w
            yield {"pcm": torch.from_numpy(pcm), "lengths": torch.tensor([w.size for w in wavs], dtype=torch.int32),
                   "starts": torch.from_numpy(starts), "items": torch.tensor(items, dtype=torch.int64)}
