"""Dataset preprocessing on the GPU: the caller of the audio front-end.

The reference's ``ljspeech.py`` (``build_from_path`` :9-37, ``_process_utterance`` :40-79) walks ``metadata.csv`` and,
per utterance, loads the wav, optionally rescales it, runs TWO CPU STFTs (``audio.spectrogram`` and
``audio.melspectrogram``) in a process pool and writes ``<name>-spec-%05d.npy`` (T, 513) and ``<name>-mel-%05d.npy``
(T, 80) plus one ``train.txt`` row ``spec|mel|n_frames|text``.  ``build_from_path`` here has the same arguments, writes
the same files and returns the same tuples, but batches the clips through ONE fused kernel launch per batch
(``audio.stft_mel_batch``: one H2D copy, one launch, one D2H copy for ``batch_clips`` utterances); ``num_workers``
threads only overlap the wav decoding and the ``np.save`` calls with the GPU work.  The reference's own
``_process_utterance`` also runs unchanged on this package's ``audio`` module (tests/test_dropin.py) -- one clip per
launch; this module is the batched equivalent.

``build_vctk_from_path`` does the same for the reference's ``vctk.py`` (the corpus of the multi-speaker preset): its
per-clip resampling (48 kHz -> ``hparams.sample_rate``) and silence trimming run as batched kernels too
(``audio.resample_batch``, ``audio.trim_bounds_batch``; csrc/resample.cu).  Both corpora share one sharded loop.

    from deepvoice3_pytorch_b200 import preprocess
    rows = preprocess.build_from_path(in_dir, out_dir, num_workers=4)
    preprocess.write_metadata(rows, out_dir)          # preprocess.py:26-35 of the reference: train.txt
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import audio


def _load(wav_path):
    wav = audio.load_wav(wav_path)
    hp = audio.hparams
    if hp.rescaling:
        wav = wav / np.abs(wav).max() * hp.rescaling_max          # ljspeech.py:59-60
    return np.ascontiguousarray(wav, dtype=np.float32)


def spectrograms_batch(wavs):
    """[float32 waveform (n_i,)] -> [(linear (T_i, 513), mel (T_i, 80))] float32, one fused launch for the whole list:
    what ``audio.spectrogram(w).T`` / ``audio.melspectrogram(w).T`` return per clip."""
    lens = [len(w) for w in wavs]
    # row pitch a multiple of 4 samples: the kernel then stages with 16-byte / bulk copies
    host = torch.zeros(len(wavs), (max(lens) + 3) // 4 * 4, dtype=torch.float32).pin_memory()
    for i, w in enumerate(wavs):
        host[i, :len(w)] = torch.from_numpy(w)
    lin, mel = audio.stft_mel_batch(host.cuda(non_blocking=True), torch.tensor(lens, dtype=torch.int32).cuda())
    lin, mel = lin.cpu().numpy(), mel.cpu().numpy()
    out = []
    for i, n in enumerate(lens):
        T = audio.num_frames(n)
        out.append((lin[i, :T].copy(), mel[i, :T].copy()))
    return out


def build_from_path(in_dir, out_dir, num_workers=1, tqdm=lambda x: x, batch_clips=64, name="ljspeech",
                    rank=None, world=None):
    """Same contract as reference ``ljspeech.build_from_path`` (:9-37): reads ``in_dir/metadata.csv`` and
    ``in_dir/wavs/*.wav``, writes the .npy pairs into ``out_dir`` and returns
    ``[(spectrogram_filename, mel_filename, n_frames, text)]`` in file order.

    Multi-GPU (one process per GPU): utterances are dealt round-robin over the ranks -- the work is independent per
    clip, so there is no data-path collective; file indices are global, every rank writes its own files, and the rows of
    all ranks are merged into file order with one ``all_gather_object`` of the (tiny) row lists.  ``rank`` / ``world``
    default to the initialised ``torch.distributed`` group, else to a single process."""
    hp = audio.hparams
    items = []
    index = 1
    with open(os.path.join(in_dir, "metadata.csv"), encoding="utf-8") as f:
        for line in f:
            parts = line.strip().split("|")
            text = parts[2]
            if len(text) < hp.min_text:
                continue
            items.append((index, os.path.join(in_dir, "wavs", "%s.wav" % parts[0]), (text,)))
            index += 1
    return _build_sharded(items, _load, spectrograms_batch, out_dir, name, num_workers, tqdm,
                          batch_clips, rank, world)


def _build_sharded(items, load, features, out_dir, name, num_workers, tqdm, batch_clips, rank, world):
    """The batched loop of both corpora.  items: [(file index, source, row tail)] in file order; ``load(source)`` runs
    on the ``num_workers`` threads one batch ahead; ``features([loaded])`` -> [(linear, mel), or None to skip the
    utterance].  Writes ``<name>-spec-%05d.npy`` / ``<name>-mel-%05d.npy`` and returns the rows
    (spec_name, mel_name, n_frames) + tail in file order, merged over the ranks (docstring of ``build_from_path``)."""
    import torch.distributed as dist
    if world is None:
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank() if world > 1 else 0
    items = items[rank::world]                       # this rank's share; indices stay global
    rows = []
    with ThreadPoolExecutor(max_workers=max(1, num_workers)) as pool:
        batches = [items[i:i + batch_clips] for i in range(0, len(items), batch_clips)]
        loads = [pool.map(load, [p for _, p, _ in b]) for b in batches[:1]]         # decode one batch ahead
        saves = []
        for bi, batch in enumerate(tqdm(batches)):
            wavs = list(loads[bi])
            if bi + 1 < len(batches):
                loads.append(pool.map(load, [p for _, p, _ in batches[bi + 1]]))
            for (idx, _, tail), feats in zip(batch, features(wavs)):
                if feats is None:
                    continue
                lin, mel = feats
                spec_name, mel_name = "%s-spec-%05d.npy" % (name, idx), "%s-mel-%05d.npy" % (name, idx)
                saves.append(pool.submit(np.save, os.path.join(out_dir, spec_name), lin, allow_pickle=False))
                saves.append(pool.submit(np.save, os.path.join(out_dir, mel_name), mel, allow_pickle=False))
                rows.append((idx, (spec_name, mel_name, lin.shape[0]) + tail))
        for s in saves:
            s.result()
    if world > 1 and dist.is_available() and dist.is_initialized():
        parts = [None] * world
        dist.all_gather_object(parts, rows)
        rows = [r for part in parts for r in part]
    return [r for _, r in sorted(rows, key=lambda ir: ir[0])]


def load_labels(path):
    """HTS label file -> [(start, end, label)]: one ``start end label`` line per entry, times in 100 ns units (what
    the reference reads with nnmnkwii's ``hts.load``)."""
    labels = []
    with open(path, encoding="utf-8") as f:
        for line in f:
            cols = line.split()
            if not cols:
                continue
            if len(cols) != 3:
                raise ValueError("%s: expected 'start end label', got %r" % (path, line.rstrip("\n")))
            labels.append((int(cols[0]), int(cols[1]), cols[2]))
    if not labels:
        raise ValueError("%s: no labels" % path)
    return labels


def start_at(labels):
    """Start time of the first non-silent label -- reference vctk.py:32-39 (its ``assert False`` raises ValueError)."""
    if labels[0][-1] != "pau":
        return labels[0][0]
    for i in range(1, len(labels)):
        if labels[i][-1] != "pau":
            return labels[i][0]
    raise ValueError("no label other than 'pau'")


def end_at(labels):
    """End time of the last non-silent label -- reference vctk.py:42-49, including its loop, which never looks at the
    first label."""
    if labels[-1][-1] != "pau":
        return labels[-1][1]
    for i in range(len(labels) - 2, 0, -1):
        if labels[i][-1] != "pau":
            return labels[i][1]
    raise ValueError("no label other than 'pau'")


def label_cut(path, sr):
    """Samples [b, e) at rate sr that vctk.py:63-65 keeps: int(start_at * 1e-7 * sr), int(end_at * 1e-7 * sr)."""
    labels = load_labels(path)
    try:
        return int(start_at(labels) * 1e-7 * sr), int(end_at(labels) * 1e-7 * sr)
    except ValueError as ex:
        raise ValueError("%s: %s" % (path, ex)) from None


TOP_DB_LABELLED, TOP_DB_UNLABELLED = 25, 15          # vctk.py:66 and :68


def vctk_utterances(in_dir, speakers=None):
    """The utterances of a VCTK tree in the reference's order (nnmnkwii's vctk data sources): speakers are the
    ``txt/pNNN`` directories sorted by number, or ``speakers`` ("225" or "p225") in the given order; per speaker the
    ``txt/pNNN/*.txt`` files sorted by name, each paired with ``wav48/pNNN/<stem>.wav`` and, when it exists,
    ``lab/pNNN/<stem>.lab``.  A transcript without a wav is skipped.  -> [(file index from 1, (wav_path, lab_path or
    None), (text, speaker_id))], text = the file decoded as UTF-8 minus its final character (the newline)."""
    import logging
    txt_root = os.path.join(in_dir, "txt")
    if speakers is None:
        speakers = sorted((d[1:] for d in os.listdir(txt_root)
                           if d.startswith("p") and d[1:].isdigit() and os.path.isdir(os.path.join(txt_root, d))),
                          key=int)
    speakers = [str(s)[1:] if str(s).startswith("p") else str(s) for s in speakers]
    items = []
    for speaker_id, spk in enumerate(speakers):
        d = os.path.join(txt_root, "p" + spk)
        for fn in sorted(f for f in os.listdir(d) if f.endswith(".txt")):
            stem = fn[:-4]
            wav = os.path.join(in_dir, "wav48", "p" + spk, stem + ".wav")
            if not os.path.exists(wav):
                logging.getLogger(__name__).warning("vctk: %s has no wav (%s); skipped", os.path.join(d, fn), wav)
                continue
            lab = os.path.join(in_dir, "lab", "p" + spk, stem + ".lab")
            with open(os.path.join(d, fn), "rb") as f:
                text = f.read().decode("utf-8")[:-1]
            items.append((len(items) + 1, (wav, lab if os.path.exists(lab) else None), (text, speaker_id)))
    return items


def _load_vctk(src):
    """(wav_path, lab_path) -> (pcm, sample rate, label cut or None): 16-bit mono files stay int16, any other format
    is ``audio.decode_wav``'s float32 mono waveform; the cut is in samples at ``hparams.sample_rate``."""
    from scipy.io import wavfile
    wav_path, lab_path = src
    sr, x = wavfile.read(wav_path)
    if not (x.dtype == np.int16 and x.ndim == 1):
        sr, x = audio.decode_wav(wav_path)
    cut = label_cut(lab_path, audio.hparams.sample_rate) if lab_path else None
    return np.ascontiguousarray(x), int(sr), cut


def _host_buffer(clips):
    """[(pcm, ...)] of one dtype -> pinned (n, pitch) tensor, rows zero-padded; pitch a multiple of 8 samples."""
    pitch = max(8, (max(len(c[0]) for c in clips) + 7) // 8 * 8)
    host = torch.zeros(len(clips), pitch, dtype=torch.from_numpy(clips[0][0][:0]).dtype).pin_memory()
    for i, c in enumerate(clips):
        host[i, :len(c[0])] = torch.from_numpy(c[0])
    return host


def _resample_trim_launch(clips):
    """The launches of ``resample_trim_batch`` and ``segment_bounds``: one H2D copy per input dtype, then per source rate
    one ``audio.resample_batch`` launch (files already at ``hparams.sample_rate`` skip it) and one
    ``audio.trim_bounds_batch`` launch on [cut] with top_db 25 or, without labels, on the whole clip with top_db 15.
    -> [(clip indices, cut offsets, resampled batch or None, bounds on the device)], nothing read back yet."""
    sr_to = audio.hparams.sample_rate
    pending = []
    for is16 in (True, False):
        rows = sorted((i for i, c in enumerate(clips) if (c[0].dtype == np.int16) == is16), key=lambda i: clips[i][1])
        if not rows:
            continue
        dev = _host_buffer([clips[i] for i in rows]).cuda(non_blocking=True)
        r0 = 0
        while r0 < len(rows):
            sr = clips[rows[r0]][1]
            r1 = r0 + 1
            while r1 < len(rows) and clips[rows[r1]][1] == sr:
                r1 += 1
            group = rows[r0:r1]
            lens = [len(clips[i][0]) for i in group]
            if sr == sr_to:
                src, resampled = dev[r0:r1], False
            else:
                (src, lens), resampled = audio.resample_batch(dev[r0:r1], lens, sr), True
            offs, segs, tops = [], [], []
            for i, n in zip(group, lens):
                cut = clips[i][2]
                b, e = (0, n) if cut is None else (min(cut[0], n), min(max(cut[1], 0), n))
                offs.append(b)
                segs.append(max(0, e - b))
                tops.append(TOP_DB_UNLABELLED if cut is None else TOP_DB_LABELLED)
            bounds = audio.trim_bounds_batch(src, segs, tops, offs)
            pending.append((group, offs, src if resampled else None, bounds))
            r0 = r1
    return pending


def segment_bounds(clips):
    """clips as in ``resample_trim_batch`` -> [(start, length)] of each trimmed segment in samples of the clip
    resampled to ``hparams.sample_rate`` (length 0: an empty segment): the same launches, reading back only the
    bounds.  ``data.WavDataset.from_vctk`` indexes a corpus with it."""
    out = [None] * len(clips)
    for group, offs, _, bounds in _resample_trim_launch(clips):
        bounds = bounds.cpu().numpy()
        for k, (i, off) in enumerate(zip(group, offs)):
            out[i] = (off + int(bounds[k, 0]), int(bounds[k, 1]) - int(bounds[k, 0]))
    return out


def resample_trim_batch(clips):
    """The GPU stages of VCTK preprocessing for one batch.  clips: [(pcm int16 / float32, sample rate, label cut or
    None)] -> [trimmed float32 segment] (possibly empty): the launches of ``_resample_trim_launch``, one readback of the
    resampled audio and the bounds, and the segments sliced on the host."""
    out = [None] * len(clips)
    for group, offs, src, bounds in _resample_trim_launch(clips):
        bounds = bounds.cpu().numpy()
        src = None if src is None else src.cpu().numpy()
        for k, (i, off) in enumerate(zip(group, offs)):
            s, e = off + int(bounds[k, 0]), off + int(bounds[k, 1])
            if src is not None:
                out[i] = src[k, s:e].copy()
            else:
                x = clips[i][0][s:e]
                out[i] = x.astype(np.float32) / float(2 ** 15) if x.dtype == np.int16 else x.astype(np.float32)
    return out


def _vctk_features(clips):
    """One batch: GPU resampling and trimming, the reference's optional rescaling (vctk.py:70-71), one fused STFT
    launch for the non-empty segments; None for an utterance whose trimmed segment is empty."""
    hp = audio.hparams
    segs = resample_trim_batch(clips)
    keep = [i for i, s in enumerate(segs) if len(s)]
    wavs = [segs[i] / np.abs(segs[i]).max() * hp.rescaling_max if hp.rescaling else segs[i] for i in keep]
    out = [None] * len(clips)
    for i, f in zip(keep, spectrograms_batch(wavs) if wavs else []):
        out[i] = f
    return out


def build_vctk_from_path(in_dir, out_dir, num_workers=1, tqdm=lambda x: x, batch_clips=64, speakers=None,
                         rank=None, world=None):
    """The reference's ``vctk.build_from_path`` (vctk.py:13-29, ``_process_utterance`` :52-87) batched on the GPU:
    reads a VCTK-Corpus tree (``txt/``, ``wav48/`` and the optional ``lab/`` of vctk_preprocess), writes
    ``vctk-spec-%05d.npy`` / ``vctk-mel-%05d.npy`` into ``out_dir`` and returns
    ``[(spectrogram_filename, mel_filename, n_frames, text, speaker_id)]`` in file order (``write_metadata`` makes the
    5-column train.txt of the ``deepvoice3_vctk`` preset).  Utterance order and speaker ids: ``vctk_utterances``.
    Per utterance: resample to ``hparams.sample_rate`` (``audio.resample_batch``), cut to the HTS labels when they
    exist and trim silence with top_db 25, otherwise trim with top_db 15 (``audio.trim_bounds_batch``), rescale when
    ``hparams.rescaling`` is set, then the fused STFT -- ``batch_clips`` utterances per set of launches.  An utterance
    whose trimmed segment is empty (the reference fails on it) gives no files and no row; its index is not reused.
    A label file without a non-'pau' label the reference accepts raises ValueError naming it.  Multi-GPU sharding,
    threads and the row merge are those of ``build_from_path``."""
    items = vctk_utterances(in_dir, speakers)
    return _build_sharded(items, _load_vctk, _vctk_features, out_dir, "vctk", num_workers, tqdm,
                          batch_clips, rank, world)


def write_metadata(metadata, out_dir):
    """``train.txt`` exactly as reference preprocess.py:26-35 writes it (and ``data.TrainTxtDataset`` reads it)."""
    with open(os.path.join(out_dir, "train.txt"), "w", encoding="utf-8") as f:
        for m in metadata:
            f.write("|".join([str(x) for x in m]) + "\n")
    frames = sum(m[2] for m in metadata)
    hours = frames * audio.hparams.hop_size / audio.hparams.sample_rate / 3600
    return frames, hours
