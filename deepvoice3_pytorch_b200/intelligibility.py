"""Intelligibility of speech (DESIGN.md section 2.20): STOI (Taal, Hendriks, Heusdens & Jensen 2011) and ESTOI (Jensen &
Taal 2016) of processed speech against clean speech, batched on the GPU (csrc/stoi.cu).

Definitions (fs = 10 kHz, frame 256, FFT 512, hop 128, 15 one-third-octave bands from 150 Hz, segments of N = 30
frames, beta = -15 dB, dynamic range 40 dB, eps = 2.220446049250313e-16):

* resampling to 10 kHz with ``audio.resample_batch`` (scipy's ``resample_poly`` semantics, rounded to fp32);
* window w(n) = 0.5 - 0.5 cos(2 pi (n + 1) / 257), n < 256 (``np.hanning(258)[1:-1]``); frames of an L-sample signal
  start at 0, 128, ... while start < L - 256;
* silent frames: e_t = 20 log10(||w x_t||_2 + eps) (fp64); frame t is kept when e_t > max(e) - 40.  The kept windowed
  frames are overlap-added at hop 128 into (K - 1) 128 + 256 samples;
* band envelopes of the frames of that signal: X[i, t] = sqrt(sum_{lo_i <= k < hi_i} |rfft_512(w y_t)(k)|^2), with
  pystoi's ``thirdoct`` edges (``band_edges``);
* segments m = N .. F of the F envelope frames (J = F - N + 1 of them): per band row x, y of a segment,
  alpha = ||x|| / (||y|| + eps), y' = min(alpha y, (1 + 10^(15/20)) x), and the correlation of the centred x and y'
  (each divided by its norm + eps).  STOI is the mean over the J x 15 (segment, band) pairs.  ESTOI normalises the rows
  of both 15 x 30 matrices (centre over time, divide by norm + eps), then the columns (centre over bands, divide by
  norm + eps), and averages (1/30) sum X^ Y^ over the segments.  The segment statistics are fp64.

Differences from pystoi and the MATLAB reference, whose parity is unpinned (neither is a dependency of this project):

* the resampler is scipy's ``resample_poly`` (Kaiser-windowed FIR), not pystoi's ``resample_oct``;
* ESTOI's normalisation is deterministic: pystoi adds eps-scaled random noise before each normalisation;
* a pair with fewer than N envelope frames gets NaN and 0 segments (pystoi returns 1e-5), so that one short clip does
  not stop a batch evaluation.

``stoi`` is the standard time-aligned measure; ``stoi_dtw`` warps two signals of different length along a DTW path,
``evaluate_vocoder`` scores copy synthesis, ``evaluate_intelligibility`` scores a TTS model against recordings.
"""

import numpy as np
import torch

from . import audio, mcd, synthesis
from ._lib import lib
from .ops import _p, _stream
from .pitch import _nanmean

FS = 10000
FRAME, NFFT, HOP = 256, 512, 128
BANDS, MIN_FREQ = 15, 150.0
N_SEG = 30
BAND_WARPS, SEG_WARPS = 8, 4      # frames per dv3_stoi_bands CTA, segments per dv3_stoi_segments CTA

_table_cache = {}


def window_fp64():
    """The 256-point analysis window in fp64: np.hanning(258)[1:-1]."""
    n = np.arange(FRAME)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * (n + 1) / (FRAME + 1))


def band_edges():
    """pystoi's ``thirdoct`` on f_k = k 10000 / 512: band i sums bins [lo_i, hi_i), lo_i the bin nearest
    150 2^((2i - 1) / 6) and hi_i the bin nearest 150 2^((2i + 1) / 6) -> (lo, hi) int arrays of 15."""
    f = np.arange(NFFT // 2 + 1) * FS / NFFT
    i = np.arange(BANDS, dtype=np.float64)
    lo = np.abs(f[None, :] - (MIN_FREQ * 2.0 ** ((2 * i - 1) / 6))[:, None]).argmin(1)
    hi = np.abs(f[None, :] - (MIN_FREQ * 2.0 ** ((2 * i + 1) / 6))[:, None]).argmin(1)
    return lo.astype(np.int64), hi.astype(np.int64)


def num_frames(n):
    """Frames of an n-sample signal at 10 kHz: len(range(0, n - 256, 128))."""
    return max(0, -(-(int(n) - FRAME) // HOP))


def _tables(device):
    """(fp32 fft_any.cuh table of N = 512 whose window is ``window_fp64`` then 256 zeros, fp64 window, int32 band
    edges) on ``device``, built once in fp64 and rounded once."""
    key = str(device)
    if key not in _table_cache:
        _, tw, sp = audio._geometry_table_fp64(NFFT, HOP)
        win = np.concatenate([window_fp64(), np.zeros(NFFT - FRAME)])
        flat = np.concatenate([win, np.stack([tw.real, tw.imag], -1).ravel(), np.stack([sp.real, sp.imag], -1).ravel()])
        lo, hi = band_edges()
        _table_cache[key] = (torch.from_numpy(flat.astype(np.float32)).to(device),
                             torch.from_numpy(window_fp64()).to(device),
                             torch.from_numpy(np.concatenate([lo, hi]).astype(np.int32)).to(device))
    return _table_cache[key]


def _check_wavs(wavs, name, device=None):
    """A non-empty list of 1-D fp32 CUDA tensors of >= 1 sample on one device, each giving at most ``mcd.MAX_FRAMES``
    frames at 10 kHz -> their lengths.  Shapes first, then devices; host values only."""
    if not isinstance(wavs, (list, tuple)) or len(wavs) == 0:
        raise ValueError("%s must be a non-empty list of 1-D waveforms" % name)
    up, down = audio.resample_ratio(audio.hparams.sample_rate, FS)
    lens = []
    for k, w in enumerate(wavs):
        if not torch.is_tensor(w) or w.dim() != 1:
            raise ValueError("%s[%d] must be a 1-D tensor" % (name, k))
        if w.dtype != torch.float32:
            raise ValueError("%s[%d] must be fp32, got %s" % (name, k, w.dtype))
        if w.numel() == 0:
            raise ValueError("%s[%d] has no samples" % (name, k))
        F = num_frames(audio.resampled_length(w.numel(), up, down))
        if F > mcd.MAX_FRAMES:
            raise ValueError("%s[%d] gives %d frames at 10 kHz, more than %d" % (name, k, F, mcd.MAX_FRAMES))
        lens.append(int(w.numel()))
    dev = wavs[0].device if device is None else device
    for k, w in enumerate(wavs):
        if not w.is_cuda or w.device != dev:
            raise ValueError("%s[%d] must be a CUDA tensor on %s (there is no CPU path), got %s" % (name, k, dev, w.device))
    return lens


def _check_pair_lists(clean, processed):
    mcd._check_pairs(clean, processed)
    a = _check_wavs(clean, "clean")
    b = _check_wavs(processed, "processed", clean[0].device)
    return a, b


class _Analysis:
    """Device buffers of the first three stages for a list of clips (resampled to 10 kHz): descriptors, per-frame
    energies / keep mask, compacted signals, band envelopes and (optionally) the DTW features."""

    def __init__(self, wavs, mask_clip, want_feat=False):
        dev = wavs[0].device
        lens = [int(w.numel()) for w in wavs]
        pad = torch.nn.utils.rnn.pad_sequence(list(wavs), batch_first=True)
        x, n10 = audio.resample_batch(pad, lens, audio.hparams.sample_rate, sr_to=FS)
        pitch = x.shape[1]
        self.F0 = [num_frames(n) for n in n10]
        cap = [(f - 1) * HOP + FRAME if f else 0 for f in self.F0]
        self.frame_off = np.concatenate([[0], np.cumsum(self.F0)[:-1]]).astype(np.int64)
        ola_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.int64)
        n = len(wavs)
        clips = np.stack([np.arange(n, dtype=np.int64) * pitch, np.array(n10, np.int64), self.frame_off, ola_off,
                          np.asarray(mask_clip, np.int64)], 1)
        self.clips = torch.from_numpy(np.ascontiguousarray(clips)).to(dev)
        table, win64, bands = _tables(dev)
        nfr = max(1, int(sum(self.F0)))
        self.energy = torch.empty(nfr, dtype=torch.float64, device=dev)
        self.keep = torch.empty(nfr, dtype=torch.int32, device=dev)
        self.kept_idx = torch.empty(nfr, dtype=torch.int32, device=dev)
        self.kept = torch.empty(n, dtype=torch.int32, device=dev)
        self.ola = torch.empty(max(1, int(sum(cap))), device=dev)
        self.frames = torch.empty(n, dtype=torch.int32, device=dev)
        self.env = torch.empty(BANDS * nfr, device=dev)
        self.feat = torch.empty(nfr, BANDS, device=dev) if want_feat else None
        st = _stream()
        lib.call("dv3_stoi_frames", _p(x), _p(self.clips), n, _p(win64), _p(self.energy), _p(self.keep),
                 _p(self.kept_idx), _p(self.kept), st)
        lib.call("dv3_stoi_overlap_add", _p(x), _p(self.clips), n, max(cap), _p(table), _p(self.kept_idx),
                 _p(self.kept), _p(self.ola), _p(self.frames), st)
        blocks = [(c, t0) for c in range(n) for t0 in range(0, max(self.F0[c] - 1, 0), BAND_WARPS)]
        blocks_d = torch.tensor(blocks, dtype=torch.int32).reshape(-1, 2).to(dev)
        lib.call("dv3_stoi_bands", _p(self.ola), _p(self.clips), _p(blocks_d), len(blocks), _p(table), _p(bands),
                 _p(self.frames), _p(self.env), _p(self.feat), st)

    def segments(self, pairs, paths, steps_d, seg_cap):
        """pairs: (clean clip, processed clip) per pair; paths: int32 (rows, 2) host array holding every pair's path
        from its path_off; steps_d: int32 device path lengths; seg_cap: host upper bounds of the segments per pair ->
        (result fp64 (P, 2) device, counts int32 (P, 2) device, per-segment values fp64 (rows, 2) device)."""
        dev = self.clips.device
        P = len(pairs)
        path_off = np.concatenate([[0], np.cumsum([len(p) for p in paths])[:-1]]).astype(np.int64)
        seg_off = np.concatenate([[0], np.cumsum(seg_cap)[:-1]]).astype(np.int64)
        pr = np.concatenate([np.asarray(pairs, np.int64).reshape(P, 2), path_off[:, None], seg_off[:, None]], 1)
        pr_d = torch.from_numpy(np.ascontiguousarray(pr)).to(dev)
        flat = np.concatenate([np.zeros((0, 2), np.int32)] + [np.asarray(p, np.int32).reshape(-1, 2) for p in paths])
        path_d = torch.from_numpy(np.ascontiguousarray(flat)).to(dev) if flat.size else None
        blocks = [(p, s0) for p in range(P) for s0 in range(0, int(seg_cap[p]), SEG_WARPS)]
        blocks_d = torch.tensor(blocks, dtype=torch.int32).reshape(-1, 2).to(dev)
        seg = torch.empty(max(1, int(sum(seg_cap))), 2, dtype=torch.float64, device=dev)
        result = torch.empty(P, 2, dtype=torch.float64, device=dev)
        counts = torch.empty(P, 2, dtype=torch.int32, device=dev)
        lib.call("dv3_stoi_segments", _p(self.env), _p(self.clips), _p(pr_d), P, _p(blocks_d), len(blocks), _p(path_d),
                 _p(steps_d), _p(self.kept), _p(seg), _p(result), _p(counts), _stream())
        return result, counts, seg


def _aligned(clean, processed):
    """The checked pairs of ``stoi`` -> (analysis, result, counts, segment values) on the device."""
    P = len(clean)
    an = _Analysis(list(clean) + list(processed), list(range(P)) * 2)
    caps = [max(f - 1, 0) for f in an.F0[:P]]
    paths = [np.repeat(np.arange(c, dtype=np.int32)[:, None], 2, 1) for c in caps]
    res, counts, seg = an.segments([(p, P + p) for p in range(P)], paths, an.frames[:P],
                                   [max(c - N_SEG + 1, 0) for c in caps])
    return an, res, counts, seg


def _host_result(res, counts):
    r = res.cpu().numpy()
    c = counts.cpu().numpy().astype(np.int64)
    return {"stoi": r[:, 0].copy(), "estoi": r[:, 1].copy(), "segments": c[:, 0].copy(), "kept_frames": c[:, 1].copy()}


def stoi(clean, processed):
    """Standard, time-aligned STOI and ESTOI (module docstring) of processed[k] against clean[k]: two lists of 1-D fp32
    CUDA waveforms at ``hparams.sample_rate``, paired by index, of equal length within a pair (as pystoi requires).  The
    silent frames are found on the clean clip and removed from both.  -> {"stoi", "estoi": fp64 (P,), "segments":
    int64 (P,), "kept_frames": int64 (P,) (the clean clip's non-silent frames)}; NaN and 0 segments for a pair with fewer
    than 30 envelope frames.  Every pair in one set of launches; a pair's bits do not depend on the rest of the batch.
    ValueError before any launch for empty or unequal lists, a waveform that is not 1-D fp32 CUDA, has no samples or
    gives more than ``mcd.MAX_FRAMES`` frames at 10 kHz, waveforms on mixed devices, and pairs of unequal length."""
    a, b = _check_pair_lists(clean, processed)
    for k, (n, m) in enumerate(zip(a, b)):
        if n != m:
            raise ValueError("pair %d has %d clean and %d processed samples; stoi needs equal lengths (stoi_dtw "
                             "compares signals of different length)" % (k, n, m))
    _, res, counts, _ = _aligned(clean, processed)
    return _host_result(res, counts)


def _warped(clean, processed, stage):
    P = len(clean)
    with stage("stoi"):
        an = _Analysis(list(clean) + list(processed), list(range(2 * P)), want_feat=True)
    with stage("dtw"):
        F = an.frames.cpu().numpy().astype(np.int64)
        ok = [p for p in range(P) if min(F[p], F[P + p]) >= N_SEG]
        paths = [np.zeros((0, 2), np.int32)] * P
        if ok:
            rows = an.frame_off
            _, _, got = mcd._dtw_path_rows(an.feat.view(-1, BANDS), BANDS, [int(rows[p]) for p in ok],
                                           [int(F[p]) for p in ok], [int(rows[P + p]) for p in ok],
                                           [int(F[P + p]) for p in ok])
            for p, path in zip(ok, got):
                paths[p] = path.astype(np.int32)
    with stage("stoi"):
        L = np.array([len(p) for p in paths], np.int64)
        steps_d = torch.from_numpy(L.astype(np.int32)).to(an.clips.device)
        res, counts, _ = an.segments([(p, P + p) for p in range(P)], paths, steps_d,
                                     [max(int(n) - N_SEG + 1, 0) for n in L])
        out = _host_result(res, counts)
    out["path_length"] = L
    out["frames"] = np.stack([F[:P], F[P:]], 1)
    return out


def stoi_dtw(clean, processed):
    """STOI and ESTOI along a DTW warping path, for signals of different length (synthesized speech against a recording
    of the same text).  This is NOT standard STOI: each side removes its own silent frames (the 40 dB rule applied to
    itself), the path is ``mcd.dtw_path``'s on the log band envelopes 10 log10(max(X^2, 1e-10)) (15 features per
    frame), and the 30-frame segments run over the path's L steps, pairing frame i of the clean side with frame j of
    the processed side.  When the two inputs are identical the path is the diagonal and the result equals ``stoi``'s bit
    for bit.  -> the keys of ``stoi`` plus "path_length": int64 (P,) (0 where not computed) and "frames": int64 (P, 2),
    the envelope frames of (clean, processed).  A pair where either side has fewer than 30 envelope frames gets NaN and
    0 segments.  ValueError before any launch as ``stoi``, except that lengths may differ."""
    _check_pair_lists(clean, processed)
    return _warped(clean, processed, synthesis.stages(None))


def evaluate_vocoder(wavs, method="griffin_lim"):
    """What phase recovery costs in intelligibility, by copy synthesis: each 1-D fp32 CUDA waveform (at
    ``hparams.sample_rate``) -> ``audio.stft_mel_batch`` linear spectrogram -> ``audio.inv_spectrogram_batch(...,
    method=method)`` -> ``stoi`` against the original over the first min(n, n') samples of each pair.  -> {"stoi",
    "estoi", "segments", "kept_frames" as ``stoi``, "mean_stoi", "mean_estoi" (over the non-NaN clips), "vocoded": the
    compared vocoded waveforms on the device}.  One method per call.  ValueError before any launch for an unknown
    method and for the waveforms ``stoi`` refuses."""
    audio.check_phase_method(method)
    lens = _check_wavs(wavs, "wavs")
    dev = wavs[0].device
    pad = torch.nn.utils.rnn.pad_sequence(list(wavs), batch_first=True)
    lin, _ = audio.stft_mel_batch(pad, torch.tensor(lens, dtype=torch.int32), want_mel=False)
    specs = [lin[k, :audio.num_frames(n)].t().cpu().numpy() for k, n in enumerate(lens)]
    rec = audio.inv_spectrogram_batch(specs, method=method)
    m = [min(n, r.size) for n, r in zip(lens, rec)]
    voc = [torch.from_numpy(np.ascontiguousarray(r[:k])).to(dev) for r, k in zip(rec, m)]
    out = stoi([w[:k] for w, k in zip(wavs, m)], voc)
    out["mean_stoi"], out["mean_estoi"] = _nanmean(out["stoi"]), _nanmean(out["estoi"])
    out["vocoded"] = voc
    return out


def evaluate_intelligibility(model, sequences, reference_wavs, speaker_ids=None, vocoder="griffin_lim", batch_size=16,
                             stage_timer=None):
    """Intelligibility of synthesized speech against recordings of the same text, in one call:

    1. synthesize every ``sequences[k]`` with ``synthesis.synthesized_audio`` (stages "synthesis" and "mel");
    2. ``stoi_dtw`` of each synthesized utterance (processed) against its reference (clean): the analysis and the
       segments in stage "stoi", the warping path in stage "dtw";
    3. -> the keys of ``stoi_dtw`` plus "mean_stoi" and "mean_estoi", the means over the utterances whose value is not
       NaN (NaN if there is none).

    reference_wavs: fp32 numpy waveforms at ``hparams.sample_rate``.  Inputs are checked and refused (ValueError before
    any launch) as ``mcd.check_evaluation`` does, and a reference that gives more than ``mcd.MAX_FRAMES`` frames at
    10 kHz is refused too.  stage_timer: optional ``name -> context manager``."""
    mcd.check_evaluation(model, sequences, reference_wavs, speaker_ids, vocoder, batch_size, 1)
    up, down = audio.resample_ratio(audio.hparams.sample_rate, FS)
    for k, w in enumerate(reference_wavs):
        if num_frames(audio.resampled_length(w.size, up, down)) > mcd.MAX_FRAMES:
            raise ValueError("reference_wavs[%d] gives more than %d frames at 10 kHz" % (k, mcd.MAX_FRAMES))
    device = next(model.parameters()).device
    stage = synthesis.stages(stage_timer)
    wavs, _ = synthesis.synthesized_audio(model, sequences, speaker_ids, vocoder, batch_size, device, stage_timer)
    with stage("stoi"):
        refs = [torch.from_numpy(np.ascontiguousarray(w)).to(device) for w in reference_wavs]
    _check_pair_lists(refs, list(wavs))
    out = _warped(refs, list(wavs), stage)
    out["mean_stoi"], out["mean_estoi"] = _nanmean(out["stoi"]), _nanmean(out["estoi"])
    return out
