"""Pitch accuracy of synthesized speech against recordings of the same text (DESIGN.md section 2.18).

* ``yin_f0``: a batched YIN F0 tracker (de Cheveigne & Kawahara 2002, steps 1-5) on the GPU, frame t centred on the
  sample of STFT frame t, so that a warping path computed on mel frames indexes F0 frames directly:
  c_t = t R + R - N / 2 (N = fft_size, R = hop_size: the "perfectrec" padding of N - R zeros on each side), and a clip
  of n samples has ``audio.num_frames(n)`` frames.  With W = N, tau_min = floor(sr / f0_max),
  tau_max = ceil(sr / f0_min) and a_t = c_t - floor((W + tau_max) / 2) (samples outside [0, n) read as zero):

  - difference function (YIN eq. 6, evaluated directly; never as e_0 + e_tau - 2 r(tau), which cancels exactly at the
    dips where the decision is made): d(tau) = sum_{j < W} (x[a_t + j] - x[a_t + j + tau])^2, tau = 1 .. tau_max;
  - CMNDF: d'(tau) = tau d(tau) / sum_{j = 1..tau} d(j), the prefix summed in order; d' = 1 where that sum is 0;
  - absolute threshold: the first tau in [tau_min, tau_max] with d'(tau) < threshold, then forward while d' keeps
    decreasing (voiced); if none passes, the frame is unvoiced and tau* is the argmin of d' over the range, ties to the
    smallest tau;
  - parabolic interpolation of d' at tau* - 1, tau*, tau* + 1 when both neighbours lie in the range and the curvature
    (y0 + y2) - 2 y1 is > 0: delta = (y0 - y2) / (2 curvature) clamped to [-1, 1]; f0 = sr / (tau* + delta);
  - aperiodicity = d'(tau*);
  - silence gate: f0 = 0 where the frame energy sum_{j < W} x[a_t + j]^2 is below 10^(silence_db / 10) times the
    clip's largest frame energy.
  YIN's step 6 (best local estimate) is not done.  f0 = 0 means unvoiced.
* ``f0_metrics``: voicing decision error (VDE), gross pitch error (GPE, |f0_a / f0_b - 1| > 0.2), F0 frame error (FFE)
  and F0 RMSE in cents over the pairs of a warping path, on the host in fp64.
* ``evaluate_pitch``: synthesize, track F0 of both sides, warp on the mel cepstra that ``mcd.mcd_dtw`` uses
  (``mcd.dtw_path``), score.

Parity with WORLD (DIO / Harvest), pYIN or librosa's ``yin`` is unpinned: none of them is installed.
"""
import ctypes
import math
import warnings

import numpy as np
import torch

from . import audio, mcd, synthesis
from ._lib import lib
from .ops import _p, _stream

MAX_TAU = 1024                # the kernel's shared-memory span is sized for lags up to this
GROSS_ERROR = 0.2             # GPE: |f0_a / f0_b - 1| above this is a gross error


def yin_params(f0_min=60.0, f0_max=500.0, threshold=0.1, silence_db=-50.0):
    """Check the tracker's parameters at ``hparams.sample_rate`` -> (tau_min, tau_max, gate = 10^(silence_db / 10)).
    ValueError for f0_min >= f0_max (or either not a positive finite number), tau_min < 2, tau_max > 1024, threshold
    outside (0, 1], silence_db > 0 or NaN."""
    sr = float(audio.hparams.sample_rate)
    for name, v in (("f0_min", f0_min), ("f0_max", f0_max)):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v <= 0:
            raise ValueError("%s must be a positive finite number, got %r" % (name, v))
    if f0_min >= f0_max:
        raise ValueError("f0_min=%r must be below f0_max=%r" % (f0_min, f0_max))
    tau_min, tau_max = int(math.floor(sr / f0_max)), int(math.ceil(sr / f0_min))
    if tau_min < 2:
        raise ValueError("f0_max=%r gives tau_min=%d at %g Hz; it must be >= 2" % (f0_max, tau_min, sr))
    if tau_max > MAX_TAU:
        raise ValueError("f0_min=%r gives tau_max=%d at %g Hz, above %d" % (f0_min, tau_max, sr, MAX_TAU))
    if isinstance(threshold, bool) or not isinstance(threshold, (int, float)) or not 0 < threshold <= 1:
        raise ValueError("threshold must lie in (0, 1], got %r" % (threshold,))
    if isinstance(silence_db, bool) or not isinstance(silence_db, (int, float)) or not silence_db <= 0:
        raise ValueError("silence_db must be <= 0, got %r" % (silence_db,))
    return tau_min, tau_max, 10.0 ** (silence_db / 10.0)


def frame_centres(n_frames):
    """Sample index on which F0 frame t (= STFT frame t) is centred, t < n_frames: t R + R - N / 2."""
    N, R = audio.hparams.fft_size, audio.hparams.hop_size
    return np.arange(int(n_frames), dtype=np.int64) * R + R - N // 2


def _check_wavs(wavs):
    """A non-empty list of 1-D fp32 CUDA tensors on one device, each of >= 1 sample and at most ``mcd.MAX_FRAMES``
    frames -> their frame counts.  Shapes first, then devices; host values only."""
    if not isinstance(wavs, (list, tuple)) or len(wavs) == 0:
        raise ValueError("wavs must be a non-empty list of 1-D waveforms")
    frames = []
    for k, w in enumerate(wavs):
        if not torch.is_tensor(w) or w.dim() != 1:
            raise ValueError("wavs[%d] must be a 1-D tensor" % k)
        if w.dtype != torch.float32:
            raise ValueError("wavs[%d] must be fp32, got %s" % (k, w.dtype))
        if w.numel() == 0:
            raise ValueError("wavs[%d] has no samples" % k)
        F = audio.num_frames_host(w.numel())
        if F > mcd.MAX_FRAMES:
            raise ValueError("wavs[%d] gives %d frames, more than %d" % (k, F, mcd.MAX_FRAMES))
        frames.append(F)
    dev = wavs[0].device
    for k, w in enumerate(wavs):
        if not w.is_cuda or w.device != dev:
            raise ValueError("wavs[%d] must be a CUDA tensor on %s (there is no CPU path), got %s" % (k, dev, w.device))
    return frames


def _yin(wavs, frames, tau_min, tau_max, threshold, gate, want_diff=False):
    """Checked waveforms -> (f0, aperiodicity, energy) flat (sum frames,) fp32 device tensors in clip order, and the
    (sum frames, 2, tau_max) d / d' tensor or None: one ``dv3_yin_f0`` call (the tracker and the gate launch)."""
    g = audio.check_geometry(mel=False)
    dev = wavs[0].device
    FB = lib.raw("dv3_yin_frames_per_cta")(int(tau_max))
    lens = [int(w.numel()) for w in wavs]
    blocks, clips = [], []
    soff = foff = 0
    for n, F in zip(lens, frames):
        for t0 in range(0, F, FB):
            blocks.append((soff, n, foff + t0, t0, min(FB, F - t0)))
        clips.append((foff, F))
        soff += n
        foff += F
    flat = torch.cat([w.contiguous() for w in wavs]).contiguous()
    blocks_d = torch.tensor(blocks, dtype=torch.int64).to(dev)
    clips_d = torch.tensor(clips, dtype=torch.int64).to(dev)
    f0 = torch.empty(foff, device=dev)
    ap = torch.empty(foff, device=dev)
    energy = torch.empty(foff, device=dev)
    diff = torch.empty(foff, 2, tau_max, device=dev) if want_diff else None
    lib.call("dv3_yin_f0", _p(flat), _p(blocks_d), len(blocks), _p(clips_d), len(clips), _p(f0), _p(ap), _p(energy),
             _p(diff), g.n_fft, g.hop, int(tau_min), int(tau_max), ctypes.c_float(threshold), ctypes.c_float(gate),
             ctypes.c_float(audio.hparams.sample_rate), _stream())
    return f0, ap, energy, diff


def yin_f0(wavs, f0_min=60.0, f0_max=500.0, threshold=0.1, silence_db=-50.0):
    """A list of 1-D fp32 CUDA waveforms at ``hparams.sample_rate`` -> list of (f0, aperiodicity) fp32 CUDA tensors of
    ``audio.num_frames(n_k)`` frames each (module docstring; f0 in Hz, 0 = unvoiced), every clip in one launch.  A clip's
    bits do not depend on the rest of the list.  ValueError before any allocation or launch for an empty list, a clip
    of 0 samples or of more than ``mcd.MAX_FRAMES`` frames, a clip that is not 1-D fp32 CUDA, clips on mixed devices,
    and the parameter errors of ``yin_params``."""
    tau_min, tau_max, gate = yin_params(f0_min, f0_max, threshold, silence_db)
    frames = _check_wavs(wavs)
    f0, ap, _, _ = _yin(list(wavs), frames, tau_min, tau_max, threshold, gate)
    offs = np.concatenate([[0], np.cumsum(frames)])
    return [(f0[offs[k]:offs[k + 1]], ap[offs[k]:offs[k + 1]]) for k in range(len(frames))]


def _host_track(f, name, k):
    f = f.detach().cpu().numpy() if torch.is_tensor(f) else np.asarray(f)
    if f.ndim != 1:
        raise ValueError("%s[%d] must be a 1-D F0 track" % (name, k))
    return f.astype(np.float64)


def f0_metrics(f0_a, f0_b, paths):
    """Pitch errors of tracks f0_a[k] against f0_b[k] (1-D, Hz, 0 = unvoiced; tensors or arrays) along paths[k], an
    (L, 2) array of 0-based frame pairs (i, j) such as ``mcd.dtw_path`` returns.  Host fp64, per utterance:

    * "vde": fraction of the L pairs whose voicing differs;
    * "gpe": fraction of the pairs voiced on both sides with |f0_a[i] / f0_b[j] - 1| > 0.2;
    * "ffe": (voicing errors + gross errors) / L;
    * "f0_rmse_cents": RMS of 1200 log2(f0_a[i] / f0_b[j]) over the pairs voiced on both sides;
    * "voiced_fraction": (n, 2), the fraction of each track's own frames that are voiced.
    "gpe" and "f0_rmse_cents" are NaN where no pair is voiced on both sides.  ValueError for lists of unequal length,
    tracks that are not 1-D, paths that are not (L >= 1, 2) or index past a track."""
    if not all(isinstance(x, (list, tuple)) for x in (f0_a, f0_b, paths)) or not \
            len(f0_a) == len(f0_b) == len(paths) or len(paths) == 0:
        raise ValueError("f0_a, f0_b and paths must be non-empty lists of equal length")
    n = len(paths)
    out = {key: np.empty(n) for key in ("vde", "gpe", "ffe", "f0_rmse_cents")}
    out["voiced_fraction"] = np.empty((n, 2))
    for k in range(n):
        fa, fb = _host_track(f0_a[k], "f0_a", k), _host_track(f0_b[k], "f0_b", k)
        p = np.asarray(paths[k])
        if p.ndim != 2 or p.shape[1] != 2 or p.shape[0] == 0 or not np.issubdtype(p.dtype, np.integer):
            raise ValueError("paths[%d] must be an (L >= 1, 2) integer array" % k)
        if p.min() < 0 or p[:, 0].max() >= fa.size or p[:, 1].max() >= fb.size:
            raise ValueError("paths[%d] indexes past its tracks (%d and %d frames)" % (k, fa.size, fb.size))
        a, b = fa[p[:, 0]], fb[p[:, 1]]
        va, vb = a > 0, b > 0
        both = va & vb
        voicing = np.count_nonzero(va != vb)
        ratio = a[both] / b[both]
        gross = np.count_nonzero(np.abs(ratio - 1.0) > GROSS_ERROR)
        L = p.shape[0]
        out["vde"][k] = voicing / L
        out["ffe"][k] = (voicing + gross) / L
        out["gpe"][k] = gross / ratio.size if ratio.size else np.nan
        out["f0_rmse_cents"][k] = math.sqrt(np.mean((1200.0 * np.log2(ratio)) ** 2)) if ratio.size else np.nan
        out["voiced_fraction"][k] = (np.count_nonzero(fa > 0) / fa.size, np.count_nonzero(fb > 0) / fb.size)
    return out


def _nanmean(x):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return float(np.nanmean(x))


def evaluate_pitch(model, sequences, reference_wavs, speaker_ids=None, vocoder="griffin_lim", batch_size=16, n_ceps=24,
                   f0_min=60.0, f0_max=500.0, threshold=0.1, silence_db=-50.0, stage_timer=None):
    """Pitch accuracy of synthesized speech against recordings of the same text, in one call:

    1. synthesize every ``sequences[k]`` with ``synthesis.tts_batch`` (stage "synthesis") and make its mels (stage
       "mel"), then the reference mels (stage "mel" again), as ``mcd.evaluate_synthesis`` does;
    2. F0 of the synthesized and the reference waveforms with ``yin_f0``, all clips in one launch (stage "f0");
    3. the warping path of each pair on the mel cepstra that ``mcd.mcd_dtw`` uses (``mcd.dtw_path``; stage "dtw");
    4. ``f0_metrics`` along each path ->
       {"f0_rmse_cents", "gpe", "vde", "ffe": fp64 (n,), "voiced_fraction": fp64 (n, 2) (synthesized, reference),
       "mcd": fp64 (n,) (bit for bit ``evaluate_synthesis``'s), "path_length": int64 (n,), "frames": int64 (n, 2),
       "frame_ratio": fp64 (n,), and "mean_f0_rmse_cents", "mean_gpe", "mean_vde", "mean_ffe", "mean_mcd": the means
       over the utterances where the value is not NaN (NaN if there is none)}.

    Inputs are checked and refused (ValueError before any launch) as ``evaluate_synthesis`` does, and the F0 parameters
    as ``yin_f0`` does.  stage_timer: optional ``name -> context manager``."""
    tau_min, tau_max, gate = yin_params(f0_min, f0_max, threshold, silence_db)
    K = mcd.check_evaluation(model, sequences, reference_wavs, speaker_ids, vocoder, batch_size, n_ceps)
    device = next(model.parameters()).device
    stage = synthesis.stages(stage_timer)
    wavs, synth = synthesis.synthesized_audio(model, sequences, speaker_ids, vocoder, batch_size, device, stage_timer)
    with stage("mel"):
        ref_wavs, ref = synthesis.wav_clips_and_mels(list(reference_wavs), device)
    n = len(synth)
    with stage("f0"):
        clips = list(wavs) + list(ref_wavs)             # the device copies the mel stage made
        frames = _check_wavs(clips)
        f0 = _yin(clips, frames, tau_min, tau_max, threshold, gate)[0].cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(frames)])
    tracks = [f0[offs[k]:offs[k + 1]] for k in range(2 * n)]
    with stage("dtw"):
        cep, lengths = mcd._cepstra_padded(list(synth) + list(ref), K)
        T_max = cep.shape[1]
        rows = [q * T_max for q in range(2 * n)]
        cost, length, paths = mcd._dtw_path_rows(cep.view(-1, K), K, rows[:n], lengths[:n], rows[n:], lengths[n:])
        res = mcd._result(cost, length)
    m = f0_metrics(tracks[:n], tracks[n:], paths)
    frames_np = np.array([[s.shape[0], r.shape[0]] for s, r in zip(synth, ref)], np.int64)
    out = {"f0_rmse_cents": m["f0_rmse_cents"], "gpe": m["gpe"], "vde": m["vde"], "ffe": m["ffe"],
           "voiced_fraction": m["voiced_fraction"], "mcd": res["mcd"], "path_length": res["path_length"],
           "frames": frames_np, "frame_ratio": frames_np[:, 0] / frames_np[:, 1]}
    for key in ("f0_rmse_cents", "gpe", "vde", "ffe", "mcd"):
        out["mean_" + key] = _nanmean(out[key])
    return out
