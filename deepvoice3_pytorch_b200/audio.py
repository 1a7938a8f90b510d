"""Audio front-end with the reference's function names (reference audio.py): ``spectrogram(y)`` and
``melspectrogram(y)`` take a float waveform and return (n_freq, n_frames) arrays in [0, 1] -- computed by ONE fused
GPU pass (csrc/stft.cu) instead of two CPU lws STFTs.  ``stft_mel_batch`` is the batched device API the
preprocessors should use (a whole shard of clips per launch; one H2D, one D2H).  ``stft_mel_targets`` runs the same
transform on a training batch's waveforms and writes the padded, decimated target layout of ``data.collate`` directly
(training from wav files, ``data.WavDataset``).

``inv_spectrogram`` (reference audio.py:37-43) recovers the phase on the same STFT frame with Griffin-Lim (the default,
csrc/stft_any.cu), with fast Griffin-Lim (``method="fast_griffin_lim"``: Griffin-Lim with momentum, as librosa and
torchaudio run it by default) or with Local Weighted Sums (``method="lws"``, csrc/lws.cu), the algorithm of the
reference's ``lws.run_lws``.  The ``lws`` package is an un-vendored dependency whose source is absent, so parity with it is unpinned.

The STFT frame is ``hparams.fft_size`` / ``hparams.hop_size``, as in the reference.  ``check_geometry`` decides which
frames are supported.  The forward transform and LWS have specialised kernels at 1024 / 256 (every reference preset;
csrc/stft.cu, csrc/lws.cu) and run the general ones of csrc/stft_any.cu and csrc/lws_any.cu at any other supported
frame; Griffin-Lim's complex STFT and the inverse STFT run the general kernels of csrc/stft_any.cu at every frame
(DESIGN.md, "Other STFT geometries").
"""
import ctypes
from collections import namedtuple

import numpy as np
import torch

from ._lib import lib, Dv3Error
from .ops import _p


class _HP:
    """Defaults of reference hparams.py / presets/*.json; override by assigning attributes."""
    sample_rate = 22050
    fft_size = 1024
    hop_size = 256
    num_mels = 80
    fmin = 125
    fmax = 7600
    preemphasis = 0.97
    min_level_db = -100
    ref_level_db = 20
    power = 1.4                   # spectrogram sharpening before phase recovery (presets/*.json)
    griffin_lim_iters = 60
    lws_iters = 30                # LWS batch iterations after the no-future initialisation (DESIGN.md section 7)
    griffin_lim_momentum = 0.99   # fast Griffin-Lim (method="fast_griffin_lim"): librosa's / torchaudio's default
    fast_griffin_lim_iters = 20   # FGLA iterations that reach Griffin-Lim-60's convergence (DESIGN.md section 7.3)
    rescaling = False             # preprocess.py: y = x / |x|.max() * rescaling_max (hparams.py:46-48)
    rescaling_max = 0.999
    min_text = 20                 # utterances with shorter transcripts are skipped (hparams.py:137)


hparams = _HP()
_basis_cache = {}

Geometry = namedtuple("Geometry", "n_fft hop bins overlap default")


def check_geometry(mel=True):
    """The STFT frame of ``hparams`` -> Geometry(n_fft, hop, bins = n_fft // 2 + 1, overlap = n_fft // hop, default),
    or Dv3Error naming the rule it breaks.  Supported: n_fft even, 256 <= n_fft <= 4096, n_fft / 2 with no prime factor
    above 5 (the length of the complex transform after real packing: radix-2/3/4/5 passes); hop divides n_fft with
    n_fft / hop in [2, 8] -- an integer overlap, the only case where the squared windows sqrt(hann * 2 hop / n_fft) sum
    to exactly 1, so that the inverse STFT can use the analysis window as its synthesis window.  ``mel``: also the
    filterbank rules of the forward path (num_mels <= 128, fmax <= sample_rate / 2).  Host values only; every audio entry
    point calls it before anything is allocated or launched.  ``default`` (1024 / 256) selects the specialised forward
    and LWS kernels (csrc/stft.cu, csrc/lws.cu); Griffin-Lim and the inverse STFT are the same at every frame."""
    hp = hparams
    N, R = check_frame(hp.fft_size, hp.hop_size)
    if mel:
        if not 0 <= hp.num_mels <= 128:
            raise Dv3Error("num_mels must lie in [0, 128], got %r" % (hp.num_mels,))
        if hp.fmax is not None and hp.fmax > hp.sample_rate / 2:
            raise Dv3Error("fmax %r lies above the Nyquist frequency %r" % (hp.fmax, hp.sample_rate / 2))
    return Geometry(N, R, N // 2 + 1, N // R, (N, R) == (1024, 256))


def check_frame(N, R):
    """The frame rules of ``check_geometry`` for one (fft_size N, hop_size R) -> (N, R) as ints, or Dv3Error naming the
    rule it breaks.  Host values only."""
    if int(N) != N or int(R) != R:
        raise Dv3Error("fft_size and hop_size must be integers, got %r / %r" % (N, R))
    N, R = int(N), int(R)
    if N % 2 or not 256 <= N <= 4096:
        raise Dv3Error("fft_size must be even and lie in [256, 4096], got %d" % N)
    m = N // 2
    for p in (2, 3, 5):
        while m % p == 0:
            m //= p
    if m != 1:
        raise Dv3Error("fft_size / 2 = %d has a prime factor above 5 (the FFT has radix-2/3/4/5 passes only)" % (N // 2))
    if R < 1 or N % R or not 2 <= N // R <= 8:
        raise Dv3Error("hop_size must divide fft_size with fft_size / hop_size in [2, 8] (an integer overlap: only then "
                       "do the squared windows sum to 1), got %d / %d" % (N, R))
    return N, R


_table_cache = {}


def _geometry_table_fp64(N, R):
    """(window w (N,), twiddles W_M^j (M,), split factors W_N^k (M + 1,)) in fp64, M = N / 2: the tables of
    csrc/fft_any.cuh.  w(i) = sqrt(hann(i + 1/2) * 2R / N), the lws window."""
    n = np.arange(N)
    win = np.sqrt(0.5 * (1.0 - np.cos(2.0 * np.pi * (n + 0.5) / N)) * 2.0 * R / N)
    M = N // 2
    tw = np.exp(-2j * np.pi * np.arange(M) / M)
    sp = np.exp(-2j * np.pi * np.arange(M + 1) / N)
    return win, tw, sp


def _geometry_table(device, N, R):
    """fft_any.cuh's table for (N, R) on ``device``: 3N + 2 fp32 values, each rounded once from fp64 (cached)."""
    key = (str(device), N, R)
    if key not in _table_cache:
        win, tw, sp = _geometry_table_fp64(N, R)
        flat = np.concatenate([win, np.stack([tw.real, tw.imag], -1).ravel(), np.stack([sp.real, sp.imag], -1).ravel()])
        _table_cache[key] = torch.from_numpy(flat.astype(np.float32)).to(device)
    return _table_cache[key]


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    lin = f / (200.0 / 3)
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-10) / 1000.0) / (np.log(6.4) / 27.0), lin)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp((np.log(6.4) / 27.0) * (m - 15.0)), (200.0 / 3) * m)


def _build_mel_basis():
    """Slaney-scale, area-normalised triangular filterbank = librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)
    (reference audio.py:71-76); (num_mels, fft_size//2+1) float32."""
    hp = hparams
    if hp.fmax is not None:
        assert hp.fmax <= hp.sample_rate // 2
    n_bins = 1 + hp.fft_size // 2
    freqs = np.linspace(0, hp.sample_rate / 2.0, n_bins)
    edges = _mel_to_hz(np.linspace(_hz_to_mel(hp.fmin), _hz_to_mel(hp.fmax or hp.sample_rate / 2.0),
                                   hp.num_mels + 2))
    basis = np.zeros((hp.num_mels, n_bins))
    for m in range(hp.num_mels):
        lo, ce, hi = edges[m], edges[m + 1], edges[m + 2]
        up = (freqs - lo) / (ce - lo)
        down = (hi - freqs) / (hi - ce)
        basis[m] = np.maximum(0.0, np.minimum(up, down)) * (2.0 / (hi - lo))
    return basis.astype(np.float32)


def _device_basis(device):
    hp = hparams
    key = (str(device), hp.sample_rate, hp.fft_size, hp.num_mels, hp.fmin, hp.fmax)
    if key not in _basis_cache:
        basis = _build_mel_basis()
        nz = basis > 0
        start = np.array([int(np.argmax(r)) if r.any() else 0 for r in nz], dtype=np.int32)
        length = np.array([int(len(r) - np.argmax(r[::-1]) - s) if r.any() else 0
                           for r, s in zip(nz, start)], dtype=np.int32)
        _basis_cache[key] = (torch.from_numpy(basis).to(device), torch.from_numpy(start).to(device),
                             torch.from_numpy(length).to(device))
    return _basis_cache[key]


def decode_wav(path):
    """-> (sample rate, float32 mono waveform): ``load_wav`` before its resampling step."""
    from scipy.io import wavfile
    sr, x = wavfile.read(path)
    if np.issubdtype(x.dtype, np.integer):
        x = x.astype(np.float32) / float(2 ** (8 * x.dtype.itemsize - 1)) if x.dtype != np.uint8 \
            else (x.astype(np.float32) - 128.0) / 128.0
    else:
        x = x.astype(np.float32)
    if x.ndim > 1:
        x = x.mean(axis=1)
    return int(sr), x


def load_wav(path):
    """float32 mono waveform in [-1, 1] at ``hparams.sample_rate`` -- reference audio.py:12-13
    (``librosa.core.load(path, sr=hparams.sample_rate)[0]``).  Host-side file plumbing (scipy): integer PCM is scaled by
    its full range, channels are averaged, and a file at another rate is resampled with a polyphase filter (librosa
    uses resampy's kaiser_best; identical output only when the rates already agree, as for the reference's datasets)."""
    sr, x = decode_wav(path)
    if sr != hparams.sample_rate:
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(int(sr), int(hparams.sample_rate))
        x = resample_poly(x, hparams.sample_rate // g, sr // g).astype(np.float32)
    return np.ascontiguousarray(x, dtype=np.float32)


def save_wav(wav, path):
    """16-bit PCM at ``hparams.sample_rate``, peak-normalised exactly like reference audio.py:16-18."""
    from scipy.io import wavfile
    wav = np.asarray(wav, dtype=np.float64)
    wav = wav * 32767 / max(0.01, np.max(np.abs(wav)))
    wavfile.write(path, hparams.sample_rate, wav.astype(np.int16))


def preemphasis(x):
    """y[n] = x[n] - c*x[n-1] on the host (reference audio.py:21-23, ``lfilter([1, -c], [1], x)``); the fused kernel
    applies the same filter on the fly, this function exists for callers that want the signal itself."""
    from scipy import signal
    return signal.lfilter([1, -hparams.preemphasis], [1], np.asarray(x))


def _linear_to_mel(spectrogram):
    """mel_basis @ |S| -- reference audio.py:64-68 (host-side helper; the kernel fuses it)."""
    return np.dot(_build_mel_basis(), spectrogram)


def num_frames(n_samples):
    g = check_geometry(mel=False)
    if g.default:
        return lib.raw("dv3_stft_num_frames")(int(n_samples))
    return lib.raw("dv3_stft_num_frames_geom")(int(n_samples), g.n_fft, g.hop)


def num_frames_host(n_samples):
    """``num_frames`` restated in Python (no CUDA library load), for DataLoader workers: frames of the padded STFT,
    ceil((n + 2*(fft - hop) - fft) / hop) + 1."""
    fft, hop = hparams.fft_size, hparams.hop_size
    return (int(n_samples) + 2 * (fft - hop) - fft + hop - 1) // hop + 1


def stft_mel_targets(wav, lengths, T_lin, r, downsample_step, lengths_dev=None):
    """Training targets of a waveform batch in ``data.collate``'s layout, in one launch (plus the peak pass when
    ``hparams.rescaling`` is on).

    wav: (B, pitch) int16 PCM (read as x / 32768, like ``load_wav``) or fp32 CUDA tensor; lengths: host sequence of
    the B clip lengths in samples; T_lin: collate's ``max_target_len``.  -> y (B, T_lin, fft_size // 2 + 1) with clip c's frame f at
    row r + f, and mel (B, T_lin / downsample_step, num_mels) = the padded mel rows 0, ds, 2*ds, ...; every other row
    zero.  Bit-identical to ``collate`` of the preprocessed .npy features.  lengths_dev: the same lengths as an int32
    tensor on wav's device (otherwise they are copied from the host).  No host synchronisation: every check below
    uses host values only, and all of them run before any launch."""
    if not (torch.is_tensor(wav) and wav.is_cuda and wav.dim() == 2):
        raise Dv3Error("stft_mel_targets needs a (B, pitch) CUDA tensor; there is no CPU path")
    if wav.dtype not in (torch.int16, torch.float32):
        raise Dv3Error("stft_mel_targets takes int16 PCM or fp32 waveforms, got %s" % wav.dtype)
    g = check_geometry()
    lengths = [int(n) for n in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
    B, pitch = wav.shape
    r, ds, T_lin = int(r), int(downsample_step), int(T_lin)
    if len(lengths) != B or not all(0 <= n <= pitch for n in lengths):
        raise Dv3Error("lengths must give 0..%d samples for each of the %d clips" % (pitch, B))
    if r < 1 or ds < 1:
        raise Dv3Error("r and downsample_step must be >= 1 (got %d, %d)" % (r, ds))
    need = r + max(num_frames_host(n) for n in lengths)
    if T_lin < need:
        raise Dv3Error("T_lin=%d is smaller than the %d rows the longest clip needs (r=%d + its frames)"
                       % (T_lin, need, r))
    wav = wav.contiguous()
    dev = wav.device
    if lengths_dev is None:
        lengths_dev = torch.tensor(lengths, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    elif not (lengths_dev.device == dev and lengths_dev.dtype == torch.int32 and lengths_dev.numel() == B):
        raise Dv3Error("lengths_dev must be an int32 tensor of %d lengths on %s" % (B, dev))
    basis, start, length = _device_basis(dev)
    y = torch.empty(B, T_lin, hparams.fft_size // 2 + 1, device=dev)      # the kernel writes every row
    mel = torch.empty(B, -(-T_lin // ds), hparams.num_mels, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    is16 = int(wav.dtype == torch.int16)
    peak = None
    if hparams.rescaling:
        peak = torch.empty(B, device=dev)
        lib.call("dv3_peak_abs_batched", _p(wav), is16, _p(lengths_dev), pitch, B, _p(peak), st)
    if g.default:
        lib.call("dv3_stft_mel_targets", _p(wav), is16, _p(lengths_dev), _p(peak), float(hparams.rescaling_max),
                 _p(basis), _p(start), _p(length), _p(y), _p(mel), B, pitch, T_lin, r, ds, hparams.num_mels,
                 float(hparams.preemphasis), float(hparams.min_level_db), float(hparams.ref_level_db), st)
    else:
        lib.call("dv3_stft_mel_geom", _p(wav), is16, _p(lengths_dev), _p(peak), float(hparams.rescaling_max),
                 _p(_geometry_table(dev, g.n_fft, g.hop)), _p(basis), _p(start), _p(length), _p(y), _p(mel), B,
                 pitch, T_lin, r, ds, hparams.num_mels, g.n_fft, g.hop, float(hparams.preemphasis),
                 float(hparams.min_level_db), float(hparams.ref_level_db), st)
    return y, mel


def stft_mel_batch(wav, lengths=None, want_linear=True, want_mel=True):
    """wav: (nclips, max_len) fp32 CUDA tensor; lengths: int32 CUDA tensor (nclips) or None (= all max_len).
    -> linear (nclips, max_frames, fft_size // 2 + 1), mel (nclips, max_frames, num_mels) in the stored (T, F) layout."""
    if not (torch.is_tensor(wav) and wav.is_cuda and wav.dtype == torch.float32 and wav.dim() == 2):
        raise Dv3Error("stft_mel_batch needs a (nclips, max_len) fp32 CUDA tensor; there is no CPU path")
    g = check_geometry()
    wav = wav.contiguous()
    nclips, max_len = wav.shape
    dev = wav.device
    if lengths is None:
        lengths = torch.full((nclips,), max_len, dtype=torch.int32, device=dev)
    lengths = lengths.to(device=dev, dtype=torch.int32).contiguous()
    max_frames = num_frames(max_len)
    basis, start, length = _device_basis(dev)
    lin = torch.empty(nclips, max_frames, hparams.fft_size // 2 + 1, device=dev) if want_linear else None
    mel = torch.empty(nclips, max_frames, hparams.num_mels, device=dev) if want_mel else None   # kernel zero-fills ragged tails

    def p(t):
        return None if t is None else ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if g.default:
        lib.call("dv3_stft_mel", p(wav), p(lengths), p(basis), p(start), p(length), p(lin), p(mel), nclips, max_len,
                 max_frames, hparams.num_mels, float(hparams.preemphasis), float(hparams.min_level_db),
                 float(hparams.ref_level_db), st)
    else:
        lib.call("dv3_stft_mel_geom", p(wav), 0, p(lengths), None, 1.0, p(_geometry_table(dev, g.n_fft, g.hop)),
                 p(basis), p(start), p(length), p(lin), p(mel), nclips, max_len, max_frames, 0, 1, hparams.num_mels,
                 g.n_fft, g.hop, float(hparams.preemphasis), float(hparams.min_level_db), float(hparams.ref_level_db),
                 st)
    return lin, mel


def resample_ratio(sr_from, sr_to=None):
    """(up, down) = sr_to / sr_from reduced by its gcd (``sr_to`` defaults to ``hparams.sample_rate``)."""
    from math import gcd
    sr_from, sr_to = int(sr_from), int(hparams.sample_rate if sr_to is None else sr_to)
    if sr_from < 1 or sr_to < 1:
        raise ValueError("sample rates must be positive, got %d -> %d" % (sr_from, sr_to))
    g = gcd(sr_from, sr_to)
    return sr_to // g, sr_from // g


def resample_filter_bank(up, down):
    """The filter of ``scipy.signal.resample_poly(x, up, down)`` for fp64 x, in polyphase form: -> (bank (ntaps, up)
    float64 with bank[j, p] = h[p + j * up], pre_remove).  h is ``firwin(2 * half_len + 1, 1 / max(up, down),
    window=('kaiser', 5.0)) * up`` with half_len = 10 * max(up, down), preceded by resample_poly's down - half_len % down
    zeros; pre_remove is the number of leading outputs resample_poly drops.  up == down == 1 is the identity."""
    from scipy.signal import firwin
    if up == 1 and down == 1:
        return np.ones((1, 1)), 0
    max_rate = max(up, down)
    half_len = 10 * max_rate
    h = firwin(2 * half_len + 1, 1.0 / max_rate, window=("kaiser", 5.0)) * up
    n_pre_pad = down - half_len % down
    h = np.concatenate([np.zeros(n_pre_pad), h])
    ntaps = -(-len(h) // up)
    h = np.concatenate([h, np.zeros(ntaps * up - len(h))])
    return np.ascontiguousarray(h.reshape(ntaps, up)), (half_len + n_pre_pad) // down


_bank_cache = {}


def _device_bank(device, up, down):
    key = (str(device), up, down)
    if key not in _bank_cache:
        bank, pre_remove = resample_filter_bank(up, down)
        _bank_cache[key] = (torch.from_numpy(bank).to(device), bank.shape[0], pre_remove)
    return _bank_cache[key]


def resampled_length(n, up, down):
    """Samples of resample_poly's output for n input samples: ceil(n * up / down)."""
    return -(-int(n) * up // down)


def _pcm_batch(wav, name):
    if not (torch.is_tensor(wav) and wav.is_cuda and wav.dim() == 2):
        raise Dv3Error("%s needs a (nclips, pitch) CUDA tensor; there is no CPU path" % name)
    if wav.dtype not in (torch.int16, torch.float32):
        raise Dv3Error("%s takes int16 PCM or fp32 waveforms, got %s" % (name, wav.dtype))
    if wav.shape[0] < 1:
        raise Dv3Error("%s needs at least one clip" % name)
    return wav.contiguous()


def _host_ints(values, n, name, what):
    values = [int(v) for v in (values.tolist() if torch.is_tensor(values) else values)]
    if len(values) != n:
        raise Dv3Error("%s: %s must give one value per clip (%d), got %d" % (name, what, n, len(values)))
    return values


def resample_batch(wav, lengths, sr_from, sr_to=None):
    """Resample a ragged batch from ``sr_from`` to ``sr_to`` (``hparams.sample_rate`` by default) in one launch: wav
    (nclips, pitch) int16 PCM (read as x / 32768, like ``load_wav``) or fp32 CUDA tensor, clip c valid for its first
    lengths[c] samples (host sequence).  -> (out (nclips, pitch_out) fp32 with clip c's ``resampled_length`` samples and
    zeros after them, the output lengths as a list).  Each output sample is scipy's ``resample_poly`` of the fp64 clip
    rounded to fp32 (csrc/resample.cu), bit-identical whatever else is in the batch."""
    wav = _pcm_batch(wav, "resample_batch")
    nclips, pitch = wav.shape
    lengths = _host_ints(lengths, nclips, "resample_batch", "lengths")
    if not all(0 <= n <= pitch for n in lengths):
        raise Dv3Error("resample_batch: lengths must lie in 0..%d" % pitch)
    up, down = resample_ratio(sr_from, sr_to)
    out_lens = [resampled_length(n, up, down) for n in lengths]
    pitch_out = max(4, (max(out_lens) + 3) // 4 * 4)
    if pitch_out >= 2 ** 31:
        raise Dv3Error("resample_batch: %d output samples per clip is too many" % pitch_out)
    dev = wav.device
    bank, ntaps, pre_remove = _device_bank(dev, up, down)
    lengths_dev = torch.tensor(lengths, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    out = torch.empty(nclips, pitch_out, device=dev)                   # the kernel writes every sample
    lib.call("dv3_resample_poly_batched", _p(wav), int(wav.dtype == torch.int16), _p(lengths_dev), pitch, _p(out),
             pitch_out, nclips, _p(bank), up, down, ntaps, pre_remove,
             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return out, out_lens


def input_span(n_in, seg_start, seg_len, up, down, ntaps, pre_remove):
    """-> (start, length): the input samples that resampled outputs [seg_start, seg_start + seg_len) of an n_in-sample
    clip read (csrc/resample.cu: output m reads x[b - j], j < ntaps, b = (m + pre_remove) * down // up), clipped to
    [0, n_in).  (0, 0) when they read none, as an empty segment does."""
    if seg_len <= 0:
        return 0, 0
    first = (seg_start + pre_remove) * down // up - (ntaps - 1)
    end = (seg_start + seg_len - 1 + pre_remove) * down // up + 1
    first, end = max(0, first), min(int(n_in), end)
    return (first, end - first) if end > first else (0, 0)


SEG_FIELDS = ("row", "n_in", "in_start", "in_len", "seg_start", "seg_len")    # dv3_resample_segments_batched's desc


def resample_segments(wav, seg, sr_from, out, seg_dev=None):
    """Part of each clip's ``resample_batch`` output, bit for bit, in one launch.  seg: host (nclips, 6) ints, one
    ``SEG_FIELDS`` row per clip: row ``row`` of wav ((rows, pitch_in) int16 PCM or fp32 CUDA tensor) holds samples
    [in_start, in_start + in_len) of a source clip of n_in samples at ``sr_from``; row ``row`` of out ((rows, pitch_out)
    fp32 CUDA tensor) gets its resampled samples [seg_start, seg_start + seg_len) in columns [0, seg_len) and zeros after
    them.  The row must hold ``input_span`` of the segment.  A clip at ``hparams.sample_rate`` runs the same launch with
    the one-tap identity bank (an exact copy).  seg_dev: seg as an int32 tensor on out's device (else it is copied from
    the host).  Every check uses host values and runs before the launch; after the first call per (rate, device) there is
    no host synchronisation."""
    wav = _pcm_batch(wav, "resample_segments")
    if not (torch.is_tensor(out) and out.is_cuda and out.dtype == torch.float32 and out.dim() == 2
            and out.is_contiguous() and out.device == wav.device):
        raise Dv3Error("resample_segments: out must be a contiguous 2-D fp32 tensor on %s" % wav.device)
    seg = [[int(v) for v in r] for r in (seg.tolist() if torch.is_tensor(seg) else seg)]
    if not 1 <= len(seg) <= 65535 or any(len(r) != len(SEG_FIELDS) for r in seg):
        raise Dv3Error("resample_segments: seg must give 1..65535 rows of %s" % (SEG_FIELDS,))
    rows_in, pitch_in = wav.shape
    rows_out, pitch_out = out.shape
    up, down = resample_ratio(sr_from)
    bank, ntaps, pre_remove = _device_bank(wav.device, up, down)
    if len({r[0] for r in seg}) != len(seg):
        raise Dv3Error("resample_segments: two clips share a row")
    for row, n_in, in_start, in_len, s0, n in seg:
        if not (0 <= row < min(rows_in, rows_out)):
            raise Dv3Error("resample_segments: row %d is not a row of both wav and out" % row)
        if not (n_in >= 0 and 0 <= s0 and 0 <= n <= pitch_out and s0 + n <= resampled_length(n_in, up, down)):
            raise Dv3Error("resample_segments: segment [%d, %d) is not inside the %d outputs of an %d-sample clip (or "
                           "longer than the %d-sample rows)" % (s0, s0 + n, resampled_length(max(n_in, 0), up, down),
                                                                n_in, pitch_out))
        if not (0 <= in_start and 0 <= in_len <= pitch_in and in_start + in_len <= n_in):
            raise Dv3Error("resample_segments: input span [%d, %d) is not inside the clip (%d samples) and its row "
                           "(%d)" % (in_start, in_start + in_len, n_in, pitch_in))
        a, m = input_span(n_in, s0, n, up, down, ntaps, pre_remove)
        if m and not (in_start <= a and a + m <= in_start + in_len):
            raise Dv3Error("resample_segments: segment [%d, %d) reads input [%d, %d), the row holds [%d, %d)"
                           % (s0, s0 + n, a, a + m, in_start, in_start + in_len))
    if seg_dev is None:
        seg_dev = torch.tensor(seg, dtype=torch.int32).pin_memory().to(out.device, non_blocking=True)
    elif not (seg_dev.device == out.device and seg_dev.dtype == torch.int32 and seg_dev.is_contiguous()
              and tuple(seg_dev.shape) == (len(seg), len(SEG_FIELDS))):
        raise Dv3Error("resample_segments: seg_dev must be a contiguous int32 (%d, %d) tensor on %s"
                       % (len(seg), len(SEG_FIELDS), out.device))
    lib.call("dv3_resample_segments_batched", _p(wav), int(wav.dtype == torch.int16), pitch_in, _p(seg_dev),
             len(seg), _p(out), pitch_out, _p(bank), up, down, ntaps, pre_remove,
             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return out


def trim_bounds_batch(wav, lengths, top_db, offsets=None):
    """Silence-trim bounds of a ragged batch in one launch: ``librosa.effects.trim(y, top_db)`` with the librosa
    0.6-0.9 defaults (frame 2048, hop 512, ref = max, centred frames with reflect padding) computed in fp64, where
    y = wav[c, offsets[c] : offsets[c] + lengths[c]].  wav as in ``resample_batch``; lengths, offsets (default 0) and
    top_db (a number, or one per clip) are host values.  -> (nclips, 2) int32 CUDA tensor of (start, end) relative to
    y, (0, 0) for a clip with no frame above the threshold (csrc/resample.cu)."""
    wav = _pcm_batch(wav, "trim_bounds_batch")
    nclips, pitch = wav.shape
    lengths = _host_ints(lengths, nclips, "trim_bounds_batch", "lengths")
    offs = [0] * nclips if offsets is None else _host_ints(offsets, nclips, "trim_bounds_batch", "offsets")
    if not all(n >= 0 and o >= 0 and o + n <= pitch for n, o in zip(lengths, offs)):
        raise Dv3Error("trim_bounds_batch: every segment must lie inside its row of %d samples" % pitch)
    dbs = [float(top_db)] * nclips if np.ndim(top_db) == 0 else [float(t) for t in top_db]
    if len(dbs) != nclips:
        raise Dv3Error("trim_bounds_batch: top_db must be a number or one value per clip")
    dev = wav.device
    ints = torch.tensor(lengths + offs, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    dbs = torch.tensor(dbs, dtype=torch.float64).pin_memory().to(dev, non_blocking=True)
    bounds = torch.empty(nclips, 2, dtype=torch.int32, device=dev)
    lib.call("dv3_trim_bounds_batched", _p(wav), int(wav.dtype == torch.int16), _p(ints),
             None if offsets is None else _p(ints[nclips:]), pitch, nclips, _p(dbs), _p(bounds),
             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return bounds


def trim_bounds_reference(y, top_db):
    """``trim_bounds_batch``'s definition restated in numpy fp64 for one segment y -> (start, end): the test oracle of
    the kernel and the host arm of bench_preprocess_vctk.py.  librosa >= 0.10 pads with zeros instead of reflecting,
    which changes the edge frames only."""
    y = np.asarray(y, dtype=np.float64)
    L = len(y)
    if L == 0:
        return 0, 0
    frame, hop = 2048, 512
    padded = y[reflect_index(np.arange(-frame // 2, L + frame // 2), L)]
    mse = np.array([np.mean(padded[hop * f: hop * f + frame] ** 2) for f in range(L // hop + 1)])
    db = 10.0 * np.log10(np.maximum(1e-10, mse))
    keep = np.flatnonzero(db - 10.0 * np.log10(np.maximum(1e-10, mse.max())) > -top_db)
    if keep.size == 0:
        return 0, 0
    return int(hop * keep[0]), int(min(L, hop * (keep[-1] + 1)))


def reflect_index(q, L):
    """Index into a length-L signal of positions q of its ``np.pad(mode='reflect')`` extension (numpy reflects again
    and again when the pad is longer than the signal): period 2 (L - 1), mirrored about 0 and L - 1."""
    q = np.asarray(q)
    if L == 1:
        return np.zeros_like(q)
    period = 2 * (L - 1)
    r = np.mod(q, period)
    return np.where(r >= L, period - r, r)


def _single(y, want_linear, want_mel):
    y = torch.as_tensor(np.asarray(y, dtype=np.float32)).view(1, -1).cuda()
    lin, mel = stft_mel_batch(y, None, want_linear, want_mel)
    return lin, mel


def spectrogram(y):
    """(fft_size//2+1, n_frames) normalised dB magnitude -- reference audio.py:31-34."""
    lin, _ = _single(y, True, False)
    return lin[0].t().cpu().numpy()


def melspectrogram(y):
    """(num_mels, n_frames) normalised dB mel spectrogram -- reference audio.py:46-51."""
    _, mel = _single(y, False, True)
    return mel[0].t().cpu().numpy()


def _amp_to_db(x):
    min_level = np.exp(hparams.min_level_db / 20 * np.log(10))
    return 20 * np.log10(np.maximum(min_level, x))


def _db_to_amp(x):
    return np.power(10.0, x * 0.05)


def _normalize(S):
    return np.clip((S - hparams.min_level_db) / -hparams.min_level_db, 0, 1)


def _denormalize(S):
    return (np.clip(S, 0, 1) * -hparams.min_level_db) + hparams.min_level_db


def inv_num_samples(n_frames):
    """Samples reconstructed from n_frames frames (the hop-aligned length whose forward STFT has n_frames frames)."""
    return (int(n_frames) - 1) * hparams.hop_size - (hparams.fft_size - 2 * hparams.hop_size)


def griffin_lim(mag, n_iter=None, momentum=0.0):
    """mag: (T, fft_size // 2 + 1) fp32 CUDA tensor of linear magnitudes -> waveform (n,) whose STFT magnitude
    approximates it.
    x <- istft(mag * exp(i*angle(stft(x)))), started from the zero-phase inverse; every arrow is one kernel launch
    (the batched kernels with one clip: ``griffin_lim_batch``, which also describes ``momentum``)."""
    momentum = _check_momentum(momentum)
    if not (torch.is_tensor(mag) and mag.is_cuda and mag.dtype == torch.float32 and mag.dim() == 2):
        raise Dv3Error("griffin_lim needs a (T, fft_size // 2 + 1) fp32 CUDA tensor; there is no CPU path")
    return griffin_lim_batch(mag[None], [mag.shape[0]], n_iter, momentum)[0]


def _check_momentum(momentum):
    """-> momentum as a float in [0, 1), else ValueError (the range torchaudio's GriffinLim accepts)."""
    if isinstance(momentum, (bool, np.bool_)) or not isinstance(momentum, (int, float, np.integer, np.floating)):
        raise ValueError("momentum must be a real number in [0, 1), got %r" % (momentum,))
    if not 0.0 <= float(momentum) < 1.0:                  # also refuses NaN
        raise ValueError("momentum must lie in [0, 1), got %r" % (momentum,))
    return float(momentum)


def _ragged_clips(mag, n_frames, name):
    """Checks of a (nclips, T_max, K) magnitude batch, K = fft_size // 2 + 1 -> (mag, n_max, frames_d, samples_d,
    stream, geometry)."""
    if not (torch.is_tensor(mag) and mag.is_cuda and mag.dtype == torch.float32 and mag.dim() == 3):
        raise Dv3Error("%s needs a (nclips, T, fft_size // 2 + 1) fp32 CUDA tensor; there is no CPU path" % name)
    g = check_geometry(mel=False)
    if mag.shape[2] != g.bins:
        raise Dv3Error("%s: magnitudes have %d bins, fft_size %d has %d" % (name, mag.shape[2], g.n_fft, g.bins))
    mag = mag.contiguous()
    nclips, T_max = mag.shape[:2]
    n_frames = [int(t) for t in n_frames]
    if len(n_frames) != nclips or not all(1 <= t <= T_max for t in n_frames):
        raise Dv3Error("n_frames must give 1..%d frames for each of the %d clips" % (T_max, nclips))
    n_samples = [inv_num_samples(t) for t in n_frames]
    if min(n_samples) < 1:
        raise Dv3Error("too few frames (%d) to reconstruct a waveform" % min(n_frames))
    dev = mag.device
    frames_d = torch.tensor(n_frames, dtype=torch.int32).to(dev)
    samples_d = torch.tensor(n_samples, dtype=torch.int32).to(dev)
    return mag, max(n_samples), frames_d, samples_d, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), g


def griffin_lim_batch(mag, n_frames, n_iter=None, momentum=0.0):
    """mag: (nclips, T_max, K) fp32 CUDA tensor (K = fft_size // 2 + 1), clip c valid for its first n_frames[c] frames -> waveforms
    (nclips, n_max), clip c valid for its first inv_num_samples(n_frames[c]) samples and zero after them.  Each clip
    comes out bit-identical to ``griffin_lim`` on that clip alone: the kernels read and write only a clip's own frames
    and samples, and the overlap-add is deterministic (csrc/stft_any.cu).

    momentum: 0 (the default) runs plain Griffin-Lim.  0 < momentum < 1 runs fast Griffin-Lim (Perraudin, Balazs &
    Sondergaard, WASPAA 2013; librosa's and torchaudio's ``momentum``): each iteration projects
    C = X - beta * X_prev, beta = momentum / (1 + momentum), instead of the new spectrum X, where X_prev is the previous
    iteration's X (0 before the first); csrc/stft_any.cu stft_complex_momentum_any_kernel.
    Any other value raises ValueError before anything is allocated or launched."""
    momentum = _check_momentum(momentum)
    mag, n_max, frames_d, samples_d, st, g = _ragged_clips(mag, n_frames, "griffin_lim_batch")
    nclips, T_max = mag.shape[:2]
    dev = mag.device
    spec = torch.zeros(nclips, T_max, g.bins, 2, device=dev)
    spec[..., 0] = mag                                   # zero phase
    x = torch.zeros(nclips, n_max, device=dev)
    tab = _geometry_table(dev, g.n_fft, g.hop)
    if momentum:
        prev = torch.zeros_like(spec)
        beta = momentum / (1.0 + momentum)               # fp64 here, rounded to fp32 once by the call

        def stft(x, spec):
            lib.call("dv3_stft_complex_momentum_geom", _p(x), _p(samples_d), n_max, _p(mag), _p(prev),
                     _p(spec), _p(frames_d), T_max, nclips, beta, _p(tab), g.n_fft, g.hop, st)
    else:
        def stft(x, spec):
            lib.call("dv3_stft_complex_geom", _p(x), _p(samples_d), n_max, _p(mag), _p(spec), _p(frames_d),
                     T_max, nclips, _p(tab), g.n_fft, g.hop, st)
    _istft(spec, x, samples_d, n_max, frames_d, T_max, nclips, st, g, tab)
    for _ in range(hparams.griffin_lim_iters if n_iter is None else n_iter):
        stft(x, spec)
        x.zero_()
        _istft(spec, x, samples_d, n_max, frames_d, T_max, nclips, st, g, tab)
    return x


def _istft(spec, x, samples_d, n_max, frames_d, T_max, nclips, st, g, tab):
    lib.call("dv3_istft_geom", _p(spec), _p(x), _p(samples_d), n_max, _p(frames_d), T_max, nclips, _p(tab), g.n_fft,
             g.hop, st)


def _lws_weights_fp64(N=1024, R=256):
    """(2Q - 1, 11) complex128 with Q = N / R, [q + Q - 1, d + 5] = beta_q(d) = (1/N) sum_n w(n) w(n - q*R)
    exp(-2 pi i d n / N), the sum over the n where both window indices lie in [0, N): the local-weighted-sum weights of
    csrc/lws.cu (N = 1024, R = 256: (7, 11)) and csrc/lws_any.cu."""
    Q = N // R
    n = np.arange(N)
    w = np.sqrt(0.5 * (1.0 - np.cos(2.0 * np.pi * (n + 0.5) / N)) * 2.0 * R / N)     # _geometry_table_fp64's window
    beta = np.zeros((2 * Q - 1, 11), dtype=np.complex128)
    for q in range(-(Q - 1), Q):
        j = n - q * R
        ok = (j >= 0) & (j < N)
        ww = np.where(ok, w * w[np.clip(j, 0, N - 1)], 0.0)
        for d in range(-5, 6):
            beta[q + Q - 1, d + 5] = np.sum(ww * np.exp(-2j * np.pi * d * n / N)) / N
    return beta


def _lws_tables_fp64(N, R):
    """csrc/lws_any.cu's weight table in fp64: beta_q(d) e^{2 pi i d q / Q} ((2Q - 1) * 11 values, [q + Q - 1][d + 5]),
    then the Q roots e^{-2 pi i r / Q}."""
    Q = N // R
    q = np.arange(-(Q - 1), Q)[:, None]
    d = np.arange(-5, 6)[None, :]
    folded = _lws_weights_fp64(N, R) * np.exp(2j * np.pi * d * q / Q)
    return np.concatenate([folded.ravel(), np.exp(-2j * np.pi * np.arange(Q) / Q)])


_lws_weight_cache = {}


def _lws_weights(device, g=None):
    """The weights as [re, im] fp32 pairs on ``device`` (computed once per device and geometry): the 77 of csrc/lws.cu
    at the default frame, csrc/lws_any.cu's table (_lws_tables_fp64) at any other."""
    key = str(device) if g is None or g.default else (str(device), g.n_fft, g.hop)
    if key not in _lws_weight_cache:
        b = _lws_weights_fp64() if g is None or g.default else _lws_tables_fp64(g.n_fft, g.hop)
        w = np.stack([b.real, b.imag], axis=-1).astype(np.float32)
        _lws_weight_cache[key] = torch.from_numpy(np.ascontiguousarray(w)).to(device)
    return _lws_weight_cache[key]


def _check_count(name, value):
    if int(value) != value or value < 0:
        raise ValueError("%s must be a non-negative integer, got %r" % (name, value))
    return int(value)


def lws(mag, n_iter=None, init_iters=1):
    """mag: (T, K) fp32 CUDA tensor of linear magnitudes -> waveform (n,) by LWS phase recovery: the one-clip case of
    ``lws_batch``."""
    n_iter = hparams.lws_iters if n_iter is None else _check_count("n_iter", n_iter)
    init_iters = _check_count("init_iters", init_iters)
    if not (torch.is_tensor(mag) and mag.is_cuda and mag.dtype == torch.float32 and mag.dim() == 2):
        raise Dv3Error("lws needs a (T, fft_size // 2 + 1) fp32 CUDA tensor; there is no CPU path")
    return lws_batch(mag[None], [mag.shape[0]], n_iter, init_iters)[0]


def lws_batch(mag, n_frames, n_iter=None, init_iters=1):
    """Local Weighted Sums phase recovery (Le Roux et al., DAFx 2010; the algorithm of the reference's ``lws.run_lws``,
    parity unpinned: csrc/lws.cu) with the contract of ``griffin_lim_batch``: mag (nclips, T_max, K), clip c valid
    for its first n_frames[c] frames -> waveforms (nclips, n_max), zero past each clip's own samples, each clip
    bit-identical to the clip alone.  The no-future initialisation (``init_iters`` in-frame passes per frame), then
    ``n_iter`` batch iterations (``hparams.lws_iters`` when None), then the inverse STFT."""
    n_iter = hparams.lws_iters if n_iter is None else _check_count("n_iter", n_iter)
    init_iters = _check_count("init_iters", init_iters)
    mag, n_max, frames_d, samples_d, st, g = _ragged_clips(mag, n_frames, "lws_batch")
    nclips, T_max = mag.shape[:2]
    dev = mag.device
    w = _lws_weights(dev, g)
    spec = torch.empty(nclips, T_max, g.bins, 2, device=dev)
    other = torch.empty_like(spec) if n_iter else None
    if g.default:
        lib.call("dv3_lws_nofuture_batched", _p(mag), _p(spec), _p(w), _p(frames_d), T_max, nclips, init_iters, st)
    else:
        lib.call("dv3_lws_nofuture_geom", _p(mag), _p(spec), _p(w), _p(frames_d), T_max, nclips, init_iters,
                 g.n_fft, g.hop, st)
    for _ in range(n_iter):
        if g.default:
            lib.call("dv3_lws_iterate_batched", _p(mag), _p(spec), _p(other), _p(w), _p(frames_d), T_max, nclips,
                     st)
        else:
            lib.call("dv3_lws_iterate_geom", _p(mag), _p(spec), _p(other), _p(w), _p(frames_d), T_max, nclips,
                     g.n_fft, g.hop, st)
        spec, other = other, spec
    x = torch.zeros(nclips, n_max, device=dev)
    _istft(spec, x, samples_d, n_max, frames_d, T_max, nclips, st, g, _geometry_table(dev, g.n_fft, g.hop))
    return x


PHASE_METHODS = ("griffin_lim", "lws", "fast_griffin_lim")


def _is_neural(method):
    """Whether method is a ``vocoder.NeuralVocoder`` instance; a string never imports the vocoder module."""
    if isinstance(method, str):
        return False
    from .vocoder import NeuralVocoder
    return isinstance(method, NeuralVocoder)


def check_phase_method(method):
    """method: one of ``PHASE_METHODS`` or a ``vocoder.NeuralVocoder`` instance, else ValueError."""
    if isinstance(method, str):
        if method not in PHASE_METHODS:
            raise ValueError("method must be one of %s or a NeuralVocoder, got %r" % (", ".join(PHASE_METHODS), method))
        return method
    if not _is_neural(method):
        raise ValueError("method must be one of %s or a NeuralVocoder, got %r" % (", ".join(PHASE_METHODS), method))
    return method


def inv_preemphasis(x):
    """y[n] = x[n] + c*y[n-1] -- reference audio.py:26-28.  x: (n,) or (nclips, n) fp32 CUDA tensor -> tensor; a numpy
    array (the reference's calling convention) is moved to the GPU and a numpy array comes back."""
    if not torch.is_tensor(x):
        return inv_preemphasis(torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()).cpu().numpy()
    x2 = x.view(1, -1) if x.dim() == 1 else x
    x2 = x2.contiguous()
    y = torch.empty_like(x2)
    lib.call("dv3_deemphasis", _p(x2), _p(y), x2.shape[0], x2.shape[1], x2.shape[1], float(hparams.preemphasis),
             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return y.view_as(x)


def inv_spectrogram(spectrogram, n_iter=None, method="griffin_lim"):
    """(K, T) normalised dB spectrogram, K = fft_size // 2 + 1 (what ``spectrogram`` returns / the model predicts,
    transposed) -> waveform
    float32 numpy array -- reference audio.py:37-43: denormalise, dB -> amplitude, ** power, phase recovery, inverse
    STFT, de-emphasis.  The one-clip case of ``inv_spectrogram_batch``."""
    return inv_spectrogram_batch([spectrogram], n_iter, method)[0]


def inv_spectrogram_batch(spectrograms, n_iter=None, method="griffin_lim"):
    """[(K, T_c) normalised dB spectrograms] -> [waveform c (float32 numpy array)], all clips in one set of launches
    per iteration.  Clip c is bit-identical to ``inv_spectrogram(spectrograms[c])``: the magnitude and de-emphasis
    kernels work element by element / causally along each clip, and the phase recovery is ``griffin_lim_batch``
    (``method="griffin_lim"``, ``hparams.griffin_lim_iters`` iterations when n_iter is None), ``lws_batch``
    (``method="lws"``, ``hparams.lws_iters``) or ``griffin_lim_batch`` with ``momentum=hparams.griffin_lim_momentum``
    (``method="fast_griffin_lim"``, ``hparams.fast_griffin_lim_iters``).  An unknown method, a negative LWS or fast
    Griffin-Lim iteration count, or a momentum outside [0, 1) raises ValueError before anything runs.

    A ``vocoder.NeuralVocoder`` instance as ``method`` vocodes the batch with ``method.vocode`` instead (no phase
    recovery, so passing n_iter with it raises ValueError)."""
    check_phase_method(method)
    if _is_neural(method):
        if n_iter is not None:
            raise ValueError("n_iter is an iteration count of phase recovery; a NeuralVocoder takes none")
        return method.vocode(spectrograms)
    if method in ("lws", "fast_griffin_lim") and n_iter is not None:
        _check_count("n_iter", n_iter)
    if method == "fast_griffin_lim":
        momentum = _check_momentum(hparams.griffin_lim_momentum)
        n_iter = hparams.fast_griffin_lim_iters if n_iter is None else n_iter
    specs = [np.asarray(s, dtype=np.float32) for s in spectrograms]
    if not specs:
        raise ValueError("inv_spectrogram_batch needs at least one spectrogram")
    K = check_geometry(mel=False).bins
    for s in specs:
        if s.ndim != 2 or s.shape[0] != K:
            raise Dv3Error("spectrograms must be (%d, T) arrays, got %s" % (K, s.shape))
    n_frames = [s.shape[1] for s in specs]
    S = np.zeros((len(specs), max(n_frames), K), dtype=np.float32)
    for c, s in enumerate(specs):
        S[c, :s.shape[1]] = s.T
    S = torch.from_numpy(S).cuda()
    amp = torch.empty_like(S)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib.call("dv3_spec_to_amp", _p(S), _p(amp), S.numel(), float(hparams.min_level_db), float(hparams.ref_level_db),
             float(hparams.power), st)
    if method == "fast_griffin_lim":
        wav = griffin_lim_batch(amp, n_frames, n_iter, momentum)
    else:
        wav = (lws_batch if method == "lws" else griffin_lim_batch)(amp, n_frames, n_iter)
    wav = inv_preemphasis(wav).cpu().numpy()
    return [wav[c, :inv_num_samples(t)].copy() for c, t in enumerate(n_frames)]
