"""Mel-cepstral distortion after dynamic time warping (MCD-DTW, Kubichek 1993): how close synthesized speech is to a
recording of the same text, in dB (DESIGN.md section 2.17).

* Mel cepstrum of a frame.  A normalised mel row S (what ``audio.stft_mel_batch`` and the model's mel output give) is
  undone to natural-log amplitude, ln A = (S (-min_level_db) + min_level_db + ref_level_db) ln10 / 20, and
  c = DCT-II_ortho(ln A).  c_1 .. c_K are kept (K = n_ceps, default 24, 1 <= K < M); the energy term c_0 is dropped.
  The affine offset of ln A is constant over the mel bins, so it only reaches c_0: the kernel needs the scale
  -min_level_db ln10 / 20 (folded into its DCT table) and the normalised mels, nothing else.
* Frame distance d(i, j) = ||c^a_i - c^b_j||_2, the squares summed over k in index order.
* DTW: D(0,0) = 0, D(i,0) = D(0,j) = +inf, D(i,j) = d(i,j) + min(D(i-1,j-1), D(i-1,j), D(i,j-1)); ties go to the
  diagonal, then to (i-1, j), then to (i, j-1).  The path length L (cells on the chosen path) rides along with the
  chosen predecessor: no N x M matrix, no backtrace.  ``dtw_path`` runs the same recursion and also keeps each cell's
  predecessor in 2 bits, then backtraces the warping path (DESIGN.md section 2.18).
* mcd = (10 sqrt(2) / ln10) D(N, M) / L, in dB, formed on the host in fp64.

This is the MFCC-style mel cepstrum of this project's filterbank, not SPTK's ``mcep`` of a WORLD envelope: numbers are
comparable between runs of this project, and parity with the SPTK-based MCD tools is unpinned.

``mel_cepstra`` and ``dtw`` run the kernels of csrc/mcd.cu, ``dtw_path`` those of csrc/pitch.cu; ``mcd_dtw`` compares
two ragged lists of mels; ``evaluate_synthesis`` synthesizes, makes mels of the synthesized and the reference audio, and
scores them.
"""
import ctypes
import math

import numpy as np
import torch

from . import audio, synthesis
from ._lib import lib
from .ops import _p, _stream

MAX_FRAMES = 16384            # frames per sequence (csrc/mcd.cu MC_MAX_FRAMES): about 190 s at 22 050 Hz / hop 256
MAX_MELS = 128                # the filterbank's limit (audio.check_geometry)
MAX_CEPS = 64                 # the DTW kernel holds a frame's cepstrum in registers
MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)
DIR_BUDGET_BYTES = 1 << 30    # dtw_path: direction words of one launch (a 16 384 x 16 384 pair needs 64 MiB)

_basis_cache = {}


def dct_basis_fp64(M, K, min_level_db=None):
    """(K, M) fp64: rows 1..K of the orthonormal DCT-II times the scale -min_level_db ln10 / 20 that takes a normalised
    mel to natural-log amplitude (``hparams.min_level_db`` by default)."""
    mld = audio.hparams.min_level_db if min_level_db is None else min_level_db
    k = np.arange(1, K + 1)[:, None]
    m = np.arange(M)[None, :]
    return math.sqrt(2.0 / M) * np.cos(np.pi * k * (m + 0.5) / M) * (-mld * math.log(10.0) / 20.0)


def _device_basis(device, M, K):
    key = (str(device), M, K, float(audio.hparams.min_level_db))
    if key not in _basis_cache:
        _basis_cache[key] = torch.from_numpy(dct_basis_fp64(M, K).astype(np.float32)).to(device)
    return _basis_cache[key]


def check_n_ceps(n_ceps, M):
    """ValueError unless 1 <= n_ceps <= min(M - 1, 64) -> int."""
    if isinstance(n_ceps, bool) or int(n_ceps) != n_ceps:
        raise ValueError("n_ceps must be an integer, got %r" % (n_ceps,))
    K = int(n_ceps)
    if not 1 <= K <= min(M - 1, MAX_CEPS):
        raise ValueError("n_ceps=%d outside [1, min(M - 1, %d)] for M=%d mel bins" % (K, MAX_CEPS, M))
    return K


def _check_frames(frames, name, width=None):
    """A non-empty list of 2-D fp32 CUDA tensors of 1..MAX_FRAMES rows and one width (``width`` if given), on one
    device -> the width.  Shapes are checked before the device, so every refusal is host-side."""
    if not isinstance(frames, (list, tuple)) or len(frames) == 0:
        raise ValueError("%s must be a non-empty list of (T, M) tensors" % name)
    W = width
    for i, f in enumerate(frames):
        if not torch.is_tensor(f) or f.dim() != 2:
            raise ValueError("%s[%d] must be a 2-D tensor" % (name, i))
        T, w = f.shape
        if W is None:
            W = int(w)
        if w != W:
            raise ValueError("%s[%d] has %d columns, expected %d" % (name, i, w, W))
        if not 1 <= T <= MAX_FRAMES:
            raise ValueError("%s[%d] has %d frames, outside [1, %d]" % (name, i, T, MAX_FRAMES))
        if f.dtype != torch.float32:
            raise ValueError("%s[%d] must be fp32, got %s" % (name, i, f.dtype))
    dev = frames[0].device
    for i, f in enumerate(frames):
        if not f.is_cuda or f.device != dev:
            raise ValueError("%s[%d] must be a CUDA tensor on %s (there is no CPU path), got %s" % (name, i, dev, f.device))
    return W


def check_mels(mels, name="mels"):
    """-> M; ValueError for anything ``mel_cepstra`` refuses (an empty list, 0 or more than MAX_FRAMES frames, mixed
    or unsupported widths, not fp32 CUDA)."""
    M = _check_frames(mels, name)
    if not 2 <= M <= MAX_MELS:
        raise ValueError("%s have %d mel bins, outside [2, %d]" % (name, M, MAX_MELS))
    return M


def _check_pairs(a, b):
    if not isinstance(a, (list, tuple)) or not isinstance(b, (list, tuple)) or len(a) == 0 or len(a) != len(b):
        raise ValueError("two non-empty lists of equal length are needed, got %s and %s"
                         % (len(a) if isinstance(a, (list, tuple)) else type(a).__name__,
                            len(b) if isinstance(b, (list, tuple)) else type(b).__name__))


def _cepstra_padded(mels, K):
    """Checked mels -> ((n, T_max, K) cepstra, host lengths): one ``dv3_mel_cepstra`` launch."""
    M = mels[0].shape[1]
    dev = mels[0].device
    lengths = [int(m.shape[0]) for m in mels]
    n, T_max = len(mels), max(lengths)
    padded = torch.nn.utils.rnn.pad_sequence([m for m in mels], batch_first=True).contiguous()
    cep = torch.empty(n, T_max, K, device=dev)
    lens = torch.tensor(lengths, dtype=torch.int32).to(dev)
    lib.call("dv3_mel_cepstra", _p(padded), _p(lens), _p(_device_basis(dev, M, K)), _p(cep), n, T_max, M, K, _stream())
    return cep, lengths


def mel_cepstra(mels, n_ceps=24):
    """A list of (T_i, M) normalised fp32 CUDA mels -> list of their (T_i, n_ceps) mel cepstra c_1..c_K (module
    docstring), all sequences in one launch.  Every value is a sum over the M bins in fixed order, so a sequence's
    cepstra do not depend on the others in the list.  ValueError before any launch for an empty list, a sequence of 0
    or more than ``MAX_FRAMES`` frames, mixed widths or M outside [2, 128], K outside [1, min(M - 1, 64)], mels that are
    not fp32 CUDA."""
    M = check_mels(mels)
    K = check_n_ceps(n_ceps, M)
    cep, lengths = _cepstra_padded(mels, K)
    return [cep[q, :n] for q, n in enumerate(lengths)]


def _work_list(a_rows, a_lens, b_rows, b_lens):
    """Host work list (P, 6) int64 (pair, a_row, N, b_row, M, ws_off), longest serial recursion first (ceil(N / 32)
    strips of M + 31 steps), and the workspace floats."""
    P = len(a_lens)
    order = sorted(range(P), key=lambda p: (-(-(-a_lens[p] // 32) * (b_lens[p] + 31)), p))
    work = np.zeros((P, 6), np.int64)
    off = 0
    for r, p in enumerate(order):
        m32 = -(-b_lens[p] // 32) * 32
        work[r] = (p, a_rows[p], a_lens[p], b_rows[p], b_lens[p], off)
        off += 2 * m32
    return work, off


def _dtw_rows(cep, K, a_rows, a_lens, b_rows, b_lens):
    """cep: (rows, K) contiguous fp32 CUDA -> (cost fp32 (P,), path length int32 (P,)) on the device."""
    work, ws_floats = _work_list(a_rows, a_lens, b_rows, b_lens)
    dev = cep.device
    P = len(a_lens)
    work_d = torch.from_numpy(work).to(dev)
    ws = torch.empty(ws_floats, device=dev)
    cost = torch.empty(P, device=dev)
    path = torch.empty(P, dtype=torch.int32, device=dev)
    lib.call("dv3_dtw_mcd", _p(cep), K, _p(work_d), _p(ws), _p(cost), _p(path), P, _stream())
    return cost, path


def _result(cost, path):
    cost = cost.cpu().numpy().astype(np.float64)
    L = path.cpu().numpy().astype(np.int64)
    return {"mcd": MCD_SCALE * cost / L, "cost": cost, "path_length": L}


def _feature_pairs(ceps_a, ceps_b):
    """The checks of ``dtw`` and ``dtw_path`` (host values only), then both sides' rows in one contiguous tensor ->
    (flat (rows, K), K, first row of each sequence, lengths, P); sequences a_0 .. a_{P-1}, then b_0 .. b_{P-1}."""
    _check_pairs(ceps_a, ceps_b)
    K = _check_frames(list(ceps_a) + list(ceps_b), "cepstra")
    if not 1 <= K <= MAX_CEPS:
        raise ValueError("cepstra have %d coefficients, outside [1, %d]" % (K, MAX_CEPS))
    seqs = list(ceps_a) + list(ceps_b)
    lens = [int(c.shape[0]) for c in seqs]
    rows = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
    flat = torch.cat([c.contiguous() for c in seqs]).contiguous()
    return flat, K, rows, lens, len(ceps_a)


def dtw(ceps_a, ceps_b):
    """Two lists of (T, K) fp32 CUDA cepstra (or any feature rows, 1 <= K <= 64), paired by index ->
    {"mcd": fp64 (P,), "cost": D(N, M) fp64 (P,), "path_length": L int64 (P,)}: the DTW of the module docstring, one
    warp per pair, longest pairs first.  A pair's result does not depend on the rest of the batch (bit for bit).
    ValueError before any launch for empty or unequal lists, sequences of 0 or more than ``MAX_FRAMES`` frames, mixed
    widths or K outside [1, 64], tensors that are not fp32 CUDA."""
    flat, K, rows, lens, P = _feature_pairs(ceps_a, ceps_b)
    return _result(*_dtw_rows(flat, K, rows[:P], lens[:P], rows[P:], lens[P:]))


def _dir_words(N, M):
    """Direction words of one pair's warping path: N rows of ceil(M / 16) 32-bit words."""
    return N * (-(-M // 16))


def _path_chunks(work, budget=None):
    """Split the work rows (in list order) into runs [r0, r1) whose direction buffers, 4 bytes a word, total at most
    ``budget`` bytes (``DIR_BUDGET_BYTES``); a run always takes at least one row.  -> list of (r0, r1)."""
    return budget_chunks([4 * _dir_words(int(w[2]), int(w[4])) for w in work], budget)


def budget_chunks(sizes, budget=None):
    """Split rows of ``sizes`` bytes each (in order) into runs [r0, r1) of at most ``budget`` bytes
    (``DIR_BUDGET_BYTES``) in all; a run always takes at least one row.  -> list of (r0, r1)."""
    budget = DIR_BUDGET_BYTES if budget is None else budget
    chunks, r0, used = [], 0, 0
    for r, b in enumerate(sizes):
        if r > r0 and used + b > budget:
            chunks.append((r0, r))
            r0, used = r, 0
        used += b
    chunks.append((r0, len(sizes)))
    return chunks


def _dtw_path_rows(cep, K, a_rows, a_lens, b_rows, b_lens):
    """``_dtw_rows`` that also returns the warping paths: per budget chunk of the work list one ``dv3_dtw_path`` and one
    ``dv3_dtw_backtrace`` launch, reusing one direction buffer.  -> (cost fp32 (P,), L int32 (P,), list of (rows_p, 2)
    int64 host arrays; rows_p = L_p wherever the cost is finite)."""
    work, ws_floats = _work_list(a_rows, a_lens, b_rows, b_lens)
    dev = cep.device
    P = len(a_lens)
    chunks = _path_chunks(work)
    path_work = np.zeros((P, 2), np.int64)
    slot = np.zeros(P, np.int64)                    # pair -> first path row of its slot
    rows = 0
    for r0, r1 in chunks:
        words = 0
        for r in range(r0, r1):
            N, M = int(work[r, 2]), int(work[r, 4])
            path_work[r] = (words, rows)
            slot[work[r, 0]] = rows
            words += _dir_words(N, M)
            rows += N + M - 1
    dir_words = max(sum(_dir_words(int(work[r, 2]), int(work[r, 4])) for r in range(r0, r1)) for r0, r1 in chunks)
    work_d = torch.from_numpy(work).to(dev)
    path_work_d = torch.from_numpy(path_work).to(dev)
    ws = torch.empty(ws_floats, device=dev)
    dirs = torch.empty(dir_words, dtype=torch.int32, device=dev)
    cost = torch.empty(P, device=dev)
    length = torch.empty(P, dtype=torch.int32, device=dev)
    path = torch.empty(rows, 2, dtype=torch.int32, device=dev)
    path_rows = torch.empty(P, dtype=torch.int32, device=dev)
    for r0, r1 in chunks:
        w = ctypes.c_void_p(work_d.data_ptr() + 48 * r0)
        pw = ctypes.c_void_p(path_work_d.data_ptr() + 16 * r0)
        lib.call("dv3_dtw_path", _p(cep), K, w, pw, _p(ws), _p(dirs), _p(cost), _p(length), r1 - r0, _stream())
        lib.call("dv3_dtw_backtrace", w, pw, _p(dirs), _p(path), _p(path_rows), r1 - r0, _stream())
    n = path_rows.cpu().numpy()
    path = path.cpu().numpy().astype(np.int64)
    paths = [np.ascontiguousarray(path[slot[p]:slot[p] + n[p]][::-1]) for p in range(P)]
    return cost, length, paths


def dtw_path(ceps_a, ceps_b):
    """``dtw`` that also returns the warping paths: -> {"mcd", "cost", "path_length"} bit for bit as ``dtw`` gives them
    (the same recursion), plus "path": list of (L_p, 2) int64 arrays of 0-based frame pairs (i, j), from (0, 0) to
    (N - 1, M - 1), monotone with unit steps, the cells the tie rule chose.  Each cell's predecessor is kept as 2 bits,
    so a pair needs N ceil(M / 16) 4-byte words of device memory (64 MiB at 16 384 x 16 384); the work list is split into
    launches whose direction buffers stay within ``DIR_BUDGET_BYTES``.  Where the cost is not finite (NaN or overflowing
    features), the path is still monotone, in the grid and from corner to corner, but its length need not equal
    "path_length".  ValueError before any launch as ``dtw``."""
    flat, K, rows, lens, P = _feature_pairs(ceps_a, ceps_b)
    cost, length, paths = _dtw_path_rows(flat, K, rows[:P], lens[:P], rows[P:], lens[P:])
    res = _result(cost, length)
    res["path"] = paths
    return res


def mcd_dtw(mels_a, mels_b, n_ceps=24):
    """Two ragged lists of (T, M) normalised fp32 CUDA mels, paired by index -> {"mcd": fp64 (P,) in dB, "cost": fp64
    (P,), "path_length": int64 (P,)}: the mel cepstra of both sides in one launch, then ``dtw``.  It serves both
    mel-vs-mel comparisons: a model's mel output against the target mel (no vocoder), and re-analysed audio.
    ValueError before any launch as ``mel_cepstra`` and ``dtw`` refuse."""
    _check_pairs(mels_a, mels_b)
    M = check_mels(list(mels_a) + list(mels_b))
    K = check_n_ceps(n_ceps, M)
    P = len(mels_a)
    cep, lengths = _cepstra_padded(list(mels_a) + list(mels_b), K)
    T_max = cep.shape[1]
    rows = [q * T_max for q in range(2 * P)]
    return _result(*_dtw_rows(cep.view(-1, K), K, rows[:P], lengths[:P], rows[P:], lengths[P:]))


def check_evaluation(model, sequences, reference_wavs, speaker_ids, vocoder, batch_size, n_ceps):
    """The checks of ``evaluate_synthesis`` (host values only, nothing allocated or launched) -> K.  ValueError for an
    unknown phase method, mismatched list lengths, malformed sequences or speaker ids (as ``tts_batch``), n_ceps outside
    [1, min(num_mels - 1, 64)], reference waveforms that are not non-empty 1-D fp32 arrays or give more than
    ``MAX_FRAMES`` frames."""
    audio.check_phase_method(vocoder)
    if not isinstance(reference_wavs, (list, tuple)) or len(reference_wavs) != len(sequences):
        raise ValueError("one reference waveform per sequence is needed: %s for %d sequences"
                         % (len(reference_wavs) if isinstance(reference_wavs, (list, tuple)) else
                            type(reference_wavs).__name__, len(sequences)))
    for k, w in enumerate(reference_wavs):
        if not isinstance(w, np.ndarray) or w.ndim != 1 or w.dtype != np.float32 or w.size == 0:
            raise ValueError("reference_wavs[%d] must be a non-empty 1-D float32 numpy array" % k)
        if audio.num_frames_host(w.size) > MAX_FRAMES:
            raise ValueError("reference_wavs[%d] gives %d frames, more than %d"
                             % (k, audio.num_frames_host(w.size), MAX_FRAMES))
    M = audio.hparams.num_mels
    if not 2 <= M <= MAX_MELS:
        raise ValueError("hparams.num_mels=%d outside [2, %d]" % (M, MAX_MELS))
    K = check_n_ceps(n_ceps, M)
    if speaker_ids is not None and getattr(model, "n_speakers", 1) > 1:
        bad = [int(s) for s in speaker_ids if not 0 <= int(s) < model.n_speakers]
        if bad:
            raise ValueError("speaker ids %s outside [0, %d)" % (bad, model.n_speakers))
    synthesis._check_inputs(model, sequences, speaker_ids, batch_size=batch_size)
    return K


def evaluate_synthesis(model, sequences, reference_wavs, speaker_ids=None, vocoder="griffin_lim", batch_size=16,
                       n_ceps=24, stage_timer=None):
    """MCD-DTW of synthesized speech against recordings of the same text, in one call:

    1. synthesize every ``sequences[k]`` (in voice ``speaker_ids[k]`` for a multi-speaker model) with
       ``synthesis.tts_batch``;
    2. turn the synthesized and the reference waveforms into normalised mels with ``audio.stft_mel_batch``, on the GPU,
       at the same STFT frame;
    3. ``mcd_dtw`` of each synthesized utterance against its reference;
    4. -> {"mcd": fp64 (n,), "path_length": int64 (n,), "frames": int64 (n, 2) (synthesized, reference),
       "frame_ratio": fp64 (n,) synthesized / reference frames, "mean_mcd": float, "median_mcd": float}.

    reference_wavs: fp32 numpy waveforms at ``hparams.sample_rate``.  Trimming silence is the caller's choice
    (``audio.trim_bounds_batch``): leading and trailing silence in a reference raises its MCD, because the warping path
    must still cover it.  A frame ratio far above 1 is the cheap sign of an attention failure that ran to
    ``max_decoder_steps``.  stage_timer: optional ``name -> context manager`` around "synthesis", "mel" (entered for the
    synthesized, then for the reference audio) and "mcd".  ValueError before any launch for an unknown phase method,
    mismatched list lengths, malformed sequences or speaker ids (as ``tts_batch``), n_ceps outside
    [1, min(num_mels - 1, 64)], reference waveforms that are not non-empty 1-D fp32 arrays or give more than
    ``MAX_FRAMES`` frames."""
    K = check_evaluation(model, sequences, reference_wavs, speaker_ids, vocoder, batch_size, n_ceps)
    device = next(model.parameters()).device
    stage = synthesis.stages(stage_timer)
    synth = synthesis.synthesized_mels(model, sequences, speaker_ids, vocoder, batch_size, device, stage_timer)
    with stage("mel"):
        ref = synthesis.wav_mels(list(reference_wavs), device)
    with stage("mcd"):
        res = mcd_dtw(synth, ref, K)
    frames = np.array([[s.shape[0], r.shape[0]] for s, r in zip(synth, ref)], np.int64)
    return {"mcd": res["mcd"], "path_length": res["path_length"], "frames": frames,
            "frame_ratio": frames[:, 0] / frames[:, 1], "mean_mcd": float(np.mean(res["mcd"])),
            "median_mcd": float(np.median(res["mcd"]))}
