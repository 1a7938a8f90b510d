"""Attention errors and token durations from DeepVoice3 alignments (DESIGN.md section 2.19).

* ``monotonic_alignment``: monotonic alignment search (MAS, the Viterbi recursion of Glow-TTS) over a batch of
  attention alignments A (B, N, L) on the GPU, with lp(t, j) = log(max(A[t, j], 1e-8)) (a NaN cell counts as the
  floor): the path from (0, 0) to (N_b - 1, L_b - 1) that at every step either stays on its token or moves to the next,
  maximising the sum of lp.  Where two predecessors score the same, the path stays on the token.  Out come each token's
  duration in decoder steps and the path's score, and from the same pass over A the per-step argmax p_t and maximum m_t
  and the per-token coverage c_j = sum_t A[t, j].
* ``attention_errors``: counts of the attention failures DeepVoice3 is known for -- skipped and repeated words,
  utterances cut short, decoders that never stop -- from those statistics, on the host in fp64.
* ``evaluate_attention``: encode and decode sentences as ``synthesis.tts_batch`` does, then MAS and the error counts of
  every utterance.  ``teacher_forced_alignment``: durations and alignment confidence of a training batch under teacher
  forcing (to distil a duration model, or to find mislabelled or badly trimmed clips).
"""
import ctypes
import math

import numpy as np
import torch

from . import mcd, synthesis
from ._lib import lib
from .ops import _p, _stream

MAX_TOKENS = 1024             # csrc/align.cu MAS_MAX_TOKENS: one column per thread


def _lengths(x, name, B, hi):
    """B integers in [1, hi] (a sequence, array or tensor) -> int list."""
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    if x.ndim != 1 or x.size != B or not np.issubdtype(x.dtype, np.integer):
        raise ValueError("%s must be %d integers, got %s of shape %s" % (name, B, x.dtype, x.shape))
    if x.min() < 1 or x.max() > hi:
        raise ValueError("%s must lie in [1, %d], got [%d, %d]" % (name, hi, x.min(), x.max()))
    return [int(v) for v in x]


def _check_alignments(aligns, step_lengths, text_lengths):
    """ValueError unless aligns is a (B, N, L) fp32 CUDA tensor with L <= 1024 and the lengths lie in [1, N] / [1, L]
    -> (steps, tokens) int lists.  Host values only."""
    if not torch.is_tensor(aligns) or aligns.dim() != 3:
        raise ValueError("aligns must be a 3-D (B, N, L) tensor")
    if aligns.dtype != torch.float32:
        raise ValueError("aligns must be fp32, got %s" % aligns.dtype)
    B, N, L = aligns.shape
    if B < 1 or N < 1 or not 1 <= L <= MAX_TOKENS:
        raise ValueError("aligns of shape %s: B, N must be >= 1 and L in [1, %d]" % (tuple(aligns.shape), MAX_TOKENS))
    if (B - 1) * aligns.stride(0) + (N - 1) * aligns.stride(1) + L >= 1 << 31 or B * N >= 1 << 31:
        raise ValueError("aligns of shape %s is too large for 32-bit indexing" % (tuple(aligns.shape),))
    steps = _lengths(step_lengths, "step_lengths", B, N)
    tokens = _lengths(text_lengths, "text_lengths", B, L)
    if not aligns.is_cuda:
        raise ValueError("aligns must be a CUDA tensor (there is no CPU path), got %s" % aligns.device)
    return steps, tokens


def _mas(aligns, steps, tokens):
    """Checked alignments -> device tensors (durations int32 (B, L), score fp32 (B,), argmax int32 (B, N), max fp32
    (B, N), coverage fp32 (B, L)): per budget chunk of rows one ``dv3_mas_forward`` and one ``dv3_mas_backtrace``
    launch, reusing one direction buffer."""
    if aligns.stride(2) != 1 or aligns.stride(1) < aligns.size(2) or aligns.stride(0) < 0:
        aligns = aligns.contiguous()
    B, N, L = aligns.shape
    dev = aligns.device
    dir_words = lib.raw("dv3_mas_dir_words")
    words = [int(dir_words(n, l)) for n, l in zip(steps, tokens)]
    chunks = mcd.budget_chunks([4 * w for w in words])
    dir_off = np.zeros(B, np.int64)
    for r0, r1 in chunks:
        dir_off[r0:r1] = np.concatenate([[0], np.cumsum(words[r0:r1 - 1], dtype=np.int64)])
    dirs = torch.empty(max(sum(words[r0:r1]) for r0, r1 in chunks), dtype=torch.int32, device=dev)
    steps_d = torch.tensor(steps, dtype=torch.int32).to(dev)
    tokens_d = torch.tensor(tokens, dtype=torch.int32).to(dev)
    dir_off_d = torch.from_numpy(dir_off).to(dev)
    durations = torch.empty(B, L, dtype=torch.int32, device=dev)
    score = torch.empty(B, device=dev)
    argmax = torch.empty(B, N, dtype=torch.int32, device=dev)
    maxv = torch.empty(B, N, device=dev)
    coverage = torch.empty(B, L, device=dev)
    sb, st = aligns.stride(0), aligns.stride(1)

    def at(t, r0, row):
        return ctypes.c_void_p(t.data_ptr() + t.element_size() * r0 * row)

    for r0, r1 in chunks:
        n = r1 - r0
        lib.call("dv3_mas_forward", at(aligns, r0, sb), sb, st, at(steps_d, r0, 1), at(tokens_d, r0, 1), n, N, L,
                 at(dir_off_d, r0, 1), _p(dirs), at(argmax, r0, N), at(maxv, r0, N), at(coverage, r0, L),
                 at(score, r0, 1), _stream())
        lib.call("dv3_mas_backtrace", at(steps_d, r0, 1), at(tokens_d, r0, 1), n, L, at(dir_off_d, r0, 1),
                 _p(dirs), at(durations, r0, L), _stream())
    return durations, score, argmax, maxv, coverage


def _mas_result(dev_out, steps, tokens):
    durations, score, argmax, maxv, coverage = (t.cpu().numpy() for t in dev_out)
    score = score.astype(np.float64)
    return {"durations": durations.astype(np.int64), "score": score,
            "score_per_step": score / np.asarray(steps, np.float64),
            "argmax": [argmax[b, :n].astype(np.int64) for b, n in enumerate(steps)],
            "max": [maxv[b, :n].copy() for b, n in enumerate(steps)],
            "coverage": [coverage[b, :l].copy() for b, l in enumerate(tokens)]}


def monotonic_alignment(aligns, step_lengths, text_lengths):
    """Monotonic alignment search and per-step statistics of a batch of alignments (module docstring).

    aligns: (B, N, L) fp32 CUDA tensor, row b valid for its first step_lengths[b] steps and text_lengths[b] tokens
    (B integers each, a sequence, array or tensor).  Strided views with unit token stride are read in place: the
    (B, N, T_text) alignments of ``incremental.decode_ragged``, one layer ``a[l]`` or the mean ``a.mean(0)`` of the
    model's (N_attn, B, T_dec, T_text) teacher-forced alignments.  L <= 1024.

    -> {"durations": int64 (B, L), each token's steps on the path (>= 1 and summing to N_b for j < L_b, 0 past it),
    "score": fp64 (B,) the path's sum of lp in fp32, "score_per_step": score / N_b (a per-utterance alignment
    confidence: log of the geometric mean of the attention weights on the path), "argmax": list of int64 (N_b,) p_t
    (ties to the lowest token), "max": list of fp32 (N_b,) m_t (NaN cells count as -inf in both), "coverage": list of
    fp32 (L_b,) c_j summed in increasing t}.  A row with N_b < L_b has no path: zero durations and a score of -inf.  A
    row's results do not depend on the rest of the batch (bit for bit).  ValueError before any launch for a tensor that
    is not 3-D fp32 CUDA, L > 1024, lengths that are not B integers in [1, N] and [1, L], or shapes past 32-bit indexing.
    """
    steps, tokens = _check_alignments(aligns, step_lengths, text_lengths)
    return _mas_result(_mas(aligns, steps, tokens), steps, tokens)


def _runs(x):
    """Lengths of the maximal runs of equal values of a non-empty 1-D array, in order."""
    edges = np.flatnonzero(x[1:] != x[:-1]) + 1
    return np.diff(np.concatenate([[0], edges, [x.size]]))


def attention_errors(argmax, max, coverage, steps, max_decoder_steps, skip_coverage=0.5, repeat_margin=1):
    """Attention-error counts per utterance, on the host in fp64, from the statistics ``monotonic_alignment`` returns.
    argmax, max: lists of (N,) arrays p_t and m_t; coverage: list of (L,) arrays c_j; steps: N per utterance.  With M_t
    the running maximum of p_t:

    * "focus_rate": mean of m_t (FastSpeech's focus rate; 1 for a one-hot attention);
    * "skips": tokens j <= M_{N-1} with c_j < skip_coverage: passed over by the attention;
    * "unreached": L - 1 - M_{N-1}, the tail the attention never got to (an utterance cut short);
    * "repeats": maximal runs of steps t >= 1 with p_t < M_{t-1} - repeat_margin: the attention went back and read again;
    * "max_dwell": the longest run of equal p_t (a stuck attention);
    * "stop_failed": N == max_decoder_steps + 1, the step at which the decoder loop gives up without a stop;
    * "finite": False where the utterance's coverage is not finite (NaN or inf alignments).

    -> dict of (n,) arrays (fp64 focus_rate, int64 counts, bool stop_failed and finite).  ValueError for lists of unequal
    or zero length, arrays that are not 1-D or do not match steps, argmax outside [0, L), max_decoder_steps < 1,
    skip_coverage not a finite number >= 0, repeat_margin not an integer >= 0."""
    if not all(isinstance(x, (list, tuple)) for x in (argmax, max, coverage)) or len(argmax) == 0 or \
            not len(argmax) == len(max) == len(coverage):
        raise ValueError("argmax, max and coverage must be non-empty lists of equal length")
    steps = np.asarray(steps)
    if steps.shape != (len(argmax),) or not np.issubdtype(steps.dtype, np.integer):
        raise ValueError("steps must hold one integer per utterance")
    if isinstance(max_decoder_steps, bool) or int(max_decoder_steps) != max_decoder_steps or max_decoder_steps < 1:
        raise ValueError("max_decoder_steps must be an integer >= 1, got %r" % (max_decoder_steps,))
    if isinstance(skip_coverage, bool) or not isinstance(skip_coverage, (int, float)) or \
            not math.isfinite(skip_coverage) or skip_coverage < 0:
        raise ValueError("skip_coverage must be a finite number >= 0, got %r" % (skip_coverage,))
    if isinstance(repeat_margin, bool) or int(repeat_margin) != repeat_margin or repeat_margin < 0:
        raise ValueError("repeat_margin must be an integer >= 0, got %r" % (repeat_margin,))
    n = len(argmax)
    out = {"focus_rate": np.empty(n), "skips": np.zeros(n, np.int64), "unreached": np.zeros(n, np.int64),
           "repeats": np.zeros(n, np.int64), "max_dwell": np.zeros(n, np.int64), "stop_failed": np.zeros(n, bool),
           "finite": np.zeros(n, bool)}
    for k in range(n):
        p = np.asarray(argmax[k])
        m = np.asarray(max[k], np.float64)
        c = np.asarray(coverage[k], np.float64)
        N = int(steps[k])
        if p.ndim != 1 or m.ndim != 1 or c.ndim != 1 or p.size != N or m.size != N or N < 1 or c.size < 1 or \
                not np.issubdtype(p.dtype, np.integer):
            raise ValueError("utterance %d: argmax and max must be 1-D of steps[%d] = %d entries (argmax integer), "
                             "coverage 1-D and non-empty" % (k, k, N))
        L = c.size
        if p.min() < 0 or p.max() >= L:
            raise ValueError("utterance %d: argmax outside [0, %d)" % (k, L))
        run_max = np.maximum.accumulate(p)
        last = int(run_max[-1])
        back = p[1:] < run_max[:-1] - int(repeat_margin)
        out["focus_rate"][k] = float(np.mean(m))
        out["skips"][k] = int(np.count_nonzero(c[:last + 1] < skip_coverage))
        out["unreached"][k] = L - 1 - last
        out["repeats"][k] = int(np.count_nonzero(back[1:] & ~back[:-1]) + (back[0] if back.size else 0))
        out["max_dwell"][k] = int(_runs(p).max())
        out["stop_failed"][k] = N == int(max_decoder_steps) + 1
        out["finite"][k] = bool(np.isfinite(c).all())
    return out


_THRESHOLDS = ("skip_coverage", "repeat_margin")


def evaluate_attention(model, sequences, speaker_ids=None, batch_size=16, stage_timer=None, durations=None, speed=1.0,
                       **thresholds):
    """Attention errors of a model's synthesis, in one call:

    1. encode and decode every ``sequences[k]`` (in voice ``speaker_ids[k]`` for a multi-speaker model) in padded
       batches of ``batch_size``, sorted by length, exactly as ``synthesis.tts_batch`` does (stages "encoder" and
       "decoder"); no post-net and no vocoder;
    2. ``monotonic_alignment`` of each batch's alignments on the device (stage "mas");
    3. ``attention_errors`` with ``thresholds`` (skip_coverage, repeat_margin) and the decoder's max_decoder_steps ->
       {"focus_rate", "skips", "unreached", "repeats", "max_dwell", "stop_failed", "finite": (n,) arrays as
       ``attention_errors`` gives them, "steps": int64 (n,) decoder steps, "durations": list of int64 (L_k,) arrays,
       "score_per_step": fp64 (n,), and the totals "total_skips", "total_repeats", "total_unreached", "stop_failures"
       and "mean_focus_rate"}, in input order.

    Every row's alignment is the one ``tts_batch`` returns for it.  Inputs are checked as ``tts_batch`` checks them
    (ValueError before any launch for malformed sequences or speaker ids, batch_size < 1, sequences longer than 1024
    tokens, unknown or malformed thresholds).  durations, speed: score duration-guided synthesis, as ``tts_batch``
    runs it; "steps" are then the durations' totals and no utterance counts as a stop failure (each stops at its
    prescribed total by construction)."""
    from .duration import guided_durations
    unknown = sorted(set(thresholds) - set(_THRESHOLDS))
    if unknown:
        raise ValueError("unknown thresholds %s (known: %s)" % (unknown, ", ".join(_THRESHOLDS)))
    if speaker_ids is not None and getattr(model, "n_speakers", 1) > 1:
        bad = [int(s) for s in speaker_ids if not 0 <= int(s) < model.n_speakers]
        if bad:
            raise ValueError("speaker ids %s outside [0, %d)" % (bad, model.n_speakers))
    max_steps = model.seq2seq.decoder.max_decoder_steps
    attention_errors([np.zeros(1, np.int64)], [np.zeros(1)], [np.zeros(1)], [1], max_steps, **thresholds)   # checks
    durs = guided_durations(model, sequences, durations, speed)
    seqs, speaker_ids = synthesis._check_inputs(model, sequences, speaker_ids, batch_size=batch_size)
    if max(s.size for s in seqs) > MAX_TOKENS:
        raise ValueError("a sequence has %d tokens, more than %d" % (max(s.size for s in seqs), MAX_TOKENS))
    stage = synthesis.stages(stage_timer)
    order = sorted(range(len(seqs)), key=lambda i: -seqs[i].size)
    res = [None] * len(seqs)
    for c in range(0, len(order), int(batch_size)):
        idx = order[c:c + int(batch_size)]
        ids = None if speaker_ids is None else [speaker_ids[i] for i in idx]
        _, aligns, _, steps, _ = synthesis._decode_chunk(model, [seqs[i] for i in idx], ids, stage,
                                                         None if durs is None else [durs[i] for i in idx])
        tokens = [seqs[i].size for i in idx]
        with stage("mas"):
            out = _mas_result(_mas(aligns, steps, tokens), steps, tokens)
        for b, i in enumerate(idx):
            res[i] = (steps[b], out["durations"][b, :tokens[b]], out["score_per_step"][b], out["argmax"][b],
                      out["max"][b], out["coverage"][b])
    steps = np.array([r[0] for r in res], np.int64)
    err = attention_errors([r[3] for r in res], [r[4] for r in res], [r[5] for r in res], steps, max_steps,
                           **thresholds)
    if durs is not None:
        err["stop_failed"][:] = False
    err.update({"steps": steps, "durations": [r[1] for r in res], "score_per_step": np.array([r[2] for r in res]),
                "total_skips": int(err["skips"].sum()), "total_repeats": int(err["repeats"].sum()),
                "total_unreached": int(err["unreached"].sum()), "stop_failures": int(err["stop_failed"].sum()),
                "mean_focus_rate": float(np.mean(err["focus_rate"]))})
    return err


def teacher_forced_steps(target_lengths, r, downsample_step):
    """Decoder steps that cover each row's own frames in a ``data.collate`` batch: ceil((r + n) / (r downsample_step))
    for a target of n frames.  Collate puts r zero frames (the initial decoder state) ahead of the n target frames, and
    decoder step s reads input frames [s r ds, (s + 1) r ds) of that layout; the step that holds the row's last frame is
    the last one counted.  Its done target is 1, as is every later one's."""
    n = np.asarray(target_lengths, np.int64)
    rd = int(r) * int(downsample_step)
    return (int(r) + n + rd - 1) // rd


@torch.no_grad()
def teacher_forced_alignment(model, batch, layer=None):
    """Durations and alignment confidence of a training batch under teacher forcing.

    batch: a dict as ``data.collate`` + ``train_step.to_device`` or ``data.wav_batch_to_device`` return it, on the
    model's device.  Runs the model's teacher-forced seq2seq forward (the model must be in eval mode; no gradient),
    then ``monotonic_alignment`` on the mean of the (N_attn, B, T_dec, T_text) alignments over the attention layers, or
    on layer ``layer`` alone.  Row b spans ``teacher_forced_steps`` of its target length and its input length in tokens.
    A multi-speaker model takes batch["speaker_ids"].

    -> the dict of ``monotonic_alignment``, plus "steps" (int64 (B,)) and "frames_per_step": r * downsample_step, the
    linear-spectrogram frames of one decoder step (durations times it are frames).  ValueError for a model in training
    mode, a layer outside [0, N_attn), a batch that lacks the collate keys, and what ``monotonic_alignment`` refuses."""
    if model.training:
        raise ValueError("teacher_forced_alignment needs the model in eval mode (model.eval())")
    missing = [k for k in ("x", "mel", "y", "text_positions", "frame_positions", "target_lengths", "input_lengths")
               if k not in batch]
    if missing:
        raise ValueError("batch lacks %s" % missing)
    dec = model.seq2seq.decoder
    n_attn = 1 if hasattr(dec, "audio_encoder_modules") else sum(a is not None for a in dec.attention)
    if layer is not None and (isinstance(layer, bool) or int(layer) != layer or not 0 <= layer < n_attn):
        raise ValueError("layer must be None or in [0, %d), got %r" % (n_attn, layer))
    if model.n_speakers > 1 and "speaker_ids" not in batch:
        raise ValueError("a multi-speaker model needs batch['speaker_ids']")
    r = dec.r
    ds = batch["y"].size(1) // batch["mel"].size(1)
    T_dec = batch["frame_positions"].size(1)
    steps = teacher_forced_steps(batch["target_lengths"].cpu().numpy(), r, ds)
    if steps.max() > T_dec:
        raise ValueError("target lengths need %d decoder steps, the batch has %d" % (steps.max(), T_dec))
    tokens = np.asarray(batch["input_lengths"], np.int64)
    spk = model._speaker_embedding(batch["speaker_ids"]) if model.n_speakers > 1 else None
    _, aligns, _, _ = model.seq2seq(batch["x"], batch["mel"], spk, batch["text_positions"], batch["frame_positions"],
                                    batch["input_lengths_dev"] if "input_lengths_dev" in batch else tokens)
    a = aligns.mean(0) if layer is None else aligns[int(layer)]
    steps_l, tokens_l = _check_alignments(a, steps, tokens)
    out = _mas_result(_mas(a, steps_l, tokens_l), steps_l, tokens_l)
    out["steps"] = steps
    out["frames_per_step"] = r * ds
    return out
