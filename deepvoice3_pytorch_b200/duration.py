"""Duration-guided synthesis (DESIGN.md section 2.22): a duration predictor trained on teacher-forced alignments, a
speaking-rate rule, and the guided decoding they drive.

* ``DurationPredictor`` reads the frozen TTS encoder's ``values`` (B, L, E) and predicts each token's log-duration in
  decoder steps; ``duration_loss`` is its fixed-order fp64 loss (csrc/duration.cu), usable under the deterministic
  mode; ``DurationPredictorStep`` trains it (clip + Adam in one CUDA graph).
* ``duration_batch`` turns a ``data.collate`` batch into a fixed-shape training batch: encoder values and the MAS
  durations of ``alignment.teacher_forced_alignment``.
* ``predict_durations`` gives one int64 duration array per sentence; ``scale_durations`` changes the speaking rate.
* ``synthesis.tts_batch`` / ``tts_stream`` / ``alignment.evaluate_attention`` take ``durations`` and ``speed``: every
  attention layer's window then follows the prescribed token path and each utterance runs exactly sum(durations)
  decoder steps (``incremental.decode_ragged``).
"""
import math

import numpy as np
import torch
from torch import nn

from . import modules, ops, synthesis
from ._lib import lib
from .incremental import check_durations, query_steps
from .ops import _device_i32, _p, _stream
from .train_step import ArenaGraphStep, check_single_process

MAX_TOKENS = 1024             # csrc/duration.cu DUR_MAX_TOKENS


# ---- speaking rate ----------------------------------------------------------------------------------------------------
def scale_durations(durations, speed):
    """Durations for speaking ``speed`` times as fast: with C_j the cumulative duration, B_0 = 0 and
    B_j = max(B_{j-1} + 1, rint(C_j / speed)) in fp64 (rint rounds half to even), d'_j = B_j - B_{j-1}.  So speed 1
    returns the input, every token keeps at least one step, and the total tracks C_L / speed.

    durations: one 1-D integer array per sequence (each entry >= 1) -> list of int64 arrays.  ValueError for a speed
    that is not a finite number > 0 or durations < 1."""
    if isinstance(speed, bool) or not isinstance(speed, (int, float, np.integer, np.floating)) or \
            not math.isfinite(speed) or speed <= 0:
        raise ValueError("speed must be a finite number > 0, got %r" % (speed,))
    if not isinstance(durations, (list, tuple)):
        raise ValueError("durations must be a list of 1-D integer arrays")
    out = []
    for d in check_durations(durations, [np.asarray(x).size if not torch.is_tensor(x) else x.numel()
                                         for x in durations]):
        target = np.rint(np.cumsum(d).astype(np.float64) / float(speed))
        b = np.empty(d.size, np.int64)
        prev = 0
        for j, c in enumerate(target):
            prev = max(prev + 1, int(c))
            b[j] = prev
        out.append(np.diff(b, prepend=0))
    return out


def guided_durations(model, sequences, durations, speed):
    """The durations a synthesis call with ``model`` runs with: None without durations (speed must then be 1), else
    the checked durations of every sequence scaled to ``speed``.  ValueError before any launch, also for a total above
    the decoder's query-position table."""
    if durations is None:
        if speed != 1.0:
            raise ValueError("speed %r needs durations (predict_durations gives them)" % (speed,))
        return None
    durs = check_durations(durations, [np.asarray(s).size for s in sequences])
    if speed != 1.0:
        durs = scale_durations(durs, speed)
    most = query_steps(model.seq2seq.decoder)
    total = max(int(d.sum()) for d in durs)
    if total > most:
        raise ValueError("durations total %d decoder steps; the query-position table holds %d" % (total, most))
    return durs


# ---- loss -------------------------------------------------------------------------------------------------------------
class _DurationLossFn(torch.autograd.Function):
    """y (B, L) fp32 (unit token stride), int32 CUDA durations (B, L) and lengths (B,) -> the mean over rows of the
    per-row mean of (y - log d)^2."""

    @staticmethod
    def forward(ctx, y, dur, lens):
        B, L = y.shape
        dev = y.device
        row = torch.empty(B, dtype=torch.float64, device=dev)
        loss = torch.empty((), device=dev)
        lib.call("dv3_duration_loss_fwd", _p(y), y.stride(0), _p(dur), dur.stride(0), _p(lens), B, L, _p(row),
                 _p(loss), _p(ops._err_flag(dev)), _stream())
        ctx.save_for_backward(y, dur, lens)
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        y, dur, lens = ctx.saved_tensors
        B, L = y.shape
        dy = torch.empty(B, L, device=y.device)
        lib.call("dv3_duration_loss_bwd", _p(y), y.stride(0), _p(dur), dur.stride(0), _p(lens), B, L,
                 _p(ops._c(d_loss)), _p(dy), _stream())
        return dy, None, None


def _check_loss_inputs(y, durations, lengths):
    """Host checks of ``duration_loss``'s arguments (values only where they are on the host) -> (B, L)."""
    if not torch.is_tensor(y) or y.dim() != 2 or y.dtype != torch.float32 or not y.is_cuda:
        raise ValueError("y must be a (B, L) float32 CUDA tensor")
    B, L = y.shape
    if not 1 <= B <= 65535 or not 1 <= L <= MAX_TOKENS:
        raise ValueError("y of shape %s: B in [1, 65535] and L in [1, %d]" % (tuple(y.shape), MAX_TOKENS))
    if tuple(durations.shape) != (B, L) or tuple(lengths.shape) != (B,):
        raise ValueError("durations must be (%d, %d) and lengths (%d,), got %s and %s"
                         % (B, L, B, tuple(durations.shape), tuple(lengths.shape)))
    for name, x in (("durations", durations), ("lengths", lengths)):
        ok = x.dtype in (torch.int32, torch.int64) if torch.is_tensor(x) else np.issubdtype(x.dtype, np.integer)
        if not ok:
            raise ValueError("%s must hold integers, got %s" % (name, x.dtype))
    host = [None if torch.is_tensor(x) and x.is_cuda else np.asarray(x.cpu() if torch.is_tensor(x) else x)
            for x in (durations, lengths)]
    _check_host_values(host[0], host[1], L)
    return B, L


def _check_host_values(durations, lengths, L):
    """ValueError for host lengths outside [1, L] or host durations below 1 within a row's length (None: on the
    device, checked by the kernels)."""
    if lengths is None:
        return
    if lengths.min() < 1 or lengths.max() > L:
        raise ValueError("lengths must lie in [1, %d], got [%d, %d]" % (L, lengths.min(), lengths.max()))
    if durations is not None:
        for b, n in enumerate(lengths):
            if durations[b, :n].min() < 1:
                raise ValueError("durations of row %d hold a value below 1" % b)


def duration_loss(y, durations, lengths):
    """The duration predictor's loss: the mean over rows of the per-row mean over the row's lengths[b] tokens of
    (y - log d)^2, y (B, L) predicted log-durations (fp32 CUDA, unit token stride), durations (B, L) and lengths (B,)
    integer arrays or tensors.  fp64 sums in a fixed order (tokens, then rows), no atomics; the gradient past a row's
    length is 0.  CUDA-tensor durations and lengths are not read back (graph capture): a value out of range sets the
    device error flag (``ops.check_index_errors()``) and that row counts 0.  ValueError before any launch for malformed
    shapes, L > 1024 and host values out of range (lengths outside [1, L], durations below 1)."""
    _check_loss_inputs(y, durations, lengths)
    dev = y.device
    if y.stride(1) != 1:
        y = y.contiguous()
    return _DurationLossFn.apply(y, _device_i32(durations, dev), _device_i32(lengths, dev))


# ---- model ------------------------------------------------------------------------------------------------------------
class _MaskRows(torch.autograd.Function):
    """x (B, C, T) -> x with every row's frames t >= lengths[b] zeroed (int64 CUDA lengths); the gradient likewise."""

    @staticmethod
    def forward(ctx, x, lengths):
        ctx.save_for_backward(lengths)
        return _mask(ops._c(x), lengths)

    @staticmethod
    def backward(ctx, g):
        return _mask(ops._c(g), ctx.saved_tensors[0]), None


def _mask(x, lengths):
    B, C, T = x.shape
    y = torch.empty_like(x)
    lib.call("dv3_mask_time", _p(x), _p(y), _p(lengths), 1, B, C, T, _stream())
    return y


class DurationPredictor(nn.Module):
    """Per-token log-duration predictor on the frozen TTS encoder's ``values`` (DESIGN.md section 2.22).

    Layers: a weight-normed 1x1 conv E -> C with ReLU, ``n_blocks`` non-causal residual Conv1dGLU blocks of width
    ``kernel_size``, then a 1x1 conv C -> 1; for a multi-speaker model (n_speakers > 1) the blocks take the TTS model's
    speaker embedding (speaker_embed_dim) through the speaker path.  All layers are the project's conv Functions (C %
    128 == 0 takes the tensor-core kernels).  Each row's frames past its length are zeroed ahead of every block, in
    training and in inference alike, so a row gets what it gets alone.  No dropout: the blocks run with p = 0, as the
    recognizer's and the speaker encoder's do.

    forward(values (B, L, E), lengths (B,) int64 CUDA, speaker_embed (B, S) or None) -> y (B, L); ValueError for
    lengths of another dtype, device or shape."""

    def __init__(self, in_dim, channels=256, n_blocks=3, kernel_size=3, n_speakers=1, speaker_embed_dim=16):
        super().__init__()
        if in_dim < 1 or channels < 1 or n_blocks < 0:
            raise ValueError("in_dim=%d, channels=%d, n_blocks=%d" % (in_dim, channels, n_blocks))
        if kernel_size < 1 or kernel_size % 2 == 0:
            raise ValueError("kernel_size=%d: the non-causal blocks keep the token count with an odd width only"
                             % kernel_size)
        self.in_dim, self.channels, self.n_speakers = int(in_dim), int(channels), int(n_speakers)
        self.speaker_embed_dim = int(speaker_embed_dim)
        C = channels
        self.proj = nn.ModuleList([modules.Conv1d(in_dim, C, 1, std_mul=2.0), nn.ReLU()])
        self.blocks = nn.ModuleList([modules.Conv1dGLU(n_speakers, speaker_embed_dim, C, C, kernel_size,
                                                       dropout=0.0, causal=False, residual=True)
                                     for _ in range(n_blocks)])
        self.out = nn.ModuleList([modules.Conv1d(C, 1, 1, std_mul=1.0)])

    def forward(self, values, lengths, speaker_embed=None):
        if not torch.is_tensor(values) or values.dim() != 3 or values.shape[2] != self.in_dim:
            raise ValueError("values must be (B, L, %d), got %s" % (self.in_dim, tuple(getattr(values, "shape", ()))))
        if not torch.is_tensor(lengths) or lengths.dtype != torch.int64 or not lengths.is_cuda or \
                tuple(lengths.shape) != (values.shape[0],):
            raise ValueError("lengths must be a (%d,) int64 CUDA tensor (dv3_mask_time reads int64), got %s"
                             % (values.shape[0], "%s %s on %s" % (lengths.dtype, tuple(lengths.shape), lengths.device)
                                if torch.is_tensor(lengths) else type(lengths).__name__))
        ops._chk(values)
        if (speaker_embed is not None) != (self.n_speakers > 1):
            raise ValueError("a multi-speaker predictor needs speaker_embed, a single-speaker one takes none")
        B, L = values.shape[:2]
        x = modules.run_conv_stack(self.proj, ops.transpose12(values))
        spk = None if speaker_embed is None else speaker_embed.unsqueeze(1).expand(B, L, speaker_embed.size(-1))
        for f in self.blocks:
            x = f(_MaskRows.apply(x, lengths), spk)
        return modules.run_conv_stack(self.out, x).reshape(B, L)


def _encode(model, text, lens, spk):
    """The TTS encoder's values of a padded token batch, in eval mode without autograd, inside a length scope."""
    ops.rng.begin_forward(False, text.device)
    try:
        with torch.no_grad(), ops.length_scope(lens, text.size(1)):
            return model.seq2seq.encoder(text, speaker_embed=spk)[1]
    finally:
        ops.rng.end_forward()


def duration_batch(model, batch, max_tokens):
    """A fixed-shape training batch of the duration predictor from a ``data.collate`` batch on the model's device:
    {"values": (B, max_tokens, E) fp32 -- the model's encoder values (eval mode, no gradient, inside a length scope),
    "durations": int32 (B, max_tokens) -- ``teacher_forced_alignment(model, batch)["durations"]``, "token_lengths":
    int32 (B,), and "speaker_embed": (B, S) for a multi-speaker model}, every row padded with zeros to max_tokens so
    that one graph shape serves every batch.  ValueError for a model in training mode, a batch longer than
    max_tokens tokens, or a row whose target has fewer decoder steps than tokens (MAS gives it no durations)."""
    from .alignment import teacher_forced_alignment
    if model.training:
        raise ValueError("duration_batch needs the model in eval mode (model.eval())")
    lens = np.asarray(batch["input_lengths"], np.int64)
    L = batch["x"].size(1)
    if not 1 <= L <= int(max_tokens) <= MAX_TOKENS:
        raise ValueError("a batch of %d tokens does not fit max_tokens=%d (at most %d)" % (L, max_tokens, MAX_TOKENS))
    tf = teacher_forced_alignment(model, batch)
    dur = tf["durations"]
    for b, n in enumerate(lens):
        if dur[b, :n].min() < 1:
            raise ValueError("row %d: %d decoder steps for %d tokens: no duration path" % (b, tf["steps"][b], n))
    dev = batch["x"].device
    spk = model._speaker_embedding(batch["speaker_ids"]) if model.n_speakers > 1 else None
    values = _encode(model, batch["x"], torch.from_numpy(lens).to(dev), spk)
    out_v = torch.zeros(values.size(0), int(max_tokens), values.size(2), device=dev)
    out_v[:, :L] = values
    out_d = np.zeros((len(lens), int(max_tokens)), np.int32)
    out_d[:, :dur.shape[1]] = dur
    res = {"values": out_v, "durations": torch.from_numpy(out_d).to(dev),
           "token_lengths": torch.from_numpy(lens.astype(np.int32)).to(dev)}
    if spk is not None:
        res["speaker_embed"] = spk.detach().contiguous()
    return res


def predict_durations(predictor, model, sequences, speaker_ids=None, batch_size=16):
    """Durations of every ``sequences[k]`` (in voice ``speaker_ids[k]`` for a multi-speaker model): the model's
    encoder values and the predictor in padded batches of ``batch_size``, each inside a length scope (so every sequence
    gets what it gets alone), then d = min(max(1, rint(exp(y))), D) in fp64 -> list of int64 arrays, in input order,
    with D = ``incremental.query_steps`` of the model's decoder: no token is given more steps than a guided decode
    can run.  Eval mode without autograd.  ValueError before any launch as ``synthesis.tts_batch``."""
    seqs, speaker_ids = synthesis._check_inputs(model, sequences, speaker_ids, batch_size=batch_size)
    if max(s.size for s in seqs) > MAX_TOKENS:
        raise ValueError("a sequence has %d tokens, more than %d" % (max(s.size for s in seqs), MAX_TOKENS))
    if (predictor.n_speakers > 1) != (model.n_speakers > 1):
        raise ValueError("the predictor and the model must both be multi-speaker or both single-speaker")
    dev = next(model.parameters()).device
    most = query_steps(model.seq2seq.decoder)
    out = [None] * len(seqs)
    was_training = predictor.training
    predictor.eval()
    try:
        for c in range(0, len(seqs), int(batch_size)):
            idx = list(range(c, min(c + int(batch_size), len(seqs))))
            lens = [seqs[i].size for i in idx]
            text = np.zeros((len(idx), max(lens)), np.int64)
            for b, i in enumerate(idx):
                text[b, :lens[b]] = seqs[i]
            text = torch.from_numpy(text).to(dev)
            lens_d = torch.tensor(lens, dtype=torch.int64).to(dev)
            spk = None if speaker_ids is None else \
                model._speaker_embedding(torch.tensor([speaker_ids[i] for i in idx]).to(dev))
            values = _encode(model, text, lens_d, spk)
            with torch.no_grad(), ops.length_scope(lens_d, text.size(1)):
                y = predictor(values, lens_d, spk).double().cpu().numpy()
            for b, i in enumerate(idx):
                yb = y[b, :lens[b]]
                if np.isnan(yb).any():
                    raise ValueError("the predictor gave NaN log-durations for sequence %d" % i)
                with np.errstate(over="ignore"):
                    out[i] = np.clip(np.rint(np.exp(yb)), 1, most).astype(np.int64)
    finally:
        predictor.train(was_training)
    return out


# ---- training ---------------------------------------------------------------------------------------------------------
class DurationPredictorStep(ArenaGraphStep):
    """One training step of a DurationPredictor: ``duration_loss`` of a batch, then clip + Adam (``ArenaGraphStep``:
    the conv_math and deterministic modes of construction, one batch shape, bit-exact checkpoints, one CUDA graph with
    use_graph).  ``step(batch)`` takes what ``duration_batch`` returns: {"values", "durations", "token_lengths"} and,
    for a multi-speaker predictor, "speaker_embed".  Single process only.  ValueError before any launch for a world
    size above 1 or a malformed batch."""

    _net_key = "predictor"
    _batch_keys = ("values", "durations", "token_lengths")

    def __init__(self, predictor, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip_thresh=None, use_graph=True):
        check_single_process("DurationPredictorStep")
        super().__init__(predictor, lr, betas, eps, clip_thresh, use_graph)
        self.predictor = predictor
        if predictor.n_speakers > 1:
            self._batch_keys = DurationPredictorStep._batch_keys + ("speaker_embed",)

    def _objective(self, batch):
        lens = batch["token_lengths"]
        y = self.predictor(batch["values"], lens.to(torch.int64), batch.get("speaker_embed"))
        return duration_loss(y, batch["durations"], lens)

    def _check_batch(self, batch):
        v = batch["values"]
        if not torch.is_tensor(v) or v.dim() != 3 or v.shape[2] != self.predictor.in_dim or v.dtype != torch.float32:
            raise ValueError("batch values %s: expected (B, L, %d) float32"
                             % (tuple(getattr(v, "shape", ())), self.predictor.in_dim))
        for k in ("durations", "token_lengths"):
            if not torch.is_tensor(batch[k]) or batch[k].dtype != torch.int32:
                raise ValueError("batch %s must be an int32 tensor" % k)
        B, L = v.shape[:2]
        if "speaker_embed" in batch and tuple(batch["speaker_embed"].shape) != (B, self.predictor.speaker_embed_dim):
            raise ValueError("batch speaker_embed must be (%d, %d)" % (B, self.predictor.speaker_embed_dim))
        if tuple(batch["durations"].shape) != (B, L) or tuple(batch["token_lengths"].shape) != (B,):
            raise ValueError("batch durations must be (%d, %d) and token_lengths (%d,)" % (B, L, B))
        if not 1 <= L <= MAX_TOKENS:
            raise ValueError("batch of %d tokens: at most %d" % (L, MAX_TOKENS))
        _check_host_values(batch["durations"].cpu().numpy(), batch["token_lengths"].cpu().numpy(), L)
