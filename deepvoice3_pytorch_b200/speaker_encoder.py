"""Speaker encoding (Arik et al., "Neural Voice Cloning with a Few Samples", NeurIPS 2018, section 3.2): a small network
that maps a few mel spectrograms of an unseen speaker straight to a speaker embedding of a trained multi-speaker model
(DESIGN.md section 2.13).  It is trained once, to regress the model's learned embedding rows
(``SpeakerEncoderStep``); after that a new voice costs one forward pass (``SpeakerEncoder.embed_batch``,
``clone_voices``).

Layers, on B speakers x N cloning samples of (T, mel_dim) normalised mel frames:

* spectral: two weight-normed 1x1 convs mel_dim -> C -> C with ReLU (``modules.run_conv_stack``: one fused launch each);
* temporal: ``n_conv`` non-causal residual ``Conv1dGLU`` blocks (the ConvBlock kernels; tensor cores at C % 128 == 0);
* pooling: the mean over each sample's own frames (``dv3_spkenc_pool_fwd`` / ``_bwd``);
* cloning-sample attention: multi-head self-attention over the valid samples of a speaker, a softmax of one score per
  sample, and the so-weighted sum of the per-sample embeddings W_e h_i + b_e (``dv3_spkenc_attn_fwd`` / ``_bwd``, one
  CTA per speaker, the L1 loss against the target rows fused in; ``dv3_spkenc_reduce`` sums the per-speaker gradient
  rows in index order).
"""
import contextlib
import math

import torch
from torch import nn

from . import modules, ops
from ._lib import lib, Dv3Error
from .ops import _p, _stream
from .train_step import ArenaGraphStep, check_single_process

MAX_SAMPLES, MAX_CHANNELS, MAX_EMBED, MAX_HEADS = 32, 256, 64, 8
_ATTN_PARAMS = ("w_q", "b_q", "w_k", "b_k", "w_v", "b_v", "w_s", "b_s", "w_e", "b_e")
# order of the parameter gradients in a partial row of dv3_spkenc_attn_bwd
_GRAD_ORDER = ("w_q", "w_k", "w_v", "b_q", "b_k", "b_v", "w_s", "b_s", "w_e", "b_e")


def _chk_index(t, what):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.int32 and t.dim() == 1 and t.is_contiguous()):
        raise Dv3Error("%s must be a contiguous int32 (n,) CUDA tensor" % what)


class _PoolFn(torch.autograd.Function):
    """x (R, C, T), lengths int32 (R,) -> (R, C): the mean over each row's first lengths[r] frames."""

    @staticmethod
    def forward(ctx, x, lengths):
        ops._chk(x)
        _chk_index(lengths, "pool lengths")
        R, C, T = x.shape
        if lengths.numel() != R:
            raise Dv3Error("pool: %d lengths for %d rows" % (lengths.numel(), R))
        y = torch.empty(R, C, device=x.device)
        lib.call("dv3_spkenc_pool_fwd", _p(x), _p(lengths), _p(y), _p(ops._err_flag(x.device)), R, C, T, _stream())
        ctx.save_for_backward(lengths)
        ctx.T = T
        return y

    @staticmethod
    def backward(ctx, dy):
        (lengths,) = ctx.saved_tensors
        dy = ops._c(dy)
        R, C = dy.shape
        dx = torch.empty(R, C, ctx.T, device=dy.device)
        lib.call("dv3_spkenc_pool_bwd", _p(dy), _p(lengths), _p(dx), _p(ops._err_flag(dy.device)), R, C, ctx.T,
                 _stream())
        return dx, None


def masked_mean(x, lengths):
    """x (R, C, T) CUDA fp32, lengths int32 (R,) in [1, T] -> (R, C) means over each row's own frames.  A length
    outside [1, T] sets the device error flag that ``ops.check_index_errors()`` raises on."""
    return _PoolFn.apply(x, lengths)


class _AttentionFn(torch.autograd.Function):
    """h (B, N, C), counts int32 (B,), target (B, S) or None -> (out (B, S), L1 loss mean |out - target| (0-dim; 0
    without a target))."""

    @staticmethod
    def forward(ctx, h, counts, target, heads, *params):
        ops._chk(h, target, *params)
        _chk_index(counts, "sample counts")
        B, N, C = h.shape
        S = params[8].shape[0]
        dev = h.device
        ws = torch.empty(B, lib.raw("dv3_spkenc_ws_floats")(N, C, S, heads), device=dev)
        out = torch.empty(B, S, device=dev)
        loss = torch.zeros((), device=dev)
        lp = torch.empty(B, device=dev) if target is not None else None
        lib.call("dv3_spkenc_attn_fwd", _p(h), _p(counts), *[_p(p) for p in params], _p(target), _p(out), _p(ws),
                 _p(lp), _p(ops._err_flag(dev)), B, N, C, S, heads, _stream())
        if target is not None:
            lib.call("dv3_spkenc_reduce", None, 0, _p(lp), 1.0 / (B * S), None, _p(loss), B, _stream())
        ctx.save_for_backward(h, counts, target, ws, *params)
        ctx.heads = heads
        ctx.set_materialize_grads(False)
        return out, loss

    @staticmethod
    def backward(ctx, d_out, d_loss):
        h, counts, target, ws = ctx.saved_tensors[:4]
        params = ctx.saved_tensors[4:]
        B, N, C = h.shape
        S = params[8].shape[0]
        dev = h.device
        d_h = torch.empty_like(h)
        P = lib.raw("dv3_spkenc_param_floats")(C, S)
        part = torch.empty(B, P, device=dev)
        grad = torch.empty(P, device=dev)
        d_out = None if d_out is None else ops._c(d_out)
        d_loss = None if (d_loss is None or target is None) else ops._c(d_loss)
        lib.call("dv3_spkenc_attn_bwd", _p(h), _p(counts), *[_p(p) for p in params], _p(target), _p(d_out),
                 _p(d_loss), 1.0 / (B * S), _p(ws), _p(d_h), _p(part), _p(ops._err_flag(dev)), B, N, C, S, ctx.heads,
                 _stream())
        lib.call("dv3_spkenc_reduce", _p(part), P, None, 0.0, _p(grad), None, B, _stream())
        by_name = dict(zip(_ATTN_PARAMS, params))
        grads, o = {}, 0
        for name in _GRAD_ORDER:
            n = by_name[name].numel()
            grads[name] = grad[o:o + n].view_as(by_name[name])
            o += n
        return (d_h, None, None, None) + tuple(grads[name] for name in _ATTN_PARAMS)


def trunk_layers(mel_dim, channels, n_conv, kernel_size, embed_dim):
    """The per-utterance trunk shared by the speaker encoder and the speaker verifier -> (spectral, temporal):
    two weight-normed 1x1 convs mel_dim -> C -> C with ReLU, and ``n_conv`` non-causal residual Conv1dGLU blocks."""
    C = channels
    spectral = nn.ModuleList([modules.Conv1d(mel_dim, C, 1, std_mul=2.0), nn.ReLU(),
                              modules.Conv1d(C, C, 1, std_mul=2.0), nn.ReLU()])
    temporal = nn.ModuleList([modules.Conv1dGLU(1, embed_dim, C, C, kernel_size, dropout=0.0, causal=False,
                                                residual=True) for _ in range(n_conv)])
    return spectral, temporal


def pooled_features(net, mels, lengths=None):
    """The trunk of ``net`` (its ``spectral`` and ``temporal`` stacks, ``mel_dim``, ``channels`` and ``_full``) over
    mels (B, N, T, mel_dim) -> pooled features (B, N, C).  lengths (B*N,) int32: each sample's own frame count.  The
    stacks then run inside ``ops.length_scope``, so a sample's features are those of the sample alone, whatever its
    padding; that is inference only (ValueError with autograd enabled)."""
    if lengths is not None and torch.is_grad_enabled():
        raise ValueError("per-sample lengths are for inference: call under torch.no_grad() (training batches are "
                         "fixed-length crops)")
    ops._chk(mels)
    B, N, T, M = mels.shape
    if M != net.mel_dim:
        raise Dv3Error("mels have %d channels, the network %d" % (M, net.mel_dim))
    if lengths is None:
        lengths, scope = net._full(B * N, T, mels.device), contextlib.nullcontext()
    else:
        _chk_index(lengths, "sample lengths")
        scope = ops.length_scope(lengths.long(), T)
    with scope:
        x = ops.transpose12(mels.view(B * N, T, M))
        x = modules.run_conv_stack(net.spectral, x)
        x = modules.run_conv_stack(net.temporal, x)
    return masked_mean(x, lengths).view(B, N, net.channels)


def check_samples(samples, mel_dim, max_samples):
    """-> ``samples`` (a list over speakers of lists of (T, mel_dim) arrays or tensors) as float32 tensors, or
    ValueError: no speakers, a speaker without samples or with more than max_samples, a sample that is not
    (T >= 1, mel_dim) floats."""
    if not isinstance(samples, (list, tuple)) or not samples:
        raise ValueError("samples must be a non-empty list over speakers of lists of (T, %d) mels" % mel_dim)
    out = []
    for k, spk in enumerate(samples):
        if not isinstance(spk, (list, tuple)) or not spk:
            raise ValueError("speaker %d has no cloning samples" % k)
        if len(spk) > max_samples:
            raise ValueError("speaker %d has %d samples, max_samples is %d" % (k, len(spk), max_samples))
        rows = []
        for j, m in enumerate(spk):
            m = torch.as_tensor(m)
            if m.dim() != 2 or m.shape[1] != mel_dim or m.shape[0] < 1 or not m.is_floating_point():
                raise ValueError("speaker %d sample %d: shape %s, expected (T >= 1, %d) floats"
                                 % (k, j, tuple(m.shape), mel_dim))
            rows.append(m.to(torch.float32))
        out.append(rows)
    return out


def pad_samples(samples, mel_dim):
    """Checked ragged samples -> (mels (n_spk, N, T, mel_dim), lengths int32 (n_spk * N,), counts int32 (n_spk,)) on the
    host, N and T the largest count and length; a padded sample slot is one zero frame, to be masked out by counts."""
    n_spk = len(samples)
    N = max(len(s) for s in samples)
    T = max(m.shape[0] for s in samples for m in s)
    mels = torch.zeros(n_spk, N, T, mel_dim)
    lengths = torch.ones(n_spk * N, dtype=torch.int32)
    for k, spk in enumerate(samples):
        for j, m in enumerate(spk):
            mels[k, j, :m.shape[0]] = m.cpu()
            lengths[k * N + j] = m.shape[0]
    counts = torch.tensor([len(s) for s in samples], dtype=torch.int32)
    return mels, lengths, counts


def _check_model(model):
    if getattr(model, "n_speakers", 1) <= 1 or not hasattr(model, "embed_speakers"):
        raise ValueError("speaker encoding needs a multi-speaker model (n_speakers=%d)" % getattr(model, "n_speakers", 1))


class SpeakerEncoder(nn.Module):
    """Speaker encoder of Arik et al. (2018), section 3.2, on this project's kernels (see the module docstring and
    DESIGN.md section 2.13 for where it departs from the paper's figure).

    forward(mels (B, N, T, mel_dim)[, lengths int32 (B*N,), counts int32 (B,)]) -> (B, speaker_embed_dim): CUDA fp32,
    every sample T frames long and every speaker N samples unless lengths / counts say otherwise."""

    def __init__(self, mel_dim=80, speaker_embed_dim=16, channels=128, n_conv=2, kernel_size=5, heads=2,
                 max_samples=32):
        super().__init__()
        if not 1 <= channels <= MAX_CHANNELS:
            raise ValueError("channels=%d outside [1, %d]" % (channels, MAX_CHANNELS))
        if not 1 <= max_samples <= MAX_SAMPLES:
            raise ValueError("max_samples=%d outside [1, %d]" % (max_samples, MAX_SAMPLES))
        if not 1 <= speaker_embed_dim <= MAX_EMBED:
            raise ValueError("speaker_embed_dim=%d outside [1, %d]" % (speaker_embed_dim, MAX_EMBED))
        if not (1 <= heads <= MAX_HEADS and channels % heads == 0):
            raise ValueError("heads=%d must divide channels=%d and be at most %d" % (heads, channels, MAX_HEADS))
        if kernel_size < 1 or kernel_size % 2 == 0:
            raise ValueError("kernel_size=%d: the non-causal blocks keep the frame count with an odd width only"
                             % kernel_size)
        if n_conv < 0 or mel_dim < 1:
            raise ValueError("n_conv=%d, mel_dim=%d" % (n_conv, mel_dim))
        self.mel_dim, self.speaker_embed_dim, self.channels = mel_dim, speaker_embed_dim, channels
        self.heads, self.max_samples = heads, max_samples
        C, S = channels, speaker_embed_dim
        self.spectral, self.temporal = trunk_layers(mel_dim, C, n_conv, kernel_size, S)

        def weight(rows, cols):
            return nn.Parameter(torch.randn(rows, cols) / math.sqrt(cols))
        self.w_q, self.w_k, self.w_v = weight(C, C), weight(C, C), weight(C, C)
        self.b_q, self.b_k, self.b_v = (nn.Parameter(torch.zeros(C)) for _ in range(3))
        self.w_s, self.b_s = nn.Parameter(torch.randn(C) / math.sqrt(C)), nn.Parameter(torch.zeros(1))
        self.w_e, self.b_e = weight(S, C), nn.Parameter(torch.zeros(S))
        self._cache = {}

    def _full(self, n, value, device):
        """A cached int32 (n,) device tensor of ``value`` (no allocation or copy per call: graph-capture safe)."""
        key = (n, value, device)
        if key not in self._cache:
            self._cache[key] = torch.full((n,), value, dtype=torch.int32, device=device)
        return self._cache[key]

    def pooled(self, mels, lengths=None):
        """mels (B, N, T, mel_dim) -> pooled features (B, N, C) (``pooled_features``)."""
        return pooled_features(self, mels, lengths)

    def attend(self, h, counts=None, target=None):
        """Cloning-sample attention of pooled features h (B, N, C) -> (embeddings (B, S), L1 loss against target)."""
        B, N, _ = h.shape
        if N > self.max_samples:
            raise ValueError("%d cloning samples per speaker, max_samples is %d" % (N, self.max_samples))
        if counts is None:
            counts = self._full(B, N, h.device)
        return _AttentionFn.apply(h, counts, target, self.heads, *[getattr(self, n) for n in _ATTN_PARAMS])

    def forward(self, mels, lengths=None, counts=None):
        """mels (B, N, T, mel_dim) -> (B, S).  lengths: as ``pooled`` (inference only); counts (B,) int32: each
        speaker's number of valid samples, the padded sample slots masked out of the attention."""
        return self.attend(self.pooled(mels, lengths), counts)[0]

    def loss(self, mels, target):
        """The training objective: mean |encoder(mels) - target| over the (B, S) rows."""
        return self.attend(self.pooled(mels), None, target)[1]

    def check_samples(self, samples):
        """-> the samples as float32 tensors, or ValueError (``check_samples``)."""
        return check_samples(samples, self.mel_dim, self.max_samples)

    def embed_batch(self, samples):
        """samples: a list over speakers of lists of (T_i, mel_dim) arrays or tensors, ragged in length and in count ->
        (n_speakers, speaker_embed_dim) embeddings, in eval mode without autograd.  Every speaker's row is what it would
        be alone: the stacks run inside ``ops.length_scope`` (each sample sees the zeros it would see alone), the pool
        averages each sample's own frames, the attention masks the padded sample slots -- bit-identical under
        ``conv_math="fp32"``, within the tensor-core tolerance otherwise."""
        mels, lengths, counts = pad_samples(self.check_samples(samples), self.mel_dim)
        dev = self.w_q.device
        was_training = self.training
        self.eval()
        try:
            with torch.no_grad():
                mels, lengths, counts = mels.to(dev), lengths.to(dev), counts.to(dev)
                return self(mels, lengths, counts)
        finally:
            self.train(was_training)


def clone_voices(model, encoder, samples):
    """Clone one new voice per entry of ``samples`` (as ``SpeakerEncoder.embed_batch`` takes them) into a multi-speaker
    model: appends the encoder's embeddings with ``model.add_speakers`` and returns the new speaker ids, which work
    directly in ``synthesis.tts_batch`` / ``tts_stream`` and as ``TrainStep(adapt_speakers=...)`` (encoding, then
    adaptation).  ValueError before any launch for a single-speaker model, an encoder of another embedding width or
    malformed samples."""
    _check_model(model)
    if encoder.speaker_embed_dim != model.speaker_embed_dim:
        raise ValueError("encoder speaker_embed_dim=%d, model %d" % (encoder.speaker_embed_dim,
                                                                     model.speaker_embed_dim))
    encoder.check_samples(samples)
    return model.add_speakers(len(samples), init=encoder.embed_batch(samples))


class SpeakerEncoderStep(ArenaGraphStep):
    """One training step of a SpeakerEncoder: the L1 regression of ``model.embed_speakers.weight[speaker_ids]``
    (detached: the multi-speaker model runs no forward and keeps every bit), then clip + Adam (``ArenaGraphStep``).

    ``step(batch)`` takes {"mels": (B, N, T, mel_dim) fp32, "speaker_ids": (B,) int64} (as ``data.SpeakerSampleBatches``
    yields them), every batch of one shape.  use_graph: one CUDA graph covers forward, backward and update.  The step
    runs in the ``ops.conv_math`` and ``ops.deterministic`` modes current at construction.  The graph reads the speaker
    table at the address it had at capture; when the table has moved since (``add_speakers`` / ``clone_voices`` install
    a new one, a ``TrainStep`` over the model re-homes it), the next ``step()`` captures a new graph.  Single process
    only.
    ValueError before any launch for a world size above 1, a single-speaker model or an encoder whose
    speaker_embed_dim differs from the model's."""

    _net_key = "encoder"

    def __init__(self, encoder, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip_thresh=None, use_graph=True):
        check_single_process("SpeakerEncoderStep")
        _check_model(model)
        if encoder.speaker_embed_dim != model.speaker_embed_dim:
            raise ValueError("encoder speaker_embed_dim=%d, model %d" % (encoder.speaker_embed_dim,
                                                                         model.speaker_embed_dim))
        super().__init__(encoder, lr, betas, eps, clip_thresh, use_graph)
        self.encoder, self.model = encoder, model

    def _objective(self, batch):
        with torch.no_grad():
            target = ops.embedding(batch["speaker_ids"], self.model.embed_speakers.weight.detach())
        return self.encoder.loss(batch["mels"], target)

    def _check_batch(self, batch):
        mels, ids = batch["mels"], batch["speaker_ids"]
        enc = self.encoder
        if mels.dim() != 4 or mels.shape[1] > enc.max_samples or mels.shape[3] != enc.mel_dim or \
                mels.dtype != torch.float32 or tuple(ids.shape) != (mels.shape[0],) or ids.dtype != torch.int64:
            raise ValueError("batch mels %s %s / speaker_ids %s %s: expected (B, N <= %d, T, %d) float32 and (B,) int64"
                             % (tuple(mels.shape), mels.dtype, tuple(ids.shape), ids.dtype, enc.max_samples,
                                enc.mel_dim))

    def _graph_key(self):
        """(address, shape) of the speaker table the targets are read from."""
        w = self.model.embed_speakers.weight
        return w.data_ptr(), tuple(w.shape), w.dtype, w.device
