"""Speaker classification (Arik et al., "Neural Voice Cloning with a Few Samples", NeurIPS 2018, section 3.3.1): a
classifier trained on real audio of a set of speakers, and the top-k accuracy with which it recognises cloned audio as
the intended speaker (DESIGN.md section 2.15).

Per utterance the trunk is the speaker encoder's (``speaker_encoder.trunk_layers`` / ``pooled_features``): two
weight-normed 1x1 convs with ReLU, ``n_conv`` non-causal residual Conv1dGLU blocks, the mean over the utterance's own
frames.  Then, with W (K, C) and c (K) plain parameters:

* logits z = W h + c over K speaker classes, the row-wise log-sum-exp and argmax (``dv3_spkcls_fwd``: a grid of
  32 x 32 (row, class) tiles, then one CTA per row);
* training loss: the mean softmax cross-entropy over the rows, its partials fused into the row pass and summed in index
  order by ``dv3_spkenc_reduce``; the gradients (``dv3_spkcls_bwd``) are written directly, with no float atomics.
"""
import math

import numpy as np
import torch
from torch import nn

from . import ops, synthesis
from ._lib import Dv3Error, lib
from .ops import _p, _stream
from .speaker_encoder import (MAX_CHANNELS, SpeakerEncoder, check_samples, pad_samples, pooled_features,
                              trunk_layers)
from .speaker_verifier import cloned_voice_mels
from .train_step import ArenaGraphStep, check_single_process

MIN_CLASSES, MAX_CLASSES = 2, 8192


def check_head(R, C, K):
    """ValueError unless the head's kernels take R rows of C channels over K classes."""
    if not 1 <= C <= MAX_CHANNELS:
        raise ValueError("C=%d channels outside [1, %d]" % (C, MAX_CHANNELS))
    if not MIN_CLASSES <= K <= MAX_CLASSES:
        raise ValueError("K=%d classes outside [%d, %d]" % (K, MIN_CLASSES, MAX_CLASSES))
    if R < 1 or R * K >= 2 ** 31:
        raise ValueError("R=%d rows x K=%d classes: R must be >= 1 and R*K below 2^31" % (R, K))


def _head_shape(h, w):
    """Features h (R, C) with contiguous rows (any row stride), weights W (K, C) -> (R, C, K, row stride in floats).
    ValueError for shapes the kernels refuse, before the device checks."""
    if h.dim() != 2 or w.dim() != 2 or h.shape[1] != w.shape[1] or h.stride(1) != 1:
        raise ValueError("features (R, C) with contiguous rows and weights (K, C): got %s strides %s and %s"
                         % (tuple(h.shape), h.stride(), tuple(w.shape)))
    (R, C), K = h.shape, w.shape[0]
    check_head(R, C, K)
    if not (h.is_cuda and h.dtype == torch.float32):
        raise Dv3Error("features must be fp32 CUDA, got %s %s" % (h.dtype, h.device))
    return R, C, K, h.stride(0)


def _chk_labels(labels, R):
    if labels is not None and not (labels.is_cuda and labels.dtype == torch.int64 and tuple(labels.shape) == (R,)
                                   and labels.is_contiguous()):
        raise ValueError("labels must be a contiguous int64 (%d,) CUDA tensor" % R)


# ---- launches -----------------------------------------------------------------------------------------------------
def logits_forward(h, w, c, labels=None):
    """Features h (R, C) (rows contiguous, any row stride), W (K, C), c (K,), int64 labels (R,) or None -> (logits
    (R, K), lse (R,), pred int32 (R,), loss partials (R,) or None: lse - z[label] per row)."""
    R, C, K, ld = _head_shape(h, w)
    ops._chk(w, c)
    _chk_labels(labels, R)
    dev = h.device
    logits = torch.empty(R, K, device=dev)
    lse = torch.empty(R, device=dev)
    pred = torch.empty(R, dtype=torch.int32, device=dev)
    lp = None if labels is None else torch.empty(R, device=dev)
    lib.call("dv3_spkcls_fwd", _p(h), ld, _p(w), _p(c), _p(labels), _p(logits), _p(lse), _p(pred), _p(lp),
             _p(ops._err_flag(dev)), R, C, K, _stream())
    return logits, lse, pred, lp


def logits_backward(h, w, logits, lse, labels=None, d_logits=None, d_loss=None, loss_scale=1.0):
    """-> (d_h (R, C) contiguous, d_w (K, C), d_c (K,)) of G = d_logits + d_loss * loss_scale * (softmax -
    onehot(labels)) (the second term with labels and d_loss)."""
    R, C, K, ld = _head_shape(h, w)
    ops._chk(w, logits, lse, d_logits, d_loss)
    _chk_labels(labels, R)
    dev = h.device
    d_h = torch.empty(R, C, device=dev)
    d_w = torch.empty(K, C, device=dev)
    d_c = torch.empty(K, device=dev)
    lib.call("dv3_spkcls_bwd", _p(h), ld, _p(w), _p(logits), _p(lse), _p(labels), _p(d_logits), _p(d_loss),
             float(loss_scale), _p(d_h), _p(d_w), _p(d_c), _p(ops._err_flag(dev)), R, C, K, _stream())
    return d_h, d_w, d_c


def mean_loss(loss_partials):
    """(R,) loss partials -> their mean, summed in index order (``dv3_spkenc_reduce`` with loss_scale 1/R)."""
    R = loss_partials.numel()
    loss = torch.empty((), device=loss_partials.device)
    lib.call("dv3_spkenc_reduce", None, 0, _p(loss_partials), 1.0 / R, None, _p(loss), R, _stream())
    return loss


class _ClassifierLossFn(torch.autograd.Function):
    """Pooled features h (B, N, C), int64 labels (B*N,) -> (logits (B*N, K), mean softmax cross-entropy over the
    B*N rows)."""

    @staticmethod
    def forward(ctx, h, labels, w, c):
        ops._chk(h)
        B, N, C = h.shape
        h2 = h.view(B * N, C)
        logits, lse, _, lp = logits_forward(h2, w, c, labels)
        loss = mean_loss(lp)
        ctx.save_for_backward(h2, labels, w, logits, lse)
        ctx.shape = (B, N, C)
        ctx.set_materialize_grads(False)
        return logits, loss

    @staticmethod
    def backward(ctx, d_logits, d_loss):
        h2, labels, w, logits, lse = ctx.saved_tensors
        R = h2.shape[0]
        d_h, d_w, d_c = logits_backward(h2, w, logits, lse, labels, None if d_logits is None else ops._c(d_logits),
                                        None if d_loss is None else ops._c(d_loss), 1.0 / R)
        return d_h.view(ctx.shape), None, d_w, d_c


# ---- model ----------------------------------------------------------------------------------------------------------
class SpeakerClassifier(nn.Module):
    """Speaker classifier of Arik et al. (2018), section 3.3.1, on this project's kernels (see the module docstring and
    DESIGN.md section 2.15 for where it departs from the paper).

    forward(mels (B, N, T, mel_dim), speaker_ids int64 (B,)) -> (logits (B*N, K), loss): the mean softmax cross-entropy
    over a batch whose row b holds N utterances of speaker speaker_ids[b], a class in [0, n_classes) (an id outside it
    sets the device error flag that ``ops.check_index_errors()`` raises on)."""

    def __init__(self, n_classes, mel_dim=80, channels=128, n_conv=2, kernel_size=5):
        super().__init__()
        if not 1 <= channels <= MAX_CHANNELS:
            raise ValueError("channels=%d outside [1, %d]" % (channels, MAX_CHANNELS))
        if not MIN_CLASSES <= n_classes <= MAX_CLASSES:
            raise ValueError("n_classes=%d outside [%d, %d]" % (n_classes, MIN_CLASSES, MAX_CLASSES))
        if kernel_size < 1 or kernel_size % 2 == 0:
            raise ValueError("kernel_size=%d: the non-causal blocks keep the frame count with an odd width only"
                             % kernel_size)
        if n_conv < 0 or mel_dim < 1:
            raise ValueError("n_conv=%d, mel_dim=%d" % (n_conv, mel_dim))
        self.n_classes, self.mel_dim, self.channels = n_classes, mel_dim, channels
        K, C = n_classes, channels
        self.spectral, self.temporal = trunk_layers(mel_dim, C, n_conv, kernel_size, C)
        self.w = nn.Parameter(torch.randn(K, C) / math.sqrt(C))
        self.c = nn.Parameter(torch.zeros(K))
        self._cache = {}

    _full = SpeakerEncoder._full

    def pooled(self, mels, lengths=None):
        """mels (B, N, T, mel_dim) -> pooled features (B, N, C) (``speaker_encoder.pooled_features``)."""
        return pooled_features(self, mels, lengths)

    def forward(self, mels, speaker_ids):
        B, N = mels.shape[:2]
        ids = torch.as_tensor(speaker_ids).to(mels.device)
        if ids.dtype != torch.int64 or tuple(ids.shape) != (B,):
            raise ValueError("speaker_ids must be (B,) int64, got %s %s" % (tuple(ids.shape), ids.dtype))
        check_head(B * N, self.channels, self.n_classes)
        labels = ids[:, None].expand(B, N).reshape(B * N)
        return _ClassifierLossFn.apply(self.pooled(mels), labels, self.w, self.c)

    def loss(self, mels, speaker_ids):
        """The mean softmax cross-entropy over the batch's B*N utterances."""
        return self(mels, speaker_ids)[1]

    def classify(self, mels):
        """mels: a list of (T_i, mel_dim) utterances (arrays or tensors) -> (logits (n, K), predicted classes int64
        (n,)), in eval mode without autograd.  The trunk runs inside ``ops.length_scope`` (``embed_tests`` of the
        verifier does the same), so every row is what that utterance gives alone: bit-identical under
        ``conv_math="fp32"``, within the tensor-core tolerance otherwise.  A prediction is the first class of largest
        logit."""
        if not isinstance(mels, (list, tuple)) or not mels:
            raise ValueError("classify takes a non-empty list of (T, %d) mels" % self.mel_dim)
        samples = check_samples([[m] for m in mels], self.mel_dim, 1)
        check_head(len(samples), self.channels, self.n_classes)
        mels, lengths, _ = pad_samples(samples, self.mel_dim)
        dev = self.w.device
        was_training = self.training
        self.eval()
        try:
            with torch.no_grad():
                h = self.pooled(mels.to(dev), lengths.to(dev))
                logits, _, pred, _ = logits_forward(h.view(h.shape[0], self.channels), self.w, self.c)
                return logits, pred.long()
        finally:
            self.train(was_training)


# ---- evaluation -----------------------------------------------------------------------------------------------------
def top_k_accuracy(logits, targets, ks=(1, 5)):
    """logits (n, K), targets (n,) in [0, K) -> {k: the fraction of rows whose target ranks below k}, host-side in fp64.
    A target's rank is the number of classes with a strictly larger logit plus the number with an equal logit and a
    lower index, so that rank 0 is the kernels' prediction (the first class of largest logit).  ValueError for
    malformed shapes, targets outside [0, K), non-finite logits or a k below 1."""
    z = np.asarray(logits.detach().cpu() if torch.is_tensor(logits) else logits, dtype=np.float64)
    t = np.asarray(targets.detach().cpu() if torch.is_tensor(targets) else targets)
    if z.ndim != 2 or z.shape[0] < 1 or t.shape != (z.shape[0],):
        raise ValueError("logits (n, K) and targets (n,): got %s and %s" % (z.shape, t.shape))
    if not np.issubdtype(t.dtype, np.integer) or ((t < 0) | (t >= z.shape[1])).any():
        raise ValueError("targets must be integer classes in [0, %d)" % z.shape[1])
    if not np.isfinite(z).all():
        raise ValueError("logits must be finite")
    ks = [int(k) for k in ks]
    if any(k < 1 for k in ks):
        raise ValueError("ks must be >= 1, got %s" % ks)
    n, K = z.shape
    zt = z[np.arange(n), t][:, None]
    rank = (z > zt).sum(1) + ((z == zt) & (np.arange(K)[None, :] < t[:, None])).sum(1)
    return {k: float((rank < k).mean()) for k in ks}


def classify_cloned_voices(model, classifier, speaker_ids, sequences, targets=None, vocoder="griffin_lim",
                           batch_size=16, stage_timer=None):
    """The paper's speaker-classification evaluation of cloned voices in one call:

    1. synthesize every ``sequences[k]`` in the voice ``speaker_ids[k]`` with ``synthesis.tts_batch``;
    2. turn the waveforms into normalised mels with ``audio.stft_mel_batch``, on the GPU;
    3. classify each synthesized utterance (``SpeakerClassifier.classify``);
    4. -> {"logits": (n_seq, K) fp32 CUDA, "predicted": int64 (n_seq,) CUDA, "targets": int list, "accuracy":
       ``top_k_accuracy(logits, targets)``}.

    targets[k]: the classifier class sequence k should be recognised as; default ``speaker_ids``, for a classifier whose
    classes are the model's own speakers (a cloned id appended by ``add_speakers`` needs an explicit target).
    stage_timer: optional ``name -> context manager`` around "synthesis", "mel" and "classification".  ValueError
    before any launch for a single-speaker model, ids out of range, a target outside [0, K), mismatched list lengths or
    malformed inputs (``speaker_verifier.cloned_voice_mels``)."""
    targets = [int(s) for s in (speaker_ids if targets is None else targets)]
    if len(targets) != len(sequences):
        raise ValueError("%d targets for %d sequences" % (len(targets), len(sequences)))
    bad = [s for s in targets if not 0 <= s < classifier.n_classes]
    if bad:
        raise ValueError("targets %s outside the classifier's classes [0, %d)" % (bad, classifier.n_classes))
    check_head(len(sequences), classifier.channels, classifier.n_classes)
    _, tests = cloned_voice_mels(model, classifier.mel_dim, speaker_ids, sequences, vocoder, batch_size,
                                 classifier.w.device, stage_timer)
    stage = synthesis.stages(stage_timer)
    with stage("classification"):
        logits, pred = classifier.classify(tests)
    return {"logits": logits, "predicted": pred, "targets": targets,
            "accuracy": top_k_accuracy(logits, np.array(targets, dtype=np.int64))}


# ---- training -------------------------------------------------------------------------------------------------------
class SpeakerClassifierStep(ArenaGraphStep):
    """One training step of a SpeakerClassifier: the mean softmax cross-entropy over the B*N utterances of a batch,
    then clip + Adam (``train_step.ArenaGraphStep``: ParameterArena + FlatAdam, the conv_math and deterministic
    modes of construction, one batch shape, bit-exact checkpoints, one CUDA graph with use_graph).

    ``step(batch)`` takes {"mels": (B, N, T, mel_dim) fp32, "speaker_ids": (B,) int64 in [0, n_classes)}, as
    ``data.SpeakerSampleBatches(dataset, B, N, T_crop)`` yields them.  Single process only.  ValueError before any
    launch for a world size above 1, a malformed batch or a speaker id outside [0, n_classes)."""

    _net_key = "classifier"

    def __init__(self, classifier, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip_thresh=None, use_graph=True):
        check_single_process("SpeakerClassifierStep")
        super().__init__(classifier, lr, betas, eps, clip_thresh, use_graph)
        self.classifier = classifier

    def _objective(self, batch):
        return self.classifier(batch["mels"], batch["speaker_ids"])[1]

    def _check_batch(self, batch):
        mels, ids = batch["mels"], batch["speaker_ids"]
        cl = self.classifier
        if mels.dim() != 4 or mels.shape[3] != cl.mel_dim or mels.dtype != torch.float32 or \
                tuple(ids.shape) != (mels.shape[0],) or ids.dtype != torch.int64:
            raise ValueError("batch mels %s %s / speaker_ids %s %s: expected (B, N, T, %d) float32 and (B,) int64"
                             % (tuple(mels.shape), mels.dtype, tuple(ids.shape), ids.dtype, cl.mel_dim))
        check_head(mels.shape[0] * mels.shape[1], cl.channels, cl.n_classes)
        bad = [i for i in ids.cpu().tolist() if not 0 <= i < cl.n_classes]
        if bad:
            raise ValueError("speaker ids %s outside the classifier's classes [0, %d)" % (bad, cl.n_classes))
