"""Speaker verification (Arik et al., "Neural Voice Cloning with a Few Samples", NeurIPS 2018, section 3.3.2, after the
end-to-end verifier of Snyder et al., 2016): a model that decides whether a test utterance comes from the speaker of a
few enrollment utterances, and the equal error rate of cloned audio against real enrollment audio (DESIGN.md section
2.14).

Per utterance the trunk is the speaker encoder's (``speaker_encoder.trunk_layers`` / ``pooled_features``): two
weight-normed 1x1 convs with ReLU, ``n_conv`` non-causal residual Conv1dGLU blocks, the mean over the utterance's own
frames.  Then, with W (D, C), c, S (D, D) and b plain parameters:

* enrollment embedding x = W mean_{i < n}(h_i) + c over a speaker's n <= max_enroll utterances, test embedding
  y = W h + c (``dv3_spkver_embed_fwd`` / ``_bwd``);
* score L(x, y) = x.y - x^T S x - y^T S y + b (``dv3_spkver_score_fwd`` / ``_bwd``: the quadratic terms once per row,
  the pairs on a grid of 32 x 32 tiles);
* training loss: 1/2 mean over same-speaker pairs of softplus(-L) + 1/2 mean over different-speaker pairs of
  softplus(L), over every (enrollment, test) pair of a batch, fused into the score kernels; ``dv3_spkenc_reduce`` sums
  every partial in index order, so there are no float atomics.
"""
import math

import numpy as np
import torch
from torch import nn

from . import audio, ops, synthesis
from ._lib import lib
from .ops import _p, _stream
from .speaker_encoder import (SpeakerEncoder, _check_model, _chk_index, check_samples, pad_samples, pooled_features,
                              trunk_layers)
from .train_step import ArenaGraphStep, check_single_process

MAX_ENROLL, MAX_CHANNELS, MAX_EMBED = 32, 256, 128


# ---- launches -----------------------------------------------------------------------------------------------------
def embed_forward(h, counts, w, c, N=None, ld=None, offset=0):
    """Rows b of h over counts[b] in [1, N] valid (C,) rows starting ``offset`` floats into row b (ld floats apart;
    default: h (B, N, C) contiguous) -> (out (B, D) = W mean + c, the means hbar (B, C))."""
    ops._chk(h, w, c)
    _chk_index(counts, "enrollment counts")
    B, C, D = counts.numel(), w.shape[1], w.shape[0]
    N = h.shape[1] if N is None else N
    ld = N * C if ld is None else ld
    hbar = torch.empty(B, C, device=h.device)
    out = torch.empty(B, D, device=h.device)
    lib.call("dv3_spkver_embed_fwd", _p(h, offset), ld, _p(counts), _p(w), _p(c), _p(hbar), _p(out),
             _p(ops._err_flag(h.device)), B, N, C, D, _stream())
    return out, hbar


def embed_backward(d_out, hbar, counts, w, d_h, N, ld=None, offset=0, partials=None):
    """Writes d_h (rows b, ``offset`` floats in, ld apart) and one partial (D*C + D) gradient row of [W, c] per row b
    into ``partials`` (B, D*C + D) -> partials."""
    B, (D, C) = counts.numel(), w.shape
    ld = N * C if ld is None else ld
    if partials is None:
        partials = torch.empty(B, D * C + D, device=d_out.device)
    lib.call("dv3_spkver_embed_bwd", _p(ops._c(d_out)), _p(hbar), _p(counts), _p(w), _p(d_h, offset), ld,
             _p(partials), _p(ops._err_flag(d_out.device)), B, N, C, D, _stream())
    return partials


def score_forward(x, y, S, bias, ids_e=None, ids_t=None):
    """-> (scores (B_e, B_t), loss partials or None): with int64 speaker ids, the partials of the balanced loss."""
    ops._chk(x, y, S, bias)
    B_e, D = x.shape
    B_t = y.shape[0]
    dev = x.device
    q = torch.empty(B_e + B_t, device=dev)
    scores = torch.empty(B_e, B_t, device=dev)
    lp = None if ids_e is None else torch.empty(lib.raw("dv3_spkver_loss_floats")(B_e, B_t), device=dev)
    lib.call("dv3_spkver_score_fwd", _p(x), _p(y), _p(S), _p(bias), _p(ids_e), _p(ids_t), _p(q), _p(q, B_e),
             _p(scores), _p(lp), B_e, B_t, D, _stream())
    return scores, lp


def score_backward(x, y, S, scores, ids_e=None, ids_t=None, d_scores=None, d_loss=None):
    """-> (dx, dy, partials (B_e + B_t, D*D + 1) of [S, b])."""
    B_e, D = x.shape
    B_t = y.shape[0]
    dx, dy = torch.empty_like(x), torch.empty_like(y)
    part = torch.empty(B_e + B_t, D * D + 1, device=x.device)
    lib.call("dv3_spkver_score_bwd", _p(x), _p(y), _p(S), _p(scores), _p(ids_e), _p(ids_t),
             _p(None if d_scores is None else ops._c(d_scores)), _p(d_loss), _p(dx), _p(dy), _p(part), B_e, B_t, D,
             _stream())
    return dx, dy, part


def reduce_rows(partials):
    """(R, P) -> (P,): the sum over the rows in index order (``dv3_spkenc_reduce``)."""
    R, P = partials.shape
    grad = torch.empty(P, device=partials.device)
    lib.call("dv3_spkenc_reduce", _p(partials), P, None, 0.0, _p(grad), None, R, _stream())
    return grad


def reduce_loss(loss_partials):
    loss = torch.empty((), device=loss_partials.device)
    lib.call("dv3_spkenc_reduce", None, 0, _p(loss_partials), 1.0, None, _p(loss), loss_partials.numel(), _stream())
    return loss


def check_trial_ids(ids):
    """The speaker ids of a training batch (enrollment row b and test row b are speaker ids[b]): ValueError unless
    they give both a same-speaker and a different-speaker pair, i.e. unless two ids differ."""
    ids = torch.as_tensor(ids)
    if ids.dim() != 1 or ids.numel() < 2 or bool((ids == ids.reshape(-1)[0]).all()):
        raise ValueError("a verifier batch needs same- and different-speaker pairs: speaker_ids %s"
                         % ids.reshape(-1).tolist())


class _VerifierLossFn(torch.autograd.Function):
    """Pooled features h (B, N, C) of a training batch (samples 0..N-2 of row b: speaker ids[b]'s enrollment, sample
    N-1: its test utterance), ids int64 (B,) -> (scores (B, B), balanced BCE loss over the B x B pairs)."""

    @staticmethod
    def forward(ctx, h, ids, n_enroll, ones, w, c, S, bias):
        ops._chk(h)
        B, N, C = h.shape
        x, hbar_e = embed_forward(h, n_enroll, w, c, N=N - 1, ld=N * C)
        y, hbar_t = embed_forward(h, ones, w, c, N=1, ld=N * C, offset=(N - 1) * C)
        scores, lp = score_forward(x, y, S, bias, ids, ids)
        loss = reduce_loss(lp)
        ctx.save_for_backward(ids, n_enroll, ones, w, S, x, y, hbar_e, hbar_t, scores)
        ctx.shape = (B, N, C)
        ctx.mark_non_differentiable(scores)
        ctx.set_materialize_grads(False)
        return scores, loss

    @staticmethod
    def backward(ctx, d_scores, d_loss):
        ids, n_enroll, ones, w, S, x, y, hbar_e, hbar_t, scores = ctx.saved_tensors
        B, N, C = ctx.shape
        D = w.shape[0]
        dx, dy, part_s = score_backward(x, y, S, scores, ids, ids, None, None if d_loss is None else ops._c(d_loss))
        d_h = torch.empty(B, N, C, device=x.device)
        part_e = torch.empty(2 * B, D * C + D, device=x.device)
        embed_backward(dx, hbar_e, n_enroll, w, d_h, N - 1, ld=N * C, partials=part_e[:B])
        embed_backward(dy, hbar_t, ones, w, d_h, 1, ld=N * C, offset=(N - 1) * C, partials=part_e[B:])
        g_s, g_e = reduce_rows(part_s), reduce_rows(part_e)
        return (d_h, None, None, None, g_e[:D * C].view(D, C), g_e[D * C:], g_s[:D * D].view(D, D), g_s[D * D:])


# ---- model ----------------------------------------------------------------------------------------------------------
class SpeakerVerifier(nn.Module):
    """End-to-end speaker verifier (see the module docstring and DESIGN.md section 2.14 for where it departs from
    Snyder et al. and the paper).

    forward(mels (B, N, T, mel_dim), speaker_ids int64 (B,)) -> (scores (B, B), loss): the training objective over a
    batch whose row b holds N - 1 enrollment utterances and one test utterance of speaker speaker_ids[b]."""

    def __init__(self, mel_dim=80, channels=128, embed_dim=128, n_conv=2, kernel_size=5, max_enroll=32):
        super().__init__()
        if not 1 <= channels <= MAX_CHANNELS:
            raise ValueError("channels=%d outside [1, %d]" % (channels, MAX_CHANNELS))
        if not 1 <= max_enroll <= MAX_ENROLL:
            raise ValueError("max_enroll=%d outside [1, %d]" % (max_enroll, MAX_ENROLL))
        if not 1 <= embed_dim <= MAX_EMBED:
            raise ValueError("embed_dim=%d outside [1, %d]" % (embed_dim, MAX_EMBED))
        if kernel_size < 1 or kernel_size % 2 == 0:
            raise ValueError("kernel_size=%d: the non-causal blocks keep the frame count with an odd width only"
                             % kernel_size)
        if n_conv < 0 or mel_dim < 1:
            raise ValueError("n_conv=%d, mel_dim=%d" % (n_conv, mel_dim))
        self.mel_dim, self.channels, self.embed_dim, self.max_enroll = mel_dim, channels, embed_dim, max_enroll
        C, D = channels, embed_dim
        self.spectral, self.temporal = trunk_layers(mel_dim, C, n_conv, kernel_size, D)
        self.w = nn.Parameter(torch.randn(D, C) / math.sqrt(C))
        self.c = nn.Parameter(torch.zeros(D))
        self.S = nn.Parameter(torch.zeros(D, D))
        self.b = nn.Parameter(torch.zeros(1))
        self._cache = {}

    _full = SpeakerEncoder._full

    def pooled(self, mels, lengths=None):
        """mels (B, N, T, mel_dim) -> pooled features (B, N, C) (``speaker_encoder.pooled_features``)."""
        return pooled_features(self, mels, lengths)

    def forward(self, mels, speaker_ids):
        B, N = mels.shape[:2]
        if N < 2 or N - 1 > self.max_enroll:
            raise ValueError("a verifier batch row holds 1 <= N - 1 <= %d enrollment utterances and a test one, N=%d"
                             % (self.max_enroll, N))
        dev = mels.device
        ids = torch.as_tensor(speaker_ids).to(dev)
        if ids.dtype != torch.int64 or tuple(ids.shape) != (B,):
            raise ValueError("speaker_ids must be (B,) int64, got %s %s" % (tuple(ids.shape), ids.dtype))
        return _VerifierLossFn.apply(self.pooled(mels), ids.contiguous(), self._full(B, N - 1, dev),
                                     self._full(B, 1, dev), self.w, self.c, self.S, self.b)

    def loss(self, mels, speaker_ids):
        """The balanced binary cross-entropy over the batch's B x B (enrollment, test) pairs.  ValueError before any
        launch unless the ids give both kinds of pair."""
        check_trial_ids(speaker_ids.cpu() if torch.is_tensor(speaker_ids) else speaker_ids)
        return self(mels, speaker_ids)[1]

    def _embed(self, samples, max_samples):
        samples = check_samples(samples, self.mel_dim, max_samples)
        mels, lengths, counts = pad_samples(samples, self.mel_dim)
        dev = self.w.device
        was_training = self.training
        self.eval()
        try:
            with torch.no_grad():
                mels, lengths, counts = mels.to(dev), lengths.to(dev), counts.to(dev)
                h = self.pooled(mels, lengths)
                return embed_forward(h, counts, self.w, self.c)[0]
        finally:
            self.train(was_training)

    def embed_enrollment(self, samples):
        """samples: a list over speakers of lists of (T_i, mel_dim) arrays or tensors, ragged in length and count (at
        most max_enroll) -> (n_spk, D) enrollment embeddings, in eval mode without autograd.  The trunk runs inside
        ``ops.length_scope``, so every row is what that speaker's utterances give alone: bit-identical under
        ``conv_math="fp32"``, within the tensor-core tolerance otherwise."""
        return self._embed(samples, self.max_enroll)

    def embed_tests(self, mels):
        """mels: a list of (T_i, mel_dim) test utterances -> (n, D) test embeddings, each what it is alone (as
        ``embed_enrollment``)."""
        if not isinstance(mels, (list, tuple)) or not mels:
            raise ValueError("tests must be a non-empty list of (T, %d) mels" % self.mel_dim)
        return self._embed([[m] for m in mels], 1)

    def score(self, enrollment, tests):
        """enrollment (n_spk, D), tests (n_test, D) embeddings -> the (n_spk, n_test) score matrix."""
        with torch.no_grad():
            return score_forward(enrollment.contiguous(), tests.contiguous(), self.S, self.b)[0]


# ---- evaluation -----------------------------------------------------------------------------------------------------
def equal_error_rate(scores, labels):
    """scores, labels (1 / True: same-speaker trial) of any matching shape -> (eer, threshold), host-side in fp64.  A
    trial is accepted when its score is >= the threshold; at every distinct score and just above the largest, the
    false-acceptance rate FAR (different-speaker trials accepted) and false-rejection rate FRR (same-speaker trials
    rejected) are counted with tied scores grouped, and the EER is where FAR and FRR cross, linearly interpolated
    between the two thresholds around the crossing.  ValueError without both kinds of trial."""
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    y = np.asarray(labels).reshape(-1).astype(bool)
    if s.shape != y.shape:
        raise ValueError("%d scores, %d labels" % (s.size, y.size))
    n_tar, n_non = int(y.sum()), int((~y).sum())
    if n_tar == 0 or n_non == 0:
        raise ValueError("the EER needs same- and different-speaker trials (%d and %d)" % (n_tar, n_non))
    if not np.isfinite(s).all():
        raise ValueError("scores must be finite")
    u = np.unique(s)
    thr = np.append(u, np.nextafter(u[-1], np.inf))
    # trials below each threshold: searchsorted over the sorted scores of each class
    far = 1.0 - np.searchsorted(np.sort(s[~y]), thr, side="left") / n_non
    frr = np.searchsorted(np.sort(s[y]), thr, side="left") / n_tar
    d = frr - far
    k = int(np.argmax(d >= 0))                  # d[0] = -FAR(min) < 0 and d[-1] = 1 > 0: a crossing exists
    a = -d[k - 1] / (d[k] - d[k - 1])
    eer = far[k - 1] + a * (far[k] - far[k - 1])
    return float(eer), float(thr[k - 1] + a * (thr[k] - thr[k - 1]))


def cloned_voice_mels(model, mel_dim, speaker_ids, sequences, vocoder, batch_size, device, stage_timer=None):
    """What the cloned-voice evaluations (``verify_cloned_voices``, ``speaker_classifier.classify_cloned_voices``)
    share.  First the checks, ValueError before any launch: a single-speaker model, an unknown phase method,
    mismatched list lengths, speaker ids outside [0, n_speakers), an evaluation network of ``mel_dim`` mel channels
    where the audio path makes another count, malformed sequences.  Then ``synthesis.synthesized_mels``: every
    ``sequences[k]`` synthesized in the voice ``speaker_ids[k]`` (stage "synthesis") and turned into normalised mels on
    ``device`` (stage "mel") -> (speaker ids as ints, list of (T_k, num_mels) mels)."""
    _check_model(model)
    audio.check_phase_method(vocoder)
    speaker_ids = [int(s) for s in speaker_ids]
    if len(speaker_ids) != len(sequences):
        raise ValueError("%d speaker_ids for %d sequences" % (len(speaker_ids), len(sequences)))
    bad = [s for s in speaker_ids if not 0 <= s < model.n_speakers]
    if bad:
        raise ValueError("speaker ids %s outside [0, %d)" % (bad, model.n_speakers))
    if mel_dim != audio.hparams.num_mels:
        raise ValueError("the evaluation network takes %d mel channels, the audio path makes %d"
                         % (mel_dim, audio.hparams.num_mels))
    return speaker_ids, synthesis.synthesized_mels(model, sequences, speaker_ids, vocoder, batch_size, device,
                                                   stage_timer)


def verify_cloned_voices(model, verifier, speaker_ids, enrollment, sequences, vocoder="griffin_lim", batch_size=16,
                         stage_timer=None):
    """The paper's speaker-verification evaluation of cloned voices in one call:

    1. synthesize every ``sequences[k]`` in the voice ``speaker_ids[k]`` with ``synthesis.tts_batch``;
    2. turn the waveforms into normalised mels with ``audio.stft_mel_batch``, on the GPU;
    3. score each synthesized utterance against every enrolled speaker's real enrollment utterances;
    4. -> {"scores": (n_enrolled, n_seq) fp64, "labels": bool (n_enrolled, n_seq), "eer": float, "threshold": float,
       "speakers": the enrolled ids, row order}.

    enrollment: {speaker id: list of (T, mel_dim) real normalised mels}; every id of speaker_ids must be enrolled, and at
    least two speakers, so that there are same- and different-speaker trials.  stage_timer: optional ``name -> context
    manager`` around "synthesis", "mel" and "scoring".  ValueError before any launch for a single-speaker model, ids out
    of range or without enrollment, mismatched list lengths or malformed inputs (``cloned_voice_mels``)."""
    speaker_ids = [int(s) for s in speaker_ids]
    if not isinstance(enrollment, dict) or len(enrollment) < 2:
        raise ValueError("enrollment must map at least two speaker ids to lists of real utterances")
    enrolled = sorted(int(k) for k in enrollment)
    missing = sorted(set(speaker_ids) - set(enrolled))
    if missing:
        raise ValueError("speakers %s have no enrollment utterances" % missing)
    samples = check_samples([enrollment[k] for k in enrolled], verifier.mel_dim, verifier.max_enroll)
    speaker_ids, tests = cloned_voice_mels(model, verifier.mel_dim, speaker_ids, sequences, vocoder, batch_size,
                                           verifier.w.device, stage_timer)
    stage = synthesis.stages(stage_timer)
    with stage("scoring"):
        scores = verifier.score(verifier.embed_enrollment(samples), verifier.embed_tests(tests))
        scores = scores.double().cpu().numpy()
    labels = np.array(enrolled)[:, None] == np.array(speaker_ids)[None, :]
    eer, thr = equal_error_rate(scores, labels)
    return {"scores": scores, "labels": labels, "eer": eer, "threshold": thr, "speakers": enrolled}


# ---- training -------------------------------------------------------------------------------------------------------
class SpeakerVerifierStep(ArenaGraphStep):
    """One training step of a SpeakerVerifier: the balanced binary cross-entropy over the B x B (enrollment, test)
    pairs of a batch, then clip + Adam (``train_step.ArenaGraphStep``: ParameterArena + FlatAdam, the conv_math
    and deterministic modes of construction, one batch shape, bit-exact checkpoints, one CUDA graph with use_graph).

    ``step(batch)`` takes {"mels": (B, N, T, mel_dim) fp32, "speaker_ids": (B,) int64}, as
    ``data.SpeakerSampleBatches(dataset, B, n_enroll + 1, T_crop)`` yields them: samples 0..N-2 of row b are its
    enrollment, sample N-1 its test utterance.  Single process only.  ValueError before any launch for a world size
    above 1 or a malformed batch, or one whose ids are all equal (no different-speaker pair)."""

    _net_key = "verifier"

    def __init__(self, verifier, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip_thresh=None, use_graph=True):
        check_single_process("SpeakerVerifierStep")
        super().__init__(verifier, lr, betas, eps, clip_thresh, use_graph)
        self.verifier = verifier

    def _objective(self, batch):
        return self.verifier(batch["mels"], batch["speaker_ids"])[1]

    def _check_batch(self, batch):
        mels, ids = batch["mels"], batch["speaker_ids"]
        v = self.verifier
        if mels.dim() != 4 or not 2 <= mels.shape[1] <= v.max_enroll + 1 or mels.shape[3] != v.mel_dim or \
                mels.dtype != torch.float32 or tuple(ids.shape) != (mels.shape[0],) or ids.dtype != torch.int64:
            raise ValueError("batch mels %s %s / speaker_ids %s %s: expected (B, 2 <= N <= %d, T, %d) float32 and (B,) "
                             "int64" % (tuple(mels.shape), mels.dtype, tuple(ids.shape), ids.dtype, v.max_enroll + 1,
                                        v.mel_dim))
        check_trial_ids(ids.cpu())
