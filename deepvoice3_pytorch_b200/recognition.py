"""Token and word error rates of synthesized speech: a CTC token recognizer trained on this project's kernels, and the
scoring of synthesized (or recorded) mels against the token sequences they should say (DESIGN.md section 2.21).

The vocabulary is the TTS model's own token ids: class 0 is the CTC blank (and the TTS padding id, never a target),
targets are ids in [1, n_vocab).  Kernels (csrc/ctc.cu):

* ``ctc_loss``: the CTC negative log-likelihood of each row (fp64 alpha recursion, one CTA per row), divided by the
  row's target length and averaged over the rows (torch's ``reduction="mean"``), with its gradient from the fused beta
  recursion -- no atomics, so it runs under the deterministic mode too.  Rows without a feasible alignment count 0
  (torch's ``zero_infinity=True``) and are flagged.
* ``greedy_decode``: the per-frame argmax, repeats collapsed and blanks dropped.
* ``edit_distance``: batched Levenshtein distances with their substitution, deletion and insertion counts.

``TokenRecognizer`` is a small non-causal convolutional acoustic model (the speaker encoder's trunk with dilated
blocks) with one class distribution per mel frame; ``TokenRecognizerStep`` trains it (clip + Adam in one CUDA graph).
``token_error_rates`` scores mels against token sequences; ``evaluate_recognition`` synthesizes with a model first.
The recognizer's floor on real recordings is the same call on their mels::

    token_error_rates(recognizer, synthesis.wav_mels(wavs, device), sequences)
"""

import numpy as np
import torch
from torch import nn

from . import audio, modules, ops, synthesis
from ._lib import lib
from .ops import _device_i32, _p, _stream
from .speaker_classifier import mean_loss
from .train_step import ArenaGraphStep, check_single_process

MAX_VOCAB = 1024              # csrc/ctc.cu CTC_MAX_VOCAB
MAX_TARGET = 1024             # target and reference tokens per row: the largest max_positions
MAX_HYP = 65535               # hypothesis tokens per edit-distance pair
WS_LIMIT = 2 << 30            # bytes of one CTC workspace
EDIT_BUDGET = 1 << 28         # bytes of packed rows and workspace per edit-distance launch


def ctc_ws_bytes(B, T, L):
    """Bytes of the CTC workspace for B rows of T frames and L target slots: lse, log p and status per row, and every
    alpha (B T (2L + 1) doubles) -- what ``dv3_ctc_ws_bytes`` returns, without the library."""
    return 8 * (B * T + 2 * B + B * T * (2 * L + 1))


def check_ctc(B, V, T, L):
    """ValueError unless the CTC kernels take B rows of V classes, T frames and L target slots."""
    if B < 1 or T < 1:
        raise ValueError("B=%d rows and T=%d frames must be >= 1" % (B, T))
    if not 2 <= V <= MAX_VOCAB:
        raise ValueError("V=%d classes outside [2, %d]" % (V, MAX_VOCAB))
    if not 0 <= L <= MAX_TARGET:
        raise ValueError("L=%d target slots outside [0, %d]" % (L, MAX_TARGET))
    if B * V * T >= 2 ** 31:
        raise ValueError("B*V*T = %d logits: past 2^31" % (B * V * T))
    if ctc_ws_bytes(B, T, max(L, 1)) > WS_LIMIT:
        raise ValueError("the CTC workspace of B=%d, T=%d, L=%d is %d bytes, above 2 GiB"
                         % (B, T, L, ctc_ws_bytes(B, T, max(L, 1))))


def _host_ints(x, name):
    """A 1-D integer sequence, array or CPU tensor -> int64 array, or None for a CUDA tensor (checked on the device)."""
    if torch.is_tensor(x):
        if x.is_cuda:
            return None
        x = x.numpy()
    x = np.asarray(x)
    if x.ndim != 1 or not np.issubdtype(x.dtype, np.integer):
        raise ValueError("%s must be a 1-D integer array, got %s of shape %s" % (name, x.dtype, x.shape))
    return x.astype(np.int64)


def _check_logits(logits):
    if not torch.is_tensor(logits) or logits.dim() != 3 or logits.dtype != torch.float32:
        raise ValueError("logits must be a (B, V, T) float32 tensor")
    if not logits.is_cuda:
        raise ValueError("logits must be a CUDA tensor (there is no CPU path), got %s" % logits.device)
    B, V, T = logits.shape
    if logits.stride(2) != 1 or (V > 1 and logits.stride(1) < T) or (B > 1 and logits.stride(0) < (V - 1) *
                                                                       logits.stride(1) + T):
        raise ValueError("logits need unit frame stride and non-overlapping rows, got strides %s" % (logits.stride(),))
    return B, V, T


def _check_lengths(x, name, B, lo, hi):
    h = _host_ints(x, name)
    if h is None:
        if tuple(x.shape) != (B,) or x.dtype not in (torch.int32, torch.int64):
            raise ValueError("%s must be (%d,) integers" % (name, B))
        return
    if h.size != B:
        raise ValueError("%s must hold %d entries, got %d" % (name, B, h.size))
    if B and (h.min() < lo or h.max() > hi):
        raise ValueError("%s must lie in [%d, %d], got [%d, %d]" % (name, lo, hi, h.min(), h.max()))


def _check_ctc_inputs(logits, frame_lengths, targets, target_lengths):
    """Host-side checks of ``ctc_loss``'s arguments (values only where they are on the host: device tensors are
    checked by the kernels, which set the error flag) -> (B, V, T, L)."""
    B, V, T = _check_logits(logits)
    if not torch.is_tensor(targets) and not isinstance(targets, np.ndarray):
        raise ValueError("targets must be a (B, L) integer tensor or array")
    if targets.ndim != 2 or targets.shape[0] != B:
        raise ValueError("targets must be (%d, L), got %s" % (B, tuple(targets.shape)))
    tgt = targets.cpu().numpy() if torch.is_tensor(targets) and not targets.is_cuda else targets
    if torch.is_tensor(tgt):
        if tgt.dtype not in (torch.int32, torch.int64):
            raise ValueError("targets must hold integers, got %s" % tgt.dtype)
    elif not np.issubdtype(tgt.dtype, np.integer):
        raise ValueError("targets must hold integers, got %s" % tgt.dtype)
    L = targets.shape[1]
    check_ctc(B, V, T, L)
    _check_lengths(frame_lengths, "frame_lengths", B, 1, T)
    _check_lengths(target_lengths, "target_lengths", B, 0, L)
    lens = _host_ints(target_lengths, "target_lengths")
    if isinstance(tgt, np.ndarray) and lens is not None:
        for b in range(B):
            row = tgt[b, :lens[b]]
            if row.size and (row.min() < 1 or row.max() >= V):
                raise ValueError("targets of row %d outside [1, %d)" % (b, V))
    return B, V, T, L


# ---- launches -------------------------------------------------------------------------------------------------------
class _CTCLossFn(torch.autograd.Function):
    """logits (B, V, T) (unit frame stride), int32 CUDA frames (B,), targets (B, L), target lengths (B,) -> (mean over
    rows of -log p_b / max(L_b, 1), int32 infeasible flags (B,))."""

    @staticmethod
    def forward(ctx, logits, frames, targets, tlen):
        B, V, T = logits.shape
        L = max(targets.shape[1], 1)
        dev = logits.device
        if targets.shape[1] == 0:
            targets = torch.zeros(B, 1, dtype=torch.int32, device=dev)
        ws = torch.empty(int(lib.raw("dv3_ctc_ws_bytes")(B, T, L)), dtype=torch.uint8, device=dev)
        nll = torch.empty(B, device=dev)
        partials = torch.empty(B, device=dev)
        infeasible = torch.empty(B, dtype=torch.int32, device=dev)
        sb, sv = logits.stride(0), logits.stride(1)
        lib.call("dv3_ctc_fwd", _p(logits), sb, sv, _p(frames), _p(targets), targets.stride(0), _p(tlen), B, V, T, L,
                 _p(ws), _p(nll), _p(partials), _p(infeasible), _p(ops._err_flag(dev)), _stream())
        loss = mean_loss(partials)
        ctx.save_for_backward(logits, frames, targets, tlen)
        ctx.ws = ws
        ctx.mark_non_differentiable(infeasible)
        return loss, infeasible

    @staticmethod
    def backward(ctx, d_loss, _):
        logits, frames, targets, tlen = ctx.saved_tensors
        B, V, T = logits.shape
        dz = torch.empty(B, V, T, device=logits.device)
        lib.call("dv3_ctc_bwd", _p(logits), logits.stride(0), logits.stride(1), _p(frames), _p(targets),
                 targets.stride(0), _p(tlen), B, V, T, targets.shape[1], _p(ctx.ws), _p(ops._c(d_loss)), 1.0 / B,
                 _p(dz), _stream())
        return dz, None, None, None


def ctc_loss(logits, frame_lengths, targets, target_lengths):
    """CTC loss of logits (B, V, T) fp32 CUDA (read in place through their strides; unit frame stride), class 0 the
    blank: row b's first frame_lengths[b] frames against its first target_lengths[b] targets (ids in [1, V)).
    Lengths and targets: integer arrays, sequences or tensors; CUDA tensors are not read back (graph capture) and an
    out-of-range value sets the device error flag (``ops.check_index_errors()``) instead.

    -> (loss: the mean over rows of -log p_b / max(L_b, 1), a 0-dim tensor with the kernels' gradient; infeasible:
    int32 (B,), 1 where a row has no alignment (T_b < L_b + its repeated adjacent labels), which then adds 0 to the loss
    and to the gradient).  ValueError before any launch for V or L above 1024, B*V*T at or past 2^31, a workspace above
    2 GiB, malformed shapes and host-side values out of range."""
    B, V, T, L = _check_ctc_inputs(logits, frame_lengths, targets, target_lengths)
    dev = logits.device
    frames = _device_i32(_host_ints(frame_lengths, "frame_lengths") if not torch.is_tensor(frame_lengths)
                         else frame_lengths, dev)
    tlen = _device_i32(_host_ints(target_lengths, "target_lengths") if not torch.is_tensor(target_lengths)
                       else target_lengths, dev)
    tgt = _device_i32(targets if torch.is_tensor(targets) else np.asarray(targets), dev)
    return _CTCLossFn.apply(logits, frames, tgt, tlen)


def greedy_decode(logits, frame_lengths):
    """Greedy CTC decoding of logits (B, V, T) fp32 CUDA: per frame t < frame_lengths[b] the first class of largest
    logit, repeats collapsed, blanks (class 0) dropped -> list of B int64 host arrays.  ValueError before any launch as
    ``ctc_loss`` (frame lengths in [1, T])."""
    B, V, T = _check_logits(logits)
    check_ctc(B, V, T, 0)
    _check_lengths(frame_lengths, "frame_lengths", B, 1, T)
    dev = logits.device
    frames = _device_i32(_host_ints(frame_lengths, "frame_lengths") if not torch.is_tensor(frame_lengths)
                         else frame_lengths, dev)
    hyps = torch.empty(B, T, dtype=torch.int32, device=dev)
    lens = torch.empty(B, dtype=torch.int32, device=dev)
    lib.call("dv3_ctc_greedy", _p(logits), logits.stride(0), logits.stride(1), _p(frames), B, V, T, _p(hyps),
             _p(lens), _p(ops._err_flag(dev)), _stream())
    h, n = hyps.cpu().numpy(), lens.cpu().numpy()
    return [h[b, :n[b]].astype(np.int64) for b in range(B)]


def _token_rows(rows, name, hi):
    if not isinstance(rows, (list, tuple)):
        raise ValueError("%s must be a list of 1-D integer arrays" % name)
    out = []
    for k, r in enumerate(rows):
        r = np.asarray(r.detach().cpu() if torch.is_tensor(r) else r)
        if r.ndim != 1 or (r.size and not np.issubdtype(r.dtype, np.integer)):
            raise ValueError("%s[%d] must be a 1-D integer array, got %s of shape %s" % (name, k, r.dtype, r.shape))
        if r.size > hi:
            raise ValueError("%s[%d] has %d tokens, more than %d" % (name, k, r.size, hi))
        if r.size and (r.min() < -2 ** 31 or r.max() >= 2 ** 31):
            raise ValueError("%s[%d] holds ids outside int32" % (name, k))
        out.append(r.astype(np.int32))
    return out


def _edit_chunks(hyps, refs):
    """Runs [r0, r1) of pairs whose packed rows and workspace stay within ``EDIT_BUDGET`` bytes (at least one pair)."""
    chunks, r0, M, N = [], 0, 0, 0
    for r, (h, f) in enumerate(zip(hyps, refs)):
        M2, N2 = max(M, h.size), max(N, f.size)
        if r > r0 and 4 * (r + 1 - r0) * (M2 + N2 + 2 * (M2 + 64)) > EDIT_BUDGET:
            chunks.append((r0, r))
            r0, M2, N2 = r, h.size, f.size
        M, N = M2, N2
    chunks.append((r0, len(hyps)))
    return chunks


def edit_distance(hyps, refs, device=None):
    """Levenshtein distances of hypothesis rows against reference rows (lists of 1-D integer arrays of equal length;
    any int32 ids) -> int64 (n, 4): (distance, substitutions, deletions, insertions), counted along the path whose
    ties prefer the diagonal (match or substitution), then a deletion (a reference token the hypothesis lacks), then an
    insertion.  Packed on the host, one ``dv3_edit_distance`` launch per chunk of pairs, on ``device`` (default: the
    current CUDA device).  ValueError before any launch for unequal or empty lists, rows that are not 1-D integers,
    references over 1024 or hypotheses over 65 535 tokens."""
    if not isinstance(hyps, (list, tuple)) or not isinstance(refs, (list, tuple)) or len(hyps) != len(refs) or \
            not hyps:
        raise ValueError("hyps and refs must be non-empty lists of equal length")
    hyps = _token_rows(hyps, "hyps", MAX_HYP)
    refs = _token_rows(refs, "refs", MAX_TARGET)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = np.empty((len(hyps), 4), np.int64)
    ws_ints = lib.raw("dv3_edit_ws_ints")
    for r0, r1 in _edit_chunks(hyps, refs):
        P = r1 - r0
        M = max(h.size for h in hyps[r0:r1])
        N = max(f.size for f in refs[r0:r1])
        hp = np.zeros((P, max(M, 1)), np.int32)
        rp = np.zeros((P, max(N, 1)), np.int32)
        for k in range(P):
            hp[k, :hyps[r0 + k].size] = hyps[r0 + k]
            rp[k, :refs[r0 + k].size] = refs[r0 + k]
        hl = np.array([h.size for h in hyps[r0:r1]], np.int32)
        rl = np.array([f.size for f in refs[r0:r1]], np.int32)
        hp_d, rp_d = torch.from_numpy(hp).to(dev), torch.from_numpy(rp).to(dev)
        hl_d, rl_d = torch.from_numpy(hl).to(dev), torch.from_numpy(rl).to(dev)
        ws = torch.empty(int(ws_ints(P, M)), dtype=torch.int32, device=dev)
        res = torch.empty(P, 4, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            lib.call("dv3_edit_distance", _p(hp_d), hp.shape[1], _p(hl_d), _p(rp_d), rp.shape[1], _p(rl_d), P, M, N,
                     _p(ws), _p(res), _p(ops._err_flag(dev)), _stream())
        out[r0:r1] = res.cpu().numpy()
    return out


# ---- model ----------------------------------------------------------------------------------------------------------
def strip_tokens(seq, strip_ids):
    """A token sequence without the ids in ``strip_ids`` -> int64 array."""
    s = np.asarray(seq, np.int64)
    return s[~np.isin(s, np.asarray(list(strip_ids), np.int64))] if len(strip_ids) else s


class TokenRecognizer(nn.Module):
    """CTC token recognizer on this project's kernels (DESIGN.md section 2.21).

    Trunk: two weight-normed 1x1 convs mel_dim -> C -> C with ReLU, then one non-causal residual Conv1dGLU block of
    width ``kernel_size`` per entry of ``dilations``; output: a 1x1 conv C -> n_vocab, one class distribution per mel
    frame (class 0 the CTC blank).  ``strip_ids`` (default: the frontends' EOS id 1, which has no sound of its own) are
    removed from every target and reference before training and scoring.

    forward(mels (B, T, mel_dim), mel_lengths (B,), tokens (B, L), token_lengths (B,)) -> (logits (B, n_vocab, T),
    loss): ``ctc_loss`` of the stripped targets (the tokens are read on the host)."""

    def __init__(self, n_vocab, mel_dim=80, channels=256, kernel_size=5, dilations=(1, 2, 4, 1, 2, 4),
                 strip_ids=(1,)):
        super().__init__()
        if not 2 <= n_vocab <= MAX_VOCAB:
            raise ValueError("n_vocab=%d outside [2, %d]" % (n_vocab, MAX_VOCAB))
        if kernel_size < 1 or kernel_size % 2 == 0:
            raise ValueError("kernel_size=%d: the non-causal blocks keep the frame count with an odd width only"
                             % kernel_size)
        if channels < 1 or mel_dim < 1 or any(int(d) < 1 for d in dilations):
            raise ValueError("channels=%d, mel_dim=%d, dilations=%s" % (channels, mel_dim, tuple(dilations)))
        self.n_vocab, self.mel_dim, self.channels = int(n_vocab), int(mel_dim), int(channels)
        self.strip_ids = tuple(int(i) for i in strip_ids)
        if 0 in self.strip_ids or any(not 0 <= i < n_vocab for i in self.strip_ids):
            raise ValueError("strip_ids %s must be token ids in [1, %d)" % (self.strip_ids, n_vocab))
        C = channels
        self.spectral = nn.ModuleList([modules.Conv1d(mel_dim, C, 1, std_mul=2.0), nn.ReLU(),
                                       modules.Conv1d(C, C, 1, std_mul=2.0), nn.ReLU()])
        self.temporal = nn.ModuleList([modules.Conv1dGLU(1, C, C, C, kernel_size, dropout=0.0, dilation=int(d),
                                                         causal=False, residual=True) for d in dilations])
        self.out = nn.ModuleList([modules.Conv1d(C, n_vocab, 1, std_mul=1.0)])

    def logits(self, mels):
        """mels (B, T, mel_dim) fp32 CUDA -> logits (B, n_vocab, T)."""
        ops._chk(mels)
        if mels.dim() != 3 or mels.shape[2] != self.mel_dim:
            raise ValueError("mels must be (B, T, %d), got %s" % (self.mel_dim, tuple(mels.shape)))
        x = ops.transpose12(mels)
        x = modules.run_conv_stack(self.spectral, x)
        x = modules.run_conv_stack(self.temporal, x)
        return modules.run_conv_stack(self.out, x)

    def strip_batch(self, tokens, token_lengths):
        """Host tokens (B, L) and lengths (B,) -> (int32 (B, L) tokens without ``strip_ids``, left-aligned and
        zero-padded, int32 (B,) lengths)."""
        tok = np.asarray(tokens.cpu() if torch.is_tensor(tokens) else tokens)
        lens = np.asarray(token_lengths.cpu() if torch.is_tensor(token_lengths) else token_lengths)
        if tok.ndim != 2 or lens.shape != (tok.shape[0],) or not np.issubdtype(tok.dtype, np.integer) or \
                not np.issubdtype(lens.dtype, np.integer):
            raise ValueError("tokens (B, L) and token_lengths (B,) must be integers, got %s and %s"
                             % (tok.shape, lens.shape))
        if tok.shape[0] and (lens.min() < 0 or lens.max() > tok.shape[1]):
            raise ValueError("token_lengths must lie in [0, %d]" % tok.shape[1])
        out = np.zeros(tok.shape, np.int32)
        n = np.zeros(tok.shape[0], np.int32)
        for b in range(tok.shape[0]):
            s = strip_tokens(tok[b, :lens[b]], self.strip_ids)
            if s.size and (s.min() < 1 or s.max() >= self.n_vocab):
                raise ValueError("tokens of row %d outside [1, %d) after stripping %s"
                                 % (b, self.n_vocab, self.strip_ids))
            out[b, :s.size] = s
            n[b] = s.size
        return out, n

    def _loss(self, mels, mel_lengths, tokens, token_lengths):
        logits = self.logits(mels)
        return logits, ctc_loss(logits, mel_lengths, tokens, token_lengths)[0]

    def forward(self, mels, mel_lengths, tokens, token_lengths):
        tok, n = self.strip_batch(tokens, token_lengths)
        dev = mels.device
        return self._loss(mels, _device_i32(_host_ints(mel_lengths, "mel_lengths") if not torch.is_tensor(mel_lengths)
                                            else mel_lengths, dev),
                          torch.from_numpy(tok).to(dev), torch.from_numpy(n).to(dev))

    def recognize(self, mels):
        """mels: a list of (T_i, mel_dim) utterances (arrays or tensors) -> list of int64 token arrays (greedy CTC), in
        eval mode without autograd.  The network runs inside ``ops.length_scope``, so every utterance gets what it
        gets alone: bit-identical under ``conv_math="fp32"``, within the tensor-core tolerance otherwise."""
        if not isinstance(mels, (list, tuple)) or not mels:
            raise ValueError("recognize takes a non-empty list of (T, %d) mels" % self.mel_dim)
        rows = []
        for k, m in enumerate(mels):
            m = torch.as_tensor(m)
            if m.dim() != 2 or m.shape[1] != self.mel_dim or m.shape[0] < 1 or not m.is_floating_point():
                raise ValueError("mel %d: shape %s, expected (T >= 1, %d) floats" % (k, tuple(m.shape), self.mel_dim))
            rows.append(m)
        T = max(m.shape[0] for m in rows)
        check_ctc(len(rows), self.n_vocab, T, 0)
        dev = self.out[0].weight_v.device
        batch = torch.zeros(len(rows), T, self.mel_dim, device=dev)
        for k, m in enumerate(rows):
            batch[k, :m.shape[0]] = m.to(dev, torch.float32)
        lengths = torch.tensor([m.shape[0] for m in rows], dtype=torch.int64).to(dev)
        was_training = self.training
        self.eval()
        try:
            with torch.no_grad():
                with ops.length_scope(lengths, T):
                    logits = self.logits(batch)
                return greedy_decode(logits, lengths)
        finally:
            self.train(was_training)


# ---- scoring ----------------------------------------------------------------------------------------------------------
def words(seq, word_sep):
    """Maximal runs of tokens between separators -> list of tuples (empty runs dropped)."""
    out, cur = [], []
    for t in np.asarray(seq).tolist():
        if t == word_sep:
            if cur:
                out.append(tuple(cur))
            cur = []
        else:
            cur.append(t)
    if cur:
        out.append(tuple(cur))
    return out


def word_ids(hyps, refs, word_sep):
    """Token rows -> (hypothesis, reference) rows of integer word ids: one id per distinct word (a tuple of tokens),
    numbered in order of first appearance over the references, then the hypotheses."""
    vocab = {}
    rw = [[vocab.setdefault(w, len(vocab)) for w in words(r, word_sep)] for r in refs]
    hw = [[vocab.setdefault(w, len(vocab)) for w in words(h, word_sep)] for h in hyps]
    return [np.array(h, np.int64) for h in hw], [np.array(r, np.int64) for r in rw]


def _rates(counts, ref_len):
    ref_len = np.asarray(ref_len, np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        per = counts[:, 0].astype(np.float64) / ref_len.astype(np.float64)
    corpus = float(counts[:, 0].sum()) / float(ref_len.sum()) if ref_len.sum() else float("nan")
    return per, corpus


def token_error_rates(recognizer, mels, sequences, word_sep=None):
    """Recognize ``mels`` (a list of (T_k, mel_dim) arrays or tensors) and score them against ``sequences`` (token id
    arrays, stripped of the recognizer's ``strip_ids`` first) -> {"hypotheses": list of int64 arrays,
    "references": the stripped references, "substitutions", "deletions", "insertions", "distance", "ref_lengths":
    int64 (n,), "ter": fp64 (n,) distance / reference length (inf or NaN for an empty reference), "corpus_ter": the sum
    of edits over the sum of reference lengths, in fp64}.  With ``word_sep`` (the id of the space token) also "wer"
    (n,), "corpus_wer", "word_distance" and "word_ref_lengths", from the same kernel on integer word ids (words are
    maximal runs between separators).  ValueError before any launch for unequal list lengths or malformed inputs."""
    if not isinstance(sequences, (list, tuple)) or not isinstance(mels, (list, tuple)) or \
            len(sequences) != len(mels) or not mels:
        raise ValueError("mels and sequences must be non-empty lists of equal length")
    refs = []
    for k, s in enumerate(sequences):
        s = np.asarray(s)
        if s.ndim != 1 or (s.size and not np.issubdtype(s.dtype, np.integer)):
            raise ValueError("sequence %d must be a 1-D integer array" % k)
        r = strip_tokens(s, recognizer.strip_ids)
        if r.size > MAX_TARGET:
            raise ValueError("sequence %d has %d tokens, more than %d" % (k, r.size, MAX_TARGET))
        refs.append(r)
    if word_sep is not None and (isinstance(word_sep, bool) or int(word_sep) != word_sep):
        raise ValueError("word_sep must be a token id, got %r" % (word_sep,))
    hyps = recognizer.recognize(mels)
    dev = recognizer.out[0].weight_v.device
    c = edit_distance(hyps, refs, dev)
    ref_len = np.array([r.size for r in refs], np.int64)
    ter, corpus = _rates(c, ref_len)
    res = {"hypotheses": hyps, "references": refs, "distance": c[:, 0], "substitutions": c[:, 1],
           "deletions": c[:, 2], "insertions": c[:, 3], "ref_lengths": ref_len, "ter": ter, "corpus_ter": corpus}
    if word_sep is not None:
        hw, rw = word_ids(hyps, refs, int(word_sep))
        cw = edit_distance(hw, rw, dev)
        wl = np.array([r.size for r in rw], np.int64)
        res["wer"], res["corpus_wer"] = _rates(cw, wl)
        res["word_distance"], res["word_ref_lengths"] = cw[:, 0], wl
    return res


def evaluate_recognition(model, recognizer, sequences, speaker_ids=None, vocoder="griffin_lim", batch_size=16,
                         word_sep=None, stage_timer=None):
    """Token (and word) error rates of a model's synthesis, in one call: ``synthesis.synthesized_mels`` (stages
    "synthesis" and "mel"), then ``token_error_rates`` (stage "recognition").  ValueError before any launch for
    malformed inputs (as ``tts_batch``), a recognizer of another mel width or vocabulary smaller than the sequences'
    ids."""
    audio.check_phase_method(vocoder)
    if audio.hparams.num_mels != recognizer.mel_dim:
        raise ValueError("synthesis makes %d mel channels, the recognizer takes %d"
                         % (audio.hparams.num_mels, recognizer.mel_dim))
    for s in sequences:
        s = np.asarray(s)
        if s.ndim == 1 and s.size and np.issubdtype(s.dtype, np.integer) and int(s.max()) >= recognizer.n_vocab:
            raise ValueError("token id %d outside the recognizer's vocabulary of %d" % (int(s.max()),
                                                                                         recognizer.n_vocab))
    synthesis._check_inputs(model, sequences, speaker_ids, batch_size=batch_size)
    dev = recognizer.out[0].weight_v.device
    mels = synthesis.synthesized_mels(model, sequences, speaker_ids, vocoder, batch_size, dev, stage_timer)
    stage = synthesis.stages(stage_timer)
    with stage("recognition"):
        return token_error_rates(recognizer, mels, sequences, word_sep)


# ---- training -------------------------------------------------------------------------------------------------------
class TokenRecognizerStep(ArenaGraphStep):
    """One training step of a TokenRecognizer: the CTC loss of a batch, then clip + Adam (``ArenaGraphStep``: the
    conv_math and deterministic modes of construction, one batch shape, bit-exact checkpoints, one CUDA graph with
    use_graph).  ``step(batch)`` takes {"mels": (B, T, mel_dim) float32, "mel_lengths": (B,) in [1, T], "tokens": (B,
    L) integers, "token_lengths": (B,) in [0, L]} on the host, as ``data.RecognizerBatches`` yields them; the tokens
    are stripped of the recognizer's ``strip_ids`` there.  Single process only.  ValueError before any launch for a
    world size above 1, a malformed batch or token ids outside [1, n_vocab) after stripping."""

    _net_key = "recognizer"
    _batch_keys = ("mels", "mel_lengths", "tokens", "token_lengths")

    def __init__(self, recognizer, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip_thresh=None, use_graph=True):
        check_single_process("TokenRecognizerStep")
        super().__init__(recognizer, lr, betas, eps, clip_thresh, use_graph)
        self.recognizer = recognizer

    def step(self, batch):
        tok, n = self.recognizer.strip_batch(batch["tokens"], batch["token_lengths"])
        ml = batch["mel_lengths"]
        ml = torch.as_tensor(ml.cpu().numpy() if torch.is_tensor(ml) else np.asarray(ml)).to(torch.int32)
        return super().step({"mels": batch["mels"], "mel_lengths": ml, "tokens": torch.from_numpy(tok),
                             "token_lengths": torch.from_numpy(n)})

    def _objective(self, batch):
        return self.recognizer._loss(batch["mels"], batch["mel_lengths"], batch["tokens"], batch["token_lengths"])[1]

    def _check_batch(self, batch):
        mels, ml = batch["mels"], batch["mel_lengths"]
        rec = self.recognizer
        if mels.dim() != 3 or mels.shape[2] != rec.mel_dim or mels.dtype != torch.float32 or \
                tuple(ml.shape) != (mels.shape[0],):
            raise ValueError("batch mels %s %s / mel_lengths %s: expected (B, T, %d) float32 and (B,)"
                             % (tuple(mels.shape), mels.dtype, tuple(ml.shape), rec.mel_dim))
        B, T = mels.shape[:2]
        check_ctc(B, rec.n_vocab, T, batch["tokens"].shape[1])
        m = ml.cpu().numpy()
        if m.min() < 1 or m.max() > T:
            raise ValueError("mel_lengths must lie in [1, %d]" % T)
