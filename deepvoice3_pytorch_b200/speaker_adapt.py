"""Embedding-only speaker adaptation (Arik et al., "Neural Voice Cloning with a Few Samples", NeurIPS 2018): every
weight of a trained multi-speaker model stays frozen and only the embedding rows of new speakers are trained, through
the full training loss.  ``TrainStep(model, adapt_speakers=ids)`` installs a ``SpeakerAdapt`` around each of its
passes (DESIGN.md section 2.12).

Inside a pass:

* every parameter has ``requires_grad`` off, so no Function launches a weight-gradient GEMM or a weight-norm backward;
  the weight norm and operand planes of the frozen network come from one ``ops.FrozenWeights`` cache, folded once;
* the looked-up embedding e (B, S) is the one tensor that takes a gradient.  The decoder's two position-rate
  projections (B x S work) reach it through autograd on the existing ops;
* every speaker-conditioned site -- the ``speaker_proj`` of each Conv1dGLU, the encoder's ``speaker_fc1`` / ``_fc2``
  -- runs its forward without autograd and becomes a ``Site``: its backward adds the collapsed gradient
  sum_t mask * sum_c W G (1-|y|)^2 as its own slot of partial rows, with one ``dv3_spk_grad_*`` launch reading the
  gradient G in the form the backward already has (csrc/spk_adapt.cu);
* after the backward, ``dv3_spk_grad_reduce`` sums every slot in index order into d_e (B, S), and
  ``dv3_spk_rows_grad`` adds the position-rate part and sums the rows of each adapted id, in row order.
"""
import ctypes

import torch
import torch.nn.functional as F

from . import ops
from ._lib import lib, Dv3Error
from .ops import _p, _stream


def check_adapt_speakers(model, ids):
    """-> the ids as a list of ints, or ValueError: empty, duplicated, out of range, not one ascending run of
    consecutive ids (the Adam leaf is a view of those rows), or a single-speaker model."""
    if getattr(model, "n_speakers", 1) <= 1 or not hasattr(model, "embed_speakers"):
        raise ValueError("speaker adaptation needs a multi-speaker model (n_speakers=%d)"
                         % getattr(model, "n_speakers", 1))
    try:
        ids = [int(i) for i in ids]
    except TypeError:
        ids = [int(ids)]
    if not ids:
        raise ValueError("adapt_speakers is empty")
    if len(set(ids)) != len(ids):
        raise ValueError("adapt_speakers has duplicates: %s" % ids)
    n = model.embed_speakers.weight.shape[0]
    if min(ids) < 0 or max(ids) >= n:
        raise ValueError("adapt_speakers %s outside [0, %d)" % (ids, n))
    if ids != list(range(ids[0], ids[0] + len(ids))):
        raise ValueError("adapt_speakers must be consecutive ascending ids (as add_speakers returns): %s" % ids)
    if model.speaker_embed_dim > 64:
        raise ValueError("speaker adaptation supports speaker_embed_dim <= 64 (got %d)" % model.speaker_embed_dim)
    return ids


class RowsArena:
    """The optimizer's view of the adapted rows: ``flat`` is the (n*S) slice of the embedding table holding rows
    [lo, lo+n) (the Adam step writes them in place), ``grad`` their gradient.  Duck-types train_step.ParameterArena
    for FlatAdam."""

    def __init__(self, table, lo, n):
        S = table.shape[1]
        assert table.is_contiguous() and table.dtype == torch.float32
        self.flat = table.data.view(-1)[lo * S:(lo + n) * S]
        self.params = [self.flat.view(n, S)]
        self.offsets = [0]
        self.numel = n * S
        self.grad = torch.zeros(n * S, device=table.device)      # written whole by dv3_spk_rows_grad every step

    def zero_grad(self):
        pass

    def all_reduce_grads(self, ranges=None):
        pass                    # single process


class Site:
    """One speaker-conditioned site of the current forward: folded weight w (C, S), its softsign output y, the dropout
    (p, seed, salt) of the stack's (B, T, S) embedding and the logical extent of its time axis."""

    def __init__(self, ctx, w, y, drop, T, ext):
        self.ctx, self.w, self.y, self.drop, self.T, self.ext = ctx, w, y, drop, T, ext
        self.anchor = ctx.anchor
        self.slot = ctx.nsites          # forward order
        ctx.nsites += 1

    def _tail(self, B, C):
        ctx = self.ctx
        p, seed_t, salt = self.drop
        ext_p, ext_m = self.ext if self.ext is not None else (None, 1)
        part = ctx.partials(B)
        at = ctypes.c_void_p(part.data_ptr() + 4 * self.slot * ctx.splits * B * ctx.S)
        return (_p(self.w), at, B, C, self.T, ctx.S, ext_p, ext_m, float(p), _p(seed_t), int(salt), _stream())

    def grad_planes(self, d_btc, npl):
        """G = the "a" half of the gate split's (npl, B, T, 2C) bf16 planes."""
        _, B, T, ld = d_btc.shape
        C = self.y.shape[1]
        lib.call("dv3_spk_grad_planes", _p(d_btc), npl, B * T * ld, ld, _p(self.y), *self._tail(B, C))

    def grad_bct(self, dab, bstride):
        """G = the "a" half of the exact path's (B, 2C, T) gate gradient."""
        B, C = self.y.shape[0], self.y.shape[1]
        lib.call("dv3_spk_grad_bct", _p(dab), bstride, _p(self.y), *self._tail(B, C))

    def grad_btc(self, g):
        """G = a (B, T, C) fp32 residual-stream gradient; y (B, T, C)."""
        B, C = self.y.shape[0], self.y.shape[2]
        lib.call("dv3_spk_grad_btc", _p(g), _p(self.y), *self._tail(B, C))


class _SpeakerResidualFn(torch.autograd.Function):
    """x + y for a site whose addend y = softsign(fc(e~)) was computed without autograd: the gradient passes to x
    unchanged and the site adds its embedding gradient from it."""

    @staticmethod
    def forward(ctx, x, y, site, anchor):
        ctx.site = site
        return x + y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        ctx.site.grad_btc(dy)
        return (dy if ctx.needs_input_grad[0] else None), None, None, None


class SpeakerAdapt:
    """State of the adaptation passes of one TrainStep (see the module docstring).

    ids: the table rows being adapted; their gradient goes to a ``RowsArena`` over them.  Or, with ids None, the anchor
    of each pass is a speaker encoder's output, which the model takes as ``speaker_embed`` (the encoder-only step of
    DESIGN.md section 2.16): ``arena`` is then the encoder's ``ParameterArena``, and ``run`` hands the per-row gradient
    to the encoder's backward."""

    def __init__(self, model, ids=None, arena=None):
        self.model = model
        self.S = model.speaker_embed_dim
        if ids is not None:
            self.ids = list(ids)
            self.lo, self.n = self.ids[0], len(self.ids)
            self.arena = RowsArena(model.embed_speakers.weight, self.lo, self.n)
            self.table = model.embed_speakers.weight    # the Parameter whose storage the Adam leaf views
        else:
            self.ids = self.table = None
            self.arena = arena
        self.frozen = ops.FrozenWeights()
        self.splits = int(lib.raw("dv3_spk_grad_splits")())
        self._rows = {}                                 # B -> arange(B): every row its own id (encoder anchor)
        self._reset()

    def _reset(self):
        self.anchor = self._partials = None
        self.nsites = 0

    def partials(self, B):
        """The pass's partial rows, one slot of (splits, B, S) per site; allocated at the first site backward, when
        the forward has created every site."""
        if self._partials is None:
            self._partials = torch.zeros(max(self.nsites, 1) * self.splits * B * self.S, device=self.arena.grad.device)
        return self._partials

    # -- per pass --------------------------------------------------------------------------------------
    def run(self, batch, inner, spk=None):
        """Forward + loss + backward (``inner(batch)``) with every parameter frozen, then the adapted rows' gradient
        into ``arena.grad``.  spk: the encoder's output e (B, S), with its autograd graph, that ``inner`` passes to the
        model as speaker_embed; the per-row gradient d(loss)/de (the position-rate part included) then runs
        ``spk.backward``.  -> the loss."""
        params = list(self.model.parameters())
        flags = [p.requires_grad for p in params]
        for p in params:
            p.requires_grad_(False)
        try:
            with ops.overrides(speaker_adapt=self, frozen_weights=self.frozen):
                loss = inner(batch)
                e = self.anchor
                B = e.shape[0]
                d_e = torch.empty(B, self.S, device=e.device)
                lib.call("dv3_spk_grad_reduce", _p(self.partials(B)), self.nsites * self.splits, _p(d_e), B, self.S,
                         _stream())
                if spk is None:
                    ids, lo, n, out = batch.get("speaker_ids"), self.lo, self.n, self.arena.grad
                else:                   # ids = arange(B): each row's own gradient
                    ids, lo, n, out = self.rows(B, e.device), 0, B, torch.empty(B, self.S, device=e.device)
                lib.call("dv3_spk_rows_grad", _p(d_e), _p(e.grad), _p(ids), lo, n, _p(out),
                         _p(ops._err_flag(e.device)), B, self.S, _stream())
                if spk is not None:
                    spk.backward(out)
                return loss
        finally:
            for p, f in zip(params, flags):
                p.requires_grad_(f)
            self._reset()

    def rows(self, B, device):
        """A cached int64 arange(B) on the device (no allocation per pass: graph-capture safe)."""
        if B not in self._rows:
            self._rows[B] = torch.arange(B, device=device)
        return self._rows[B]

    # -- hooks called by the model (through ops.speaker_adapt) ----------------------------------------------
    def embed(self, table, speaker_ids):
        """The lookup (range-checked on the device), as the one tensor of the pass that takes a gradient."""
        with torch.no_grad():
            e = table(speaker_ids)
        return self.anchor_of(e)

    def anchor_of(self, e):
        """e (B, S) cut from its autograd graph, as the one tensor of the pass that takes a gradient."""
        e = e.detach().requires_grad_(True)
        self.anchor = e
        return e

    def dropout(self, e_btc, p, training):
        """The stack's dropout of the time-expanded embedding, without autograd; the result carries the (p, seed,
        salt) its sites regenerate the mask from."""
        with torch.no_grad():
            live = training and p > 0.0
            y = ops.dropout(e_btc.detach(), p, training)
            y._dv3_drop = (float(p), ops.rng.seed, ops.rng.salt) if live else (0.0, None, 0)
        return y

    def _site(self, fc, y, e_btc):
        v, g = fc.weight_v, fc.weight_g
        C, S = v.shape
        w = self.frozen.get("fp32", v.view(C, S, 1), g.view(C, 1, 1))[1]        # w_b: (1, C, S)
        return Site(self, w, y, e_btc._dv3_drop, e_btc.shape[1], _extent_of(e_btc.shape[1]))

    def block_site(self, proj, e_btc):
        """Conv1dGLU: -> (softsign(proj(e~)) (B, C, T), Site)."""
        with torch.no_grad():
            y = F.softsign(proj.forward_bct(ops.transpose12(e_btc)))
        return y, self._site(proj, y, e_btc)

    def residual_site(self, x, fc, e_btc):
        """Encoder speaker_fc1 / speaker_fc2: -> x + softsign(fc(e~))."""
        with torch.no_grad():
            y = F.softsign(fc(e_btc)).contiguous()
        site = self._site(fc, y, e_btc)
        return _SpeakerResidualFn.apply(x, y, site, site.anchor)


def _extent_of(T):
    """(device address, mult) of the logical extent of a time axis of T frames in a bucketed batch, else None: the
    active extent axis (encoder: text, converter: mel frames), the decoder steps outside one."""
    ext = ops._extent
    if ext is None:
        return None
    axis = ops.EXT_DEC if ext["axis"] is None else ext["axis"]
    T0 = ext["padded"][axis]
    if T % T0 != 0:
        raise Dv3Error("speaker site of %d frames does not fit a padded extent of %d" % (T, T0))
    return ops._ext_ptr(axis), T // T0
