"""One data-parallel training step of the hot path.

What the reference does per step (train.py:621-779) -- H2D of the batch, model forward, the four losses,
backward, ``clip_grad_norm_``, ``Adam.step`` -- restated around three ideas:

* **flat arenas**: every trainable parameter is a view into one contiguous fp32 buffer and every gradient a view
  into another, so the optimizer (clip + Adam) is two kernel launches over ~26 M floats and the data-parallel
  exchange is ONE NCCL all-reduce of the gradient arena over NVLink (the path is straight data-parallel over
  utterances: no other collective exists);
* **no host synchronisation inside the step**: the clip coefficient, learning rate and dropout seed live in
  device memory, the loss is returned as a device scalar;
* **graph capture**: because of the above the whole step (forward, loss, backward, optimizer) can be captured
  once in a CUDA graph and replayed, which removes the ~1.5 k kernel-launch / autograd dispatch overhead that
  dominates once the convolutions run on tensor cores.
"""
import contextlib
import ctypes
import math
import os
import time

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F

from . import data, ops
from ._lib import lib
from .weight_bank import WeightBank


def noam_learning_rate_decay(init_lr, global_step, warmup_steps=4000):
    """reference lrschedule.py:5-11."""
    warmup_steps = float(warmup_steps)
    step = global_step + 1.0
    return init_lr * warmup_steps ** 0.5 * min(step * warmup_steps ** -1.5, step ** -0.5)


def step_learning_rate_decay(init_lr, global_step, anneal_rate=0.98, anneal_interval=30000):
    """reference lrschedule.py:14-17: x anneal_rate every anneal_interval steps."""
    return init_lr * anneal_rate ** (global_step // anneal_interval)


def cyclic_cosine_annealing(init_lr, global_step, T, M):
    """reference lrschedule.py:20-35: M cosine cycles of T // M steps each over T steps (arXiv:1704.00109)."""
    TdivM = T // M
    return float(init_lr / 2.0 * (np.cos(np.pi * ((global_step - 1) % TdivM) / TdivM) + 1.0))


def sequence_mask(lengths, max_len):
    """(B,) int64 device tensor -> (B, max_len) float mask (reference train.py:261-271)."""
    return (torch.arange(max_len, device=lengths.device)[None, :] < lengths[:, None]).float()


def guided_attention_mask(input_lengths, target_lengths, max_target_len, max_input_len, g):
    """W[b,t,n] = 1 - exp(-(n/N_b - t/T_b)^2 / (2 g^2)) inside (T_b, N_b), 0 outside -- computed on the device
    from the two length vectors (the reference builds it with numba on the host and uploads it every step,
    train.py:585-601, 734-738)."""
    dev = input_lengths.device
    N = input_lengths.double()[:, None, None]
    T = target_lengths.double()[:, None, None]
    n = torch.arange(max_input_len, device=dev, dtype=torch.float64)[None, None, :]
    t = torch.arange(max_target_len, device=dev, dtype=torch.float64)[None, :, None]
    W = 1.0 - torch.exp(-(n / N - t / T) ** 2 / (2 * g * g))
    W = W * (n < N) * (t < T)
    return W.float()


def spec_loss(y_hat, y, mask, masked_loss_weight, binary_divergence_weight, eps=1e-8, priority_bin=None,
              priority_w=0.0):
    """reference train.py:547-582 (torch ops; TrainStep(fused_loss=False) -- the default is csrc/loss.cu)."""
    w = masked_loss_weight

    def l1_of(a, b):
        l1 = (a - b).abs().mean()
        if w > 0:
            mask_ = mask.expand_as(a)
            l1 = w * ((a * mask_ - b * mask_).abs().sum() / mask_.sum()) + (1 - w) * l1
        return l1

    l1 = l1_of(y_hat, y)
    if priority_bin is not None and priority_w > 0:
        l1 = (1 - priority_w) * l1 + priority_w * l1_of(y_hat[:, :, :priority_bin], y[:, :, :priority_bin])
    if binary_divergence_weight <= 0:
        return l1, y_hat.new_zeros(())
    logits = torch.log(y_hat + eps) - torch.log(1 - y_hat + eps)
    z = -y * logits + torch.log1p(torch.exp(logits))
    if w > 0:
        mask_ = mask.expand_as(z)
        bd = w * ((z * mask_).sum() / mask_.sum()) + (1 - w) * z.mean()
    else:
        bd = z.mean()
    return l1, bd


def priority_bin_of(priority_freq, sample_rate, linear_dim):
    """reference train.py:722."""
    return int(priority_freq / (sample_rate * 0.5) * linear_dim)


def training_loss(outs, batch, r=1, downsample_step=4, masked_loss_weight=0.5, binary_divergence_weight=0.1,
                  guided_attention_sigma=0.2, use_guided_attention=True, priority_freq=3000, priority_freq_weight=0.0,
                  sample_rate=22050):
    """Total loss of one step (reference train.py:665-740).  outs = (mel, linear, attention, done) predictions; a
    seq2seq-only step passes linear = None (mel + done + attention losses), a postnet-only step everything but linear
    as None (linear loss only)."""
    if batch.get("extents") is not None:
        raise ValueError("training_loss does not take a batch padded to a bucket (extents): use fused_training_loss")
    mel_out, lin_out, attn, done_hat = outs
    mel, y, done = batch["mel"], batch["y"], batch["done"]
    tl = batch["target_lengths"]
    dec_mask = tgt_mask = None
    if masked_loss_weight > 0:
        dec_mask = sequence_mask(tl // (r * downsample_step), mel.size(1)).unsqueeze(-1)
        tgt_mask = sequence_mask(tl, y.size(1)).unsqueeze(-1) if downsample_step > 1 else dec_mask
        dec_mask, tgt_mask = dec_mask[:, r:, :], tgt_mask[:, r:, :]
    w = binary_divergence_weight
    loss = 0.0
    if mel_out is not None:
        l1, bd = spec_loss(mel_out[:, :-r, :], mel[:, r:, :], dec_mask, masked_loss_weight, w)
        loss = (1 - w) * l1 + w * bd
        loss = loss + F.binary_cross_entropy(done_hat, done)
    if lin_out is not None:
        l1, bd = spec_loss(lin_out[:, :-r, :], y[:, r:, :], tgt_mask, masked_loss_weight, w,
                           priority_bin=priority_bin_of(priority_freq, sample_rate, lin_out.size(-1)),
                           priority_w=priority_freq_weight)
        loss = loss + (1 - w) * l1 + w * bd
    if use_guided_attention and attn is not None:
        soft = guided_attention_mask(batch["input_lengths_dev"], tl // r // downsample_step, attn.size(-2),
                                     attn.size(-1), guided_attention_sigma)
        loss = loss + (attn * soft).mean()
    return loss


class _FusedLossFn(torch.autograd.Function):
    """All four training losses and their gradients in 3 kernel launches (csrc/loss.cu).  Predictions passed as None
    (a seq2seq-only or postnet-only step) leave their loss out and get no launch.  terms: optional float
    (ops.TERM_COUNT,) device block the kernels add the per-term losses to.  det: the fixed-order kernels
    (dv3_spec_loss_det / dv3_aux_loss_det) with the loss scratch of ops.det_scratch."""

    @staticmethod
    def forward(ctx, mel_out, lin_out, attn, done_hat, mel, y, done, target_lengths, input_lengths, r,
                downsample_step, w, bw, sigma, use_attn, pbin, pw, ext, terms, det):
        dev = target_lengths.device
        vp = lambda t: ctypes.c_void_p(t.data_ptr())
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        # a batch padded to a bucket: the kernels read the logical extents (ops.EXT_* slots)
        at = (lambda slot: ctypes.c_void_p(ext.data_ptr() + 8 * slot)) if ext is not None else (lambda slot: None)
        tp = (lambda slot: ctypes.c_void_p(terms.data_ptr() + 4 * slot)) if terms is not None else (lambda slot: None)
        loss = torch.zeros(1, device=dev)
        dec_len = (target_lengths // (r * downsample_step)).contiguous()
        g_mel = g_lin = g_attn = g_done = None
        spec, aux, scratch = "dv3_spec_loss_terms", "dv3_aux_loss_terms", ()
        if det:
            spec, aux, scratch = "dv3_spec_loss_det", "dv3_aux_loss_det", (vp(ops.det_scratch.loss(dev)),)
        if mel_out is not None:
            mel_out = mel_out.contiguous()
            g_mel = torch.empty_like(mel_out)
            B, Td, Dm = mel_out.shape
            lib.call(spec, vp(mel_out), vp(mel.contiguous()), vp(dec_len), at(ops.EXT_MEL), vp(g_mel),
                     vp(loss), tp(ops.TERM_MEL_L1), *scratch, B, Td, Dm, r, float(w), float(bw), 0, 0.0, st)
        if lin_out is not None:
            lin_out = lin_out.contiguous()
            g_lin = torch.empty_like(lin_out)
            B, Tl, Dl = lin_out.shape
            lin_len = target_lengths.contiguous() if downsample_step > 1 else dec_len
            lib.call(spec, vp(lin_out), vp(y.contiguous()), vp(lin_len),
                     at(ops.EXT_LIN if downsample_step > 1 else ops.EXT_MEL), vp(g_lin), vp(loss), tp(ops.TERM_LIN_L1),
                     *scratch, B, Tl, Dl, r, float(w), float(bw), int(pbin), float(pw), st)
        if done_hat is not None:
            attn, done_hat = attn.contiguous(), done_hat.contiguous()
            g_attn, g_done = torch.empty_like(attn), torch.empty_like(done_hat)
            A, B, Td, Ts = attn.shape
            dec_len_attn = (target_lengths // r // downsample_step).contiguous()
            assert ext is None or (done_hat.numel() == B * Td and ops.EXT_TEXT == ops.EXT_DEC + 1)
            lib.call(aux, vp(done_hat), vp(done.contiguous()), vp(g_done), done_hat.numel(), vp(attn),
                     vp(g_attn), vp(input_lengths.contiguous()), vp(dec_len_attn), at(ops.EXT_DEC), A, B, Td, Ts,
                     float(sigma), int(use_attn), vp(loss), tp(ops.TERM_DONE), *scratch, st)
        ctx.save_for_backward(g_mel, g_lin, g_attn, g_done)
        return loss[0]

    @staticmethod
    def backward(ctx, gout):
        return tuple(None if g is None else g * gout for g in ctx.saved_tensors) + (None,) * 16


def fused_training_loss(outs, batch, r=1, downsample_step=4, masked_loss_weight=0.5, binary_divergence_weight=0.1,
                        guided_attention_sigma=0.2, use_guided_attention=True, priority_freq=3000,
                        priority_freq_weight=0.0, sample_rate=22050, terms=None, deterministic=None):
    """Same value and gradients as ``training_loss`` (reference train.py:665-740), computed by csrc/loss.cu.  A batch
    padded to a bucket (``data.pad_to_bucket``: it carries ``extents``) gives the loss and gradients of the unpadded
    batch: the padding leaves every mean and its gradient is 0.  terms: a zeroed float (ops.TERM_COUNT,) CUDA tensor
    that receives the per-term losses (L1 and binary-divergence parts of the mel and linear losses, done BCE, guided
    attention) without a launch of their own.  deterministic (None: ``ops.deterministic``): sum the losses in a fixed
    order (DESIGN.md section 2.10); the gradients are the same bits either way."""
    mel_out, lin_out, attn, done_hat = outs
    det = ops.is_deterministic() if deterministic is None else bool(deterministic)
    ext = batch.get("extents")
    if ext is not None and not (ext.is_cuda and ext.dtype == torch.int64 and ext.shape == (4,) and ext.is_contiguous()):
        raise ValueError("batch['extents'] must be a contiguous int64 (4,) CUDA tensor")
    if terms is not None and not (terms.is_cuda and terms.dtype == torch.float32 and terms.shape == (ops.TERM_COUNT,)):
        raise ValueError("terms must be a float32 (%d,) CUDA tensor" % ops.TERM_COUNT)
    pbin = priority_bin_of(priority_freq, sample_rate, lin_out.size(-1)) if lin_out is not None else 0
    return _FusedLossFn.apply(mel_out, lin_out, attn, done_hat, batch["mel"], batch.get("y"), batch.get("done"),
                              batch["target_lengths"], batch.get("input_lengths_dev"), r, downsample_step,
                              masked_loss_weight, binary_divergence_weight, guided_attention_sigma,
                              use_guided_attention, pbin, priority_freq_weight, ext, terms, det)


class ParameterArena:
    """Re-homes the trainable parameters of ``model`` into one flat fp32 buffer (and their gradients into
    another).  ``state_dict`` / ``load_state_dict`` keep working: parameters stay nn.Parameters, only their
    storage moves."""

    def __init__(self, model, params=None):
        params = list(model.get_trainable_parameters()) if params is None else list(params)
        assert all(p.dtype == torch.float32 for p in params), "fp32 parameters only"
        self.params = params
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4            # keep every view 16-byte aligned
        self.numel = n
        dev = params[0].device
        self.flat = torch.zeros(n, device=dev)
        self.grad = torch.zeros(n, device=dev)
        for p, o in zip(params, offs):
            self.flat[o:o + p.numel()].view_as(p).copy_(p.data)
            p.data = self.flat[o:o + p.numel()].view_as(p)
            p.grad = self.grad[o:o + p.numel()].view_as(p)
        self.offsets = offs

    def zero_grad(self):
        self.grad.zero_()

    def broadcast(self, model=None, src=0):
        """Replica consistency at start-up (what DistributedDataParallel does at construction): every rank takes
        rank ``src``'s parameter arena, plus -- when ``model`` is given -- the parameters outside the arena (frozen
        position tables / embeddings) and the buffers."""
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        dist.broadcast(self.flat, src)
        if model is not None:
            inside = {id(p) for p in self.params}
            for t in list(model.parameters()) + list(model.buffers()):
                if id(t) not in inside:
                    dist.broadcast(t.data, src)

    def all_reduce_grads(self, ranges=None):
        """The exchange step of the data-parallel path: sum the flat gradient arena (or the given [lo, hi) slices of
        it) over all ranks (NCCL over NVLink on GPUs; gloo in the CPU tests).  The 1/world average is applied by the
        optimizer (hyper[3])."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            if ranges is None:
                dist.all_reduce(self.grad)
            else:
                for lo, hi in ranges:
                    if hi > lo:
                        dist.all_reduce(self.grad[lo:hi])

    def range_of(self, params):
        """[lo, hi) of the arena slice holding ``params`` (must be consecutive arena entries), or None if empty."""
        ids = {id(p) for p in params}
        idx = [i for i, p in enumerate(self.params) if id(p) in ids]
        if not idx:
            return None
        assert idx == list(range(idx[0], idx[-1] + 1)), "bucket parameters are not contiguous in the arena"
        last = idx[-1]
        return self.offsets[idx[0]], self.offsets[last] + (self.params[last].numel() + 3) // 4 * 4


def gradient_buckets(model, arena):
    """Bucket plan of the overlapped gradient exchange.  The backward pass finishes the post-net first, then the
    decoder, then the encoder from its last layer to its first (the encoder holds ~60 % of the parameters), so:
      "postnet"     everything under model.postnet        -- final when d(loss)/d(postnet input) exists
      "encoder_hi" / "encoder_mid"  encoder.convolutions[hi:] / [mid:hi]  -- final when the gradient entering layer
                    hi / mid exists
      "rest"        all other slices (decoder, first encoder layers, embeddings): reduced after backward()
    -> ({tag: (lo, hi)}, [rest ranges])."""
    tagged = {}
    post = arena.range_of(list(model.postnet.parameters())) if hasattr(model, "postnet") else None
    if post:
        tagged["postnet"] = post
    enc = getattr(getattr(model, "seq2seq", None), "encoder", None)
    if enc is not None and hasattr(enc, "grad_bucket_splits") and hasattr(enc, "convolutions"):
        layers = list(enc.convolutions)
        splits = sorted(enc.grad_bucket_splits(), key=lambda ti: ti[1])
        for (tag, lo_i), hi_i in zip(splits, [i for _, i in splits[1:]] + [len(layers)]):
            r = arena.range_of([p for m in layers[lo_i:hi_i] for p in m.parameters()])
            if r:
                tagged[tag] = r
    cuts = sorted(tagged.values())
    rest, pos = [], 0
    for lo, hi in cuts:
        if lo > pos:
            rest.append((pos, lo))
        pos = max(pos, hi)
    if pos < arena.numel:
        rest.append((pos, arena.numel))
    return tagged, rest


def arena_parts(model, arena):
    """[lo, hi) arena ranges of ``model.seq2seq``'s and ``model.postnet``'s parameters, plus whatever lies between or
    after them (the speaker embedding) as parts of their own: the units that keep their own Adam step count."""
    cuts = sorted(r for r in (arena.range_of(list(getattr(model, name).parameters()))
                              for name in ("seq2seq", "postnet") if hasattr(model, name)) if r)
    parts, pos = [], 0
    for lo, hi in cuts:
        if lo > pos:
            parts.append((pos, lo))
        parts.append((lo, hi))
        pos = hi
    if pos < arena.numel:
        parts.append((pos, arena.numel))
    return parts


class FlatAdam:
    """torch.optim.Adam(betas, eps, weight_decay, amsgrad) + clip_grad_norm_(clip) over a ParameterArena in two
    launches.

    parts: [lo, hi) arena ranges that keep their own step count (bias-correction clock); default one part.  State
    loaded for only some parts (a checkpoint of a seq2seq-only or postnet-only run) resumes those at their step and
    starts the others at 0, as torch.optim.Adam does for parameters it has no state for.  While all clocks agree the
    update is one launch over the arena; otherwise one per part (``split_update()``; a captured CUDA graph keeps the
    plan it was captured with, and TrainStep.load_state_dict drops its graphs when the plan changes).
    State loaded for parameters outside the arena (the other part, in a seq2seq-only or postnet-only run) is kept
    as it is and written back by ``state_dict()``, as torch.optim.Adam keeps state for parameters without gradients.
    index / n_index: position of each arena parameter in the optimizer's parameter list (the indices of the checkpoint
    format) and that list's length; default the arena's own parameters."""

    def __init__(self, arena, lr=5e-4, betas=(0.5, 0.9), eps=1e-6, clip_thresh=0.1, weight_decay=0.0, amsgrad=False,
                 parts=None, index=None, n_index=None):
        if weight_decay < 0:
            raise ValueError("weight_decay=%r < 0" % weight_decay)
        self.arena = arena
        self.lr, self.betas, self.eps, self.clip = lr, betas, eps, clip_thresh
        self.weight_decay, self.amsgrad = float(weight_decay), bool(amsgrad)
        dev = arena.flat.device
        self.m = torch.zeros_like(arena.flat)
        self.v = torch.zeros_like(arena.flat)
        self.vmax = torch.zeros_like(arena.flat) if self.amsgrad else None
        self.parts = list(parts) if parts else [(0, arena.numel)]
        self.part_t = [0] * len(self.parts)
        self._part_of = [next(k for k, (lo, hi) in enumerate(self.parts) if lo <= o < hi) for o in arena.offsets]
        self.index = list(range(len(arena.params))) if index is None else list(index)
        self.n_index = len(self.index) if n_index is None else int(n_index)
        nh = 4 * len(self.parts)
        self.hyper = torch.zeros(nh, device=dev)
        # ring of pinned staging slots: the host may run several steps ahead of the stream, so a slot is only
        # rewritten after the copy that last read it has completed (event wait, normally already signalled)
        self._slots = [torch.zeros(nh).pin_memory() if dev.type == "cuda" else torch.zeros(nh) for _ in range(4)]
        self._events = [None] * 4
        self._n = 0
        self._foreign = {}          # loaded state of parameters outside the arena: list index -> torch Adam state
        self.sumsq = torch.zeros(1, device=dev)
        self._scratch = torch.zeros(lib.raw("dv3_sumsq_scratch_floats")(), device=dev) if dev.type == "cuda" else None

    def split_update(self):
        """True when the parts' step counts differ: one update launch per part instead of one over the arena."""
        return len(set(self.part_t)) > 1

    @property
    def t(self):
        """Step count (of the part that has taken the most steps)."""
        return max(self.part_t)

    def set_hyper(self, lr, grad_scale=1.0):
        """Host-side scalar prep; the async H2D copy of 16 bytes per part is the only thing the stream sees.
        hyper[4k:4k+4] = {lr, bias correction 1, bias correction 2, grad_scale} of part k."""
        self.part_t = [t + 1 for t in self.part_t]
        self._n += 1
        b1, b2 = self.betas
        i = self._n % 4
        if self._events[i] is not None:
            self._events[i].synchronize()
        h = self._slots[i]
        for k, t in enumerate(self.part_t):
            h[4 * k], h[4 * k + 1], h[4 * k + 2], h[4 * k + 3] = lr, 1.0 - b1 ** t, 1.0 - b2 ** t, grad_scale
        self.hyper.copy_(h, non_blocking=True)
        self._events[i] = torch.cuda.Event()
        self._events[i].record()

    def apply(self):
        """Device-only part (graph-capturable): grad norm -> clip -> Adam."""
        a = self.arena
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        lib.call("dv3_sumsq", ctypes.c_void_p(a.grad.data_ptr()), a.numel, ctypes.c_void_p(self.sumsq.data_ptr()),
                 ctypes.c_void_p(self._scratch.data_ptr()), st)
        if not self.split_update():
            plan = [(0, a.numel, 0)]
        else:
            plan = [(lo, hi, k) for k, (lo, hi) in enumerate(self.parts)]
        for lo, hi, k in plan:
            at = lambda t: ctypes.c_void_p(t.data_ptr() + 4 * lo) if t is not None else None
            lib.call("dv3_adam_clip_opts", at(a.flat), at(a.grad), at(self.m), at(self.v), at(self.vmax), hi - lo,
                     ctypes.c_void_p(self.hyper.data_ptr() + 16 * k), ctypes.c_void_p(self.sumsq.data_ptr()),
                     self.betas[0], self.betas[1], self.eps, float(self.clip), self.weight_decay, st)

    def grad_norm(self):
        return self.sumsq.sqrt() * self.hyper[3]

    # -- checkpoint format of torch.optim.Adam (what reference train.py:save_checkpoint stores under "optimizer",
    #    train.py:787-810, and load_checkpoint restores, :843-860): parameter index[j] of the optimizer's list <->
    #    state = {step, exp_avg, exp_avg_sq[, max_exp_avg_sq]}; parameters that have not stepped have no state
    def state_dict(self):
        a = self.arena
        state = {}
        for p, o, i, k in zip(a.params, a.offsets, self.index, self._part_of):
            if self.part_t[k] == 0:
                continue
            n = p.numel()
            state[i] = {"step": torch.tensor(float(self.part_t[k])),
                        "exp_avg": self.m[o:o + n].view_as(p).clone(),
                        "exp_avg_sq": self.v[o:o + n].view_as(p).clone()}
            if self.amsgrad:
                state[i]["max_exp_avg_sq"] = self.vmax[o:o + n].view_as(p).clone()
        for i, st in self._foreign.items():
            state[i] = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in st.items()}
        group = {"lr": self.lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay,
                 "amsgrad": self.amsgrad, "maximize": False, "foreach": None, "capturable": False,
                 "differentiable": False, "fused": None, "decoupled_weight_decay": False,
                 "params": list(range(self.n_index))}
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        """Accepts a torch.optim.Adam state_dict over the same parameter list (e.g. from a reference checkpoint, whole
        or partial).  Every part resumes at the step count of its parameters' state, or at 0 if it has none."""
        a = self.arena
        groups = sd["param_groups"]
        ids = [i for g in groups for i in g["params"]]
        if len(ids) != self.n_index:
            raise ValueError("optimizer state has %d parameters, the model %d" % (len(ids), self.n_index))
        g0 = groups[0]
        if float(g0.get("weight_decay", 0)) != self.weight_decay or bool(g0.get("amsgrad", False)) != self.amsgrad:
            raise ValueError("optimizer state has weight_decay=%r amsgrad=%r, this optimizer weight_decay=%r amsgrad=%r"
                             % (g0.get("weight_decay", 0), g0.get("amsgrad", False), self.weight_decay, self.amsgrad))
        self.lr, self.betas, self.eps = g0["lr"], tuple(g0["betas"]), g0["eps"]
        mine = set(self.index)
        self._foreign = {j: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in sd["state"][ids[j]].items()}
                         for j in range(self.n_index) if j not in mine and ids[j] in sd["state"]}
        steps = [set() for _ in self.parts]
        self.m.zero_()
        self.v.zero_()
        if self.vmax is not None:
            self.vmax.zero_()
        for j, p, o, k in zip(self.index, a.params, a.offsets, self._part_of):
            st = sd["state"].get(ids[j])
            if st is None:                      # parameter that never received a gradient
                continue
            n = p.numel()
            if tuple(st["exp_avg"].shape) != tuple(p.shape):
                raise ValueError("optimizer state %d has shape %s, parameter %s" % (ids[j], tuple(st["exp_avg"].shape),
                                                                                   tuple(p.shape)))
            self.m[o:o + n].view_as(p).copy_(st["exp_avg"])
            self.v[o:o + n].view_as(p).copy_(st["exp_avg_sq"])
            if self.vmax is not None:
                self.vmax[o:o + n].view_as(p).copy_(st["max_exp_avg_sq"])
            steps[k].add(int(st["step"]))
        for k, s in enumerate(steps):
            if len(s) > 1:
                raise ValueError("step counts differ within arena part %d (%s): not representable in a flat Adam"
                                 % (k, sorted(s)))
        self.part_t = [s.pop() if s else 0 for s in steps]


def check_train_mode(model, train_seq2seq, train_postnet):
    """ValueError for a training mode the reference would assert on or crash in later (train.py:615, 690, 699)."""
    if not (train_seq2seq or train_postnet):
        raise ValueError("train_seq2seq and train_postnet are both False: nothing to train")
    if train_seq2seq and train_postnet:
        return
    if getattr(model, "n_speakers", 1) > 1:
        raise ValueError("seq2seq-only / postnet-only training needs a single-speaker model (n_speakers=%d)"
                         % model.n_speakers)
    if train_postnet and getattr(model, "use_decoder_state_for_postnet_input", False):
        raise ValueError("postnet-only training feeds the converter ground-truth mels, but this model was built with "
                         "use_decoder_state_for_postnet_input=True (its converter reads decoder states)")


class TrainStep:
    """model + losses + flat optimizer (+ NCCL gradient all-reduce when torch.distributed is initialised): reference
    train.py's ``train()``.

    train_seq2seq / train_postnet: the reference's two-stage training (train.py:655-740).  Seq2seq-only runs
    ``model.seq2seq`` and the mel + done + guided-attention losses; postnet-only runs ``model.postnet`` on the
    ground-truth mel and the linear loss.  The arena, the optimizer state and the gradient norm then cover only the
    trained part; the other part's parameters keep their bits.  weight_decay / amsgrad: torch.optim.Adam's.

    The step runs in the ``ops.conv_math`` mode current at construction ("tc", "tc1" or "fp32"): its weight bank and
    captured graphs hold that mode's kernels and operand planes, so ``step()`` under another mode raises ValueError.

    deterministic (None: ``ops.deterministic`` at construction): every step runs the fixed-order kernels of DESIGN.md
    section 2.10 whatever ``ops.deterministic`` says later, eager or captured; the step owns their scratch, which is
    allocated by the eager passes before a capture and so lies outside every graph pool."""

    def __init__(self, model, init_lr=5e-4, betas=(0.5, 0.9), eps=1e-6, clip_thresh=0.1, r=1, downsample_step=4,
                 masked_loss_weight=0.5, binary_divergence_weight=0.1, guided_attention_sigma=0.2,
                 use_guided_attention=True, priority_freq=3000, priority_freq_weight=0.0, sample_rate=22050,
                 lr_schedule=noam_learning_rate_decay, use_graph=False, fused_loss=True, weight_bank=None,
                 train_seq2seq=True, train_postnet=True, weight_decay=0.0, amsgrad=False, deterministic=None):
        check_train_mode(model, train_seq2seq, train_postnet)
        self.math = ops.math_mode()
        self.deterministic = ops.is_deterministic() if deterministic is None else bool(deterministic)
        self._det_scratch = ops.DetScratch() if self.deterministic else None
        self.model = model
        self.train_seq2seq, self.train_postnet = bool(train_seq2seq), bool(train_postnet)
        # the module whose parameters are trained and checkpointed (reference save_checkpoint, train.py:787-808)
        self.trained = model if self.train_seq2seq and self.train_postnet else \
            (model.seq2seq if self.train_seq2seq else model.postnet)
        trainable = list(model.get_trainable_parameters())
        own = {id(p) for p in self.trained.parameters()}
        index = [i for i, p in enumerate(trainable) if id(p) in own]
        self.arena = ParameterArena(model, [trainable[i] for i in index])
        self.opt = FlatAdam(self.arena, init_lr, betas, eps, clip_thresh, weight_decay, amsgrad,
                            arena_parts(model, self.arena), index, len(trainable))
        self.init_lr, self.lr_schedule = init_lr, lr_schedule
        self.loss_kw = dict(r=r, downsample_step=downsample_step, masked_loss_weight=masked_loss_weight,
                            binary_divergence_weight=binary_divergence_weight,
                            guided_attention_sigma=guided_attention_sigma,
                            use_guided_attention=use_guided_attention, priority_freq=priority_freq,
                            priority_freq_weight=priority_freq_weight, sample_rate=sample_rate)
        self.loss_fn = fused_training_loss if fused_loss else training_loss
        # per-term losses of the last step (ops.TERM_* slots); outside every graph pool, like the bucket loss scalars
        self._terms = torch.zeros(ops.TERM_COUNT, device=self.arena.flat.device)
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.global_step = 0
        self.use_graph = use_graph
        self._graph = None
        self._static = None
        self._loss = None
        self.launches_per_step = None       # dv3 kernel launches inside one captured step (graph mode)
        # graph mode with batches of other shapes than the first: one graph per bucket (data.bucket_shape), all in
        # one memory pool; the first shape keeps its own exact graph
        self._pool = None
        self._graph_key = None
        self._buckets = {}                  # bucket key -> (graph, static inputs, loss buffer, launches)
        self.capture_seconds = 0.0          # wall time spent warming up and capturing graphs
        if weight_bank is None:
            weight_bank = os.environ.get("DV3_WEIGHT_BANK", "1") == "1"
        self.bank = WeightBank(ops._npl()) if weight_bank else None
        self.arena.broadcast(model)             # replicas start from rank 0's weights (no-op for world == 1)
        # overlapped gradient exchange (world > 1): buckets are all-reduced on a communication stream as soon as the
        # backward pass has finished them; only the last ("rest") bucket is exposed
        self.buckets, self.rest_ranges = gradient_buckets(model, self.arena)
        self.overlap_comm = self.world > 1 and os.environ.get("DV3_OVERLAP_COMM", "1") == "1" and \
            self.arena.flat.is_cuda
        self._comm = torch.cuda.Stream(device=self.arena.flat.device) if self.overlap_comm else None
        self._reduced = set()
        # capture the NCCL collectives inside the step's CUDA graph (so clip + Adam stay in the graph too)
        self.graph_comm = self.overlap_comm and os.environ.get("DV3_GRAPH_COMM", "1") == "1"

    # -- checkpointing: the reference's checkpoint keys (train.py:787-810) ---------------------------------
    def state_dict(self, global_epoch=0):
        """The reference's checkpoint: in a partial mode the trained part's state_dict (model.seq2seq or
        model.postnet), with optimizer state for its parameters only."""
        return {"state_dict": self.trained.state_dict(), "optimizer": self.opt.state_dict(),
                "global_step": self.global_step, "global_epoch": global_epoch}

    def load_state_dict(self, ckpt, load_optimizer=True):
        """Resume from ``state_dict()`` or from a reference checkpoint (same keys), of the whole model or of
        model.seq2seq / model.postnet alone, in any mode.  Restores the Adam moments, the bias-correction steps (parts
        without optimizer state start at step 0) and the position in the learning-rate schedule."""
        sd = ckpt["state_dict"]
        target = self.model
        for part in (self.model.seq2seq, self.model.postnet):
            if set(sd) == set(part.state_dict()):
                target = part
        target.load_state_dict(sd)      # copies into the arena views in place
        if load_optimizer and ckpt.get("optimizer") is not None:
            split = self.opt.split_update()
            self.opt.load_state_dict(ckpt["optimizer"])
            if self.opt.split_update() != split:       # captured graphs hold the other update plan: capture anew
                self._graph = self._static = self._loss = self._graph_key = self._pool = None
                self._buckets = {}
                self.launches_per_step = None
        self.global_step = int(ckpt.get("global_step", 0))
        return int(ckpt.get("global_epoch", 0))

    # -- pieces -------------------------------------------------------------------------------
    def _forward_backward(self, batch):
        self.arena.zero_grad()
        ops.grad_sink = True          # kernels accumulate parameter gradients straight into the arena
        ops.weight_bank = self.bank   # weight norm of all layers: 2 launches up front, 1 per bucket in the backward
        ops.grad_boundary_cb = self._bucket_ready if self.overlap_comm else None
        self._reduced = set()
        det_outer = (ops.deterministic, ops.det_scratch)
        ops.deterministic = self.deterministic
        if self.deterministic:
            ops.det_scratch = self._det_scratch
        try:
            if self.bank is not None:
                self.bank.begin_step()
            return self._forward_backward_inner(batch)
        finally:
            ops.deterministic, ops.det_scratch = det_outer
            ops.grad_sink = False
            ops.weight_bank = None
            ops.grad_boundary_cb = None
            if self.bank is not None:
                self.bank.end_step()

    def _bucket_ready(self, tag):
        """Called from the backward pass (ops.grad_boundary hook): the parameter gradients of bucket ``tag`` are final
        -- finish their weight-norm backward and start their all-reduce on the communication stream."""
        rng = self.buckets.get(tag)
        if rng is None or tag in self._reduced:
            return
        self._reduced.add(tag)
        if self.bank is not None:
            self.bank.end_backward()
        main = torch.cuda.current_stream()
        self._comm.wait_stream(main)
        with torch.cuda.stream(self._comm):
            self.arena.all_reduce_grads([rng])

    def _forward_backward_inner(self, batch):
        ext = batch.get("extents")          # a batch padded to a bucket (data.pad_to_bucket)
        scope = ops.extent_scope(ext, data.batch_extents(batch)) if ext is not None else contextlib.nullcontext()
        with scope:
            outs = self._forward(batch)
            if self.loss_fn is fused_training_loss:
                self._terms.zero_()
                loss = self.loss_fn(outs, batch, terms=self._terms, **self.loss_kw)
            else:
                loss = self.loss_fn(outs, batch, **self.loss_kw)
        loss.backward()
        if self.bank is not None:
            self.bank.end_backward()
        return loss.detach()

    def _forward(self, batch):
        """-> (mel, linear, attention, done) predictions; the parts this mode does not run are None."""
        m = self.model
        if self.train_seq2seq and self.train_postnet:
            return m(batch["x"], batch["mel"], speaker_ids=batch.get("speaker_ids"),
                     text_positions=batch["text_positions"], frame_positions=batch["frame_positions"],
                     input_lengths=batch["input_lengths_dev"])
        mel = batch["mel"]
        if self.train_seq2seq:                  # reference train.py:690-697
            mel_out, attn, done_hat, _ = m.seq2seq(batch["x"], mel, text_positions=batch["text_positions"],
                                                   frame_positions=batch["frame_positions"],
                                                   input_lengths=batch["input_lengths_dev"])
            return mel_out.reshape(mel.size(0), -1, mel.size(-1)), None, attn, done_hat
        with ops.extent_axis(ops.EXT_MEL):      # reference train.py:698-700
            return None, m.postnet(mel), None, None

    def _mode_batch(self, batch):
        """A postnet-only step reads no text: its batch keeps zero text positions, so that graphs and buckets follow
        the mel / linear axes alone."""
        if self.train_seq2seq:
            return batch
        return {k: (v[:, :0] if k in ("x", "text_positions") and torch.is_tensor(v) else v) for k, v in batch.items()}

    def loss_terms(self):
        """The per-term losses of the last step under the tags reference train.py logs (:761-776), for the terms this
        mode has, plus "gradient norm" when clipping is on.  Device scalars (no host sync), valid until the next
        ``step()``; on a data-parallel run, this rank's losses and the norm of the averaged gradient."""
        if self.loss_fn is not fused_training_loss:
            raise ValueError("loss_terms() needs the fused loss kernels (TrainStep(fused_loss=True))")
        t, w = self._terms, self.loss_kw["binary_divergence_weight"]
        out = {}
        if self.train_seq2seq:
            out["mel loss"] = (1 - w) * t[ops.TERM_MEL_L1] + w * t[ops.TERM_MEL_BD]
            out["mel_l1_loss"], out["mel_binary_div_loss"] = t[ops.TERM_MEL_L1], t[ops.TERM_MEL_BD]
            out["done_loss"] = t[ops.TERM_DONE]
        if self.train_postnet:
            out["linear_loss"] = (1 - w) * t[ops.TERM_LIN_L1] + w * t[ops.TERM_LIN_BD]
            out["linear_l1_loss"], out["linear_binary_div_loss"] = t[ops.TERM_LIN_L1], t[ops.TERM_LIN_BD]
        if self.train_seq2seq and self.loss_kw["use_guided_attention"]:
            out["attn_loss"] = t[ops.TERM_ATTN]
        if self.opt.clip > 0:
            out["gradient norm"] = self.opt.grad_norm()[0]
        return out

    def _exchange_and_update(self):
        """Gradient exchange (sum; the 1/world average is folded into hyper[3]) + clip + Adam."""
        if self.overlap_comm:
            main = torch.cuda.current_stream()
            self._comm.wait_stream(main)
            with torch.cuda.stream(self._comm):         # buckets whose boundary never fired + everything else
                pending = [r for t, r in self.buckets.items() if t not in self._reduced]
                self.arena.all_reduce_grads(pending + self.rest_ranges)
            main.wait_stream(self._comm)
        else:
            self.arena.all_reduce_grads()
        self.opt.apply()          # (fresh dropout masks per step: the model's forward draws a new seed itself)

    # -- public -------------------------------------------------------------------------------
    @property
    def graphs_captured(self):
        return (self._graph is not None) + len(self._buckets)

    def step(self, batch):
        """batch: dict of DEVICE tensors (x, text_positions, frame_positions int64; mel, y, done fp32;
        target_lengths, input_lengths_dev int64) + host numpy ``input_lengths``.  Returns the loss (device).

        Batches may differ in shape from step to step (``data.collate`` pads each to its own longest utterance).  In
        graph mode the first shape runs its own exact graph; any other is padded to its bucket (``data.bucket_shape``,
        ``data.pad_to_bucket``) and replays that bucket's graph, with the loss, gradients and update of the unpadded
        batch.  A batch that already carries ``extents`` is its own bucket."""
        if ops.math_mode() != self.math:
            raise ValueError("TrainStep was built with ops.conv_math = %r and cannot step under %r: its weight bank and "
                             "CUDA graphs hold that mode's kernels (build a new TrainStep)" % (self.math, ops.conv_math))
        self.model.train()
        batch = self._mode_batch(batch)
        lr = self.lr_schedule(self.init_lr, self.global_step) if self.lr_schedule else self.init_lr
        self.opt.set_hyper(lr, 1.0 / self.world)
        if not self.use_graph:
            loss = self._forward_backward(batch)
            self._exchange_and_update()
        else:
            loss = self._graph_step(batch)
        self.global_step += 1
        return loss

    def _shape_key(self, batch):
        return tuple((k, tuple(v.shape)) for k, v in sorted(batch.items()) if torch.is_tensor(v))

    def _warm_up(self, static):
        """Two eager passes on a side stream before a capture (allocator, NCCL, weight-bank tables); they do not
        consume dropout seeds."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            dev = self.arena.flat.device
            ops.rng.seed_tensor(dev)
            seed0 = ops.rng.base.clone()
            for _ in range(2):
                self._forward_backward(static)
                if self.world > 1 and self.overlap_comm:    # NCCL communicators / bucket tables exist before capture
                    pend = [r for t, r in self.buckets.items() if t not in self._reduced]
                    with torch.cuda.stream(self._comm):
                        self._comm.wait_stream(s)
                        self.arena.all_reduce_grads(pend + self.rest_ranges)
                    s.wait_stream(self._comm)
            ops.rng.base.copy_(seed0)           # the warm-up passes do not consume dropout seeds
        torch.cuda.current_stream().wait_stream(s)

    def _bucket_step(self, batch):
        """A batch of another shape than the first graph's: pad it to its bucket and replay (capturing on first use)
        that bucket's graph."""
        if self.loss_fn is not fused_training_loss:
            raise ValueError("TrainStep(use_graph=True, fused_loss=False) needs every batch in the shape of the first "
                             "one: padding to a bucket is supported by the fused loss kernels only")
        if self.world > 1:
            raise ValueError("TrainStep(use_graph=True) with world_size > 1 needs every batch in the shape of the "
                             "first one (pad the batches to one shape, or train in eager mode)")
        r, ds = self.loss_kw["r"], self.loss_kw["downsample_step"]
        if batch.get("extents") is not None:                      # already padded by the caller: its own bucket
            key = ("padded", self._shape_key(batch))
            shape = None
        else:
            ext = data.batch_extents(batch)
            shape = data.bucket_shape(ext[1], ext[0])
            key = ("bucket", shape, int(batch["x"].shape[0]), "speaker_ids" in batch)
        rec = self._buckets.get(key)
        if rec is None:
            t0 = time.perf_counter()
            if shape is None:
                static = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
            else:
                static = data.pad_to_bucket(batch, shape[0], shape[1], r, ds)
            out = torch.zeros((), device=self.arena.flat.device)   # outside the graph pool: read after the replay
            self._warm_up(static)
            graph = torch.cuda.CUDAGraph()
            n0 = lib.raw("dv3_launch_count")()
            with torch.cuda.graph(graph, pool=self._pool):
                out.copy_(self._forward_backward(static))
                self._exchange_and_update()
            rec = self._buckets[key] = (graph, static, out, int(lib.raw("dv3_launch_count")() - n0))
            torch.cuda.synchronize()
            self.capture_seconds += time.perf_counter() - t0
        graph, static, out, _ = rec
        if shape is None:
            for k, v in batch.items():
                if torch.is_tensor(v):
                    static[k].copy_(v, non_blocking=True)
        else:
            data.pad_to_bucket(batch, shape[0], shape[1], r, ds, out=static)
        graph.replay()
        return out

    def _graph_step(self, batch):
        if self._graph is not None and self._shape_key(batch) != self._graph_key:
            return self._bucket_step(batch)
        if self._graph is None:
            t0 = time.perf_counter()
            self._pool = torch.cuda.graph_pool_handle()
            self._graph_key = self._shape_key(batch)
            # static input buffers; warm up on a side stream, then capture forward+loss+backward (+update when
            # there is no collective to run in between)
            self._static = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
            self._warm_up(self._static)
            self._graph = torch.cuda.CUDAGraph()
            n0 = lib.raw("dv3_launch_count")()
            capture_all = self.world == 1 or self.graph_comm
            with torch.cuda.graph(self._graph, pool=self._pool):
                self._loss = self._forward_backward(self._static)
                if capture_all:                     # NCCL all-reduces are captured as graph nodes on the comm stream
                    self._exchange_and_update()
            self.launches_per_step = int(lib.raw("dv3_launch_count")() - n0) + (0 if capture_all else 2)
            torch.cuda.synchronize()
            self.capture_seconds += time.perf_counter() - t0
        for k, v in batch.items():
            if torch.is_tensor(v):
                self._static[k].copy_(v, non_blocking=True)
        self._graph.replay()
        if self.world > 1 and not self.graph_comm:
            self._exchange_and_update()
        return self._loss


def make_synthetic_batch(B=16, T_text=128, T_mel=800, downsample_step=4, r=1, n_speakers=1, n_vocab=149,
                         mel_dim=80, linear_dim=513, seed=1234, pin=False):
    """Synthetic batch of SURVEY.md section 8(d), on the HOST (what collate_fn would hand to the step)."""
    gen = torch.Generator().manual_seed(seed)
    T_dec = T_mel // downsample_step // r
    b = {
        "x": torch.randint(2, n_vocab, (B, T_text), generator=gen),
        "text_positions": torch.arange(1, T_text + 1)[None, :].repeat(B, 1),
        "frame_positions": torch.arange(1, T_dec + 1)[None, :].repeat(B, 1),
        "mel": torch.rand(B, T_dec, mel_dim * r, generator=gen),
        "y": torch.rand(B, T_mel, linear_dim, generator=gen),
        "done": torch.cat([torch.zeros(B, T_dec - 1, 1), torch.ones(B, 1, 1)], dim=1),
        "target_lengths": torch.full((B,), T_mel, dtype=torch.int64),
        "input_lengths_dev": torch.full((B,), T_text, dtype=torch.int64),
    }
    if n_speakers > 1:
        b["speaker_ids"] = torch.randint(0, n_speakers, (B,), generator=gen)
    if pin:
        b = {k: v.pin_memory() for k, v in b.items()}
    b["input_lengths"] = np.full(B, T_text, dtype=np.int64)
    return b


def to_device(batch, device, non_blocking=True):
    return {k: (v.to(device, non_blocking=non_blocking) if torch.is_tensor(v) else v) for k, v in batch.items()}
