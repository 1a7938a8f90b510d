"""torch.autograd Functions over the dv3b200 C ABI (include/dv3b200.h).

PyTorch is plumbing here: it owns device memory, the current stream and autograd bookkeeping.  All
arithmetic happens in csrc/*.cu.  Every function requires CUDA fp32 tensors and raises otherwise --
there is no CPU fallback.
"""
import collections
import contextlib
import ctypes
import os

import numpy as np
import torch

from ._lib import lib, Dv3Error

MODE_GLU, MODE_HIGHWAY = 0, 1

# Arithmetic of the ConvBlock / conv / attention contractions:
#   "tc"     (default) wgmma tensor cores, every fp32 operand split into a 16-bit (hi, lo) pair, hi*hi + hi*lo + lo*hi
#            with fp32 accumulation in registers (csrc/tc_gemm.cu, tc_attn.cu): fp16 pairs (22-bit operands) in the forward
#            GEMMs, bf16 pairs in the gradient GEMMs.  Full-depth preset models match the fp32 oracle at rtol 1e-3 /
#            atol 1e-4 (tests/test_gpu_models.py).  Shapes the tensor-core kernels do not cover (C % 128 != 0, tiny
#            GEMMs) run on the exact-fp32 kernels automatically.  ("bf16x3" is accepted as an alias.)
#   "tc1"    opt-in single pass (DESIGN.md section 2.7): the conv GEMMs take one 16-bit plane per operand and issue one
#            MMA per K-step with fp32 accumulation -- fp16 operands (TF32-class: 11-bit significands) in the forward GEMMs,
#            bf16 operands (bf16-autocast class) in the data- and weight-gradient GEMMs.  Everything else keeps the "tc"
#            arithmetic: the attention kernels, the exact-fp32 fallback shapes, the losses, the optimizer, the
#            autoregressive step kernels.  Dropout masks are the same bits as in "tc".
#   "fp32"   exact-fp32 CUDA-core kernels everywhere (csrc/conv.cu, bgemm.cu): much slower, the strict reference mode.
# A TrainStep records the mode it was built in: its captured graphs hold that mode's kernels and planes.
conv_math = os.environ.get("DV3_CONV_MATH", "tc")

# Bit-reproducible training (DESIGN.md section 2.10): "0" (default) the training step sums its losses, bias gradients
# and embedding / position-table gradients with float atomics, whose order differs from run to run; "1" every one of
# those sums is formed in an order fixed by the tensor shapes (the dv3_*_det entry points), so the same build, GPU model,
# world size, conv_math, graph / eager setting, seed and batches give the same bits.  The autograd Functions read the
# switch in their forward and keep it for their backward.
deterministic = os.environ.get("DV3_DETERMINISTIC", "0")


def is_deterministic():
    """ops.deterministic as a bool ("0" / "1", or a bool); an unknown value raises."""
    if deterministic in ("0", 0, False):
        return False
    if deterministic in ("1", 1, True):
        return True
    raise Dv3Error("unknown ops.deterministic %r (DV3_DETERMINISTIC is \"0\" or \"1\")" % (deterministic,))


# The module attributes that select how the Functions run (each is described where it is defined below).
_STATE = ("conv_math", "deterministic", "det_scratch", "grad_sink", "weight_bank", "grad_boundary_cb",
          "frozen_weights", "speaker_adapt")


@contextlib.contextmanager
def overrides(**state):
    """Set some of the execution-state attributes (``_STATE``) for the body of a ``with`` block and restore each to
    the value it had on entry, on exit or exception.  An unknown name raises ValueError before anything is set."""
    unknown = sorted(set(state) - set(_STATE))
    if unknown:
        raise ValueError("ops.overrides: unknown execution state %s (one of %s)" % (unknown, ", ".join(_STATE)))
    scope = globals()
    outer = {k: scope[k] for k in state}
    scope.update(state)
    try:
        yield
    finally:
        scope.update(outer)


# ----------------------------------------------------------------------------------------------
# plumbing
# ----------------------------------------------------------------------------------------------
def _chk(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise Dv3Error("dv3b200 ops need CUDA tensors (got %s); there is no CPU path" % t.device)
        if t.dtype != torch.float32:
            raise Dv3Error("dv3b200 ops are fp32 (got %s)" % t.dtype)
        if not t.is_contiguous():
            raise Dv3Error("dv3b200 ops need contiguous tensors")


def _p(t, offset=0):
    """Device address of t's data, ``offset`` fp32 elements in (None for None)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr() + 4 * offset)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device_i32(x, dev):
    """An integer array, sequence or tensor as a contiguous int32 tensor on ``dev``."""
    if torch.is_tensor(x):
        return x.to(dev, torch.int32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(x, np.int32)).to(dev)


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


class DropoutState:
    """Step seed in device memory + call-site salts.

    keep(i) = f(seed[0], salt, i).  ``base`` is a persistent int64[1] device tensor that is bumped IN PLACE at the
    start of every training forward (a device-side add, so a captured CUDA graph gets fresh masks on every replay);
    ``seed`` is the snapshot of it that the kernels of the current forward -- and of its backward, through the
    autograd contexts, which hold the tensor -- read.  Salts are handed out in call order and restart with every
    outermost forward (``begin_forward``), so a replayed graph sees the same sequence."""

    GOLD = 0x9E3779B97F4A7C15 & 0x7FFFFFFFFFFFFFFF

    def __init__(self):
        self.base = None
        self.seed = None
        self.salt = 0
        self.depth = 0

    def _init(self, s, device):
        self.base = torch.tensor([int(s) & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=device)
        self.seed = self.base.clone()

    def seed_tensor(self, device):
        if self.seed is None or self.seed.device != device:
            s = torch.initial_seed()
            if torch.distributed.is_available() and torch.distributed.is_initialized():
                s += 0x632BE59BD9B4E019 * torch.distributed.get_rank()      # different masks on every replica
            self._init(s, device)
        return self.seed

    def manual_seed(self, s, device):
        self._init(s, device)

    def next_salt(self):
        self.salt += 1
        return self.salt

    def start_forward(self):
        self.salt = 0

    def advance(self):
        """New masks from here on: bump the persistent seed in place, snapshot it for the coming forward."""
        if self.base is not None:
            self.base.add_(self.GOLD)
            self.seed = self.base.clone()

    # -- called by the model containers around their forward ------------------------------------------------
    def begin_forward(self, training, device):
        """Outermost forward of a model (or of model.seq2seq / model.postnet called on their own, reference
        train.py:691-700): restart the salts and, in training, draw a new step seed."""
        self.depth += 1
        if self.depth == 1:
            self.salt = 0
            if training and device.type == "cuda":
                self.seed_tensor(device)
                self.advance()

    def end_forward(self):
        self.depth -= 1


rng = DropoutState()


class DetScratch:
    """Device scratch of the deterministic kernels: the partial-sum rows of the bias gradients (reused by every layer --
    a layer's reduction is ordered before the next layer's partials on the stream) and the block partials + ticket of
    the loss kernels.  Buffers grow on demand but never during a CUDA-graph capture: a captured launch keeps the address
    it was given, so a TrainStep sizes its scratch in the eager warm-up passes that precede every capture, and outgrown
    buffers stay alive for the graphs that hold them."""

    def __init__(self):
        self._bias = {}       # device -> list of buffers, the last one current
        self._loss = {}

    @staticmethod
    def _growable(what):
        if torch.cuda.is_current_stream_capturing():
            raise Dv3Error("deterministic mode: %s scratch must exist before a CUDA-graph capture (run the step "
                           "eagerly once, as TrainStep's warm-up does)" % what)

    def bias(self, floats, device):
        bufs = self._bias.setdefault(device, [])
        if not bufs or bufs[-1].numel() < floats:
            self._growable("bias-gradient")
            bufs.append(torch.empty(max(int(floats), 1 << 18), device=device, dtype=torch.float32))
        return bufs[-1]

    def loss(self, device):
        if device not in self._loss:
            self._growable("loss")
            self._loss[device] = torch.zeros(lib.raw("dv3_loss_det_scratch_floats")(), device=device)
        return self._loss[device]


# the scratch of Functions called outside a TrainStep; a TrainStep installs its own around its passes
det_scratch = DetScratch()


def _bias_scratch(B, nch, T, tiled, device):
    """-> (pointer, floats) of the partial rows a deterministic bias-gradient call needs."""
    lib.load()
    fn = lib.raw("dv3_bias_det_scratch_floats")
    buf = det_scratch.bias(fn(B, nch, T, int(tiled)), device)
    return _p(buf), buf.numel()


def forward_scope(fn):
    """Decorator for the ``forward`` of a module the reference's train.py may call on its own (model.postnet,
    train.py:700): draws the dropout seed / restarts the salts when it is the outermost forward."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, x, *a, **kw):
        rng.begin_forward(self.training, x.device)
        try:
            return fn(self, x, *a, **kw)
        finally:
            rng.end_forward()
    return wrapped


def _drop_args(p, training, device):
    """-> (p_eff, seed tensor | None, salt) ; consumes a salt only when dropout is live."""
    if training and p > 0.0:
        return float(p), rng.seed_tensor(device), rng.next_salt()
    return 0.0, None, 0


# ----------------------------------------------------------------------------------------------
# weight-norm packing helpers
# ----------------------------------------------------------------------------------------------
# How the plain conv Functions run a weight-normed layer.  A ConvTranspose1d(k=2, s=2) is a 1x1 conv with 2*Cout
# output rows ordered (j, co) followed by a time interleave (conv_transpose1d_k2s2); all it changes is this record:
#   dims(v) -> (M, N, k)     output rows, input channels and taps of the layer's GEMM
#   fp32, tc                 the weight-norm fold kinds (_FOLDS) of the exact-fp32 and the tensor-core path
#   wgrad(M, N, k, tc) -> (msplit, s_m, s_mh, s_n, s_j, tap_major_k): where the weight-gradient GEMM writes element
#                            (m, n, j) of a partial (include/dv3b200.h), and how _wn_bwd reads the partials back
#   bias(b), dbias(db)       the GEMM's bias rows from the layer's bias, and the layer's bias gradient from theirs
#   banked                   the WeightBank and the gradient sink may take the layer: both assume a (Cout, Cin, k) v
#                            and one bias row per GEMM row
_Layout = collections.namedtuple("_Layout", "dims fp32 tc wgrad bias dbias banked")
# v (Cout, Cin, k); the tensor-core partials are tap-major [j][M][N]: contiguous float4 stores from the GEMM epilogue
_CONV = _Layout(lambda v: tuple(v.shape), "fp32", "tc",
                lambda M, N, k, tc: (M, N, 0, 1, M * N, k) if tc else (M, N * k, 0, k, 1, 0),
                lambda b: b, lambda db: db, True)
# v (Cin, Cout, 2) normalised over Cin; GEMM element (m = (j, co), ci) is v[ci, co, j] on both paths
_CONVT = _Layout(lambda v: (v.shape[2] * v.shape[1], v.shape[0], 1), "convt_fp32", "convt_tc",
                 lambda M, N, k, tc: (M // 2, 2, 1, M, 0, 0),
                 lambda b: b.repeat(2), lambda db: db if db is None else db[:db.numel() // 2] + db[db.numel() // 2:],
                 False)
_CONVT_S = {}


def _convt_layout(s):
    """The _CONVT record of a ConvTranspose1d(k = s, stride = s), v (Cin, Cout, s): s*Cout GEMM rows ordered (j, co);
    the bias gradient adds the s row blocks in j order."""
    if s == 2:
        return _CONVT
    if s not in _CONVT_S:
        def dbias(db):
            if db is None:
                return db
            parts = db.view(s, -1)
            out = parts[0].clone()
            for j in range(1, s):
                out += parts[j]
            return out
        _CONVT_S[s] = _Layout(_CONVT.dims, "convt_fp32", "convt_s_tc", lambda M, N, k, tc: (M // s, s, 1, M, 0, 0),
                              lambda b: b.repeat(s), dbias, False)
    return _CONVT_S[s]


def _wn_buffers(lay, v, npl):
    """Outputs of a layer's weight-norm fold, for its GEMM (M, N, k) = lay.dims(v): (w_f [k][N][M], w_b [k][M][N],
    inv, scale) fp32 on the exact-fp32 path (npl = 0); (inv, wfwd [npl][k][M][pad8(N)] fp16 planes of the forward
    GEMM, wbwd [npl][k][N][pad8(M)] bf16 planes of the data gradient, scale) on the tensor-core path.  inv and scale
    have one entry per normalised row of v."""
    M, N, k = lay.dims(v)
    dev = v.device
    inv = torch.empty(v.shape[0], device=dev)
    if npl == 0:
        return torch.empty(k, N, M, device=dev), torch.empty(k, M, N, device=dev), inv, torch.empty_like(inv)
    return (inv, torch.empty(npl, k, M, _pad8(N), device=dev, dtype=torch.float16),
            torch.empty(npl, k, N, _pad8(M), device=dev, dtype=torch.bfloat16), torch.empty_like(inv))


def _fold_fp32(v, g, npl, out):
    w_f, w_b, inv, scale = out
    Cout, Cin, k = v.shape
    lib.call("dv3_weightnorm_fwd", _p(v), _p(g), _p(inv), _p(scale), _p(w_f), _p(w_b), Cout, Cin, k,
             1, Cout, Cin * Cout, Cin, 1, Cout * Cin, _stream())


def _fold_convt_fp32(v, g, npl, out):
    w_f, w_b, inv, scale = out
    Cin, Cout, s = v.shape
    lib.call("dv3_weightnorm_fwd", _p(v), _p(g), _p(inv), _p(scale), _p(w_f), _p(w_b), Cin, Cout, s,
             s * Cout, 1, Cout, 1, Cin, Cout * Cin, _stream())


def _fold_tc(v, g, npl, out):
    inv, wfwd, wbwd, scale = out
    Cout, Cin, k = v.shape
    lib.call("dv3_tc_weightnorm_fwd", _p(v), _p(g), _p(inv), _p(scale), _p(wfwd), npl, _p(wbwd), Cout, Cin, k,
             _stream())


def _fold_convt_tc(v, g, npl, out):
    inv, wfwd, wbwd, scale = out
    lib.call("dv3_tc_weightnorm_convt_fwd", _p(v), _p(g), _p(inv), _p(scale), _p(wfwd), npl, _p(wbwd), v.shape[0],
             v.shape[1], _stream())


def _fold_convt_s_tc(v, g, npl, out):
    inv, wfwd, wbwd, scale = out
    lib.call("dv3_tc_weightnorm_convt_s_fwd", _p(v), _p(g), _p(inv), _p(scale), _p(wfwd), npl, _p(wbwd), v.shape[0],
             v.shape[1], v.shape[2], _stream())


_FOLDS = {"fp32": (_CONV, _fold_fp32), "tc": (_CONV, _fold_tc),
          "convt_fp32": (_CONVT, _fold_convt_fp32), "convt_tc": (_CONVT, _fold_convt_tc),
          "convt_s_tc": (_CONVT, _fold_convt_s_tc)}


def _fold(kind, v, g, npl=0, out=None):
    """Weight norm of a layer by fold kind (_FOLDS) on the current stream into ``out`` (new buffers of _wn_buffers when
    None) -> out."""
    lay, fold = _FOLDS[kind]
    out = out or _wn_buffers(lay, v, npl)
    fold(v, g, npl, out)
    return out


def _fp32_weights(v, g, lay):
    """-> (w_f, w_b, inv) of the exact-fp32 weight norm, from the frozen-weight cache when it holds the layer."""
    return (_frozen(lay.fp32, v, g) or _fold(lay.fp32, v, g))[:3]


class FrozenWeights:
    """Weight norm and operand planes of layers whose parameters take no gradient, folded once and reused by every
    pass (installed as ``ops.frozen_weights`` by an embedding-only ``TrainStep(adapt_speakers=...)``).  A layer is
    folded the first time a Function sees it -- in an eager pass, never inside a CUDA-graph capture -- into persistent
    buffers; ``refresh()`` refolds every layer in place (the buffers keep their addresses, so captured graphs stay
    valid), and ``stale()`` tells from the parameters' version counters whether one was written since its fold."""

    def __init__(self):
        self.entries = {}           # (kind, v.data_ptr(), v.shape, npl) -> [v, g, npl, buffers, versions]

    def get(self, kind, v, g, npl=0):
        key = (kind, v.data_ptr(), tuple(v.shape), npl)
        e = self.entries.get(key)
        if e is None:
            if torch.cuda.is_current_stream_capturing():
                raise Dv3Error("frozen weights: layer %s first seen during a CUDA-graph capture (warm up first)"
                               % (tuple(v.shape),))
            e = self.entries[key] = [kind, v, g, npl, _fold(kind, v, g, npl), (v._version, g._version)]
        return e[4]

    def stale(self):
        return any((v._version, g._version) != ver for _, v, g, _, _, ver in self.entries.values())

    def refresh(self):
        for e in self.entries.values():
            kind, v, g, npl, bufs, _ = e
            _fold(kind, v, g, npl, bufs)
            e[5] = (v._version, g._version)


frozen_weights = None


def _frozen(kind, v, g, npl=0):
    """Cached fold of a frozen layer (``frozen_weights`` installed and neither parameter takes a gradient), or None."""
    if frozen_weights is None or v.requires_grad or g.requires_grad:
        return None
    return frozen_weights.get(kind, v, g, npl)


# Gradient sink (set by train_step.TrainStep): parameter gradients are accumulated by the kernels straight into the
# pre-allocated ``.grad`` views of the flat gradient arena and the autograd Functions return None for them, which
# removes one ``grad += new`` elementwise kernel per parameter per step (~130 launches).  Off by default: plain
# autograd semantics (Functions return dv, dg, dbias).
grad_sink = False


# Gradient-bucket boundaries (set by train_step.TrainStep in data-parallel runs): ``grad_boundary(x, tag)`` marks a tensor
# whose gradient, once computed, proves that every parameter gradient of the layers AFTER it is final -- the training
# step then starts the NCCL all-reduce of that parameter bucket while the rest of the backward pass still runs.
grad_boundary_cb = None


def grad_boundary(x, tag):
    if grad_boundary_cb is not None and x.requires_grad:
        cb = grad_boundary_cb

        def _hook(grad, tag=tag, cb=cb):
            cb(tag)
            return None
        x.register_hook(_hook)
    return x


# Batched weight norm (weight_bank.WeightBank), installed by train_step.TrainStep for the duration of one
# forward/backward: operand planes of every layer are prepared up front, the weight-norm backward is deferred to one
# launch after loss.backward().  None: every Function normalises / reduces its own layer.
weight_bank = None


def _sink(*params):
    """The .grad buffers to accumulate into, or None when the sink is off / a parameter is not a leaf (e.g. the views
    ``linear`` passes) / not every buffer exists."""
    if not grad_sink or any(not p.is_leaf or p.grad is None or not p.grad.is_contiguous() for p in params):
        return None
    return [p.grad for p in params]


def _wn_bwd(partials, nsplit, v, g, inv, tap_major_k=0, out=None, accumulate=False):
    """tap_major_k = 0: partials in v's layout; = k (> 0): partials as [j][R][X] (tensor-core weight gradient)."""
    dv, dg = out if out is not None else (torch.empty_like(v), torch.empty_like(g))
    R, k = v.shape[0], tap_major_k or 1
    lib.call("dv3_weightnorm_bwd", _p(partials), v.numel(), nsplit, int(tap_major_k > 0), _p(v), _p(g), _p(inv),
             _p(dv), _p(dg), R, v.numel() // R // k, k, int(accumulate), _stream())
    return dv, dg


def _wgrad_conv(dab, x, k, dilation, causal, p, seed_ptr, salt, lay):
    """Exact-fp32 weight gradient -> partials [nsplit][M*Cin*k] in v's layout (lay.wgrad)."""
    B, M, T = dab.shape
    Cin = x.shape[1]
    nsplit = lib.raw("dv3_conv1d_wgrad_nsplit")(B, M, Cin, T, k)
    numel = M * Cin * k
    partials = torch.empty(nsplit, numel, device=x.device, dtype=torch.float32)
    lib.call("dv3_conv1d_wgrad", _p(dab), _p(x), _p(partials), numel, B, M, Cin, T, k, dilation,
             int(causal), p, seed_ptr, salt, *lay.wgrad(M, Cin, k, False)[:5], _stream())
    return partials, nsplit


# ----------------------------------------------------------------------------------------------
# fused ConvBlock (Conv1dGLU / HighwayConv1d)
# ----------------------------------------------------------------------------------------------
def _gate_addend(mode, residual, dy, s):
    """(addmode, e1, e2, alpha) of a gated block's data-gradient GEMM: the gradient that reaches x around the conv --
    sqrt(0.5) * dy through the GLU residual, dy * (1 - s) through the highway carry gate, nothing for a plain GLU."""
    if mode == MODE_GLU:
        return (1, dy, None, 0.7071067811865476) if residual else (0, None, None, 0.0)
    return 2, dy, s, 0.0


class _ConvBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, v, g, bias, spk, k, dilation, causal, mode, residual, p_drop, training, site, anchor):
        _chk(x, v, g, bias, spk)
        B, C, T = x.shape
        assert v.shape == (2 * C, C, k), "ConvBlock needs in_channels == out_channels"
        w_f, w_b, inv = _fp32_weights(v, g, _CONV)
        p, seed_t, salt = _drop_args(p_drop, training, x.device)
        seed_ptr = _p(seed_t)
        need_bwd = any(ctx.needs_input_grad)
        y = torch.empty_like(x)
        a = torch.empty_like(x) if need_bwd else None
        s = torch.empty_like(x) if need_bwd else None
        lib.call("dv3_convblock_fwd", _p(x), _p(w_f), _p(bias), _p(spk), _p(y), _p(a), _p(s), B, C, T, k,
                 dilation, int(causal), mode, int(residual), p, seed_ptr, salt, _stream())
        if need_bwd:
            ctx.save_for_backward(x, v, g, a, s, w_b, inv)
            ctx.cfg = (k, dilation, causal, mode, residual, p, salt, spk is not None, x.device)
            ctx.seed_t = seed_t
            ctx.det = is_deterministic()
            ctx.site = site
        return y

    @staticmethod
    def backward(ctx, dy):
        x, v, g, a, s, w_b, inv = ctx.saved_tensors
        k, dilation, causal, mode, residual, p, salt, has_spk, dev = ctx.cfg
        seed_ptr = _p(ctx.seed_t)          # the forward's own seed snapshot
        dy = _c(dy)
        B, C, T = x.shape
        dab = torch.empty(B, 2 * C, T, device=dev, dtype=torch.float32)
        dbias = torch.zeros(2 * C, device=dev, dtype=torch.float32)
        if ctx.det:
            lib.call("dv3_convblock_gate_bwd_det", _p(dy), _p(a), _p(s), _p(x), _p(dab), _p(dbias),
                     *_bias_scratch(B, 2 * C, T, False, dev), B, C, T, mode, int(residual), _stream())
        else:
            lib.call("dv3_convblock_gate_bwd", _p(dy), _p(a), _p(s), _p(x), _p(dab), _p(dbias), B, C, T, mode,
                     int(residual), _stream())
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            addmode, e1, e2, alpha = _gate_addend(mode, residual, dy, s)
            lib.call("dv3_conv1d_dgrad", _p(dab), _p(w_b), _p(dx), B, 2 * C, C, T, k, dilation,
                     int(causal), p, seed_ptr, salt, addmode, _p(e1), _p(e2), alpha, _stream())
        dv = dg = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            partials, nsplit = _wgrad_conv(dab, x, k, dilation, causal, p, seed_ptr, salt, _CONV)
            dv, dg = _wn_bwd(partials, nsplit, v, g, inv)
        dspk = dab[:, :C, :] if has_spk and ctx.needs_input_grad[4] else None
        if ctx.site is not None:            # speaker adaptation: d_e from the "a" half of the gate gradient
            ctx.site.grad_bct(dab, 2 * C * T)
        return dx, dv, dg, dbias, dspk, None, None, None, None, None, None, None, None, None


# The weight-gradient GEMM (+ the weight-norm backward that consumes it) and the data-gradient GEMM of a block are
# independent: run the former on a side stream so the two overlap -- most layers launch only 32-128 CTAs on 132 SMs.
# Fork/join with stream waits, which a CUDA-graph capture records as graph edges.
_side_streams = {}


class _SideStream:
    """with _SideStream(dev): ...   work inside is ordered after everything already on the current stream; the
    current stream waits for it at join()."""

    def __init__(self, dev):
        if dev not in _side_streams:
            _side_streams[dev] = torch.cuda.Stream(device=dev)
        self.side = _side_streams[dev]
        self.main = torch.cuda.current_stream(dev)
        self.ctx = torch.cuda.stream(self.side)

    def __enter__(self):
        self.side.wait_stream(self.main)
        self.ctx.__enter__()
        return self

    def __exit__(self, *a):
        self.ctx.__exit__(*a)

    def join(self):
        self.main.wait_stream(self.side)


def _pad8(n):
    return (n + 7) // 8 * 8


def _tc_weights(v, g, npl, lay):
    """Tensor-core weight operands of a layer -> (inv, wfwd, wbwd, bank record or None, side or None), as _wn_buffers
    lays them out.  Without a weight-bank record the per-layer weight norm is started on the side stream -- it depends
    only on the parameters, so it overlaps the caller's activation split; the caller joins ``side`` before its GEMM.
    Only a banked layout asks the bank: it registers every layer it is asked about as a (Cout, Cin, k) conv."""
    bank = weight_bank.weights_for(v, g, npl) if weight_bank is not None and lay.banked else None
    if bank is not None:                                                              # planes prepared for this step
        return bank.inv, bank.wfwd, bank.wbwd, bank, None
    fz = _frozen(lay.tc, v, g, npl)
    if fz is not None:
        return fz[0], fz[1], fz[2], None, None
    out = _wn_buffers(lay, v, npl)    # allocated on the main stream, written on the side stream
    side = _SideStream(v.device)
    side.keep = out[3]                # the scale, written and read on the side stream: must outlive the caller's join
    with side:
        _fold(lay.tc, v, g, npl, out)
    return out[0], out[1], out[2], None, side


class _TCWeightGrad:
    """Weight and bias gradients of a weight-normed tensor-core layer whose GEMM is (M, N, k) = lay.dims(v), bias rows
    [M]: ``dbias`` is where the gradient split sums the bias gradient; start() runs the weight-gradient GEMM and the
    weight-norm backward on the side stream, finish() joins it after the data gradient.  With the gradient sink (a
    banked layout) they are accumulated into .grad (a weight-bank layer's reduction deferred to
    WeightBank.end_backward()) and finish() returns None for them."""

    def __init__(self, ctx, v, g, lay):
        self.ctx, self.v, self.g, self.lay = ctx, v, g, lay
        self.sink = _sink(v, g, ctx.bias_param) if ctx.bias_param is not None and lay.banked else None
        self.dbias = self.sink[2] if self.sink else torch.zeros(lay.dims(v)[0], device=v.device) \
            if ctx.needs_input_grad[3] else None          # a frozen bias: no bias gradient at all
        self.side = self.dv = self.dg = self.partials = None

    def start(self, d_planes, x_wg, inv, B, T, dilation, causal, npl):
        ctx, v, g, sink = self.ctx, self.v, self.g, self.sink
        if not (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            return
        M, N, k = self.lay.dims(v)
        nsplit = lib.raw("dv3_tc_wgrad_nsplit")(B, M, N, T, k)
        msplit, s_m, s_mh, s_n, s_j, tap_major_k = self.lay.wgrad(M, N, k, True)
        numel = v.numel()
        # allocated on the main stream (and held until finish()), computed on the side stream
        partials = weight_bank.partials_for(ctx.bank, nsplit, numel) if (sink and ctx.bank is not None) else None
        deferred = partials is not None
        if not deferred:
            partials = torch.empty(nsplit, numel, device=v.device)
        self.partials = partials
        self.dv, self.dg = (sink[0], sink[1]) if sink else (torch.empty_like(v), torch.empty_like(g))
        self.side = _SideStream(v.device)
        with self.side:
            lib.call("dv3_tc_wgrad_mn_npl", _p(d_planes), _p(x_wg), npl, _p(partials), numel, B, M, N, T, k,
                     dilation, int(causal), msplit, s_m, s_mh, s_n, s_j, _stream())
            if not deferred:
                _wn_bwd(partials, nsplit, v, g, inv, tap_major_k=tap_major_k, out=(self.dv, self.dg),
                        accumulate=bool(sink))

    def finish(self):
        if self.side is not None:
            self.side.join()
        if self.sink:                 # already accumulated into the .grad arena views
            return None, None, None
        return self.dv, self.dg, self.lay.dbias(self.dbias)


class _ConvBlockTCFn(torch.autograd.Function):
    """Same contract as _ConvBlockFn on the tensor-core path: operands are 16-bit planes, npl per operand (fp16 in the
    forward GEMM, bf16 in the gradient GEMMs)."""

    @staticmethod
    def forward(ctx, x, v, g, bias, spk, k, dilation, causal, mode, residual, p_drop, training, extent, site, anchor):
        _chk(x, v, g, bias, spk)
        B, C, T = x.shape
        dev = x.device
        bf = torch.bfloat16
        npl = _npl()
        need_bwd = any(ctx.needs_input_grad)
        need_w = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        p, seed_t, salt = _drop_args(p_drop, training, dev)
        inv, wfwd, wbwd, bank, side = _tc_weights(v, g, npl, _CONV)
        x_btc = torch.empty(npl, B, T, C, device=dev, dtype=torch.float16)        # forward operand (fp16)
        x_wg = torch.empty(npl, B, T, C, device=dev, dtype=bf) if need_w else None  # weight-gradient operand
        seed_ptr = _p(seed_t)
        y = torch.empty_like(x)
        a = torch.empty_like(x) if need_bwd else None
        s = torch.empty_like(x) if need_bwd else None
        ext_p, ext_m = extent if extent is not None and k > 1 else (None, 1)   # frames past it enter the conv as 0
        lib.call("dv3_tc_split_input_ext", _p(x), _p(x_btc), npl, _p(x_wg), B, C, T, p, seed_ptr, salt, ext_p, ext_m,
                 _stream())
        if side is not None:
            side.join()
        lib.call("dv3_tc_convblock_fwd", _p(x_btc), _p(wfwd), npl, _p(bias), _p(spk), _p(x), _p(y), _p(a), _p(s),
                 B, C, T, k, dilation, int(causal), mode, int(residual), None, _stream())
        if need_bwd:
            ctx.save_for_backward(x, v, g, a, s, x_wg, wbwd, inv)
            ctx.cfg = (k, dilation, causal, mode, residual, p, salt, spk is not None, dev)
            ctx.seed_t = seed_t
            ctx.bias_param = bias if bias.is_leaf else None
            ctx.bank = bank
            ctx.extent = extent
            ctx.npl = npl
            ctx.det = is_deterministic()
            ctx.site = site
        return y

    @staticmethod
    def backward(ctx, dy):
        x, v, g, a, s, x_wg, wbwd, inv = ctx.saved_tensors
        npl = ctx.npl                       # the forward's plane count, whatever ops.conv_math says now
        k, dilation, causal, mode, residual, p, salt, has_spk, dev = ctx.cfg
        seed_ptr = _p(ctx.seed_t)          # the forward's own seed snapshot
        dy = _c(dy)
        B, C, T = x.shape
        d_btc = torch.empty(npl, B, T, 2 * C, device=dev, dtype=torch.bfloat16)
        wg = _TCWeightGrad(ctx, v, g, _CONV)
        # the gradient past the extent is taken as 0 (see ops.extent_frames)
        ext_p, ext_m = ctx.extent if ctx.extent is not None else (None, 1)
        if ctx.det and wg.dbias is not None:
            lib.call("dv3_tc_gate_bwd_split_det", _p(dy), _p(a), _p(s), _p(x), _p(d_btc), npl, _p(wg.dbias),
                     *_bias_scratch(B, 2 * C, T, True, dev), B, C, T, mode, int(residual), ext_p, ext_m, _stream())
        else:
            lib.call("dv3_tc_gate_bwd_split_npl", _p(dy), _p(a), _p(s), _p(x), _p(d_btc), npl, None, _p(wg.dbias), B,
                     C, T, mode, int(residual), ext_p, ext_m, _stream())
        wg.start(d_btc, x_wg, inv, B, T, dilation, causal, npl)
        if ctx.site is not None:            # speaker adaptation: d_e straight from the "a" half of the planes
            ctx.site.grad_planes(d_btc, npl)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            addmode, e1, e2, alpha = _gate_addend(mode, residual, dy, s)
            lib.call("dv3_tc_conv", _p(d_btc), _p(wbwd), npl, _p(dx), B, 2 * C, C, T, k, dilation, int(causal), 1,
                     None, 0, p, seed_ptr, salt, addmode, _p(e1), _p(e2), alpha, None, _stream())
        dv, dg, dbias = wg.finish()
        dspk = None
        if has_spk and ctx.needs_input_grad[4]:     # d_a = hi (+ lo * 2^-11) of the (B,T,2C) planes, back to (B,C,T)
            da = d_btc[0, :, :, :C].float()
            if npl == 2:
                da = da + d_btc[1, :, :, :C].float() * (1.0 / 2048.0)
            dspk = transpose12(da.contiguous())
        return (dx, dv, dg, dbias, dspk) + (None,) * 10


class _Conv1dTCFn(torch.autograd.Function):
    """Plain weight-normed conv (+ReLU) on the tensor-core path (1x1 convs, projections, and in the _CONVT layout the
    ConvTranspose upsamplers)."""

    @staticmethod
    def forward(ctx, x, v, g, bias, k, dilation, causal, relu, extent, lay):
        _chk(x, v, g, bias)
        B, Cin, T = x.shape
        Cout = lay.dims(v)[0]
        dev, bf = x.device, torch.bfloat16
        need_bwd = any(ctx.needs_input_grad)
        Cinp = _pad8(Cin)
        npl = _npl()
        inv, wfwd, wbwd, bank, side = _tc_weights(v, g, npl, lay)
        need_w = need_bwd and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2])
        x_btc = torch.empty(npl, B, T, Cinp, device=dev, dtype=torch.float16)
        x_wg = torch.empty(npl, B, T, Cinp, device=dev, dtype=bf) if need_w else None
        y = torch.empty(B, Cout, T, device=dev)
        ext_p, ext_m = extent if extent is not None and k > 1 else (None, 1)
        lib.call("dv3_tc_split_input_ext", _p(x), _p(x_btc), npl, _p(x_wg), B, Cin, T, 0.0, None, 0, ext_p, ext_m,
                 _stream())
        if side is not None:
            side.join()
        lib.call("dv3_tc_conv", _p(x_btc), _p(wfwd), npl, _p(y), B, Cin, Cout, T, k, dilation, int(causal), 0,
                 _p(lay.bias(bias)), int(relu), 0.0, None, 0, 0, None, None, 0.0, None, _stream())
        if need_bwd:
            ctx.save_for_backward(v, g, x_wg, wbwd, inv, y if relu else None)
            ctx.cfg = (B, Cin, Cout, T, k, dilation, causal, relu, lay)
            ctx.bias_param = bias if bias.is_leaf else None
            ctx.bank = bank
            ctx.extent = extent
            ctx.npl = npl
            ctx.det = is_deterministic()
        return y

    @staticmethod
    def backward(ctx, dy):
        v, g, x_wg, wbwd, inv, y = ctx.saved_tensors
        B, Cin, Cout, T, k, dilation, causal, relu, lay = ctx.cfg
        npl = ctx.npl
        dy = _c(dy)
        dev = dy.device
        g_btc = torch.empty(npl, B, T, _pad8(Cout), device=dev, dtype=torch.bfloat16)
        wg = _TCWeightGrad(ctx, v, g, lay)
        ext_p, ext_m = ctx.extent if ctx.extent is not None else (None, 1)
        if ctx.det and wg.dbias is not None:
            lib.call("dv3_tc_grad_split_det", _p(dy), _p(y), _p(g_btc), npl, _p(wg.dbias),
                     *_bias_scratch(B, Cout, T, True, dev), B, Cout, T, int(relu), ext_p, ext_m, _stream())
        else:
            lib.call("dv3_tc_grad_split_npl", _p(dy), _p(y), _p(g_btc), npl, None, _p(wg.dbias), B, Cout, T,
                     int(relu), ext_p, ext_m, _stream())
        wg.start(g_btc, x_wg, inv, B, T, dilation, causal, npl)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(B, Cin, T, device=dev)
            lib.call("dv3_tc_conv", _p(g_btc), _p(wbwd), npl, _p(dx), B, Cout, Cin, T, k, dilation, int(causal), 1, None,
                     0, 0.0, None, 0, 0, None, None, 0.0, None, _stream())
        dv, dg, dbias = wg.finish()
        return (dx, dv, dg, dbias) + (None,) * 6


def math_mode():
    """conv_math normalised: "tc" (also for its alias "bf16x3"), "tc1" or "fp32"; an unknown value raises."""
    if conv_math in ("tc", "bf16x3"):
        return "tc"
    if conv_math not in ("tc1", "fp32"):
        raise Dv3Error("unknown conv_math %r" % (conv_math,))
    return conv_math


def _tc_selected():
    """Whether conv_math selects the tensor-core kernels; an unknown value raises."""
    return math_mode() != "fp32"


def _npl():
    """16-bit operand planes of the tensor-core conv GEMMs in the current mode: 1 single pass ("tc1"), 2 hi / lo pairs."""
    return 1 if math_mode() == "tc1" else 2


# 16 keeps the 16-wide speaker projections of the multi-speaker model on tensor cores (measured: vctk step 11.8 -> 10.6 ms)
TC_MIN_CHANNELS = int(os.environ.get("DV3_TC_MIN_CHANNELS", "16"))


def _use_tc_conv(x, Cin, Cout, k):
    """Tensor cores for plain convs when the mode asks for it, the shape is supported and the GEMM is big enough to
    amortise the operand-split passes."""
    if not _tc_selected() or not x.is_cuda:
        return False
    B, _, T = x.shape
    if not lib.raw("dv3_tc_conv_supported")(B, Cin, Cout, T, int(k)):
        return False
    if k > 1 and Cin % 128 != 0:          # the data gradient swaps the roles of Cin / Cout
        return False
    return min(Cin, Cout) >= TC_MIN_CHANNELS and B * T >= 512


def tc_supported(B, C, T, k):
    return bool(lib.raw("dv3_tc_supported")(B, C, T, k))


def convblock(x, v, g, bias, spk=None, k=3, dilation=1, causal=False, mode=MODE_GLU, residual=True,
              p_drop=0.0, training=False, extent=None, site=None):
    """Fused weight-normed dilated conv + gate.  x (B,C,T); v (2C,C,k); g (2C,1,1); bias (2C);
    spk (B,C,T) already softsign'ed (or None).  extent (``extent_frames``): frames past it are taken as 0 in the conv
    input (k > 1) and in the incoming gradient.  site: a speaker-adaptation site (speaker_adapt.Site) whose embedding
    gradient the backward adds from the block's gate gradient; spk then takes no gradient of its own."""
    if causal:
        extent = None
    anchor = None if site is None else site.anchor
    if _tc_selected() and x.is_cuda and tc_supported(x.shape[0], x.shape[1], x.shape[2], int(k)):
        return _ConvBlockTCFn.apply(_c(x), v, g, bias, None if spk is None else _c(spk), int(k), int(dilation),
                                    bool(causal), int(mode), bool(residual), float(p_drop), bool(training), extent,
                                    site, anchor)
    x = _fp32_extent_in(_c(x), k, extent)
    y = _ConvBlockFn.apply(x, v, g, bias, None if spk is None else _c(spk), int(k), int(dilation),
                           bool(causal), int(mode), bool(residual), float(p_drop), bool(training), site, anchor)
    return extent_grad_mask(y, extent)


# ----------------------------------------------------------------------------------------------
# plain weight-normed Conv1d (+ReLU)
# ----------------------------------------------------------------------------------------------
class _Conv1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, v, g, bias, k, dilation, causal, relu, lay):
        _chk(x, v, g, bias)
        B, Cin, T = x.shape
        Cout, N, kv = lay.dims(v)
        assert (N, kv) == (Cin, k)
        w_f, w_b, inv = _fp32_weights(v, g, lay)
        y = torch.empty(B, Cout, T, device=x.device, dtype=torch.float32)
        lib.call("dv3_conv1d_fwd", _p(x), _p(w_f), _p(lay.bias(bias)), _p(y), B, Cin, Cout, T, k, dilation,
                 int(causal), int(relu), _stream())
        if any(ctx.needs_input_grad):
            ctx.save_for_backward(x, v, g, w_b, inv, y if relu else None)
            ctx.cfg = (k, dilation, causal, relu, lay)
            ctx.det = is_deterministic()
        return y

    @staticmethod
    def backward(ctx, dy):
        x, v, g, w_b, inv, y = ctx.saved_tensors
        k, dilation, causal, relu, lay = ctx.cfg
        dy = _c(dy)
        B, Cout, T = dy.shape
        Cin = x.shape[1]
        dbias = torch.zeros(Cout, device=x.device, dtype=torch.float32)
        dyr = torch.empty_like(dy) if relu else dy
        if ctx.det:
            lib.call("dv3_bias_act_bwd_det", _p(dy), _p(y), _p(dyr), _p(dbias),
                     *_bias_scratch(B, Cout, T, False, x.device), B, Cout, T, int(relu), _stream())
        else:
            lib.call("dv3_bias_act_bwd", _p(dy), _p(y), _p(dyr), _p(dbias), B, Cout, T, int(relu), _stream())
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            lib.call("dv3_conv1d_dgrad", _p(dyr), _p(w_b), _p(dx), B, Cout, Cin, T, k, dilation, int(causal),
                     0.0, None, 0, 0, None, None, 0.0, _stream())
        dv = dg = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            partials, nsplit = _wgrad_conv(dyr, x, k, dilation, causal, 0.0, None, 0, lay)
            dv, dg = _wn_bwd(partials, nsplit, v, g, inv)
        return dx, dv, dg, lay.dbias(dbias), None, None, None, None, None


def conv1d(x, v, g, bias, k=1, dilation=1, causal=False, relu=False, extent=None):
    """Weight-normed Conv1d with 'same' (or causal) padding, optional fused ReLU.  x (B,Cin,T).  extent: as
    ``convblock``."""
    return _conv1d(_CONV, x, v, g, bias, k, dilation, causal, relu, extent)


def _conv1d(lay, x, v, g, bias, k, dilation, causal, relu, extent):
    """conv1d of a layer whose parameters are in layout ``lay`` (_CONV, _CONVT)."""
    if causal:
        extent = None
    M, N, _ = lay.dims(v)
    if _use_tc_conv(x, N, M, k):
        return _Conv1dTCFn.apply(_c(x), v, g, bias, int(k), int(dilation), bool(causal), bool(relu), extent, lay)
    y = _Conv1dFn.apply(_fp32_extent_in(_c(x), k, extent), v, g, bias, int(k), int(dilation), bool(causal),
                        bool(relu), lay)
    return extent_grad_mask(y, extent)


# ----------------------------------------------------------------------------------------------
# layout, lookups, position encodings, dropout
# ----------------------------------------------------------------------------------------------
class _TransposeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        _chk(x)
        B, R, C = x.shape
        y = torch.empty(B, C, R, device=x.device, dtype=torch.float32)
        lib.call("dv3_transpose", _p(x), _p(y), B, R, C, _stream())
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        B, C, R = dy.shape
        dx = torch.empty(B, R, C, device=dy.device, dtype=torch.float32)
        lib.call("dv3_transpose", _p(dy), _p(dx), B, C, R, _stream())
        return dx


def transpose12(x):
    """(B, R, C) -> contiguous (B, C, R) -- the (B,T,C) <-> (B,C,T) layout change."""
    return _TransposeFn.apply(_c(x))


_err_flags = {}


def _err_flag(device):
    f = _err_flags.get(device)
    if f is None:
        f = torch.zeros(1, dtype=torch.int32, device=device)
        _err_flags[device] = f
    return f


def check_index_errors(device=None):
    """Raise if any lookup kernel saw an out-of-range id since the last call (one D2H sync)."""
    for dev, f in _err_flags.items():
        if device is not None and dev != device:
            continue
        if int(f.item()) != 0:
            f.zero_()
            raise IndexError("dv3b200: embedding / position index out of range")


class _EmbeddingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, table, padding_idx):
        _chk(table)
        assert ids.dtype == torch.int64 and ids.is_cuda
        ids = ids.contiguous()
        N, (V, D) = ids.numel(), table.shape
        out = torch.empty(*ids.shape, D, device=table.device, dtype=torch.float32)
        lib.call("dv3_embedding_fwd", _p(ids), _p(table), _p(out), N, D, V, _p(_err_flag(table.device)),
                 _stream())
        ctx.save_for_backward(ids)
        ctx.cfg = (V, D, -1 if padding_idx is None else int(padding_idx))
        ctx.det = is_deterministic()
        return out

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        V, D, pad = ctx.cfg
        dy = _c(dy)
        dtable = torch.zeros(V, D, device=dy.device, dtype=torch.float32)
        lib.call("dv3_embedding_bwd_det" if ctx.det else "dv3_embedding_bwd", _p(ids), _p(dy), _p(dtable), ids.numel(),
                 D, V, pad, _stream())
        return None, dtable, None


def embedding(ids, table, padding_idx=None):
    return _EmbeddingFn.apply(ids, table, padding_idx)


class _SinusoidFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, table, w):
        _chk(table, w)
        assert pos.dtype == torch.int64 and pos.is_cuda and pos.dim() == 2
        pos = pos.contiguous()
        B, T = pos.shape
        P, D = table.shape
        out = torch.empty(B, T, D, device=table.device, dtype=torch.float32)
        lib.call("dv3_sinusoid_fwd", _p(pos), _p(table), _p(w), w.numel(), _p(out), B, T, D, P,
                 _p(_err_flag(table.device)), _stream())
        ctx.save_for_backward(pos, table, w)
        ctx.det = is_deterministic()
        return out

    @staticmethod
    def backward(ctx, dy):
        pos, table, w = ctx.saved_tensors
        dy = _c(dy)
        B, T = pos.shape
        P, D = table.shape
        dtable = torch.zeros_like(table) if ctx.needs_input_grad[1] else None
        dw = torch.zeros_like(w) if ctx.needs_input_grad[2] else None
        if dtable is not None or dw is not None:
            lib.call("dv3_sinusoid_bwd_det" if ctx.det else "dv3_sinusoid_bwd", _p(pos), _p(table), _p(w), w.numel(),
                     _p(dy), _p(dtable), _p(dw), B, T, D, P, _stream())
        return None, dtable, dw


def sinusoidal_encoding(pos, table, w):
    """pos int64 (B,T); table (P,D) raw position table; w fp32 tensor with 1 or B position rates."""
    return _SinusoidFn.apply(pos, table, w)


class _DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p, seed_t, salt):
        _chk(x)
        y = torch.empty_like(x)
        lib.call("dv3_dropout", _p(x), _p(y), x.numel(), p, _p(seed_t), salt, _stream())
        ctx.cfg = (p, seed_t, salt)
        return y

    @staticmethod
    def backward(ctx, dy):
        p, seed_t, salt = ctx.cfg
        dy = _c(dy)
        dx = torch.empty_like(dy)
        lib.call("dv3_dropout", _p(dy), _p(dx), dy.numel(), p, _p(seed_t), salt, _stream())
        return dx, None, None, None


def dropout(x, p, training):
    if not training or p <= 0.0:
        return x
    return _DropoutFn.apply(_c(x), float(p), rng.seed_tensor(x.device), rng.next_salt())


# Embedding-only speaker adaptation (speaker_adapt.SpeakerAdapt, installed by TrainStep(adapt_speakers=...) for the
# duration of one forward/backward): the speaker-conditioned sites run through it.  None: the plain autograd chain.
speaker_adapt = None


def speaker_dropout(e_btc, p, training):
    """A stack's dropout of its time-expanded speaker embedding (B, T, S)."""
    if speaker_adapt is None:
        return dropout(e_btc, p, training)
    return speaker_adapt.dropout(e_btc, p, training)


def speaker_residual(x, fc, e_btc):
    """x + softsign(fc(e_btc)): the encoder's speaker_fc1 / speaker_fc2 sites (reference deepvoice3.py:84, 101)."""
    if speaker_adapt is None:
        return x + torch.nn.functional.softsign(fc(e_btc))
    return speaker_adapt.residual_site(x, fc, e_btc)


# ----------------------------------------------------------------------------------------------
# ConvTranspose1d(k=2, stride=2) and Linear on the conv kernels
# ----------------------------------------------------------------------------------------------
class _Interleave2Fn(torch.autograd.Function):
    """x (B, 2C, T) with rows ordered (j, c) -> y (B, C, 2T), y[b, c, 2t + j] = x[b, j*C + c, t]: the time interleave
    after the 1x1 conv of a ConvTranspose1d(k=2, s=2).  A permutation: its adjoint is its inverse."""

    @staticmethod
    def forward(ctx, x):
        return _interleave2(x, 0)

    @staticmethod
    def backward(ctx, dy):
        return _interleave2(_c(dy), 1)


def _interleave2(x, inverse):
    B, R, T = x.shape
    C, T = (R, T // 2) if inverse else (R // 2, T)
    y = torch.empty((B, 2 * C, T) if inverse else (B, C, 2 * T), device=x.device)
    lib.call("dv3_interleave2", _p(x), _p(y), B, C, T, inverse, _stream())
    return y


def conv_transpose1d_k2s2(x, v, g, bias, extent=None):
    """Weight-normed ConvTranspose1d(k=2, s=2), v (Cin, Cout, 2): y[b,co,2t+j] = bias[co] + sum_ci x[b,ci,t] w[ci,co,j],
    w = g*v/||v|| over dim 0 (= Cin).  Runs as the 1x1 conv with 2*Cout output rows ordered (j,co) (_CONVT) followed
    by the time interleave.  extent: of x's time axis; the incoming gradient past it (2x in output frames) is taken
    as 0."""
    return _Interleave2Fn.apply(_conv1d(_CONVT, x, v, g, bias, 1, 1, False, False, extent))


class _InterleaveFn(torch.autograd.Function):
    """x (B, s*C, T) with rows ordered (j, c) -> y (B, C, s*T), y[b, c, s*t + j] = x[b, j*C + c, t], s in [3, 8]: the
    time interleave after the 1x1 conv of a ConvTranspose1d(k=s, stride=s) (s = 2 keeps _Interleave2Fn).  A
    permutation: its adjoint is its inverse."""

    @staticmethod
    def forward(ctx, x, s):
        ctx.s = s
        return interleave(x, s, 0)

    @staticmethod
    def backward(ctx, dy):
        return interleave(_c(dy), ctx.s, 1), None


def interleave(x, s, inverse=0):
    """The stride-s time interleave (B, s*C, T) -> (B, C, s*T) (dv3_interleave), or its inverse with inverse=1."""
    _chk(x)
    B, R, T = x.shape
    C, T = (R, T // s) if inverse else (R // s, T)
    y = torch.empty((B, s * C, T) if inverse else (B, C, s * T), device=x.device)
    lib.call("dv3_interleave", _p(x), _p(y), B, C, T, s, inverse, _stream())
    return y


def conv_transpose1d(x, v, g, bias, stride, extent=None):
    """Weight-normed ConvTranspose1d(k = stride = s), s in [2, 8], v (Cin, Cout, s):
    y[b,co,s*t+j] = bias[co] + sum_ci x[b,ci,t] w[ci,co,j], w = g*v/||v|| over dim 0 (= Cin).  The 1x1 conv with s*Cout
    output rows ordered (j,co) followed by the stride-s time interleave; s = 2 is ``conv_transpose1d_k2s2``."""
    s = int(stride)
    if s == 2:
        return conv_transpose1d_k2s2(x, v, g, bias, extent=extent)
    if not 2 <= s <= 8 or v.dim() != 3 or v.shape[2] != s:
        raise Dv3Error("conv_transpose1d: stride %d must lie in [2, 8] and equal the kernel size of v %s"
                       % (s, tuple(v.shape)))
    return _InterleaveFn.apply(_conv1d(_convt_layout(s), x, v, g, bias, 1, 1, False, False, extent), s)


def linear(x, v, g, bias):
    """Weight-normed Linear over the last dim (reference modules.py:80-85): x (..., Cin) -> (..., Cout).
    Runs on the conv kernels in channel-major layout: (N,Cin) -> (1,Cin,N) -> 1x1 conv -> back."""
    shp = x.shape
    Cin, Cout = shp[-1], v.shape[0]
    x2 = x.reshape(1, -1, Cin)
    y = conv1d(transpose12(x2), v.view(Cout, Cin, 1), g.view(Cout, 1, 1), bias)
    return transpose12(y).reshape(*shp[:-1], Cout)


# ----------------------------------------------------------------------------------------------
# length scope of a padded inference batch
# ----------------------------------------------------------------------------------------------
_length_scope = None          # (lengths int64 (B,) on the device, T of the scope) while a scope is active


class length_scope:
    """``with ops.length_scope(lengths, T):`` -- the stacks run inside (``modules.run_conv_stack`` and the deepvoice3
    converter) zero every row's frames past its own length before each conv whose kernel spans more than one frame,
    so that each row of a padded batch sees the zeros it would see alone.  ``lengths`` counts frames at time length
    ``T``; a stack running at T' = mult*T (after the converter's 2x upsamplers) masks from mult*lengths[b].
    Inference only: entering with grad enabled raises.  Scopes do not nest."""

    def __init__(self, lengths, T):
        self.lengths, self.T = lengths, int(T)

    def __enter__(self):
        global _length_scope
        if torch.is_grad_enabled():
            raise RuntimeError("ops.length_scope is for inference: enter it under torch.no_grad()")
        if _length_scope is not None:
            raise RuntimeError("ops.length_scope does not nest")
        lengths = self.lengths
        if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64 and lengths.dim() == 1):
            raise Dv3Error("length_scope needs an int64 (B,) CUDA tensor of lengths")
        _length_scope = (lengths.contiguous(), self.T)
        return self

    def __exit__(self, *exc):
        global _length_scope
        _length_scope = None
        return False


# ----------------------------------------------------------------------------------------------
# logical extents of a training batch padded to a bucket shape
# ----------------------------------------------------------------------------------------------
EXT_DEC, EXT_TEXT, EXT_MEL, EXT_LIN = 0, 1, 2, 3    # slots of the int64[4] extents: decoder steps, text positions,
                                                    # mel frames (= decoder steps * r), linear frames
_extent = None          # {"ext", "padded", "axis", "keymask"} while an extent scope is active

# slots of the per-term loss block of dv3_spec_loss_terms / dv3_aux_loss_terms (DV3_TERM_* in include/dv3b200.h)
TERM_MEL_L1, TERM_MEL_BD, TERM_LIN_L1, TERM_LIN_BD, TERM_DONE, TERM_ATTN, TERM_COUNT = 0, 1, 2, 3, 4, 5, 6


class extent_scope:
    """``with ops.extent_scope(extents, padded):`` -- the forward of a training batch that was padded past its own
    longest utterance to a bucket shape (``data.pad_to_bucket``).  ``extents`` is an int64[4] CUDA tensor of the
    batch's logical sizes (slots EXT_*), ``padded`` the host tuple of the padded sizes in the same slots.  The kernels
    read the extents from device memory, so one captured CUDA graph serves every batch of its bucket.  Inside:

    * the encoder's and the converter's stacks (whichever container selects the axis with ``extent_axis``) zero the
      frames t >= mult*extent before each conv whose kernel spans more than one frame, forward and backward
      (``mask_time``);
    * attention masks the keys s >= the logical text length and scales its context by the logical Ts*sqrt(1/Ts);
    * ``train_step.fused_training_loss`` divides its means by the logical sizes and leaves the padding out.

    Works with autograd and under graph capture.  Per-row masking of an inference batch is ``length_scope``."""

    def __init__(self, extents, padded):
        self.ext, self.padded = extents, tuple(int(v) for v in padded)

    def __enter__(self):
        global _extent
        ext = self.ext
        if _extent is not None or _length_scope is not None:
            raise RuntimeError("ops.extent_scope does not nest, nor run inside a length_scope")
        if not (torch.is_tensor(ext) and ext.is_cuda and ext.dtype == torch.int64 and ext.shape == (4,) and
                ext.is_contiguous()):
            raise Dv3Error("extent_scope needs a contiguous int64 (4,) CUDA tensor of logical extents")
        if len(self.padded) != 4:
            raise Dv3Error("extent_scope needs the 4 padded sizes")
        _extent = {"ext": ext, "padded": self.padded, "axis": None, "keymask": {}}
        return self

    def __exit__(self, *exc):
        global _extent
        _extent = None
        return False


class extent_axis:
    """``with ops.extent_axis(EXT_TEXT):`` -- the time axis of the stacks run inside (the encoder on text positions,
    the converter on mel frames) for the masking of an active ``extent_scope``; a no-op without one.  Stacks run
    outside an axis (the causal decoder: padded frames come after the valid ones) are not masked."""

    def __init__(self, slot):
        self.slot = slot

    def __enter__(self):
        if _extent is not None:
            self.prev = _extent["axis"]
            _extent["axis"] = self.slot
        return self

    def __exit__(self, *exc):
        if _extent is not None:
            _extent["axis"] = self.prev
        return False


def _ext_ptr(slot):
    """Device address of one extent."""
    ext = _extent["ext"]
    return ctypes.c_void_p(ext.data_ptr() + slot * ext.element_size())


def extent_frames(x):
    """(device address of the logical extent, mult) of the time axis of a stack activation x (B,C,T) inside an
    ``extent_scope`` and an ``extent_axis`` (mult = T // padded T: 2 and 4 after the converter's upsamplers), else
    None.  The conv stacks (``modules.run_conv_stack``) hand it to every layer they run: the tensor-core kernels read
    it in their operand-split passes, the exact-fp32 path masks with ``dv3_mask_frames``."""
    if _extent is None or _extent["axis"] is None:
        return None
    _chk(x)
    T, T0 = x.shape[2], _extent["padded"][_extent["axis"]]
    if T % T0 != 0:
        raise Dv3Error("x %s does not fit a padded extent of %d frames" % (tuple(x.shape), T0))
    return _ext_ptr(_extent["axis"]), T // T0


class _MaskFramesFn(torch.autograd.Function):
    """y = x with frames t >= mult*extent zeroed in every row; the mask is its own adjoint.  grad_only: the forward
    is the identity and only the gradient is masked (what leaves a stack, or enters an exact-fp32 layer's backward,
    must be 0 past the extent)."""

    @staticmethod
    def forward(ctx, x, ext_ptr, mult, grad_only):
        ctx.cfg = (ext_ptr, mult)
        if grad_only:
            return x.view_as(x)
        B, C, T = x.shape
        y = torch.empty_like(x)
        lib.call("dv3_mask_frames", _p(x), _p(y), ext_ptr, mult, B, C, T, _stream())
        return y

    @staticmethod
    def backward(ctx, dy):
        ext_ptr, mult = ctx.cfg
        dy = _c(dy)
        B, C, T = dy.shape
        dx = torch.empty_like(dy)
        lib.call("dv3_mask_frames", _p(dy), _p(dx), ext_ptr, mult, B, C, T, _stream())
        return dx, None, None, None


def extent_grad_mask(x, extent):
    """x unchanged; its gradient zeroed past the extent (``extent_frames``; None: x itself)."""
    return x if extent is None else _MaskFramesFn.apply(x, extent[0], extent[1], True)


def _fp32_extent_in(x, k, extent):
    """Exact-fp32 layer inside an extent scope: the input of a conv spanning more than one frame is masked (forward and
    backward); the tensor-core Functions do the same inside their operand splits."""
    if extent is None or k <= 1:
        return x
    return _MaskFramesFn.apply(x, extent[0], extent[1], False)


def mask_time(x):
    """x (B,C,T) -> a new tensor with frames t >= mult*lengths[b] zeroed (mult = T // T_scope); x itself when no
    length scope is active.  Never writes into x."""
    if _length_scope is None:
        return x
    lengths, T0 = _length_scope
    _chk(x)
    B, C, T = x.shape
    if B != lengths.numel() or T % T0 != 0:
        raise Dv3Error("mask_time: x %s does not fit a length scope of %d rows at T = %d" % (tuple(x.shape),
                                                                                          lengths.numel(), T0))
    y = torch.empty_like(x)
    lib.call("dv3_mask_time", _p(x), _p(y), _p(lengths), T // T0, B, C, T, _stream())
    return y


# ----------------------------------------------------------------------------------------------
# attention core (channel-major): q (B,E,Td), k (B,E,Ts), v (B,E,Ts) -> out (B,E,Td), probs (B,Td,Ts)
# ----------------------------------------------------------------------------------------------
def _bgemm(A, sA, Bm, sB, C, sCb, ldc, batch, M, N, K, alpha=1.0, accumulate=False, ts_ptr=None):
    """ts_ptr (device address of a key count): alpha = Ts*sqrt(1/Ts) of that count instead of ``alpha``."""
    if ts_ptr is not None:
        lib.call("dv3_bgemm_ctx_scale", _p(A), sA[0], sA[1], sA[2], _p(Bm), sB[0], sB[1], sB[2], _p(C), sCb, ldc,
                 batch, M, N, K, ts_ptr, int(accumulate), _stream())
        return
    lib.call("dv3_bgemm", _p(A), sA[0], sA[1], sA[2], _p(Bm), sB[0], sB[1], sB[2], _p(C), sCb, ldc, batch, M, N,
             K, float(alpha), int(accumulate), _stream())


class _AttentionCoreFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, mask, p_drop, training, ts_ptr):
        _chk(q, k, v)
        B, E, Td = q.shape
        Ts = k.shape[2]
        dev = q.device
        scores = torch.empty(B, Td, Ts, device=dev, dtype=torch.float32)
        # S[t,s] = sum_e q[e,t] k[e,s]                       (reference deepvoice3.py:143, no 1/sqrt(d))
        _bgemm(q, (E * Td, 1, Td), k, (E * Ts, Ts, 1), scores, Td * Ts, Ts, B, Td, Ts, E)
        p, seed_t, salt = _drop_args(p_drop, training, dev)
        seed_ptr = _p(seed_t)
        probs = torch.empty_like(scores)
        pd = torch.empty_like(scores) if p > 0 else None
        lib.call("dv3_softmax_fwd", _p(scores), _p(mask), _p(probs), _p(pd), B * Td, Ts, Td, p, seed_ptr, salt,
                 _stream())
        pv = pd if pd is not None else probs
        scale = Ts * (1.0 / Ts) ** 0.5                         # deepvoice3.py:170-171
        out = torch.empty(B, E, Td, device=dev, dtype=torch.float32)
        # O[e,t] = scale * sum_s v[e,s] pd[t,s]
        _bgemm(v, (E * Ts, Ts, 1), pv, (Td * Ts, 1, Ts), out, E * Td, Td, B, E, Td, Ts, alpha=scale, ts_ptr=ts_ptr)
        ctx.save_for_backward(q, k, v, probs, pd)
        ctx.cfg = (p, salt, scale, ts_ptr)
        ctx.seed_t = seed_t
        ctx.mark_non_differentiable()
        return out, probs

    @staticmethod
    def backward(ctx, dout, dprobs_ext):
        q, k, v, probs, pd = ctx.saved_tensors
        p, salt, scale, ts_ptr = ctx.cfg
        B, E, Td = q.shape
        Ts = k.shape[2]
        dev = q.device
        dout = _c(dout)
        seed_ptr = _p(ctx.seed_t)          # the forward's own seed snapshot
        pv = pd if pd is not None else probs
        # dPd[t,s] = scale * sum_e dO[e,t] v[e,s]
        dpd = torch.empty(B, Td, Ts, device=dev, dtype=torch.float32)
        _bgemm(dout, (E * Td, 1, Td), v, (E * Ts, Ts, 1), dpd, Td * Ts, Ts, B, Td, Ts, E, alpha=scale, ts_ptr=ts_ptr)
        # dV[e,s] = scale * sum_t dO[e,t] pd[t,s]
        dv = torch.empty_like(v)
        _bgemm(dout, (E * Td, Td, 1), pv, (Td * Ts, Ts, 1), dv, E * Ts, Ts, B, E, Ts, Td, alpha=scale, ts_ptr=ts_ptr)
        ds = torch.empty_like(dpd)
        dpe = _c(dprobs_ext) if dprobs_ext is not None else None
        lib.call("dv3_softmax_bwd", _p(probs), _p(dpd), _p(dpe), _p(ds), B * Td, Ts, p, seed_ptr, salt, _stream())
        # dq[e,t] = sum_s k[e,s] dS[t,s] ; dk[e,s] = sum_t q[e,t] dS[t,s]
        dq = torch.empty_like(q)
        _bgemm(k, (E * Ts, Ts, 1), ds, (Td * Ts, 1, Ts), dq, E * Td, Td, B, E, Td, Ts)
        dk = torch.empty_like(k)
        _bgemm(q, (E * Td, Td, 1), ds, (Td * Ts, Ts, 1), dk, E * Ts, Ts, B, E, Ts, Td)
        return dq, dk, dv, None, None, None, None


tc_attention = os.environ.get("DV3_TC_ATTN", "1") == "1"      # 0: attention on the exact-fp32 bgemm + softmax kernels


class _AttentionTCFn(torch.autograd.Function):
    """The same contract on the fused tensor-core kernels (csrc/tc_attn.cu): one launch forward, two backward."""

    @staticmethod
    def forward(ctx, q, k, v, mask, p_drop, training, ts_ptr):
        _chk(q, k, v)
        B, E, Td = q.shape
        Ts = k.shape[2]
        dev = q.device
        p, seed_t, salt = _drop_args(p_drop, training, dev)
        scale = Ts * (1.0 / Ts) ** 0.5                         # deepvoice3.py:170-171
        probs = torch.empty(B, Td, Ts, device=dev, dtype=torch.float32)
        out = torch.empty(B, E, Td, device=dev, dtype=torch.float32)
        if ts_ptr is not None:
            lib.call("dv3_tc_attn_fwd_ext", _p(q), _p(k), _p(v), _p(mask), _p(probs), _p(out), B, E, Td, Ts, ts_ptr,
                     p, _p(seed_t), salt, _stream())
        else:
            lib.call("dv3_tc_attn_fwd", _p(q), _p(k), _p(v), _p(mask), _p(probs), _p(out), B, E, Td, Ts, scale, p,
                     _p(seed_t), salt, _stream())
        ctx.save_for_backward(q, k, v, probs)
        ctx.cfg = (p, salt, scale, ts_ptr)
        ctx.seed_t = seed_t
        return out, probs

    @staticmethod
    def backward(ctx, dout, dprobs_ext):
        q, k, v, probs = ctx.saved_tensors
        p, salt, scale, ts_ptr = ctx.cfg
        B, E, Td = q.shape
        Ts = k.shape[2]
        dev = q.device
        dout = _c(dout)
        dpe = _c(dprobs_ext) if dprobs_ext is not None else None
        ds = torch.empty(B, Td, Ts, device=dev, dtype=torch.float32)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        if ts_ptr is not None:
            lib.call("dv3_tc_attn_bwd_ext", _p(dout), _p(q), _p(k), _p(v), _p(probs), _p(dpe), _p(ds), _p(dq), _p(dk),
                     _p(dv), B, E, Td, Ts, ts_ptr, p, _p(ctx.seed_t), salt, _stream())
        else:
            lib.call("dv3_tc_attn_bwd", _p(dout), _p(q), _p(k), _p(v), _p(probs), _p(dpe), _p(ds), _p(dq), _p(dk),
                     _p(dv), B, E, Td, Ts, scale, p, _p(ctx.seed_t), salt, _stream())
        return dq, dk, dv, None, None, None, None


def _extent_key_mask(B, Ts, device):
    """(B, Ts) uint8, 1 at keys s >= the logical text length of the active extent scope (built once per scope)."""
    km = _extent["keymask"].get((B, Ts))
    if km is None:
        ext = _extent["ext"]
        s = torch.arange(Ts, device=device)
        km = (s[None, :] >= ext[EXT_TEXT:EXT_TEXT + 1]).to(torch.uint8).expand(B, Ts).contiguous()
        _extent["keymask"][(B, Ts)] = km
    return km


def attention_core(q, k, v, mask=None, p_drop=0.0, training=False):
    """mask: (B, Ts) uint8/bool, 1 = padding.  Returns (out (B,E,Td), probs (B,Td,Ts)).  Inside an
    ``extent_scope`` the keys past the logical text length are masked too and the context scale is the logical one."""
    if mask is not None:
        mask = mask.to(torch.uint8).contiguous()
    B, E, Td = q.shape
    ts_ptr = None
    if _extent is not None:
        km = _extent_key_mask(B, k.shape[2], k.device)
        mask = km if mask is None else (mask | km)
        ts_ptr = _ext_ptr(EXT_TEXT)
    tc = (_tc_selected() and tc_attention and q.is_cuda and
          lib.raw("dv3_tc_attn_supported")(B, E, Td, k.shape[2]))
    fn = _AttentionTCFn if tc else _AttentionCoreFn
    return fn.apply(_c(q), _c(k), _c(v), mask, float(p_drop), bool(training), ts_ptr)
