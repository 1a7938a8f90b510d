"""Batched weight normalisation for the training step (csrc/wn_batched.cu).

The reference re-evaluates ``w = g * v / ||v||`` in a forward-pre-hook of every conv on every call
(``modules.py:85,100,109`` -- old-style ``weight_norm``).  Per layer that is two tiny launches in the forward (norm,
pack into the bf16 operand planes) and one in the backward (split-K reduction + g/v gradient): 127 latency-bound
launches per step.  Weights do not depend on activations, so ``TrainStep`` lets a ``WeightBank``

* prepare every registered layer's operand planes with TWO launches before the forward pass, and
* fold every layer's weight-norm backward into ONE launch after ``loss.backward()``,

using a device-resident table of ``Dv3WnEntry`` records (include/dv3b200.h).  Layers register themselves the first
time the tensor-core autograd Functions see them (that step runs the per-layer path); buffers are persistent, so the
whole thing is CUDA-graph capturable from the second step on.  A bank packs the operand planes of the mode it was built
in (``npl``: 2 planes per operand in ``ops.conv_math = "tc"``, 1 in ``"tc1"``).
"""
import ctypes

import torch

from ._lib import lib, Dv3Error


class Dv3WnEntry(ctypes.Structure):
    _fields_ = [("v", ctypes.c_void_p), ("g", ctypes.c_void_p), ("inv_norm", ctypes.c_void_p),
                ("scale", ctypes.c_void_p), ("wfwd", ctypes.c_void_p), ("wbwd", ctypes.c_void_p),
                ("partials", ctypes.c_void_p), ("dv", ctypes.c_void_p), ("dg", ctypes.c_void_p),
                ("split_stride", ctypes.c_longlong), ("Cout", ctypes.c_int), ("Cin", ctypes.c_int),
                ("k", ctypes.c_int), ("nsplit", ctypes.c_int), ("blk_norm", ctypes.c_int),
                ("blk_pack", ctypes.c_int), ("blk_bwd", ctypes.c_int), ("pack_gx", ctypes.c_int)]


def _pad8(n):
    return (n + 7) // 8 * 8


class _Layer:
    """Persistent per-layer buffers: what dv3_tc_weightnorm_fwd would allocate on every call."""

    def __init__(self, v, g, npl=2):
        Cout, Cin, k = v.shape
        dev, bf = v.device, torch.bfloat16
        self.v, self.g = v, g
        self.Cout, self.Cin, self.k = Cout, Cin, k
        self.inv = torch.empty(Cout, device=dev)
        self.scale = torch.empty(Cout, device=dev)
        self.wfwd = torch.empty(npl, k, Cout, _pad8(Cin), device=dev, dtype=torch.float16)
        self.wbwd = torch.empty(npl, k, Cin, _pad8(Cout), device=dev, dtype=bf)
        self.partials = None
        self.nsplit = 0
        self.partials_by_shape = {}      # (nsplit, numel) -> buffer: graphs captured at other shapes keep theirs
        self.prepared = False
        self.pending = False

    def entry(self):
        e = Dv3WnEntry()
        e.v, e.g = self.v.data_ptr(), self.g.data_ptr()
        e.inv_norm, e.scale = self.inv.data_ptr(), self.scale.data_ptr()
        e.wfwd, e.wbwd = self.wfwd.data_ptr(), self.wbwd.data_ptr()
        e.Cout, e.Cin, e.k = self.Cout, self.Cin, self.k
        e.pack_gx = (self.Cin * self.k + 31) // 32
        return e


def _upload(entries, device):
    arr = (Dv3WnEntry * len(entries))(*entries)
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
    return host.to(device)


class WeightBank:
    def __init__(self, npl=2):
        if npl not in (1, 2):
            raise Dv3Error("WeightBank: npl must be 1 or 2")
        self.npl = npl                   # operand planes packed per layer (the mode the bank was built in)
        self.layers = {}                 # v.data_ptr() -> _Layer, in registration (= forward) order
        self.active = False              # inside TrainStep._forward_backward
        self.fresh = False               # operand planes match the current parameter values
        self._fwd = None                 # (device table, n, norm_blocks, pack_blocks, layers)
        self._bwd = {}                   # pending-set key -> (device table, n, blocks); one entry per gradient bucket

    # -- forward ------------------------------------------------------------------------------------
    def begin_step(self):
        """Normalise + pack every registered layer (2 launches).  Call before the forward pass."""
        self.active = True
        self.fresh = False
        if not self.layers:
            return
        if self._fwd is None or self._fwd[1] != len(self.layers):
            if torch.cuda.is_current_stream_capturing():
                raise Dv3Error("WeightBank: a layer registered during CUDA-graph capture (warm up first)")
            ents, nb, pb = [], 0, 0
            layers = list(self.layers.values())
            for L in layers:
                e = L.entry()
                e.blk_norm, e.blk_pack = nb, pb
                nb += (L.Cout * 32 + 255) // 256
                pb += e.pack_gx * ((L.Cout + 31) // 32)
                ents.append(e)
            self._fwd = (_upload(ents, layers[0].v.device), len(ents), nb, pb, layers)
        tab, n, nb, pb, layers = self._fwd
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        lib.call("dv3_tc_weightnorm_fwd_batched_npl", ctypes.c_void_p(tab.data_ptr()), n, nb, pb, self.npl, st)
        for L in layers:
            L.prepared = True
        self.fresh = True

    def weights_for(self, v, g, npl=2):
        """The prepared (wfwd, wbwd, inv) record of parameter pair (v, g) with ``npl`` planes per operand, or None ->
        caller runs the per-layer kernels (first step, bank idle, or a bank built for the other plane count).  Unknown
        layers are registered for the next step."""
        if not self.active or npl != self.npl:
            return None
        L = self.layers.get(v.data_ptr())
        if L is None:
            if v.dim() == 3 and v.is_leaf and g.is_leaf and not torch.cuda.is_current_stream_capturing():
                self.layers[v.data_ptr()] = _Layer(v, g, self.npl)
            return None
        if not (self.fresh and L.prepared) or tuple(L.v.shape) != tuple(v.shape):
            return None
        return L

    # -- backward -----------------------------------------------------------------------------------
    def partials_for(self, L, nsplit, numel):
        """Persistent split-K partial buffer of layer L when its weight-norm backward can be deferred to
        end_backward(); None -> the caller reduces immediately."""
        if not self.active or L.pending or L.v.grad is None or L.g.grad is None:
            return None
        if L.partials is None or L.nsplit != nsplit or L.partials.shape[1] != numel:
            buf = L.partials_by_shape.get((nsplit, numel))
            if buf is None:
                if torch.cuda.is_current_stream_capturing():
                    return None
                buf = L.partials_by_shape[(nsplit, numel)] = torch.empty(nsplit, numel, device=L.v.device)
            L.partials = buf
            L.nsplit = nsplit
        L.pending = True
        return L.partials

    def end_backward(self):
        """dv / dg of every layer whose weight gradient was deferred, accumulated into .grad (1 launch)."""
        pend = [L for L in self.layers.values() if L.pending]
        if not pend:
            return
        key = tuple((L.v.data_ptr(), L.nsplit, L.partials.data_ptr(), L.v.grad.data_ptr(), L.g.grad.data_ptr())
                    for L in pend)
        if key not in self._bwd:
            if torch.cuda.is_current_stream_capturing():
                raise Dv3Error("WeightBank: backward table changed during CUDA-graph capture (warm up first)")
            ents, blocks = [], 0
            for L in pend:
                e = L.entry()
                e.partials, e.split_stride, e.nsplit = L.partials.data_ptr(), L.partials.shape[1], L.nsplit
                e.dv, e.dg = L.v.grad.data_ptr(), L.g.grad.data_ptr()
                e.blk_bwd = blocks
                blocks += L.Cout
                ents.append(e)
            self._bwd[key] = (_upload(ents, pend[0].v.device), len(ents), blocks)
        tab, n, blocks = self._bwd[key]
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        lib.call("dv3_weightnorm_bwd_batched", ctypes.c_void_p(tab.data_ptr()), n, blocks, 1, st)
        for L in pend:
            L.pending = False

    def end_step(self):
        self.active = False
        self.fresh = False
        for L in self.layers.values():
            L.pending = False
