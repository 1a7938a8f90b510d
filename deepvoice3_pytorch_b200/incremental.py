"""Autoregressive (incremental) decoding on the device -- SURVEY.md section 8(f)3.

Reference behaviour: ``Decoder.incremental_forward`` (deepvoice3.py:367-485, nyanko.py:250-338) feeds one frame at a
time through ``Conv1d.incremental_forward`` (conv.py:17-46: a ring buffer of the last (k-1)*dilation+1 inputs times
the linearised weight), the gate epilogues (modules.py:145-167, 200-226) and the attention layer with its monotonic
window (deepvoice3.py:150-156), until every utterance raised its done flag.

Here one decoder step is a fixed sequence of matrix-vector kernels (csrc/incremental.cu) whose loop state -- step
counter, ring buffers, monotonic-attention cursor, output arrays indexed by the step -- lives in device memory, so the
sequence is captured ONCE in a CUDA graph and replayed; the host looks at the done flags every ``CHECK_EVERY`` steps
and discards the few frames computed past the reference's stopping point.  Weight norm is folded once per call, the
key / value projections are hoisted out of the loop (the reference recomputes them every step, deepvoice3.py:136-141).
Quirks kept on purpose: the "average" alignment is first_layer * 2**(n-1) / n (``ave_alignment + ave_alignment``,
deepvoice3.py:446) and the monotonic cursor follows batch row 0 only (deepvoice3.py:443).

``decode_ragged`` is the batched form for rows of different text lengths (``synthesis.tts_batch``): row b attends to
its own text_lengths[b] keys with its own monotonic cursor and stops by the reference's rule applied to it alone, so
every row gets what ``decode`` gives for that row on its own, bit for bit (every step kernel works per row).

``decode_stream`` is continuous batching (``synthesis.tts_stream``): a fixed set of decoder slots, each with its own
step counter; when a slot's utterance stops (the stop rule runs on the device, per row), the host gathers it at the next
check and one ``dv3_inc_refill`` launch resets the slot and loads the next waiting utterance into it.

Both take per-token durations (DESIGN.md section 2.22): guided decoding centres every attention layer's window on a
prescribed token path (token j for steps S_j <= t < S_{j+1}, S_j the sum of the first j durations) instead of on the
previous argmax, and stops each row after exactly its total of steps.
"""
import contextlib
import ctypes
import os

import numpy as np
import torch
from torch import nn

from . import ops
from ._lib import lib
from .conv import Conv1d as _Conv1d, WNLinear
from .modules import Conv1dGLU, HighwayConv1d

CHECK_EVERY = 16
_P, _LL, _I, _F = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float


class Dv3IncStep(ctypes.Structure):
    _fields_ = [("x", _P), ("x_ld", _LL), ("x_t", _LL), ("add", _P), ("add_ld", _LL), ("add_t", _LL),
                ("ring", _P), ("w", _P), ("bias", _P), ("spk", _P), ("spk_ld", _LL),
                ("res1", _P), ("res1_ld", _LL), ("res1_t", _LL), ("res2", _P), ("res2_ld", _LL), ("res2_t", _LL),
                ("y", _P), ("y_ld", _LL), ("y_t", _LL), ("y2", _P), ("y2_ld", _LL), ("y2_t", _LL),
                ("yadd", _P), ("yadd_ld", _LL), ("yadd_t", _LL), ("t_ptr", _P),
                ("B", _I), ("Cin", _I), ("Cout", _I), ("k", _I), ("dilation", _I), ("mode", _I), ("act", _I),
                ("vec4", _I), ("y2_mode", _I)]


class Dv3IncAttn(ctypes.Structure):
    _fields_ = [("q", _P), ("q_ld", _LL), ("keys", _P), ("values", _P), ("ctx", _P), ("ctx_ld", _LL),
                ("align", _P), ("align_ld", _LL), ("align_t", _LL), ("last_attended", _P), ("t_ptr", _P),
                ("align_scale", _F), ("B", _I), ("E", _I), ("Ts", _I), ("window_backward", _I),
                ("window_ahead", _I)]


class Dv3IncRefill(ctypes.Structure):
    _fields_ = [("dst", _P), ("src", _P), ("row_bytes", _LL), ("dst_row_stride", _LL), ("src_row_stride", _LL)]


class _Rows:
    """(B, C) rows of a float32 buffer that may advance with the step: row b of step t = ptr + b*ld + t*t (floats)."""

    def __init__(self, tensor, C, ld=None, t=0, offset=0):
        assert tensor.dtype == torch.float32 and tensor.is_contiguous()
        self.tensor, self.C = tensor, C
        self.ld = C if ld is None else ld
        self.t, self.offset = t, offset

    @property
    def ptr(self):
        return self.tensor.data_ptr() + 4 * self.offset

    def aligned16(self):
        return self.ptr % 16 == 0 and self.ld % 4 == 0 and self.t % 4 == 0


def _folded_weight(m):
    """w = v * g/||v|| (old-style weight_norm, dim 0) linearised like reference conv.py:51-60: (Cout, k, Cin)."""
    v, g = m.weight_v.detach(), m.weight_g.detach()
    w = v * (g / torch.norm_except_dim(v, 2, 0))
    if w.dim() == 2:                       # WNLinear (out, in)
        return w.unsqueeze(1).contiguous()
    return w.transpose(1, 2).contiguous()


class StepProgram:
    """The launch sequence of one decoder step + its device-resident state.

    slots=True: every row has its own step counter (``t`` is int32 (B,)) and runs the ``_slots`` step kernels; the step
    ends with the device-side stop rule (``stop_rule``) and a per-row advance that holds rows which stopped."""

    def __init__(self, B, device, slots=False):
        self.B, self.dev, self.slots = B, device, slots
        self.calls = []                     # (entry point name, ctypes struct, extra arguments)
        self.keep = []                      # tensors the structs point into
        self.t = torch.zeros(B if slots else 1, dtype=torch.int32, device=device)
        self.rings, self.cursors = [], []   # the per-row history a new utterance starts from zero
        self.stop = None                    # slots: int32 (B,) stop steps, 0 while the row runs
        self.total = None                   # guided slots: int32 (B,) prescribed step counts (the stop rule)
        self.graph = None

    def buf(self, *shape):
        t = torch.zeros(*shape, device=self.dev, dtype=torch.float32)
        self.keep.append(t)
        return t

    def conv(self, x, m, mode=0, act=0, add=None, spk=None, res1=None, res2=None, y=None, y2=None, y2_mode=0,
             yadd=None):
        """One conv / linear step of module m (Conv1d | WNLinear) on rows x -> rows y (allocated when None)."""
        w = _folded_weight(m)
        bias = m.bias.detach().contiguous()
        Cout, k, Cin = w.shape
        d = m.dilation[0] if isinstance(m, _Conv1d) else 1
        assert x.C == Cin, "step input has %d channels, layer expects %d" % (x.C, Cin)
        C = Cout // 2 if mode else Cout
        if y is None:
            y = _Rows(self.buf(self.B, C), C)
        s = Dv3IncStep()
        s.x, s.x_ld, s.x_t = x.ptr, x.ld, x.t
        if add is not None:
            s.add, s.add_ld, s.add_t = add.ptr, add.ld, add.t
        if k > 1:
            ring = self.buf(self.B, (k - 1) * d + 1, Cin)
            self.rings.append(ring)
            s.ring = ring.data_ptr()
        s.w, s.bias = w.data_ptr(), bias.data_ptr()
        if spk is not None:
            s.spk, s.spk_ld = spk.ptr, spk.ld
        if res1 is not None:
            s.res1, s.res1_ld, s.res1_t = res1.ptr, res1.ld, res1.t
        if res2 is not None:
            s.res2, s.res2_ld, s.res2_t = res2.ptr, res2.ld, res2.t
        s.y, s.y_ld, s.y_t = y.ptr, y.ld, y.t
        if y2 is not None:
            s.y2, s.y2_ld, s.y2_t, s.y2_mode = y2.ptr, y2.ld, y2.t, y2_mode
        if yadd is not None:
            s.yadd, s.yadd_ld, s.yadd_t = yadd.ptr, yadd.ld, yadd.t
        s.t_ptr = self.t.data_ptr()
        s.B, s.Cin, s.Cout, s.k, s.dilation, s.mode, s.act = self.B, Cin, Cout, k, d, mode, act
        s.vec4 = int(Cin % 4 == 0 and x.aligned16() and (add is None or add.aligned16()))
        self.keep += [w, bias]
        self.calls.append(("dv3_inc_conv_step_slots" if self.slots else "dv3_inc_conv_step", s, ()))
        return y

    def cursor(self, per_row):
        """Monotonic-attention cursors: int[2] (row 0 leads, ``decode``) or int[2][B] (one per row)."""
        la = torch.zeros(2 * self.B if per_row else 2, dtype=torch.int32, device=self.dev)
        self.cursors.append(la)
        return la

    def attention(self, q, keys_bet, values_bte, ctx, align, align_scale, last_attended, window_backward, window_ahead,
                  text_len=None, path=None):
        """text_len: int32 (B,) device tensor -> the per-row (ragged) step, last_attended then holds [2][B] cursors.
        path: int32 (B, n) device tensor -> the guided step: row b's window centre at step t is path[b, t]."""
        a = Dv3IncAttn()
        B, E, Ts = keys_bet.shape
        a.q, a.q_ld = q.ptr, q.ld
        a.keys, a.values = keys_bet.data_ptr(), values_bte.data_ptr()
        a.ctx, a.ctx_ld = ctx.ptr, ctx.ld
        if align is not None:
            a.align, a.align_ld, a.align_t = align.ptr, align.ld, align.t
        if last_attended is not None:
            a.last_attended = last_attended.data_ptr()
        a.t_ptr = self.t.data_ptr()
        a.align_scale = align_scale
        a.B, a.E, a.Ts, a.window_backward, a.window_ahead = B, E, Ts, window_backward, window_ahead
        self.keep += [keys_bet, values_bte]
        if path is not None:
            assert text_len is not None and last_attended is None and path.dtype == torch.int32
            self.keep += [text_len, path]
            name = "dv3_inc_attn_step_slots_path" if self.slots else "dv3_inc_attn_step_path"
            self.calls.append((name, a, (ctypes.c_void_p(text_len.data_ptr()), ctypes.c_void_p(path.data_ptr()),
                                         path.stride(0))))
        elif text_len is None:
            assert not self.slots, "the slot program attends per row: it needs text_len"
            self.calls.append(("dv3_inc_attn_step", a, ()))
        else:
            self.keep.append(text_len)
            name = "dv3_inc_attn_step_slots" if self.slots else "dv3_inc_attn_step_rows"
            self.calls.append((name, a, (ctypes.c_void_p(text_len.data_ptr()),)))

    def stop_rule(self, dones, min_steps, max_steps):
        """slots: apply the reference stop rule to row b's done flag dones[b, t[b]] at the end of every step.  Rows
        start idle (stop = -1: held at step 0) until ``dv3_inc_refill`` loads them."""
        assert self.slots and dones.size(1) > max_steps
        self.stop = torch.full((self.B,), -1, dtype=torch.int32, device=self.dev)
        self._stop_args = (ctypes.c_void_p(dones.data_ptr()), dones.size(1), ctypes.c_void_p(self.t.data_ptr()),
                           ctypes.c_void_p(self.stop.data_ptr()), self.B, min_steps, max_steps)

    def stop_rule_total(self, total):
        """guided slots: stop row b once it has run total[b] (int32 (B,) device) steps; rows start idle as with
        ``stop_rule``."""
        assert self.slots and total.dtype == torch.int32
        self.stop = torch.full((self.B,), -1, dtype=torch.int32, device=self.dev)
        self.total = total

    # -- execution --------------------------------------------------------------------------------
    def _launch_step(self):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        for name, s, extra in self.calls:
            lib.call(name, ctypes.byref(s), *extra, st)
        if self.slots:
            if self.total is not None:
                lib.call("dv3_inc_stop_rows_total", ctypes.c_void_p(self.t.data_ptr()),
                         ctypes.c_void_p(self.stop.data_ptr()), ctypes.c_void_p(self.total.data_ptr()), self.B, st)
            else:
                lib.call("dv3_inc_stop_rows", *self._stop_args, st)
            lib.call("dv3_inc_advance_rows", ctypes.c_void_p(self.t.data_ptr()),
                     ctypes.c_void_p(self.stop.data_ptr()), self.B, st)
        else:
            lib.call("dv3_inc_advance", ctypes.c_void_p(self.t.data_ptr()), st)

    def run(self, n_steps, use_graph=True):
        if use_graph and self.graph is None:
            # capture_begin/_end directly: the torch.cuda.graph() context manager also runs gc.collect() and
            # empty_cache(), which cost more than the whole utterance (measured: 80-400 ms per call)
            self.graph = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream(device=self.dev)
            side.wait_stream(torch.cuda.current_stream(self.dev))
            with torch.cuda.stream(side):
                self.graph.capture_begin()
                try:
                    self._launch_step()
                finally:
                    self.graph.capture_end()
            torch.cuda.current_stream(self.dev).wait_stream(side)
        for _ in range(n_steps):
            if use_graph:
                self.graph.replay()
            else:
                self._launch_step()


class ModuleStepper:
    """Stateful single-layer stepping for the module-level API (``Conv1d.incremental_forward`` & co., reference
    conv.py:17-46 / modules.py:142-143, 197-198): weight folded and ring buffer allocated at creation."""

    def __init__(self, conv, B, mode=0, spk=None, residual=False):
        dev = conv.weight_v.device
        if not conv.weight_v.is_cuda:
            raise RuntimeError("incremental_forward runs on the GPU only (no CPU fallback)")
        self.prog = StepProgram(B, dev)
        Cin = conv.weight_v.shape[1]
        self.x = self.prog.buf(B, Cin)
        rows = _Rows(self.x, Cin)
        spk_rows = None
        if spk is not None:
            spk = spk.detach().to(torch.float32).contiguous()
            self.prog.keep.append(spk)
            spk_rows = _Rows(spk, spk.size(-1))
        self.y = self.prog.conv(rows, conv, mode=mode, spk=spk_rows, res1=rows if residual else None)
        self.B = B

    @torch.no_grad()
    def step(self, frame):
        self.x.copy_(frame.reshape(self.B, -1))
        self.prog.run(1, use_graph=False)
        return self.y.tensor.clone().view(self.B, 1, -1)


def _run_stack(prog, layers, cur, spk_of=None, last_y=None, last_y2=None, last_yadd=None):
    """[Conv1d | ReLU | Conv1dGLU | HighwayConv1d] one step each (Conv1d + ReLU fused); the LAST op may be given an
    explicit destination ``last_y`` and a second output ``last_y2 = y + last_yadd``."""
    layers = list(layers)
    ops_ = []
    i = 0
    while i < len(layers):
        f = layers[i]
        if isinstance(f, _Conv1d):
            relu = i + 1 < len(layers) and isinstance(layers[i + 1], nn.ReLU)
            ops_.append((f, 1 if relu else 0))
            i += 2 if relu else 1
        elif isinstance(f, (Conv1dGLU, HighwayConv1d)):
            ops_.append((f, 0))
            i += 1
        else:
            raise NotImplementedError("no incremental step for %s" % type(f).__name__)
    for n, (f, relu) in enumerate(ops_):
        last = n == len(ops_) - 1
        kw = dict(y=last_y if last else None)
        if last and last_y2 is not None:
            kw.update(y2=last_y2, y2_mode=2, yadd=last_yadd)
        if isinstance(f, _Conv1d):
            cur = prog.conv(cur, f, act=relu, **kw)
        elif isinstance(f, Conv1dGLU):
            cur = prog.conv(cur, f.conv, mode=1, spk=spk_of(f) if spk_of else None,
                            res1=cur if f.residual else None, **kw)
        else:
            cur = prog.conv(cur, f.conv, mode=2, **kw)
    return cur


def _stop_step(done, min_steps, max_steps):
    """Number of decoder steps the reference loop runs given done flags (B, n) of the steps computed so far, or None
    if it would still be running: break after step n if all(done > .5) and n > min_steps, or if n > max_steps."""
    flags = (done > 0.5).all(dim=0).tolist()
    for n in range(1, len(flags) + 1):
        if (flags[n - 1] and n > min_steps) or n > max_steps:
            return n
    return None


def _row_stop_steps(done, min_steps, max_steps):
    """The stop rule of ``_stop_step`` applied to every row alone: [N_b or None] for done flags (B, n)."""
    return [_stop_step(done[b:b + 1], min_steps, max_steps) for b in range(done.size(0))]


@torch.no_grad()
def decode(decoder, encoder_out, text_positions, speaker_embed=None, initial_input=None, test_inputs=None,
           use_graph=None):
    """-> outputs (B, N, in_dim*r), alignments (B, N, T_text), dones [N x (B,1,1)], decoder_states (B, N, C): what
    the reference's Decoder.incremental_forward returns."""
    return _decode(decoder, encoder_out, text_positions, speaker_embed, initial_input, test_inputs, use_graph)


def check_durations(durations, lengths):
    """durations: one 1-D integer array (sequence or tensor) per row, of lengths[b] entries each >= 1 -> list of int64
    arrays.  ValueError otherwise (host values only)."""
    if not isinstance(durations, (list, tuple)) or len(durations) != len(lengths):
        raise ValueError("durations must be a list of %d arrays, one per sequence" % len(lengths))
    out = []
    for b, (d, n) in enumerate(zip(durations, lengths)):
        d = np.asarray(d.detach().cpu() if torch.is_tensor(d) else d)
        if d.ndim != 1 or (d.size and not np.issubdtype(d.dtype, np.integer)):
            raise ValueError("durations[%d] must be a 1-D integer array, got %s of shape %s" % (b, d.dtype, d.shape))
        if d.size != int(n):
            raise ValueError("durations[%d] has %d entries for a sequence of %d tokens" % (b, d.size, int(n)))
        if d.size and d.min() < 1:
            raise ValueError("durations[%d] holds a duration below 1 step: %d" % (b, int(d.min())))
        out.append(d.astype(np.int64))
    return out


def path_table(durations, steps=None):
    """Per-row durations (int64 arrays, each >= 1) -> (path int64 (B, steps), totals [B]): row b attends token j at
    steps S_j <= t < S_{j+1} (S_j the sum of its first j durations); past its total S_{L_b} it holds its last token,
    the step a row that has stopped keeps recomputing.  steps defaults to the largest total."""
    totals = [int(d.sum()) for d in durations]
    T = max(totals) if steps is None else int(steps)
    path = np.empty((len(durations), T), np.int64)
    for b, d in enumerate(durations):
        row = np.repeat(np.arange(d.size, dtype=np.int64), d)[:T]
        path[b, :row.size] = row
        path[b, row.size:] = d.size - 1
    return path, totals


def query_steps(decoder):
    """The most decoder steps the query-position table holds: steps t = 0.. read positions t + 1."""
    return decoder.embed_query_positions.num_embeddings - 1


@torch.no_grad()
def decode_ragged(decoder, encoder_out, text_positions, text_lengths, speaker_embed=None, initial_input=None,
                  test_inputs=None, use_graph=None, durations=None):
    """Batched decode of rows with text_lengths (B,) valid keys each (encoder outputs padded to T_text).
    -> outputs (B, N, in_dim*r), alignments (B, N, T_text), dones (B, N), decoder_states (B, N, C), steps [B]:
    row b is valid for its first steps[b] decoder steps (and its first text_lengths[b] alignment columns; the rest are
    0) and there equals ``decode`` run on that row alone with its encoder outputs cut to text_lengths[b].  Free-running,
    row b stops by the reference rule applied to its own done flags; rows that stopped keep computing until the last
    one does, their extra frames are not part of the result.  Teacher-forced (test_inputs (B, N, in_dim*r)), every row
    runs N steps.

    durations: guided decoding -- one integer array per row, durations[b] of text_lengths[b] entries >= 1 (in decoder
    steps).  Every attention layer centres its window on token j of row b for steps S_j <= t < S_{j+1}, and row b runs
    exactly steps[b] = S_{L_b} steps (the sum of its durations): the done flags are computed and returned but do not
    stop it, and min / max_decoder_steps do not apply.  ValueError before any launch for malformed durations, a total
    above the query-position table (``query_steps``) or teacher-forced inputs."""
    guide = None
    if durations is not None:
        if test_inputs is not None:
            raise ValueError("durations guide a free-running decode; teacher-forced inputs take none")
        lens = np.asarray(text_lengths.cpu() if torch.is_tensor(text_lengths) else text_lengths).reshape(-1)
        path, totals = path_table(check_durations(durations, lens))
        if max(totals) > query_steps(decoder):
            raise ValueError("durations total %d decoder steps; the query-position table holds %d"
                             % (max(totals), query_steps(decoder)))
        guide = (path, totals)
    return _decode(decoder, encoder_out, text_positions, speaker_embed, initial_input, test_inputs, use_graph,
                   text_lengths=text_lengths, guide=guide)


def _constants(decoder, keys, values, text_positions, speaker_embed, Tmax):
    """The per-utterance constants of the step program, for B rows (call in exact-fp32 mode):
    [(keys (B, E, Ts), values (B, Ts, E))] per attention layer (key-position embedding added, projected once), the
    query-position table (B, Tmax, C) and ``addend(f)``: the softsign speaker addend (B, C) of GLU block f, or None."""
    nyanko = hasattr(decoder, "audio_encoder_modules")
    B = keys.size(0)
    if nyanko:
        if text_positions is not None:
            keys = keys + decoder.embed_keys_positions(text_positions)
    else:
        w = decoder._position_rate(decoder.key_position_rate, decoder.speaker_proj1, speaker_embed)
        keys = keys + decoder.embed_keys_positions(text_positions, w)
    frame_pos = torch.arange(1, Tmax + 1, device=keys.device).view(1, -1).repeat(B, 1)
    if nyanko:
        pos_table = decoder.embed_query_positions(frame_pos)
    else:
        w2 = decoder._position_rate(decoder.query_position_rate, decoder.speaker_proj2, speaker_embed)
        pos_table = decoder.embed_query_positions(frame_pos, w2)
    pos_table = pos_table.contiguous()                     # (B, Tmax, C)
    att_layers = [decoder.attention] if nyanko else [a for a in decoder.attention if a is not None]
    kv = []
    for att in att_layers:
        k_ = keys if att.key_projection is None else att.key_projection(keys)
        v_ = values if att.value_projection is None else att.value_projection(values)
        kv.append((k_.transpose(1, 2).contiguous(), v_.contiguous()))

    def addend(f):
        if f.speaker_proj is None or speaker_embed is None:
            return None
        return torch.nn.functional.softsign(f.speaker_proj(speaker_embed)).contiguous()     # (B, C)
    return kv, pos_table, addend


def _build_program(decoder, prog, Tmax, E, kv, pos_table, spk_of, text_len, frames, test_inputs=None, path=None):
    """Record one decoder step into prog (B rows): input frame t of ``frames`` (B, Tmax + 1, Fr) -- or of test_inputs
    (B, Tmax, Fr) -- to output frame t + 1.  spk_of(f) -> _Rows of GLU block f's speaker addend, or None; text_len:
    int32 (B,) per-row attention lengths, or None (``decode``); path: int32 (B, Tmax) guided window centres, or None.
    -> states (B, Tmax, Cs), aligns (B, Tmax, Ts),
    dones (B, Tmax)."""
    nyanko = hasattr(decoder, "audio_encoder_modules")
    B, Ts = prog.B, kv[0][0].size(2)
    Fr = decoder.in_dim * decoder.r
    C = pos_table.size(-1)
    prog.keep += [pos_table]
    states = prog.buf(B, Tmax, C if not nyanko else decoder.last_conv.in_channels)
    Cs = states.size(-1)
    aligns = prog.buf(B, Tmax, Ts)
    dones = prog.buf(B, Tmax)
    if test_inputs is not None:
        prog.keep.append(test_inputs)
        cur = _Rows(test_inputs, Fr, ld=Tmax * Fr, t=Fr)
    else:
        cur = _Rows(frames, Fr, ld=(Tmax + 1) * Fr, t=Fr)
    pos_rows = _Rows(pos_table, C, ld=Tmax * C, t=C)
    states_rows = _Rows(states, Cs, ld=Tmax * Cs, t=Cs)
    align_rows = _Rows(aligns, Ts, ld=Tmax * Ts, t=Ts)

    def cursor(force):
        return prog.cursor(text_len is not None) if force and path is None else None

    if nyanko:
        D = C
        cat = prog.buf(B, 2 * D)
        q_in = _Rows(prog.buf(B, D), D)
        _run_stack(prog, decoder.audio_encoder_modules, cur, last_y=_Rows(cat, D, ld=2 * D, offset=D),
                   last_y2=q_in, last_yadd=pos_rows)
        att = decoder.attention
        q = prog.conv(q_in, att.query_projection)
        ctx = _Rows(prog.buf(B, E), E)
        prog.attention(q, kv[0][0], kv[0][1], ctx, align_rows, 1.0, cursor(decoder.force_monotonic_attention),
                       att.window_backward, att.window_ahead, text_len, path)
        prog.conv(ctx, att.out_projection, res1=q_in, y=_Rows(cat, D, ld=2 * D))
        cur = _run_stack(prog, decoder.audio_decoder_modules, _Rows(cat, 2 * D), last_y=states_rows)
    else:
        cur = _run_stack(prog, decoder.preattention, cur, spk_of)
        n_att = len(kv)
        n_conv = len(decoder.convolutions)
        ai = 0
        for idx, (f, att) in enumerate(zip(decoder.convolutions, decoder.attention)):
            dst = states_rows if idx == n_conv - 1 else None
            residual = cur
            if att is None:
                cur = prog.conv(cur, f.conv, mode=1, spk=spk_of(f), res1=residual, y=dst)
                continue
            q_in = _Rows(prog.buf(B, C), C)                # x + frame position encoding
            prog.conv(cur, f.conv, mode=1, spk=spk_of(f), y2=q_in, y2_mode=2, yadd=pos_rows)
            q = prog.conv(q_in, att.query_projection)
            ctx = _Rows(prog.buf(B, E), E)
            first = ai == 0
            prog.attention(q, kv[ai][0], kv[ai][1], ctx, align_rows if first else None,
                           float(2 ** (n_att - 1)) / n_att, cursor(decoder.force_monotonic_attention[idx]),
                           att.window_backward, att.window_ahead, text_len, path)
            cur = prog.conv(ctx, att.out_projection, res1=q_in, res2=residual, y=dst)
            ai += 1
    xraw = _Rows(prog.buf(B, Fr), Fr)
    prog.conv(states_rows, decoder.last_conv, y=xraw,
              y2=_Rows(frames, Fr, ld=(Tmax + 1) * Fr, t=Fr, offset=Fr), y2_mode=1)
    prog.conv(xraw, decoder.fc, act=2, y=_Rows(dones, 1, ld=Tmax, t=1))
    return states, aligns, dones


def _decode(decoder, encoder_out, text_positions, speaker_embed, initial_input, test_inputs, use_graph,
            text_lengths=None, guide=None):
    """guide: (path int (B, n), steps [B]) -- the guided decode of ``decode_ragged``: the window centres of every step
    t < n and each row's step count."""
    if decoder.training:
        raise RuntimeError("incremental_forward only supports eval mode")     # reference conv.py:19-20
    if use_graph is None:
        use_graph = os.environ.get("DV3_INC_GRAPH", "1") == "1"
    keys, values = encoder_out
    if not keys.is_cuda:
        raise RuntimeError("incremental decoding runs on the GPU only (no CPU fallback)")
    B, Ts, E = keys.shape
    dev = keys.device
    ragged = text_lengths is not None
    if ragged:
        text_len = torch.as_tensor(text_lengths).to(device=dev, dtype=torch.int32).reshape(-1).contiguous()
        lens_host = text_len.tolist()
        if len(lens_host) != B or min(lens_host) < 1 or max(lens_host) > Ts:
            raise ValueError("text_lengths must hold B = %d lengths in [1, %d], got %s" % (B, Ts, lens_host))
    else:
        text_len = None
    Fr = decoder.in_dim * decoder.r
    with ops.overrides(conv_math="fp32"):       # one-off set-up GEMMs (projections) in exact fp32
        path = None
        if test_inputs is not None:
            test_inputs = test_inputs.to(torch.float32).contiguous()
            assert test_inputs.size(-1) == Fr
            Tmax = test_inputs.size(1)
        elif guide is not None:
            assert ragged
            path = torch.from_numpy(np.ascontiguousarray(guide[0], np.int32)).to(dev)
            Tmax = path.size(1)
        else:
            Tmax = decoder.max_decoder_steps + 1
        kv, pos_table, addend = _constants(decoder, keys, values, text_positions, speaker_embed, Tmax)

        def spk_of(f):
            s = addend(f)
            if s is None:
                return None
            prog.keep.append(s)
            return _Rows(s, s.size(-1))

        prog = StepProgram(B, dev)
        frames = prog.buf(B, Tmax + 1, Fr)                     # frame 0 = initial input, frame t+1 = output of step t
        if initial_input is not None:
            frames[:, 0] = initial_input.reshape(B, Fr)
        states, aligns, dones = _build_program(decoder, prog, Tmax, E, kv, pos_table, spk_of, text_len, frames,
                                               test_inputs, path)

    # ---- run ---------------------------------------------------------------------------------------
    def stop_steps(done):
        """-> steps per row once every row has stopped, else None (decode: all rows stop together)."""
        if ragged:
            steps = _row_stop_steps(done, decoder.min_decoder_steps, decoder.max_decoder_steps)
            return None if None in steps else steps
        n = _stop_step(done, decoder.min_decoder_steps, decoder.max_decoder_steps)
        return None if n is None else [n] * B

    if test_inputs is not None:
        prog.run(Tmax, use_graph)
        steps = [Tmax] * B
    elif guide is not None:
        prog.run(Tmax, use_graph)
        steps = [int(n) for n in guide[1]]
    else:
        steps, done_steps = None, 0
        while steps is None:
            n = min(CHECK_EVERY, Tmax - done_steps)
            prog.run(n, use_graph)
            done_steps += n
            steps = stop_steps(dones[:, :done_steps])
            assert steps is not None or done_steps < Tmax
    N = max(steps)
    if ragged:
        return (frames[:, 1:N + 1].contiguous(), aligns[:, :N].clone(), dones[:, :N].clone(),
                states[:, :N].contiguous(), steps)
    outputs = frames[:, 1:N + 1].contiguous()
    done_list = [dones[:, t].reshape(B, 1, 1).clone() for t in range(N)]
    return outputs, aligns[:, :N].clone(), done_list, states[:, :N].contiguous()


def _refill_table(entries, device):
    """[(dst tensor, src tensor or None, row_bytes, byte offset)] -> the Dv3IncRefill table on the device: row b is
    row_bytes from the offset of dst's b-th slice along dim 0; src (dst's shape) holds one row per refilled slot."""
    table = (Dv3IncRefill * len(entries))()
    for e, (dst, src, row_bytes, offset) in zip(table, entries):
        stride = dst.stride(0) * dst.element_size()
        assert dst.is_contiguous() and row_bytes % 4 == 0 and stride % 4 == 0 and offset % 4 == 0
        e.dst, e.row_bytes, e.dst_row_stride = dst.data_ptr() + offset, row_bytes, stride
        if src is not None:
            assert src.is_contiguous() and src.shape[1:] == dst.shape[1:] and src.dtype == dst.dtype
            e.src, e.src_row_stride = src.data_ptr(), stride
    return torch.frombuffer(bytearray(table), dtype=torch.uint8).to(device)


def _reset_entries(prog, frames):
    """Refill-table entries that return a slot of a slot program to the state of a fresh one: zero ring rows, cursors
    (int[2][B]), step counter and stop step, and a zero go frame frames[b, 0]."""
    B = prog.B
    entries = [(r, None, r[0].numel() * 4, 0) for r in prog.rings]
    entries += [(c, None, 4, half * B * 4) for c in prog.cursors for half in (0, 1)]
    return entries + [(prog.t, None, 4, 0), (prog.stop, None, 4, 0), (frames, None, frames.size(2) * 4, 0)]


@torch.no_grad()
def decode_stream(decoder, slots, requests, use_graph=None, stats=None, stage_timer=None, guided_steps=None):
    """Continuous batching: decode many utterances on a fixed set of ``slots`` decoder rows, refilling a row with the
    next waiting utterance as soon as its own one stops.

    requests: iterable of (request_id, keys (T, E), values (T, E), text_positions (T,), speaker_embed (D,) or None) --
    one utterance's encoder outputs -- consumed lazily, as slots free up.  Yields, in completion order,
    (request_id, outputs (N, in_dim*r), alignment (N, T), dones (N,), decoder_states (N, C), N): what ``decode`` gives
    for that utterance alone (free-running, from a zero go frame), bit for bit -- every step kernel computes row b from
    row b's own data at its own step t[b], and a refilled slot starts from the zeros of a fresh program.

    The step program is built and captured once, for ``slots`` rows with the longest text the key-position table holds
    and max_decoder_steps + 1 frames.  Every ``CHECK_EVERY`` steps the host reads the slots' stop steps (set on the
    device by the reference stop rule), gathers the finished utterances and reloads their slots in one launch.
    stats: optional dict, filled with "replays" (steps of the program), "useful_steps" (sum of N), "slots" and
    "refills" [(replays so far, slots reloaded, slots mid-decode)].  stage_timer: optional ``name -> context
    manager`` around the decoder work ("decoder"); pulling requests happens outside it.

    Guided decoding: requests of six entries, the last one the utterance's durations ((T,) integers >= 1, every
    request or none).  Each slot then carries its path row and step total (loaded by the same refill), attends as
    ``decode_ragged(..., durations=...)`` does and stops after exactly N = sum(durations) steps (``dv3_inc_stop_rows_total``);
    each utterance is what ``decode_ragged`` gives it with those durations.  The program is then sized for
    ``guided_steps`` steps -- the largest total, when the caller knows it -- or, by default, for the query-position
    table (``query_steps``); a request whose total exceeds that raises ValueError when it is loaded, and so does a
    guided_steps outside [1, query_steps]."""
    if decoder.training:
        raise RuntimeError("incremental_forward only supports eval mode")     # reference conv.py:19-20
    S = int(slots)
    if S < 1:
        raise ValueError("slots must be >= 1, got %r" % (slots,))
    if use_graph is None:
        use_graph = os.environ.get("DV3_INC_GRAPH", "1") == "1"
    stage = stage_timer or (lambda name: contextlib.nullcontext())
    it = iter(requests)
    waiting = []

    def take(n):
        got, waiting[:] = waiting[:n], waiting[n:]
        while len(got) < n:
            r = next(it, None)
            if r is None:
                break
            got.append(r)
        return got

    first = take(1)
    if not first:
        return
    waiting[:] = first
    keys0 = first[0][1]
    if not keys0.is_cuda:
        raise RuntimeError("incremental decoding runs on the GPU only (no CPU fallback)")
    dev, E = keys0.device, keys0.size(-1)
    multi = first[0][4] is not None
    guided = len(first[0]) > 5 and first[0][5] is not None
    Tp = decoder.embed_keys_positions.num_embeddings - 1      # the longest text: positions 1..Tp index the table
    if guided and guided_steps is not None and not 1 <= int(guided_steps) <= query_steps(decoder):
        raise ValueError("guided_steps=%r outside [1, %d]" % (guided_steps, query_steps(decoder)))
    Tmax = decoder.max_decoder_steps + 1 if not guided else \
        query_steps(decoder) if guided_steps is None else int(guided_steps)
    Fr = decoder.in_dim * decoder.r
    if stats is not None:
        stats.update(replays=0, useful_steps=0, slots=S, refills=[])

    def constants(reqs):
        """per-request constants of a group, padded to its longest text, in exact fp32 as ``_decode`` computes them"""
        G, L = len(reqs), max(r[1].size(0) for r in reqs)
        keys = torch.zeros(G, L, E, device=dev)
        values = torch.zeros(G, L, E, device=dev)
        tpos = torch.zeros(G, L, dtype=torch.long, device=dev)
        for g, r in enumerate(reqs):
            k, v, p = r[1:4]
            if (k.size(0) > Tp or (r[4] is not None) != multi or k.shape != v.shape
                    or p.shape != k.shape[:1] or (len(r) > 5 and r[5] is not None) != guided):
                raise ValueError("request %r: keys / values (T, %d), T <= %d, text_positions (T,), and a speaker "
                                 "embedding and durations for every request or for none" % (r[0], E, Tp))
            keys[g, :k.size(0)], values[g, :k.size(0)], tpos[g, :k.size(0)] = k, v, p
        spk = torch.stack([r[4] for r in reqs]) if multi else None
        with ops.overrides(conv_math="fp32"):
            kv, pos_table, addend = _constants(decoder, keys, values, tpos, spk, Tmax)
            return kv, pos_table, [addend(f) for f in spk_layers] if spk_layers else []

    # ---- the slot program: per-request constants live in slot buffers, loaded from staging by dv3_inc_refill ----
    spk_layers, spk_slot = [], []
    prog = StepProgram(S, dev, slots=True)
    text_len = torch.ones(S, dtype=torch.int32, device=dev)     # idle slots attend one (zero) key
    with stage("decoder"):
        kv0, pos0, _ = constants(first)                         # the shapes of the slot buffers
        kv_slot = [(torch.zeros(S, k.size(1), Tp, device=dev), torch.zeros(S, Tp, v.size(2), device=dev))
                   for k, v in kv0]
        pos_slot = torch.zeros(S, Tmax, pos0.size(-1), device=dev)
        # guided: each slot's window centres and step total (idle slots: token 0, held at step 0)
        path_slot = torch.zeros(S, Tmax, dtype=torch.int32, device=dev) if guided else None
        total_slot = torch.ones(S, dtype=torch.int32, device=dev) if guided else None

        def spk_of(f):
            if f.speaker_proj is None or not multi:
                return None
            buf = torch.zeros(S, f.speaker_proj.out_features, device=dev)
            spk_layers.append(f)
            spk_slot.append(buf)
            return _Rows(buf, buf.size(-1))

        with ops.overrides(conv_math="fp32"):
            frames = prog.buf(S, Tmax + 1, Fr)
            states, aligns, dones = _build_program(decoder, prog, Tmax, E, kv_slot, pos_slot, spk_of, text_len,
                                                   frames, path=path_slot)
        prog.keep += spk_slot
        if guided:
            prog.stop_rule_total(total_slot)
        else:
            prog.stop_rule(dones, decoder.min_decoder_steps, decoder.max_decoder_steps)

        # staging: row i holds the constants of the i-th slot of the next refill
        kv_stage = [(torch.zeros_like(k), torch.zeros_like(v)) for k, v in kv_slot]
        pos_stage, len_stage = torch.zeros_like(pos_slot), torch.ones_like(text_len)
        spk_stage = [torch.zeros_like(b) for b in spk_slot]
        slot_list = torch.zeros(S, dtype=torch.int32, device=dev)
        entries = _reset_entries(prog, frames)
        entries += [(text_len, len_stage, 4, 0), (pos_slot, pos_stage, pos_slot[0].numel() * 4, 0)]
        for (k, v), (ks, vs) in zip(kv_slot, kv_stage):
            entries += [(k, ks, k[0].numel() * 4, 0), (v, vs, v[0].numel() * 4, 0)]
        entries += [(b, bs, b[0].numel() * 4, 0) for b, bs in zip(spk_slot, spk_stage)]
        if guided:
            path_stage, total_stage = torch.zeros_like(path_slot), torch.ones_like(total_slot)
            entries += [(path_slot, path_stage, Tmax * 4, 0), (total_slot, total_stage, 4, 0)]
            prog.keep += [path_stage, total_stage]
        table = _refill_table(entries, dev)
        prog.keep += [table, slot_list, kv_stage, pos_stage, len_stage, spk_stage]

    occupant = [None] * S                                       # (request_id, text length) per slot
    replays = 0

    def load(free):
        """load the next waiting requests into the free slots (one refill launch); -> slots loaded"""
        reqs = take(len(free))
        if not reqs:
            return []
        if guided:
            durs = check_durations([r[5] if len(r) > 5 else None for r in reqs], [r[1].size(0) for r in reqs])
            path, totals = path_table(durs, Tmax)
            if max(totals) > Tmax:
                raise ValueError("request %r: durations total %d decoder steps; the program holds %d"
                                 % (reqs[int(np.argmax(totals))][0], max(totals), Tmax))
        with stage("decoder"):
            kv, pos, spk = constants(reqs)
            G = len(reqs)
            for (k, v), (ks, vs) in zip(kv, kv_stage):
                ks[:G, :, :k.size(2)] = k
                vs[:G, :v.size(1)] = v
            pos_stage[:G] = pos
            for s, ss in zip(spk, spk_stage):
                ss[:G] = s
            lens = [r[1].size(0) for r in reqs]
            len_stage[:G] = torch.tensor(lens, dtype=torch.int32)
            if guided:
                path_stage[:G] = torch.from_numpy(path.astype(np.int32))
                total_stage[:G] = torch.tensor(totals, dtype=torch.int32)
            slot_list[:G] = torch.tensor(free[:G], dtype=torch.int32)
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            lib.call("dv3_inc_refill", ctypes.c_void_p(table.data_ptr()), len(entries),
                     ctypes.c_void_p(slot_list.data_ptr()), G, st)
        for b, r, n in zip(free, reqs, lens):
            occupant[b] = (r[0], n)
        return free[:G]

    load(list(range(S)))
    while any(o is not None for o in occupant):
        with stage("decoder"):
            prog.run(CHECK_EVERY, use_graph)
            replays += CHECK_EVERY
            stop = prog.stop.tolist()
        free = []
        for b in range(S):
            if occupant[b] is None or stop[b] <= 0:
                continue
            rid, L = occupant[b]
            n = stop[b]
            out = (rid, frames[b, 1:n + 1].clone(), aligns[b, :n, :L].clone(), dones[b, :n].clone(),
                   states[b, :n].clone(), n)
            occupant[b] = None
            free.append(b)
            if stats is not None:
                stats["useful_steps"] += n
            yield out
        if free:
            busy = sum(o is not None for o in occupant)
            loaded = load(free)
            if stats is not None and loaded:
                stats["refills"].append((replays, loaded, busy))
        if stats is not None:
            stats["replays"] = replays
