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
"""
import ctypes
import os

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
    """The launch sequence of one decoder step + its device-resident state."""

    def __init__(self, B, device):
        self.B, self.dev = B, device
        self.calls = []                     # (entry point name, ctypes struct, extra arguments)
        self.keep = []                      # tensors the structs point into
        self.t = torch.zeros(1, dtype=torch.int32, device=device)
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
        self.calls.append(("dv3_inc_conv_step", s, ()))
        return y

    def attention(self, q, keys_bet, values_bte, ctx, align, align_scale, last_attended, window_backward, window_ahead,
                  text_len=None):
        """text_len: int32 (B,) device tensor -> the per-row (ragged) step, last_attended then holds [2][B] cursors."""
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
        if text_len is None:
            self.calls.append(("dv3_inc_attn_step", a, ()))
        else:
            self.keep.append(text_len)
            self.calls.append(("dv3_inc_attn_step_rows", a, (ctypes.c_void_p(text_len.data_ptr()),)))

    # -- execution --------------------------------------------------------------------------------
    def _launch_step(self):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        for name, s, extra in self.calls:
            lib.call(name, ctypes.byref(s), *extra, st)
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


@torch.no_grad()
def decode_ragged(decoder, encoder_out, text_positions, text_lengths, speaker_embed=None, initial_input=None,
                  test_inputs=None, use_graph=None):
    """Batched decode of rows with text_lengths (B,) valid keys each (encoder outputs padded to T_text).
    -> outputs (B, N, in_dim*r), alignments (B, N, T_text), dones (B, N), decoder_states (B, N, C), steps [B]:
    row b is valid for its first steps[b] decoder steps (and its first text_lengths[b] alignment columns; the rest are
    0) and there equals ``decode`` run on that row alone with its encoder outputs cut to text_lengths[b].  Free-running,
    row b stops by the reference rule applied to its own done flags; rows that stopped keep computing until the last
    one does, their extra frames are not part of the result.  Teacher-forced (test_inputs (B, N, in_dim*r)), every row
    runs N steps."""
    return _decode(decoder, encoder_out, text_positions, speaker_embed, initial_input, test_inputs, use_graph,
                   text_lengths=text_lengths)


def _decode(decoder, encoder_out, text_positions, speaker_embed, initial_input, test_inputs, use_graph,
            text_lengths=None):
    if decoder.training:
        raise RuntimeError("incremental_forward only supports eval mode")     # reference conv.py:19-20
    if use_graph is None:
        use_graph = os.environ.get("DV3_INC_GRAPH", "1") == "1"
    nyanko = hasattr(decoder, "audio_encoder_modules")
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
    old_math = ops.conv_math
    ops.conv_math = "fp32"                       # one-off set-up GEMMs (projections) in exact fp32
    try:
        # ---- per-utterance constants --------------------------------------------------------------
        if nyanko:
            if text_positions is not None:
                keys = keys + decoder.embed_keys_positions(text_positions)
        else:
            w = decoder._position_rate(decoder.key_position_rate, decoder.speaker_proj1, speaker_embed)
            keys = keys + decoder.embed_keys_positions(text_positions, w)
        if test_inputs is not None:
            test_inputs = test_inputs.to(torch.float32).contiguous()
            assert test_inputs.size(-1) == Fr
            Tmax = test_inputs.size(1)
        else:
            Tmax = decoder.max_decoder_steps + 1
        frame_pos = torch.arange(1, Tmax + 1, device=dev).view(1, -1).repeat(B, 1)
        if nyanko:
            pos_table = decoder.embed_query_positions(frame_pos)
        else:
            w2 = decoder._position_rate(decoder.query_position_rate, decoder.speaker_proj2, speaker_embed)
            pos_table = decoder.embed_query_positions(frame_pos, w2)
        pos_table = pos_table.contiguous()                     # (B, Tmax, C)
        C = pos_table.size(-1)
        att_layers = [decoder.attention] if nyanko else [a for a in decoder.attention if a is not None]
        kv = []
        for att in att_layers:
            k_ = keys if att.key_projection is None else att.key_projection(keys)
            v_ = values if att.value_projection is None else att.value_projection(values)
            kv.append((k_.transpose(1, 2).contiguous(), v_.contiguous()))

        def spk_of(f):
            if f.speaker_proj is None or speaker_embed is None:
                return None
            s = torch.nn.functional.softsign(f.speaker_proj(speaker_embed)).contiguous()     # (B, C)
            prog.keep.append(s)
            return _Rows(s, s.size(-1))

        # ---- the step program ---------------------------------------------------------------------
        prog = StepProgram(B, dev)
        prog.keep += [pos_table]
        frames = prog.buf(B, Tmax + 1, Fr)                     # frame 0 = initial input, frame t+1 = output of step t
        if initial_input is not None:
            frames[:, 0] = initial_input.reshape(B, Fr)
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
            if not force:
                return None
            la = torch.zeros(2 * B if ragged else 2, dtype=torch.int32, device=dev)
            prog.keep.append(la)
            return la

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
                           att.window_backward, att.window_ahead, text_len)
            prog.conv(ctx, att.out_projection, res1=q_in, y=_Rows(cat, D, ld=2 * D))
            cur = _run_stack(prog, decoder.audio_decoder_modules, _Rows(cat, 2 * D), last_y=states_rows)
        else:
            cur = _run_stack(prog, decoder.preattention, cur, spk_of)
            n_att = len(att_layers)
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
                               att.window_backward, att.window_ahead, text_len)
                cur = prog.conv(ctx, att.out_projection, res1=q_in, res2=residual, y=dst)
                ai += 1
        xraw = _Rows(prog.buf(B, Fr), Fr)
        prog.conv(states_rows, decoder.last_conv, y=xraw,
                  y2=_Rows(frames, Fr, ld=(Tmax + 1) * Fr, t=Fr, offset=Fr), y2_mode=1)
        prog.conv(xraw, decoder.fc, act=2, y=_Rows(dones, 1, ld=Tmax, t=1))
    finally:
        ops.conv_math = old_math

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
