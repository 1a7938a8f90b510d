"""DeepVoice3 networks with the reference's classes, constructor arguments, attribute names and
``forward`` signatures (reference deepvoice3_pytorch/deepvoice3.py), running on the dv3b200 kernels.

Internally the teacher-forced path stays in the channel-major (B, C, T) layout end to end: the attention
layer consumes queries/keys/values as (B, E, T) so the reference's per-layer transposes disappear; the
public ``forward`` methods still take and return the reference's (B, T, C) tensors.
"""
import math

import torch
from torch import nn

from . import ops
from .modules import (Conv1d, ConvTranspose1d, Embedding, Linear, SinusoidalEncoding, Conv1dGLU,
                      get_mask_from_lengths, mask_conv_input, run_conv_stack)

SQRT_HALF = math.sqrt(0.5)


def expand_speaker_embed(inputs_btc, speaker_embed=None, tdim=1):
    """(B, N) -> (B, T, N) stride-0 expansion over the time axis of ``inputs`` (reference deepvoice3.py:13-21)."""
    if speaker_embed is None:
        return None
    ss = speaker_embed.size()
    return speaker_embed.unsqueeze(1).expand(ss[0], inputs_btc.size(tdim), ss[-1])


def _conv_recipe(in_channels, convolutions, n_speakers, speaker_embed_dim, causal, residual, dropout):
    """1x1 Conv1d + ReLU whenever the width changes, then a Conv1dGLU per entry; std_mul follows
    the reference's 1.0 -> 2.0 -> 4.0 progression (deepvoice3.py:44-61, 214-231, 553-569)."""
    layers, std_mul = [], 1.0
    for (out_channels, kernel_size, dilation) in convolutions:
        if in_channels != out_channels:
            layers.append(Conv1d(in_channels, out_channels, kernel_size=1, padding=0, dilation=1,
                                 std_mul=std_mul))
            layers.append(nn.ReLU(inplace=True))
            in_channels = out_channels
            std_mul = 2.0
        layers.append(Conv1dGLU(n_speakers, speaker_embed_dim, in_channels, out_channels, kernel_size,
                                causal=causal, dilation=dilation, dropout=dropout, std_mul=std_mul,
                                residual=residual))
        in_channels = out_channels
        std_mul = 4.0
    return layers, in_channels, std_mul


class Encoder(nn.Module):
    def __init__(self, n_vocab, embed_dim, n_speakers, speaker_embed_dim, padding_idx=None,
                 embedding_weight_std=0.1, convolutions=((64, 5, .1),) * 7, max_positions=512, dropout=0.1,
                 apply_grad_scaling=False):
        super().__init__()
        if apply_grad_scaling:
            raise NotImplementedError("apply_grad_scaling is dead code in the reference (GradMultiply uses "
                                      "removed autograd APIs, modules.py:67-77) and no builder enables it")
        self.dropout = dropout
        self.num_attention_layers = None
        self.apply_grad_scaling = apply_grad_scaling
        self.embed_tokens = Embedding(n_vocab, embed_dim, padding_idx, embedding_weight_std)
        if n_speakers > 1:
            self.speaker_fc1 = Linear(speaker_embed_dim, embed_dim, dropout=dropout)
            self.speaker_fc2 = Linear(speaker_embed_dim, embed_dim, dropout=dropout)
        self.n_speakers = n_speakers
        layers, in_channels, std_mul = _conv_recipe(embed_dim, convolutions, n_speakers, speaker_embed_dim,
                                                    causal=False, residual=True, dropout=dropout)
        layers.append(Conv1d(in_channels, embed_dim, kernel_size=1, padding=0, dilation=1, std_mul=std_mul,
                             dropout=dropout))
        self.convolutions = nn.ModuleList(layers)

    def grad_bucket_splits(self):
        """[(tag, index into ``convolutions``)]: layers [index, next index) form one gradient bucket of the
        data-parallel step.  The encoder holds 60 % of the parameters and its backward runs last, from the last layer
        down: "encoder_hi" is final (and its all-reduce starts) two thirds into the encoder's backward, "encoder_mid"
        shortly before its end; only the first layers are left for the exposed bucket."""
        n = len(self.convolutions)
        hi, mid = n * 3 // 5, n // 4
        return [("encoder_hi", hi), ("encoder_mid", mid)] if 0 < mid < hi < n else []

    def forward(self, text_sequences, text_positions=None, lengths=None, speaker_embed=None):
        """-> keys, values, both (B, T_text, embed_dim) (reference deepvoice3.py:69-105)."""
        assert self.n_speakers == 1 or speaker_embed is not None
        x = self.embed_tokens(text_sequences.long())
        x = ops.dropout(x, self.dropout, self.training)
        speaker_embed_btc = expand_speaker_embed(x, speaker_embed)
        if speaker_embed_btc is not None:
            speaker_embed_btc = ops.speaker_dropout(speaker_embed_btc, self.dropout, self.training)
            x = ops.speaker_residual(x, self.speaker_fc1, speaker_embed_btc)
        input_embedding = x
        x = run_conv_stack(self.convolutions, ops.transpose12(x), speaker_embed_btc,
                           boundaries={i: tag for tag, i in self.grad_bucket_splits()})
        keys = ops.transpose12(x)
        if speaker_embed_btc is not None:
            keys = ops.speaker_residual(keys, self.speaker_fc2, speaker_embed_btc)
        values = (keys + input_embedding) * SQRT_HALF
        return keys, values


class AttentionLayer(nn.Module):
    def __init__(self, conv_channels, embed_dim, dropout=0.1, window_ahead=3, window_backward=1,
                 key_projection=True, value_projection=True):
        super().__init__()
        self.query_projection = Linear(conv_channels, embed_dim)
        if key_projection:
            self.key_projection = Linear(embed_dim, embed_dim)
            # The reference tries to share the q/k init here (deepvoice3.py:118-119) but assigns to the
            # weight-norm-derived ``.weight``, which the pre-hook overwrites: a no-op, deliberately not "fixed".
        else:
            self.key_projection = None
        self.value_projection = Linear(embed_dim, embed_dim) if value_projection else None
        self.out_projection = Linear(embed_dim, conv_channels)
        self.dropout = dropout
        self.window_ahead = window_ahead
        self.window_backward = window_backward

    def forward_bct(self, query_bct, keys_bct, values_bct, mask=None):
        """Channel-major core: query (B,C,Td), keys (B,E,Ts), values (B,E,Ts) -> (B,C,Td), probs (B,Td,Ts).
        No 1/sqrt(d) scaling, -inf mask on padded keys, probabilities returned pre-dropout, context scaled
        by Ts*sqrt(1/Ts), output (x + residual)*sqrt(.5) -- reference deepvoice3.py:132-176."""
        v = values_bct if self.value_projection is None else self.value_projection.forward_bct(values_bct)
        k = keys_bct if self.key_projection is None else self.key_projection.forward_bct(keys_bct)
        q = self.query_projection.forward_bct(query_bct)
        ctx, probs = ops.attention_core(q, k, v, mask, self.dropout, self.training)
        x = self.out_projection.forward_bct(ctx)
        return (x + query_bct) * SQRT_HALF, probs

    def forward(self, query, encoder_out, mask=None, last_attended=None):
        """Reference signature: query (B,Td,C); encoder_out = (keys (B,E,Ts) pre-transposed, values (B,Ts,E))."""
        keys, values = encoder_out
        if last_attended is not None:
            # reference deepvoice3.py:150-156: scores outside [last_attended - window_backward, last_attended +
            # window_ahead) are set to -inf.  The window is the same for every query row, so it folds into the key mask.
            Ts = keys.size(-1)
            s = torch.arange(Ts, device=keys.device)
            backward, ahead = last_attended - self.window_backward, last_attended + self.window_ahead
            win = torch.zeros(Ts, dtype=torch.bool, device=keys.device)
            if backward > 0:
                win |= s < backward
            if ahead < Ts:
                win |= s >= ahead
            win = win[None, :].expand(keys.size(0), Ts)
            mask = win if mask is None else (mask.bool() | win)
        x, probs = self.forward_bct(ops.transpose12(query), keys, ops.transpose12(values), mask)
        return ops.transpose12(x), probs


class Decoder(nn.Module):
    def __init__(self, embed_dim, n_speakers, speaker_embed_dim, in_dim=80, r=5, max_positions=512,
                 padding_idx=None, preattention=((128, 5, 1),) * 4, convolutions=((128, 5, 1),) * 4,
                 attention=True, dropout=0.1, use_memory_mask=False, force_monotonic_attention=False,
                 query_position_rate=1.0, key_position_rate=1.29, window_ahead=3, window_backward=1,
                 key_projection=True, value_projection=True):
        super().__init__()
        self.dropout = dropout
        self.in_dim = in_dim
        self.r = r
        self.query_position_rate = query_position_rate
        self.key_position_rate = key_position_rate
        if isinstance(attention, bool):
            attention = [attention] * len(convolutions)

        self.embed_query_positions = SinusoidalEncoding(max_positions, convolutions[0][0])
        self.embed_keys_positions = SinusoidalEncoding(max_positions, embed_dim)
        if n_speakers > 1:
            self.speaker_proj1 = Linear(speaker_embed_dim, 1, dropout=dropout)
            self.speaker_proj2 = Linear(speaker_embed_dim, 1, dropout=dropout)
        else:
            self.speaker_proj1, self.speaker_proj2 = None, None

        layers, in_channels, std_mul = _conv_recipe(in_dim * r, preattention, n_speakers, speaker_embed_dim,
                                                    causal=True, residual=True, dropout=dropout)
        self.preattention = nn.ModuleList(layers)

        self.convolutions = nn.ModuleList()
        self.attention = nn.ModuleList()
        for i, (out_channels, kernel_size, dilation) in enumerate(convolutions):
            assert in_channels == out_channels
            self.convolutions.append(
                Conv1dGLU(n_speakers, speaker_embed_dim, in_channels, out_channels, kernel_size, causal=True,
                          dilation=dilation, dropout=dropout, std_mul=std_mul, residual=False))
            self.attention.append(
                AttentionLayer(out_channels, embed_dim, dropout=dropout, window_ahead=window_ahead,
                               window_backward=window_backward, key_projection=key_projection,
                               value_projection=value_projection) if attention[i] else None)
            in_channels = out_channels
            std_mul = 4.0
        self.last_conv = Conv1d(in_channels, in_dim * r, kernel_size=1, padding=0, dilation=1, std_mul=std_mul,
                                dropout=dropout)
        self.fc = Linear(in_dim * r, 1)

        self.max_decoder_steps = 200
        self.min_decoder_steps = 10
        self.use_memory_mask = use_memory_mask
        if isinstance(force_monotonic_attention, bool):
            self.force_monotonic_attention = [force_monotonic_attention] * len(convolutions)
        else:
            self.force_monotonic_attention = force_monotonic_attention

    def _position_rate(self, rate, proj, speaker_embed):
        if proj is None:
            return rate
        return rate * torch.sigmoid(proj(speaker_embed)).view(-1)

    def forward(self, encoder_out, inputs=None, text_positions=None, frame_positions=None, speaker_embed=None,
                lengths=None):
        """Teacher-forced decoder (reference deepvoice3.py:277-365).
        -> outputs (B,T,in_dim*r), alignments (N_attn,B,T,T_text), done (B,T,1), decoder_states (B,T,C)."""
        if inputs is None:                 # inference: autoregressive decoding (reference deepvoice3.py:280-284)
            assert text_positions is not None
            self.start_fresh_sequence()
            return self.incremental_forward(encoder_out, text_positions, speaker_embed)
        if inputs.size(-1) == self.in_dim:
            inputs = inputs.reshape(inputs.size(0), inputs.size(1) // self.r, -1)
        assert inputs.size(-1) == self.in_dim * self.r

        speaker_embed_btc = expand_speaker_embed(inputs, speaker_embed)
        if speaker_embed_btc is not None:
            speaker_embed_btc = ops.speaker_dropout(speaker_embed_btc, self.dropout, self.training)

        keys, values = encoder_out
        mask = get_mask_from_lengths(keys, lengths) if (self.use_memory_mask and lengths is not None) else None

        if text_positions is not None:
            w = self._position_rate(self.key_position_rate, self.speaker_proj1, speaker_embed)
            keys = keys + self.embed_keys_positions(text_positions, w)
        frame_pos_bct = None
        if frame_positions is not None:
            w = self._position_rate(self.query_position_rate, self.speaker_proj2, speaker_embed)
            frame_pos_bct = ops.transpose12(self.embed_query_positions(frame_positions, w))

        keys_bct = ops.transpose12(keys)          # the reference's "transpose only once"
        values_bct = ops.transpose12(values)

        x = ops.dropout(inputs, self.dropout, self.training)
        x = run_conv_stack(self.preattention, ops.transpose12(x), speaker_embed_btc)

        alignments = []
        for f, attention in zip(self.convolutions, self.attention):
            if attention is None:
                # x = (f(x) + x) * sqrt(.5): the block kernel's own residual epilogue
                x = f(x, speaker_embed_btc, fuse_residual=True)
                continue
            residual = x
            x = f(x, speaker_embed_btc)
            q = x if frame_pos_bct is None else x + frame_pos_bct
            x, alignment = attention.forward_bct(q, keys_bct, values_bct, mask)
            alignments.append(alignment)
            x = (x + residual) * SQRT_HALF

        decoder_states = ops.transpose12(x)
        x = ops.transpose12(self.last_conv(x))
        outputs = torch.sigmoid(x)
        done = torch.sigmoid(self.fc(x))
        return outputs, torch.stack(alignments), done, decoder_states

    def incremental_forward(self, encoder_out, text_positions, speaker_embed=None, initial_input=None,
                            test_inputs=None):
        """Autoregressive decoding (reference deepvoice3.py:367-485) as a CUDA-graph-replayed step program;
        see incremental.py.  -> outputs (B,N,in_dim*r), alignments (B,N,T_text), dones [N x (B,1,1)], states."""
        from .incremental import decode
        return decode(self, encoder_out, text_positions, speaker_embed, initial_input, test_inputs)

    def start_fresh_sequence(self):
        """All step state (ring buffers, cursors) is created per incremental_forward call; only the module-level
        steppers need clearing (reference deepvoice3.py:487-490)."""
        for m in list(self.preattention) + list(self.convolutions) + [self.last_conv]:
            if hasattr(m, "clear_buffer"):
                m.clear_buffer()


class Converter(nn.Module):
    def __init__(self, n_speakers, speaker_embed_dim, in_dim, out_dim, convolutions=((256, 5, 1),) * 4,
                 time_upsampling=1, dropout=0.1):
        super().__init__()
        self.dropout = dropout
        self.in_dim = in_dim
        self.out_dim = out_dim
        self.n_speakers = n_speakers
        c = convolutions[0][0]

        def glu(dilation, std_mul):
            return Conv1dGLU(n_speakers, speaker_embed_dim, c, c, kernel_size=3, causal=False,
                             dilation=dilation, dropout=dropout, std_mul=std_mul, residual=True)

        def up(std_mul):
            return ConvTranspose1d(c, c, kernel_size=2, padding=0, stride=2, std_mul=std_mul)

        head = [Conv1d(in_dim, c, kernel_size=1, padding=0, dilation=1, std_mul=1.0)]
        if time_upsampling == 4:      # reference deepvoice3.py:515-534
            head += [up(1.0), glu(1, 1.0), glu(3, 4.0), up(4.0), glu(1, 1.0), glu(3, 4.0)]
        elif time_upsampling == 2:    # :535-546
            head += [up(1.0), glu(1, 1.0), glu(3, 4.0)]
        elif time_upsampling == 1:    # :547-554
            head += [glu(3, 4.0)]
        else:
            raise ValueError("Not supported")
        # the tail restarts the std_mul progression at 4.0 (reference deepvoice3.py:558)
        tail, std_mul, in_channels = [], 4.0, c
        for (out_channels, kernel_size, dilation) in convolutions:
            if in_channels != out_channels:
                tail.append(Conv1d(in_channels, out_channels, kernel_size=1, padding=0, dilation=1,
                                   std_mul=std_mul))
                tail.append(nn.ReLU(inplace=True))
                in_channels = out_channels
                std_mul = 2.0
            tail.append(Conv1dGLU(n_speakers, speaker_embed_dim, in_channels, out_channels, kernel_size,
                                  causal=False, dilation=dilation, dropout=dropout, std_mul=std_mul,
                                  residual=True))
            in_channels = out_channels
            std_mul = 4.0
        tail.append(Conv1d(in_channels, out_dim, kernel_size=1, padding=0, dilation=1, std_mul=std_mul,
                           dropout=dropout))
        self.convolutions = nn.ModuleList(head + tail)

    @ops.forward_scope
    def forward(self, x, speaker_embed=None):
        """x (B, T, in_dim) -> (B, T*upsampling, out_dim) (reference deepvoice3.py:582-604)."""
        assert self.n_speakers == 1 or speaker_embed is not None
        x = ops.transpose12(x)
        layers = list(self.convolutions)
        # The speaker embedding is re-expanded (and re-dropped) whenever the time axis grows
        # (reference deepvoice3.py:595-598), so run the stack in segments of constant T.
        i = 0
        while i < len(layers):
            if _is_upsampler(layers[i]):
                x = layers[i](mask_conv_input(layers[i], x), extent=ops.extent_frames(x))
                i += 1
                continue
            j = i
            while j < len(layers) and not _is_upsampler(layers[j]):
                j += 1
            spk = expand_speaker_embed(x, speaker_embed, tdim=-1)
            if spk is not None:
                spk = ops.speaker_dropout(spk, self.dropout, self.training)
            x = run_conv_stack(layers[i:j], x, spk)
            i = j
        return torch.sigmoid(ops.transpose12(x))


def _is_upsampler(m):
    from .conv import ConvTranspose1d as _CT
    return isinstance(m, _CT)
