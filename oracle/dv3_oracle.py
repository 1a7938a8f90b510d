"""TEST INFRASTRUCTURE ONLY.  Functional CPU restatement of the reference's training-time forward.

Everything is a pure function of a reference-keyed ``state_dict`` (old-style weight-norm keys
``*.weight_g`` / ``*.weight_v``), a spec from ``oracle/specs.py`` and the inputs; gradients come from
torch autograd on CPU.  Works in fp32 (the parity target) or fp64 (error yardstick).
Dropout is not drawn here: parity runs use dropout=0 exactly as the reference's own incremental
tests do with ``.eval()`` (reference tests/test_deepvoice3.py:184-235).  ``conv1d_glu``,
``highway_conv1d`` and ``attention_core`` take an optional explicit multiplicative mask ``drop``
(0 or 1/(1-p) per element, e.g. ``oracle/dropout_mask.py``'s restatement of the device mask) at the
reference's dropout site: the conv input only (the residual / highway carry stay unmasked), and
the attention probabilities after they are returned, before P.V.  ``drop=None`` is the
dropout-free forward, unchanged.

PARITY: pinned.  ``tests/golden/make_golden.py`` runs the live reference modules
(/root/reference/deepvoice3_pytorch, importable in the build container) and stores their outputs;
``tests/test_oracle_golden.py`` checks every function below against those vectors.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

SQRT_HALF = math.sqrt(0.5)


# ----------------------------------------------------------------------------------------------
# leaf ops
# ----------------------------------------------------------------------------------------------
def weight_norm(v, g):
    """w = g * v / ||v||, norm over every dim but 0 (torch.nn.utils.weight_norm, dim=0), as applied
    by the factories at reference modules.py:80-85 (Linear), 94-100 (Conv1d), 103-109
    (ConvTranspose1d -- dim 0 is the *input* channel there)."""
    dims = tuple(range(1, v.dim()))
    return g * v / v.pow(2).sum(dims, keepdim=True).sqrt()


def _w(sd, prefix):
    return weight_norm(sd[prefix + ".weight_v"], sd[prefix + ".weight_g"])


def linear(sd, prefix, x):
    """reference modules.py:80-85; x (..., Cin) -> (..., Cout)."""
    return F.linear(x, _w(sd, prefix), sd[prefix + ".bias"])


def conv1d(sd, prefix, x, k=1, dilation=1, causal=False):
    """reference conv.py:7-15 (training forward = nn.Conv1d.forward); x (B, Cin, T).
    causal: pad (k-1)*d both sides and keep the first T (modules.py:126,155) == left pad only."""
    T = x.size(-1)
    pad = (k - 1) * dilation if causal else (k - 1) // 2 * dilation
    y = F.conv1d(x, _w(sd, prefix), sd[prefix + ".bias"], padding=pad, dilation=dilation)
    return y[:, :, :T] if causal else y


def conv_transpose1d(sd, prefix, x):
    """reference modules.py:103-109, k=2, stride=2: (B, Cin, T) -> (B, Cout, 2T)."""
    return F.conv_transpose1d(x, _w(sd, prefix), sd[prefix + ".bias"], stride=2)


def conv1d_glu(sd, prefix, x, k, dilation, causal, residual, speaker_embed_btc=None, drop=None):
    """reference modules.py:145-164; ``drop`` (B,C,T) multiplies the conv input only (modules.py:147)."""
    y = conv1d(sd, prefix + ".conv", x if drop is None else x * drop, k, dilation, causal)
    a, b = y.split(y.size(1) // 2, dim=1)
    if (prefix + ".speaker_proj.weight_v") in sd:
        a = a + F.softsign(linear(sd, prefix + ".speaker_proj", speaker_embed_btc)).transpose(1, 2)
    y = a * torch.sigmoid(b)
    return (y + x) * SQRT_HALF if residual else y


def highway_conv1d(sd, prefix, x, k, dilation, causal, drop=None):
    """reference modules.py:200-226, glu=False branch (the only one the builders use); ``drop`` (B,C,T)
    multiplies the conv input only (modules.py:214), the carry (1 - t) * x takes x unmasked."""
    y = conv1d(sd, prefix + ".conv", x if drop is None else x * drop, k, dilation, causal)
    a, b = y.split(y.size(1) // 2, dim=1)
    t = torch.sigmoid(b)
    return t * a + (1 - t) * x


def position_table(n_position, d, position_rate=1.0, sinusoidal=True, dtype=torch.float32):
    """reference modules.py:10-24: table[pos,i] = rate*pos / 10000^(2(i//2)/d), row 0 zero; computed
    in float64 and cast to float32 (numpy -> .float()), sin on even / cos on odd columns of rows>=1."""
    pos = np.arange(n_position, dtype=np.float64)[:, None]
    i = np.arange(d)
    tab = position_rate * pos / np.power(10000.0, 2 * (i // 2) / d)[None, :]
    tab[0] = 0.0
    tab = torch.from_numpy(tab).float()
    if sinusoidal:
        tab[1:, 0::2] = torch.sin(tab[1:, 0::2])
        tab[1:, 1::2] = torch.cos(tab[1:, 1::2])
    return tab.to(dtype)


def sinusoidal_encoding(table, positions, w):
    """reference modules.py:27-31,45-64: y = w*table, sin/cos on rows >= 1, then an embedding lookup.
    ``w`` is a python scalar, or a (B,) tensor (one rate per utterance -- multi-speaker)."""
    def enc(wi):
        y = wi * table
        y = torch.cat([y[:1], torch.stack([torch.sin(y[1:, 0::2]), torch.cos(y[1:, 1::2])],
                                          dim=-1).flatten(1)], dim=0)
        return y
    # padding_idx only matters for the gradient (row 0 gets none), reference modules.py:40
    if np.isscalar(w) or w.numel() == 1:
        return F.embedding(positions, enc(w), padding_idx=0)
    return torch.stack([F.embedding(positions[b], enc(w[b]), padding_idx=0)
                        for b in range(w.numel())])


def memory_mask(lengths, max_len=None):
    """reference modules.py:232-241: True where the text position is padding."""
    lengths = torch.as_tensor(np.asarray(lengths))
    max_len = int(lengths.max()) if max_len is None else max_len
    return ~(torch.arange(max_len)[None, :] < lengths[:, None])


def attention_core(query, keys_bct, values, mask=None, drop=None):
    """reference deepvoice3.py:142-171 between the projections: query (B,Td,E); keys_bct (B,E,Ts);
    values (B,Ts,E); mask (B,Ts) bool, True = padding; drop (B,Td,Ts) multiplies the probabilities
    after they are returned and before P.V (deepvoice3.py:161-165).  -> (context (B,Td,E), probs)."""
    x = torch.bmm(query, keys_bct)  # no 1/sqrt(d)
    if mask is not None:
        x = x.masked_fill(mask[:, None, :], -float("inf"))
    probs = F.softmax(x, dim=-1)
    x = torch.bmm(probs if drop is None else probs * drop, values)
    s = values.size(1)
    return x * (s * math.sqrt(1.0 / s)), probs


def attention_layer(sd, prefix, query, keys_bct, values, mask=None):
    """reference deepvoice3.py:132-176 (training path; no window, dropout omitted).
    query (B,Td,C); keys_bct (B,E,Ts) pre-transposed; values (B,Ts,E); mask (B,Ts) bool."""
    residual = query
    if (prefix + ".value_projection.weight_v") in sd:
        values = linear(sd, prefix + ".value_projection", values)
    if (prefix + ".key_projection.weight_v") in sd:
        keys_bct = linear(sd, prefix + ".key_projection", keys_bct.transpose(1, 2)).transpose(1, 2)
    x, probs = attention_core(linear(sd, prefix + ".query_projection", query), keys_bct, values, mask)
    x = linear(sd, prefix + ".out_projection", x)
    return (x + residual) * SQRT_HALF, probs


def run_stack(sd, prefix, layers, x, speaker_embed=None, dropout_reexpand=True):
    """Run a spec layer list on x (B,C,T).  The speaker embedding (B,S) is re-expanded over the
    current T before each GLU block (reference deepvoice3.py:13-21, 595-598)."""
    for layer in layers:
        kind, idx = layer[0], layer[1]
        p = "%s.%d" % (prefix, idx)
        if kind == "conv":
            x = conv1d(sd, p, x, layer[4], layer[5])
        elif kind == "convT":
            x = conv_transpose1d(sd, p, x)
        elif kind == "relu":
            x = F.relu(x)
        elif kind == "sigmoid":
            x = torch.sigmoid(x)
        elif kind == "glu":
            _, _, C, k, d, causal, residual = layer
            spk = None
            if speaker_embed is not None:
                spk = speaker_embed[:, None, :].expand(-1, x.size(-1), -1)
            x = conv1d_glu(sd, p, x, k, d, causal, residual, spk)
        elif kind == "hw":
            _, _, C, k, d, causal = layer
            x = highway_conv1d(sd, p, x, k, d, causal)
        else:
            raise ValueError(kind)
    return x


# ----------------------------------------------------------------------------------------------
# networks
# ----------------------------------------------------------------------------------------------
def dv3_encoder(sd, spec, text, speaker_embed=None, prefix="seq2seq.encoder"):
    """reference deepvoice3.py:69-105."""
    x = F.embedding(text.long(), sd[prefix + ".embed_tokens.weight"], padding_idx=spec["padding_idx"])
    spk_btc = None
    if speaker_embed is not None:
        spk_btc = speaker_embed[:, None, :].expand(-1, x.size(1), -1)
        x = x + F.softsign(linear(sd, prefix + ".speaker_fc1", spk_btc))
    input_embedding = x
    x = run_stack(sd, prefix + ".convolutions", spec["encoder"], x.transpose(1, 2), speaker_embed)
    keys = x.transpose(1, 2)
    if spk_btc is not None:
        keys = keys + F.softsign(linear(sd, prefix + ".speaker_fc2", spk_btc))
    values = (keys + input_embedding) * SQRT_HALF
    return keys, values


def dv3_decoder(sd, spec, encoder_out, inputs, text_positions=None, frame_positions=None,
                speaker_embed=None, lengths=None, prefix="seq2seq.decoder"):
    """reference deepvoice3.py:277-365 (teacher-forced forward)."""
    in_dim, r = spec["mel_dim"], spec["r"]
    if inputs.size(-1) == in_dim:
        inputs = inputs.reshape(inputs.size(0), inputs.size(1) // r, -1)
    assert inputs.size(-1) == in_dim * r
    keys, values = encoder_out
    mask = memory_mask(lengths) if (spec["use_memory_mask"] and lengths is not None) else None
    if text_positions is not None:
        w = spec["key_position_rate"]
        if speaker_embed is not None:
            w = w * torch.sigmoid(linear(sd, prefix + ".speaker_proj1", speaker_embed)).view(-1)
        keys = keys + sinusoidal_encoding(sd[prefix + ".embed_keys_positions.weight"],
                                          text_positions, w)
    frame_pos_embed = None
    if frame_positions is not None:
        w = spec["query_position_rate"]
        if speaker_embed is not None:
            w = w * torch.sigmoid(linear(sd, prefix + ".speaker_proj2", speaker_embed)).view(-1)
        frame_pos_embed = sinusoidal_encoding(sd[prefix + ".embed_query_positions.weight"],
                                              frame_positions, w)
    keys = keys.transpose(1, 2)
    x = run_stack(sd, prefix + ".preattention", spec["preattention"], inputs.transpose(1, 2),
                  speaker_embed)
    alignments = []
    for layer, has_attn in zip(spec["decoder"], spec["attention"]):
        residual = x
        x = run_stack(sd, prefix + ".convolutions", [layer], x, speaker_embed)
        if has_attn:
            q = x.transpose(1, 2)
            q = q if frame_pos_embed is None else q + frame_pos_embed
            q, a = attention_layer(sd, "%s.attention.%d" % (prefix, layer[1]), q, keys, values, mask)
            x = q.transpose(1, 2)
            alignments.append(a)
        x = (x + residual) * SQRT_HALF
    decoder_states = x.transpose(1, 2)
    x = conv1d(sd, prefix + ".last_conv", x).transpose(1, 2)
    outputs = torch.sigmoid(x)
    done = torch.sigmoid(linear(sd, prefix + ".fc", x))
    return outputs, torch.stack(alignments), done, decoder_states


def dv3_converter(sd, spec, x, speaker_embed=None, prefix="postnet"):
    """reference deepvoice3.py:582-604."""
    x = run_stack(sd, prefix + ".convolutions", spec["converter"], x.transpose(1, 2), speaker_embed)
    return torch.sigmoid(x.transpose(1, 2))


def nyanko_encoder(sd, spec, text, prefix="seq2seq.encoder"):
    """reference nyanko.py:60-71."""
    x = F.embedding(text.long(), sd[prefix + ".embed_tokens.weight"], padding_idx=spec["padding_idx"])
    x = run_stack(sd, prefix + ".convnet", spec["encoder"], x.transpose(1, 2)).transpose(1, 2)
    keys, values = x.split(x.size(-1) // 2, dim=-1)
    return keys, values


def nyanko_decoder(sd, spec, encoder_out, inputs, text_positions=None, frame_positions=None,
                   lengths=None, prefix="seq2seq.decoder"):
    """reference nyanko.py:177-248."""
    in_dim, r = spec["mel_dim"], spec["r"]
    if inputs.size(-1) == in_dim:
        inputs = inputs.reshape(inputs.size(0), inputs.size(1) // r, -1)
    keys, values = encoder_out
    mask = memory_mask(lengths) if (spec["use_memory_mask"] and lengths is not None) else None
    if text_positions is not None:
        keys = keys + F.embedding(text_positions, sd[prefix + ".embed_keys_positions.weight"],
                                  padding_idx=spec["padding_idx"])
    keys = keys.transpose(1, 2)
    x = run_stack(sd, prefix + ".audio_encoder_modules", spec["audio_encoder"],
                  inputs.transpose(1, 2))
    Q = x
    q = x.transpose(1, 2)
    if frame_positions is not None:
        q = q + F.embedding(frame_positions, sd[prefix + ".embed_query_positions.weight"],
                            padding_idx=spec["padding_idx"])
    R, alignments = attention_layer(sd, prefix + ".attention", q, keys, values, mask)
    x = torch.cat((R.transpose(1, 2), Q), dim=1)
    x = run_stack(sd, prefix + ".audio_decoder_modules", spec["audio_decoder"], x)
    decoder_states = x.transpose(1, 2)
    x = conv1d(sd, prefix + ".last_conv", x).transpose(1, 2)
    outputs = torch.sigmoid(x)
    done = torch.sigmoid(linear(sd, prefix + ".fc", x))
    return outputs, alignments.unsqueeze(0), done, decoder_states


def nyanko_converter(sd, spec, x, prefix="postnet"):
    """reference nyanko.py:401-402 (the Sequential ends in nn.Sigmoid)."""
    return run_stack(sd, prefix + ".convnet", spec["converter"], x.transpose(1, 2)).transpose(1, 2)


def model_forward(sd, spec, text, mel, speaker_ids=None, text_positions=None,
                  frame_positions=None, input_lengths=None):
    """reference deepvoice3_pytorch/__init__.py:65-97 + 112-126."""
    B = text.size(0)
    speaker_embed = None
    if speaker_ids is not None:
        assert spec["n_speakers"] > 1
        speaker_embed = F.embedding(speaker_ids, sd["embed_speakers.weight"])
    if spec["kind"] == "deepvoice3":
        enc = dv3_encoder(sd, spec, text, speaker_embed)
        mel_out, align, done, states = dv3_decoder(
            sd, spec, enc, mel, text_positions, frame_positions, speaker_embed, input_lengths)
    else:
        enc = nyanko_encoder(sd, spec, text)
        mel_out, align, done, states = nyanko_decoder(
            sd, spec, enc, mel, text_positions, frame_positions, input_lengths)
    mel_out = mel_out.reshape(B, -1, spec["mel_dim"])
    post_in = states.reshape(B, mel_out.size(1), -1) \
        if spec["use_decoder_state_for_postnet_input"] else mel_out
    if spec["kind"] == "deepvoice3":
        linear_out = dv3_converter(sd, spec, post_in, speaker_embed)
    else:
        linear_out = nyanko_converter(sd, spec, post_in)
    assert linear_out.size(-1) == spec["linear_dim"]
    return mel_out, linear_out, align, done


# ----------------------------------------------------------------------------------------------
# training-step harness pieces (reference train.py) used by bench.py's cpu_baseline and tests
# ----------------------------------------------------------------------------------------------
def sequence_mask(lengths, max_len):
    """reference train.py:261-271."""
    return (torch.arange(max_len)[None, :] < lengths[:, None]).to(torch.float32)


def spec_loss(y_hat, y, mask, masked_loss_weight=0.5, binary_divergence_weight=0.1, eps=1e-8, priority_bin=None,
              priority_w=0.0):
    """reference train.py:547-582 (pinned: tests/golden/train_fns.npz ``specloss*``)."""
    w = masked_loss_weight

    def l1_of(a, b):
        l1 = (a - b).abs().mean()
        if w > 0:
            mask_ = mask.expand_as(a)
            l1 = w * (((a * mask_) - (b * mask_)).abs().sum() / mask_.sum()) + (1 - w) * l1
        return l1

    l1 = l1_of(y_hat, y)
    if priority_bin is not None and priority_w > 0:          # train.py:559-567
        l1 = (1 - priority_w) * l1 + priority_w * l1_of(y_hat[:, :, :priority_bin], y[:, :, :priority_bin])
    if binary_divergence_weight <= 0:
        return l1, y.new_zeros(1)
    logits = torch.log(y_hat + eps) - torch.log(1 - y_hat + eps)
    z = -y * logits + torch.log1p(torch.exp(logits))
    if w > 0:
        mask_ = mask.expand_as(z)
        bd = w * ((z * mask_).sum() / mask_.sum()) + (1 - w) * z.mean()
    else:
        bd = z.mean()
    return l1, bd


def guided_attentions(input_lengths, target_lengths, max_target_len, max_input_len, g=0.2):
    """reference train.py:585-601: W[b,t,n] = 1-exp(-(n/N - t/T)^2 / (2 g^2)) inside (T_b, N_b)."""
    B = len(input_lengths)
    W = np.zeros((B, max_target_len, max_input_len), dtype=np.float32)
    for b in range(B):
        N, T = int(input_lengths[b]), int(target_lengths[b])
        n = np.arange(N, dtype=np.float64)[None, :] / N
        t = np.arange(T, dtype=np.float64)[:, None] / T
        W[b, :T, :N] = (1 - np.exp(-(n - t) ** 2 / (2 * g * g))).astype(np.float32)
    return W


def training_loss(outs, mel, y, done, input_lengths, target_lengths, r=1, downsample_step=4,
                  masked_loss_weight=0.5, binary_divergence_weight=0.1, guided_sigma=0.2, use_guided_attention=True,
                  priority_freq=3000, priority_freq_weight=0.0, sample_rate=22050):
    """reference train.py:665-740: total loss of one step (both seq2seq and postnet trained).  Pinned by the ``step*``
    cases of tests/golden/train_fns.npz, which come from running the reference's train() itself."""
    mel_out, lin_out, attn, done_hat = outs
    tl = torch.as_tensor(np.asarray(target_lengths))
    dec_mask = tgt_mask = None
    if masked_loss_weight > 0:
        dec_mask = sequence_mask(tl // (r * downsample_step), mel.size(1)).unsqueeze(-1)
        tgt_mask = sequence_mask(tl, y.size(1)).unsqueeze(-1) if downsample_step > 1 else dec_mask
        dec_mask, tgt_mask = dec_mask[:, r:, :], tgt_mask[:, r:, :]
    w = binary_divergence_weight
    l1, bd = spec_loss(mel_out[:, :-r, :], mel[:, r:, :], dec_mask, masked_loss_weight, w)
    mel_loss = (1 - w) * l1 + w * bd
    done_loss = F.binary_cross_entropy(done_hat, done)
    pbin = int(priority_freq / (sample_rate * 0.5) * lin_out.size(-1))          # train.py:722
    l1, bd = spec_loss(lin_out[:, :-r, :], y[:, r:, :], tgt_mask, masked_loss_weight, w, priority_bin=pbin,
                       priority_w=priority_freq_weight)
    lin_loss = (1 - w) * l1 + w * bd
    loss = mel_loss + lin_loss + done_loss
    if use_guided_attention:
        dec_lengths = np.asarray(target_lengths) // r // downsample_step
        soft = torch.from_numpy(guided_attentions(np.asarray(input_lengths), dec_lengths,
                                                  attn.size(-2), attn.size(-1), guided_sigma))
        loss = loss + (attn * soft.to(attn.dtype)).mean()
    return loss
