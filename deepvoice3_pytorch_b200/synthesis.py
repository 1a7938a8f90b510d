"""Batched text-to-speech synthesis: many utterances per set of launches, each exactly as if synthesized alone.

Reference synthesis.py:42-73 (``tts``) runs one sentence per call: text ids -> ``model(...)`` (encoder, autoregressive
decoder, converter) -> ``audio.inv_spectrogram``.  ``tts_batch`` runs the same four stages on padded batches:

* encoder and converter inside an ``ops.length_scope``: every row's frames past its own length are zeroed before each
  conv that spans several frames, so each row sees the zero padding it would see alone;
* ``incremental.decode_ragged``: per-row attention length, context scale, monotonic cursor and stopping step;
* ``audio.inv_spectrogram_batch``: Griffin-Lim (or LWS, ``vocoder="lws"``, or fast Griffin-Lim,
  ``vocoder="fast_griffin_lim"``) over a ragged batch of clips with a deterministic overlap-add.

``tts_stream`` runs the decoder with continuous batching instead (``incremental.decode_stream``): a fixed set of decoder
slots, each refilled with the next waiting utterance as soon as its own one stops, so no slot idles until the longest
utterance of a chunk is done.  Finished utterances go through the post-net and vocoder in groups and are yielded as
they complete.

Both take ``durations`` (one integer array per sequence, in decoder steps) and ``speed`` for duration-guided synthesis
(DESIGN.md section 2.22): every attention layer's window follows the prescribed token path and each utterance runs
exactly sum(durations) decoder steps; ``speed`` rescales the durations (``duration.scale_durations``).

Every kernel on this path computes a row from that row's data alone, in an order that does not depend on the batch,
so with ``ops.conv_math = "fp32"`` each result is bit-identical to the one-utterance path.  In the default tensor-core
mode the batch's larger GEMMs may take the tensor-core kernels where a short single sentence runs on the exact-fp32 ones
(``ops._use_tc_conv``), so results then agree to the tensor-core tolerance instead.
"""
import contextlib

import numpy as np
import torch

from . import audio, incremental, ops


def stages(stage_timer):
    """The ``stage_timer`` argument of the synthesis and evaluation calls as a callable ``name -> context manager``
    (None: no timing)."""
    return stage_timer or (lambda name: contextlib.nullcontext())


def _check_inputs(model, sequences, speaker_ids, **counts):
    """-> int64 token arrays, int speaker ids; counts: name=value arguments that must be >= 1 (batch_size, slots)."""
    if len(sequences) == 0:
        raise ValueError("synthesis needs at least one sequence")
    seqs = []
    max_len = model.seq2seq.decoder.embed_keys_positions.num_embeddings - 1      # positions 1..L index the table
    for i, s in enumerate(sequences):
        s = np.asarray(s)
        if s.ndim != 1 or s.size == 0:
            raise ValueError("sequence %d must be a non-empty 1-D array of token ids, got shape %s" % (i, s.shape))
        if not np.issubdtype(s.dtype, np.integer):
            raise ValueError("sequence %d must hold integer token ids, got %s" % (i, s.dtype))
        if s.size > max_len:
            raise ValueError("sequence %d has %d tokens; the position tables hold %d" % (i, s.size, max_len))
        seqs.append(s.astype(np.int64))
    if speaker_ids is not None:
        if model.n_speakers <= 1:
            raise ValueError("speaker_ids given for a single-speaker model")
        speaker_ids = [int(x) for x in speaker_ids]
        if len(speaker_ids) != len(seqs):
            raise ValueError("%d speaker_ids for %d sequences" % (len(speaker_ids), len(seqs)))
    elif model.n_speakers > 1:
        raise ValueError("a multi-speaker model needs speaker_ids")
    for name, value in counts.items():
        if int(value) < 1:
            raise ValueError("%s must be >= 1, got %r" % (name, value))
    if model.training:
        raise RuntimeError("incremental_forward only supports eval mode")         # as incremental.decode
    if not next(model.parameters()).is_cuda:
        raise RuntimeError("incremental decoding runs on the GPU only (no CPU fallback)")
    return seqs, speaker_ids


@torch.no_grad()
def _synthesize_chunk(model, seqs, speaker_ids, stage, vocoder, durations=None):
    """seqs: list of int64 arrays -> [(waveform, alignment, spectrogram, mel)] for one padded batch."""
    outputs, aligns, states, steps, spk = _decode_chunk(model, seqs, speaker_ids, stage, durations)
    aligns = aligns.cpu().numpy()
    post = _postnet_vocode(model, outputs, states, steps, spk, stage, vocoder)
    return [(w, aligns[b, :steps[b], :s.size], lin, mel) for b, (s, (w, lin, mel)) in enumerate(zip(seqs, post))]


@torch.no_grad()
def _decode_chunk(model, seqs, speaker_ids, stage, durations=None):
    """The encoder and ``incremental.decode_ragged`` of ``tts_batch`` on one padded batch (stages "encoder" and
    "decoder"), guided by ``durations`` (one int64 array per row) when given: seqs: list of int64 arrays -> (outputs (B, N, in_dim*r), alignments (B, N, T_text) on the device,
    decoder states (B, N, C), steps [B], speaker embeddings (B, D) or None)."""
    dev = next(model.parameters()).device
    B = len(seqs)
    lens = [s.size for s in seqs]
    L = max(lens)
    text = np.zeros((B, L), dtype=np.int64)
    tpos = np.zeros((B, L), dtype=np.int64)
    for b, s in enumerate(seqs):
        text[b, :s.size] = s
        tpos[b, :s.size] = np.arange(1, s.size + 1)
    text, tpos = torch.from_numpy(text).to(dev), torch.from_numpy(tpos).to(dev)
    text_len = torch.tensor(lens, dtype=torch.int64).to(dev)
    ops.rng.begin_forward(False, dev)
    try:
        spk = None if speaker_ids is None else model._speaker_embedding(torch.tensor(speaker_ids).to(dev))
        dec = model.seq2seq.decoder
        with stage("encoder"), ops.length_scope(text_len, L):
            keys, values = model.seq2seq.encoder(text, speaker_embed=spk)
        with stage("decoder"):
            outputs, aligns, _, states, steps = incremental.decode_ragged(dec, (keys, values), tpos, text_len, spk,
                                                                          durations=durations)
    finally:
        ops.rng.end_forward()
    return outputs, aligns, states, steps, spk


@torch.no_grad()
def _postnet_vocode(model, outputs, states, steps, spk, stage, vocoder="griffin_lim"):
    """Decoder outputs (B, N, in_dim*r) and states (B, N, C), row b valid for its first steps[b] decoder steps ->
    [(waveform, spectrogram, mel)] of each row, denormalised and cut to its own frames; the waveform's phase recovered
    with ``vocoder`` (an ``audio.inv_spectrogram`` method)."""
    B = outputs.size(0)
    ops.rng.begin_forward(False, outputs.device)
    try:
        with stage("converter"):
            mel = outputs.reshape(B, -1, model.mel_dim)
            r = mel.size(1) // outputs.size(1)
            post_in = states.reshape(B, mel.size(1), -1) if model.use_decoder_state_for_postnet_input else mel
            frames = torch.tensor(steps, dtype=torch.int64).to(outputs.device) * r
            with ops.length_scope(frames, mel.size(1)):
                linear = model.postnet(post_in, spk)
            up = linear.size(1) // mel.size(1)
            mel, linear = mel.cpu().numpy(), linear.cpu().numpy()
    finally:
        ops.rng.end_forward()
    lin_rows = [linear[b, :steps[b] * r * up] for b in range(B)]
    with stage("vocoder"):
        wavs = audio.inv_spectrogram_batch([x.T for x in lin_rows], method=vocoder)
    return [(wavs[b], audio._denormalize(lin_rows[b]), audio._denormalize(mel[b, :steps[b] * r])) for b in range(B)]


def tts_batch(model, sequences, speaker_ids=None, batch_size=16, stage_timer=None, vocoder="griffin_lim",
              durations=None, speed=1.0):
    """Synthesize many utterances at once.

    model: a ``MultiSpeakerTTSModel`` in eval mode on CUDA.  sequences: list of 1-D token-id arrays (what a text
    frontend's ``text_to_sequence`` returns).  speaker_ids: one id per sequence for a multi-speaker model, else None.
    Sequences are sorted by length and synthesized in padded batches of ``batch_size`` (similar lengths share a batch,
    which bounds the decoder steps spent on rows that already stopped).

    -> list, in input order, of (waveform, alignment (N_b, L_b), spectrogram, mel): what reference ``synthesis.tts``
    returns for that sequence synthesized alone -- the same decoder steps, the denormalised linear and mel spectrograms
    cut to the row's own frames, and its waveform (see the module docstring for when this is bit-exact).

    stage_timer: optional callable ``name -> context manager`` wrapped around each stage ("encoder", "decoder",
    "converter", "vocoder") of every batch, e.g. to time them.  vocoder: the phase recovery of
    ``audio.inv_spectrogram``, "griffin_lim" (the default), "lws" (the reference's algorithm) or "fast_griffin_lim"
    (Griffin-Lim with momentum); checked first.

    durations: duration-guided synthesis -- one integer array per sequence, one entry >= 1 per token, in decoder steps
    (from ``duration.predict_durations``, from ``alignment.teacher_forced_alignment`` of a recording, or the
    "durations" of ``alignment.evaluate_attention``); sequence k then runs exactly sum(durations[k]) decoder steps with
    every attention window on the prescribed token (``incremental.decode_ragged``).  speed: speaking rate, applied to
    the durations with ``duration.scale_durations``; a speed other than 1 needs durations.  ValueError before any
    launch for malformed durations or speed, or a total above the query-position table."""
    from .duration import guided_durations
    audio.check_phase_method(vocoder)
    durs = guided_durations(model, sequences, durations, speed)
    seqs, speaker_ids = _check_inputs(model, sequences, speaker_ids, batch_size=batch_size)
    stage = stages(stage_timer)
    order = sorted(range(len(seqs)), key=lambda i: -seqs[i].size)
    out = [None] * len(seqs)
    for c in range(0, len(order), int(batch_size)):
        idx = order[c:c + int(batch_size)]
        ids = None if speaker_ids is None else [speaker_ids[i] for i in idx]
        chunk = _synthesize_chunk(model, [seqs[i] for i in idx], ids, stage, vocoder,
                                  None if durs is None else [durs[i] for i in idx])
        for i, res in zip(idx, chunk):
            out[i] = res
    return out


def wav_mels(wavs, device):
    """fp32 host waveforms -> list of their (T_k, num_mels) normalised mels on ``device``: one padded batch through
    ``audio.stft_mel_batch``, each clip cut to its own ``audio.num_frames``."""
    return wav_clips_and_mels(wavs, device)[1]


def wav_clips_and_mels(wavs, device):
    """``wav_mels`` that also returns the waveforms as they were copied to ``device``: -> (list of 1-D fp32 views of
    the padded device batch, one per clip at its own length, list of mels)."""
    lens = [len(w) for w in wavs]
    pad = np.zeros((len(wavs), max(lens)), np.float32)
    for k, w in enumerate(wavs):
        pad[k, :lens[k]] = w
    pad = torch.from_numpy(pad).to(device)
    _, mel = audio.stft_mel_batch(pad, torch.tensor(lens, dtype=torch.int32), want_linear=False)
    return [pad[k, :n] for k, n in enumerate(lens)], [mel[k, :audio.num_frames(n)] for k, n in enumerate(lens)]


def synthesized_audio(model, sequences, speaker_ids, vocoder, batch_size, device, stage_timer=None):
    """What the evaluations of synthesized speech share (``mcd.evaluate_synthesis``, ``pitch.evaluate_pitch``,
    ``speaker_verifier``'s and ``speaker_classifier``'s cloned-voice evaluations): every ``sequences[k]`` synthesized
    with ``tts_batch`` (in voice ``speaker_ids[k]`` for a multi-speaker model, None for a single-speaker one; stage
    "synthesis") and turned into normalised mels on ``device`` with ``wav_clips_and_mels`` (stage "mel") -> (list of
    the waveforms on ``device``, list of their (T_k, num_mels) mels).  ValueError before any launch for an unknown phase
    method or malformed inputs (as ``tts_batch``)."""
    audio.check_phase_method(vocoder)
    _check_inputs(model, sequences, speaker_ids, batch_size=batch_size)
    stage = stages(stage_timer)
    with stage("synthesis"):
        wavs = [w for w, _, _, _ in tts_batch(model, sequences, speaker_ids, batch_size=batch_size, vocoder=vocoder)]
    with stage("mel"):
        return wav_clips_and_mels(wavs, device)


def synthesized_mels(model, sequences, speaker_ids, vocoder, batch_size, device, stage_timer=None):
    """``synthesized_audio`` without the waveforms -> list of (T_k, num_mels) mels."""
    return synthesized_audio(model, sequences, speaker_ids, vocoder, batch_size, device, stage_timer)[1]


def tts_stream(model, sequences, speaker_ids=None, slots=16, post_batch=16, stage_timer=None, stats=None,
               vocoder="griffin_lim", durations=None, speed=1.0):
    """Synthesize many utterances with continuous batching; a generator of (index, (waveform, alignment, spectrogram,
    mel)) in completion order, each item what ``tts_batch`` gives for that sequence (bit for bit in exact-fp32 mode).

    The encoder runs on groups of ``slots`` waiting sequences (inside a length scope) as the decoder needs them; the
    decoder is ``incremental.decode_stream`` on ``slots`` rows; finished utterances go through the post-net (inside a
    length scope on their frames) and the vocoder in groups of ``post_batch``, the last partial group when the decoder
    is done.  Inputs are checked as ``tts_batch`` checks them, before the first item.  stage_timer, vocoder: as for
    ``tts_batch``; stats: a dict ``decode_stream`` fills (decoder occupancy); durations, speed: duration-guided
    synthesis as for ``tts_batch`` (each slot then stops after its utterance's total of steps)."""
    from .duration import guided_durations
    audio.check_phase_method(vocoder)
    durs = guided_durations(model, sequences, durations, speed)
    seqs, speaker_ids = _check_inputs(model, sequences, speaker_ids, slots=slots, post_batch=post_batch)
    stage = stages(stage_timer)
    return _stream(model, seqs, speaker_ids, int(slots), int(post_batch), stage, stats, vocoder, durs)


@torch.no_grad()
def _encode(model, idx, seqs, speaker_ids, stage):
    """Encode one padded group -> [(index, keys (T, E), values (T, E), text_positions (T,), speaker_embed or None)]."""
    dev = next(model.parameters()).device
    lens = [s.size for s in seqs]
    L = max(lens)
    text = np.zeros((len(seqs), L), dtype=np.int64)
    for b, s in enumerate(seqs):
        text[b, :s.size] = s
    text = torch.from_numpy(text).to(dev)
    text_len = torch.tensor(lens, dtype=torch.int64).to(dev)
    ops.rng.begin_forward(False, dev)
    try:
        spk = None if speaker_ids is None else model._speaker_embedding(torch.tensor(speaker_ids).to(dev))
        with stage("encoder"), ops.length_scope(text_len, L):
            keys, values = model.seq2seq.encoder(text, speaker_embed=spk)
    finally:
        ops.rng.end_forward()
    return [(i, keys[b, :n], values[b, :n], torch.arange(1, n + 1, device=dev), None if spk is None else spk[b])
            for b, (i, n) in enumerate(zip(idx, lens))]


def _stream(model, seqs, speaker_ids, slots, post_batch, stage, stats, vocoder="griffin_lim", durations=None):
    def requests():
        for g in range(0, len(seqs), slots):
            idx = list(range(g, min(g + slots, len(seqs))))
            reqs = _encode(model, idx, [seqs[i] for i in idx],
                           None if speaker_ids is None else [speaker_ids[i] for i in idx], stage)
            yield from reqs if durations is None else (r + (durations[r[0]],) for r in reqs)

    def flush(group):
        N = max(r[5] for r in group)
        Fr, Cs = group[0][1].size(1), group[0][4].size(1)
        outputs = group[0][1].new_zeros(len(group), N, Fr)
        states = group[0][4].new_zeros(len(group), N, Cs)
        for b, r in enumerate(group):
            outputs[b, :r[5]], states[b, :r[5]] = r[1], r[4]
        spk = None if speaker_ids is None else \
            model._speaker_embedding(torch.tensor([speaker_ids[r[0]] for r in group]).to(outputs.device))
        post = _postnet_vocode(model, outputs, states, [r[5] for r in group], spk, stage, **vocoder_kw)
        for r, (w, lin, mel) in zip(group, post):
            yield r[0], (w, r[2].cpu().numpy(), lin, mel)

    vocoder_kw = {} if vocoder == "griffin_lim" else {"vocoder": vocoder}     # the default: the six-argument call
    group = []
    # guided: the program holds the longest total, not the whole query-position table
    guided_kw = {} if durations is None else {"guided_steps": max(int(d.sum()) for d in durations)}
    for r in incremental.decode_stream(model.seq2seq.decoder, slots, requests(), stats=stats, stage_timer=stage,
                                       **guided_kw):
        group.append(r)
        if len(group) == post_batch:
            yield from flush(group)
            group = []
    if group:
        yield from flush(group)
