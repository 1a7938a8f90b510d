"""Top-level containers: the seq2seq (encoder + attention decoder) wrapper and the full TTS model that adds the
speaker table and the post-net.  Public surface (attribute names, call signatures, return tuples) follows what
reference train.py / synthesis.py touch (SURVEY.md section 8b); see reference deepvoice3_pytorch/__init__.py:11-126.
"""
import torch
from torch import nn

from . import ops
from .modules import Embedding


class AttentionSeq2Seq(nn.Module):
    """text -> (keys, values) -> teacher-forced attention decoder."""

    def __init__(self, encoder, decoder):
        super().__init__()
        self.encoder, self.decoder = encoder, decoder
        attn = self.decoder.attention
        if isinstance(attn, nn.ModuleList):          # deepvoice3 decoders: one optional layer per conv block
            self.encoder.num_attention_layers = len([a for a in attn if a is not None])

    def forward(self, text_sequences, mel_targets=None, speaker_embed=None, text_positions=None,
                frame_positions=None, input_lengths=None):
        # reference train.py:691-694 also calls model.seq2seq(...) on its own: a new dropout seed per training
        # forward is drawn by whichever container is outermost (ops.DropoutState.begin_forward)
        ops.rng.begin_forward(self.training, text_sequences.device)
        try:
            with ops.extent_axis(ops.EXT_TEXT):             # masks the padding of a bucketed batch (ops.extent_scope)
                memory = self.encoder(text_sequences, lengths=input_lengths, speaker_embed=speaker_embed)
            # -> mel (B, T//r, mel_dim*r), alignments (N, B, T_dec, T_text), done (B, T//r, 1), decoder states
            return self.decoder(memory, mel_targets, text_positions=text_positions,
                                frame_positions=frame_positions, speaker_embed=speaker_embed, lengths=input_lengths)
        finally:
            ops.rng.end_forward()


class MultiSpeakerTTSModel(nn.Module):
    """seq2seq + converter ("postnet"), optionally conditioned on a learned speaker embedding."""

    def __init__(self, seq2seq, postnet, mel_dim=80, linear_dim=513, n_speakers=1, speaker_embed_dim=16,
                 padding_idx=None, trainable_positional_encodings=False,
                 use_decoder_state_for_postnet_input=False, speaker_embedding_weight_std=0.01,
                 freeze_embedding=False):
        super().__init__()
        self.seq2seq, self.postnet = seq2seq, postnet
        self.mel_dim, self.linear_dim = mel_dim, linear_dim
        self.n_speakers, self.speaker_embed_dim = n_speakers, speaker_embed_dim
        self.trainable_positional_encodings = trainable_positional_encodings
        self.use_decoder_state_for_postnet_input = use_decoder_state_for_postnet_input
        self.freeze_embedding = freeze_embedding
        self.speaker_embedding_weight_std = speaker_embedding_weight_std
        if n_speakers > 1:
            self.embed_speakers = Embedding(n_speakers, speaker_embed_dim, padding_idx=None,
                                            std=speaker_embedding_weight_std)

    def add_speakers(self, n, init="mean"):
        """Append ``n`` rows to the speaker table and return their ids [n_speakers, n_speakers + n): one contiguous
        block at the end, the existing rows bit-identical, the state_dict keys unchanged (a model built with
        n_speakers + n loads the result strictly).  init: "mean" (the mean of the existing rows, in fp64, rounded
        once), "normal" (the builder's N(0, speaker_embedding_weight_std) init from the torch RNG) or an
        (n, speaker_embed_dim) tensor of the table's dtype.  Raises ValueError, changing nothing, for a
        single-speaker model, n < 1 or a malformed init.  Train the new rows with TrainStep(adapt_speakers=ids)."""
        if self.n_speakers <= 1 or not hasattr(self, "embed_speakers"):
            raise ValueError("add_speakers needs a multi-speaker model (n_speakers=%d)" % self.n_speakers)
        if isinstance(n, bool) or not isinstance(n, int) or n < 1:
            raise ValueError("add_speakers: n=%r must be an int >= 1" % (n,))
        old = self.embed_speakers.weight
        S = self.speaker_embed_dim
        if torch.is_tensor(init):
            if tuple(init.shape) != (n, S) or init.dtype != old.dtype:
                raise ValueError("add_speakers: init of shape %s dtype %s, expected (%d, %d) %s"
                                 % (tuple(init.shape), init.dtype, n, S, old.dtype))
            rows = init.detach().to(old.device)
        elif init == "mean":
            rows = old.detach().double().mean(0, keepdim=True).to(old.dtype).expand(n, S)
        elif init == "normal":
            rows = torch.empty(n, S, dtype=old.dtype).normal_(0, self.speaker_embedding_weight_std).to(old.device)
        else:
            raise ValueError("add_speakers: init must be \"mean\", \"normal\" or a tensor (got %r)" % (init,))
        ids = list(range(self.n_speakers, self.n_speakers + n))
        with torch.no_grad():
            table = torch.cat([old.detach(), rows], 0)
        self.embed_speakers.weight = nn.Parameter(table, requires_grad=old.requires_grad)
        self.embed_speakers.num_embeddings = table.shape[0]
        self.n_speakers += n
        return ids

    # -- optimiser view ---------------------------------------------------------------------------------
    def _frozen_parameters(self):
        dec, enc = self.seq2seq.decoder, self.seq2seq.encoder
        frozen = []
        if not self.trainable_positional_encodings:
            frozen += list(dec.embed_query_positions.parameters()) + list(dec.embed_keys_positions.parameters())
        if self.freeze_embedding:
            frozen += list(enc.embed_tokens.parameters())
        return {id(p) for p in frozen}

    def get_trainable_parameters(self):
        """All parameters but the position tables (unless trainable) and, if frozen, the text embedding."""
        skip = self._frozen_parameters()
        return (p for p in self.parameters() if id(p) not in skip)

    def make_generation_fast_(self):
        """The reference strips the weight-norm hooks here so inference stops re-normalising every call
        (__init__.py:39-46).  Nothing to strip in this implementation: the incremental decoder folds g*v/||v|| once
        per utterance (incremental.py) and the parameters keep their reference names."""
        return None

    # -- forward ------------------------------------------------------------------------------------------
    def _speaker_embedding(self, speaker_ids, speaker_embed=None):
        if speaker_embed is not None:
            if speaker_ids is not None:
                raise ValueError("pass speaker_ids or speaker_embed, not both")
            if self.n_speakers <= 1 or speaker_embed.dim() != 2 or speaker_embed.shape[1] != self.speaker_embed_dim:
                raise ValueError("speaker_embed of shape %s: expected (B, %d) on a multi-speaker model (n_speakers=%d)"
                                 % (tuple(speaker_embed.shape), self.speaker_embed_dim, self.n_speakers))
            if ops.speaker_adapt is not None:        # frozen model: e is the one tensor with a gradient
                return ops.speaker_adapt.anchor_of(speaker_embed)
            return speaker_embed
        if speaker_ids is None:
            return None
        assert self.n_speakers > 1
        if ops.speaker_adapt is not None:            # embedding-only adaptation: e is the one tensor with a gradient
            return ops.speaker_adapt.embed(self.embed_speakers, speaker_ids)
        return self.embed_speakers(speaker_ids)

    def forward(self, text_sequences, mel_targets=None, speaker_ids=None, text_positions=None,
                frame_positions=None, input_lengths=None, speaker_embed=None):
        """-> mel_outputs (B, T, mel_dim), linear_outputs (B, T*ds, linear_dim), alignments (N, B, T_dec, T_text),
        done (B, T_dec, 1).  speaker_embed (B, speaker_embed_dim): the speakers' embeddings themselves, used instead of
        looking ``speaker_ids`` up in the table (e.g. a speaker encoder's output, which then takes the gradient)."""
        # dropout: call-site salts restart and (in training) a new step seed is drawn with every forward, so
        # model(...) / loss.backward() / optimizer.step() loops get fresh masks without any TrainStep
        ops.rng.begin_forward(self.training, text_sequences.device)
        try:
            batch = text_sequences.size(0)
            spk = self._speaker_embedding(speaker_ids, speaker_embed)
            mel, alignments, done, states = self.seq2seq(text_sequences, mel_targets, spk, text_positions,
                                                         frame_positions, input_lengths)
            mel = mel.reshape(batch, -1, self.mel_dim)    # un-group the r frames per decoder step
            post_in = states.reshape(batch, mel.size(1), -1) if self.use_decoder_state_for_postnet_input else mel
            post_in = ops.grad_boundary(post_in, "postnet")     # its gradient ready <=> the postnet's backward is done
            with ops.extent_axis(ops.EXT_MEL):
                linear = self.postnet(post_in, spk)
            assert linear.size(-1) == self.linear_dim
            return mel, linear, alignments, done
        finally:
            ops.rng.end_forward()
