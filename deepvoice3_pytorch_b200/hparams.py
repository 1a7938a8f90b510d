"""From the reference's hyper-parameter sets (``hparams.py`` / ``presets/*.json``) to this package's objects.

``train.py`` is the caller and stays the reference's (or the user's) -- but the two mappings it applies are needed by
anybody who switches packages, so they are restated here:

* ``build_model(hp, n_vocab)``: hparams -> builder kwargs, reference train.py:812-840 (``build_model``).  Note what the
  reference does NOT forward: ``query_position_rate`` / ``key_position_rate`` / ``embedding_weight_std`` of the preset
  are ignored and the builder defaults (1.0 / 1.29 / 0.1) apply -- kept, because checkpoints were trained that way.
* ``train_step_kwargs(hp)``: the optimiser / loss settings ``train.py`` reads in its loop (train.py:704-759, 939-946)
  and passes to torch.optim.Adam (train.py:975-979) as keyword arguments of ``train_step.TrainStep``.
"""
import json

from . import builder
from . import train_step as _ts

_BUILDER_KEYS = {
    # builder kwarg                      hparams name
    "n_speakers": "n_speakers", "speaker_embed_dim": "speaker_embed_dim", "embed_dim": "text_embed_dim",
    "mel_dim": "num_mels", "r": "outputs_per_step", "downsample_step": "downsample_step",
    "padding_idx": "padding_idx", "dropout": "dropout", "kernel_size": "kernel_size",
    "encoder_channels": "encoder_channels", "decoder_channels": "decoder_channels",
    "converter_channels": "converter_channels", "use_memory_mask": "use_memory_mask",
    "trainable_positional_encodings": "trainable_positional_encodings",
    "force_monotonic_attention": "force_monotonic_attention",
    "use_decoder_state_for_postnet_input": "use_decoder_state_for_postnet_input", "max_positions": "max_positions",
    "speaker_embedding_weight_std": "speaker_embedding_weight_std", "freeze_embedding": "freeze_embedding",
    "window_ahead": "window_ahead", "window_backward": "window_backward", "key_projection": "key_projection",
    "value_projection": "value_projection",
}


def load_preset(path):
    """A ``presets/*.json`` file of the reference as a plain dict."""
    with open(path) as f:
        return json.load(f)


def builder_kwargs(hp, n_vocab):
    """-> (builder function name, kwargs) exactly as reference train.py:812-840 assembles them."""
    kw = {k: hp[h] for k, h in _BUILDER_KEYS.items()}
    kw["n_vocab"] = n_vocab
    kw["linear_dim"] = hp["fft_size"] // 2 + 1
    return hp["builder"], kw


def build_model(hp, n_vocab):
    name, kw = builder_kwargs(hp, n_vocab)
    return getattr(builder, name)(**kw)


def train_step_kwargs(hp):
    """Keyword arguments of ``TrainStep`` for this hyper-parameter set.  The training mode (train_seq2seq /
    train_postnet) is a command-line choice of train.py, not an hparam: pass it alongside."""
    schedule = hp.get("lr_schedule")
    if schedule is not None and not callable(schedule):
        base = getattr(_ts, schedule)          # reference: getattr(lrschedule, hparams.lr_schedule)
        extra = dict(hp.get("lr_schedule_kwargs") or {})
        schedule = (lambda lr, step, _f=base, _kw=extra: _f(lr, step, **_kw)) if extra else base
    return dict(init_lr=hp["initial_learning_rate"], betas=(hp["adam_beta1"], hp["adam_beta2"]), eps=hp["adam_eps"],
                clip_thresh=hp["clip_thresh"], r=hp["outputs_per_step"], downsample_step=hp["downsample_step"],
                masked_loss_weight=hp["masked_loss_weight"], binary_divergence_weight=hp["binary_divergence_weight"],
                guided_attention_sigma=hp["guided_attention_sigma"], use_guided_attention=hp["use_guided_attention"],
                priority_freq=hp.get("priority_freq", 3000), priority_freq_weight=hp.get("priority_freq_weight", 0.0),
                sample_rate=hp.get("sample_rate", 22050), lr_schedule=schedule,
                weight_decay=hp.get("weight_decay", 0.0), amsgrad=hp.get("amsgrad", False))
