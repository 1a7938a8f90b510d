"""deepvoice3_pytorch_b200 -- H100-native drop-in for the training hot path of r9y9/deepvoice3_pytorch.

Mirrors the reference package surface: ``MultiSpeakerTTSModel``, ``AttentionSeq2Seq`` (tts_model.py) and
``builder.{deepvoice3, nyanko, deepvoice3_multispeaker}``, with identical ``state_dict`` keys.  All arithmetic runs in
hand-written sm_90a kernels behind a C ABI (include/dv3b200.h, csrc/); there is no CPU fallback.
"""
__version__ = "0.1.0"

from .tts_model import AttentionSeq2Seq, MultiSpeakerTTSModel  # noqa: F401
