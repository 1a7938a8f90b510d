"""Fine-tuning a speaker encoder through the training loss on the deepvoice3_vctk preset (random weights): four arms on
the same batches, alternating over rounds, in "tc" and "tc1", at B = 16, T_text 128, T_mel 800, N = 8 cloning
samples of T_crop = 128 frames:

  (a) TrainStep(speaker_encoder=enc, train_model=True, use_graph=True): the joint step, model + encoder;
  (b) TrainStep(speaker_encoder=enc, train_model=False, use_graph=True): the encoder-only step, model frozen;
  (c) the plain multi-speaker TrainStep(use_graph=True) with table lookup, on the same TTS batches;
  (d) SpeakerEncoderStep at the same B x N x T_crop (the encoder regressing table rows).

Reports ms/step (median and min-max over rounds), launches per step, and the encoder's added cost in the joint step,
(a) - (c), next to (d), with the card's name and power limit read in the same run.  Prints one JSON line.
Writes nothing to the tree.

    python bench_speaker_joint.py [--steps 20] [--rounds 3]
"""
import argparse
import json

import numpy as np
import torch

from bench import PRESETS
from bench_speaker_adapt import card, time_steps
from deepvoice3_pytorch_b200 import builder, ops
from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder, SpeakerEncoderStep
from deepvoice3_pytorch_b200.train_step import TrainStep, make_synthetic_batch, to_device

PRESET = "deepvoice3_vctk"
B, T_TEXT, T_MEL, N, T_CROP = 16, 128, 800, 8, 128


def _model(kw, seed=0):
    torch.manual_seed(seed)
    return getattr(builder, PRESETS[PRESET][0])(**kw).cuda().train()


def _encoder(kw, seed=1):
    torch.manual_seed(seed)
    return SpeakerEncoder(mel_dim=kw.get("mel_dim", 80), speaker_embed_dim=kw["speaker_embed_dim"]).cuda()


def _batches(kw, n=4):
    out = []
    gen = torch.Generator().manual_seed(7)
    for i in range(n):
        h = make_synthetic_batch(B=B, T_text=T_TEXT, T_mel=T_MEL, n_speakers=kw["n_speakers"], linear_dim=513, seed=i)
        h["speaker_mels"] = torch.rand(B, N, T_CROP, kw.get("mel_dim", 80), generator=gen)
        out.append(to_device(h, "cuda"))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maths", default="tc,tc1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speaker_joint.py needs a CUDA device")
    _, kw, extra = PRESETS[PRESET]
    res = {"preset": PRESET, "card": card(), "B": B, "T_text": T_TEXT, "T_mel": T_MEL, "N": N, "T_crop": T_CROP,
           "runs": []}
    for math in args.maths.split(","):
        ops.conv_math = math
        batches = _batches(kw)
        enc_batches = [{"mels": b["speaker_mels"], "speaker_ids": b["speaker_ids"]} for b in batches]
        steps = {"a_joint_graph": TrainStep(_model(kw), speaker_encoder=_encoder(kw), train_model=True,
                                            use_graph=True, **extra),
                 "b_frozen_graph": TrainStep(_model(kw), speaker_encoder=_encoder(kw), train_model=False,
                                             use_graph=True, **extra),
                 "c_table_graph": TrainStep(_model(kw), use_graph=True, **extra),
                 "d_encoder_step": SpeakerEncoderStep(_encoder(kw), _model(kw), use_graph=True)}
        feeds = {k: (enc_batches if k == "d_encoder_step" else batches) for k in steps}
        for k, st in steps.items():
            time_steps(st.step, feeds[k], args.warmup)
        ms = {k: [] for k in steps}
        for _ in range(args.rounds):
            for k, st in steps.items():
                ms[k].append(time_steps(st.step, feeds[k], args.steps)[0])
        med = {k: float(np.median(v)) for k, v in ms.items()}
        run = {"math": math,
               "ms_per_step": {k: {"median": round(med[k], 3), "min": round(min(v), 3), "max": round(max(v), 3)}
                               for k, v in ms.items()},
               "launches_per_step": {k: st.launches_per_step for k, st in steps.items()},
               "encoder_added_ms_a_minus_c": round(med["a_joint_graph"] - med["c_table_graph"], 3),
               "encoder_step_ms_d": round(med["d_encoder_step"], 3)}
        res["runs"].append(run)
        del steps
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
