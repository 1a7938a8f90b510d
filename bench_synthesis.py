#!/usr/bin/env python
"""Batched synthesis benchmark: ``synthesis.tts_batch`` against a loop of one-utterance synthesis (what reference
synthesis.py does: one ``model(...)`` + ``inv_spectrogram`` per sentence) over the same token sequences.

    python bench_synthesis.py [--preset deepvoice3_ljspeech] [--batch 16] [--utterances 32] [--steps 100]

Random weights (seeded); text lengths are drawn in 20..190 tokens.  The decoder's done bias is forced strongly
negative and max_decoder_steps set so that every utterance runs exactly ``--steps`` decoder steps: the work is fixed
and equal in both arms.  Reports utterances/s and seconds of audio per second of each arm, split into encoder /
decoder / converter / vocoder time (each stage ends in a device synchronise), with the card's name and power limit
read in the same run.  Before printing it checks that both arms produced the same waveforms bit for bit.  With
``--conv-math fp32`` that holds for the timed outputs.  In the default tensor-core mode a batch's larger GEMMs may take
the tensor-core kernels where a single short sentence runs on the exact-fp32 ones, so the timed waveforms differ
slightly (reported relative to their peak), and the bit-for-bit check reruns the first batch in fp32 mode.
Prints one JSON line.
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


class StageTimer:
    def __init__(self):
        self.t = {"encoder": 0.0, "decoder": 0.0, "converter": 0.0, "vocoder": 0.0}

    @contextlib.contextmanager
    def __call__(self, name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        try:
            yield
        finally:
            torch.cuda.synchronize()
            self.t[name] += time.perf_counter() - t0


def synthesize_alone(model, seq, speaker_id, stage):
    """One utterance through the same stages as ``model(...)`` in inference + ``audio.inv_spectrogram``."""
    from deepvoice3_pytorch_b200 import audio
    text = torch.from_numpy(seq).unsqueeze(0).cuda()
    tpos = torch.arange(1, text.size(-1) + 1).unsqueeze(0).cuda()
    with torch.no_grad():
        spk = None if speaker_id is None else model._speaker_embedding(torch.tensor([speaker_id]).cuda())
        with stage("encoder"):
            memory = model.seq2seq.encoder(text, speaker_embed=spk)
        with stage("decoder"):
            outputs, _, _, states = model.seq2seq.decoder(memory, None, text_positions=tpos, speaker_embed=spk)
        with stage("converter"):
            mel = outputs.reshape(1, -1, model.mel_dim)
            post_in = states.reshape(1, mel.size(1), -1) if model.use_decoder_state_for_postnet_input else mel
            linear = model.postnet(post_in, spk)[0].cpu().numpy()
    with stage("vocoder"):
        return audio.inv_spectrogram(linear.T)


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power, clock = [x.strip() for x in out.stdout.strip().split(",")]
    except Exception as ex:                    # the measurement stays valid; say what could not be read
        power = clock = "unknown (%s)" % type(ex).__name__
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="deepvoice3_ljspeech")
    ap.add_argument("--batch", type=int, default=16, choices=[1, 4, 16, 32])
    ap.add_argument("--utterances", type=int, default=32)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--conv-math", default="tc", choices=["tc", "fp32"])
    ap.add_argument("--no-single", action="store_true", help="skip the one-utterance loop (and the output check)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_synthesis.py measures the GPU path; no GPU found")
    from test_gpu_models import preset_kwargs
    from deepvoice3_pytorch_b200 import audio, builder, ops
    from deepvoice3_pytorch_b200.synthesis import tts_batch
    ops.conv_math = a.conv_math
    bname, kw = preset_kwargs(a.preset)
    torch.manual_seed(1234)
    model = getattr(builder, bname)(dropout=0.0, **kw).cuda().eval()
    dec = model.seq2seq.decoder
    dec.max_decoder_steps = a.steps - 1            # stop rule: n > max_decoder_steps -> exactly --steps steps
    with torch.no_grad():
        dec.fc.bias.fill_(-30.0)                   # done never > .5
    rng = np.random.RandomState(1)
    lengths = rng.randint(20, 191, size=a.utterances)
    seqs = [rng.randint(2, 149, size=n).astype(np.int64) for n in lengths]
    spk = [int(x) for x in rng.randint(0, kw["n_speakers"], size=a.utterances)] if kw["n_speakers"] > 1 else None

    out = {"metric": "batched text-to-speech synthesis", "unit": "utterances/s", "preset": a.preset,
           "batch": a.batch, "utterances": a.utterances, "decoder_steps": a.steps,
           "text_tokens": [int(lengths.min()), int(lengths.max())], "conv_math": a.conv_math,
           "griffin_lim_iters": audio.hparams.griffin_lim_iters, "weights": "random (seeded)", "card": card()}

    def report(timer, wall, wavs):
        audio_s = sum(w.size for w in wavs) / audio.hparams.sample_rate
        return {"utterances_per_s": a.utterances / wall, "audio_s_per_s": audio_s / wall, "wall_s": wall,
                "stage_s": {k: round(v, 4) for k, v in timer.t.items()}}

    # warm-up: module loads, graph capture paths, allocator (a full batch of the longest shape is not needed)
    tts_batch(model, seqs[:min(a.batch, 4)], speaker_ids=spk[:min(a.batch, 4)] if spk else None, batch_size=a.batch)
    timer = StageTimer()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = tts_batch(model, seqs, speaker_ids=spk, batch_size=a.batch, stage_timer=timer)
    torch.cuda.synchronize()
    batched = [r[0] for r in res]
    out["batched"] = report(timer, time.perf_counter() - t0, batched)
    assert all(r[1].shape[0] == a.steps for r in res), "an utterance did not run exactly --steps steps"
    out["value"] = out["batched"]["utterances_per_s"]

    if not a.no_single:
        synthesize_alone(model, seqs[0], spk[0] if spk else None, lambda n: contextlib.nullcontext())   # warm-up
        timer = StageTimer()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        single = [synthesize_alone(model, s, spk[i] if spk else None, timer) for i, s in enumerate(seqs)]
        torch.cuda.synchronize()
        out["single"] = report(timer, time.perf_counter() - t0, single)
        out["speedup"] = out["single"]["wall_s"] / out["batched"]["wall_s"]
        assert all(x.shape == y.shape for x, y in zip(batched, single)), "waveform lengths differ between arms"
        out["max_waveform_diff_rel_peak"] = max(float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-12))
                                                for x, y in zip(batched, single))
        if a.conv_math == "fp32":
            assert all(np.array_equal(x, y) for x, y in zip(batched, single)), "waveforms differ between arms"
            out["check"] = "all waveforms bit-identical between the arms"
        else:
            # tensor-core mode: a batch's GEMMs can take the tensor-core kernels where a short single sentence runs on
            # the exact-fp32 ones, and the free-running decoder carries that difference along -- so the bit-for-bit
            # check of the batching itself runs the first batch of utterances again through both arms in fp32 mode
            n = min(a.utterances, max(a.batch, 4))
            ops.conv_math = "fp32"
            try:
                xs = [r[0] for r in tts_batch(model, seqs[:n], speaker_ids=spk[:n] if spk else None,
                                              batch_size=a.batch)]
                ys = [synthesize_alone(model, s, spk[i] if spk else None, lambda _: contextlib.nullcontext())
                      for i, s in enumerate(seqs[:n])]
            finally:
                ops.conv_math = a.conv_math
            assert all(np.array_equal(x, y) for x, y in zip(xs, ys)), "fp32 waveforms differ between arms"
            out["check"] = "fp32 mode, first %d utterances: waveforms bit-identical between the arms" % n
    print(json.dumps(out))


if __name__ == "__main__":
    main()
