#!/usr/bin/env python
"""Continuous-batching synthesis benchmark: ``synthesis.tts_stream`` (decoder slots refilled as their utterances stop)
against ``synthesis.tts_batch`` (sorted, padded chunks that run until their last row stops) on the same sequences, with
``--slots`` decoder rows in both (``batch_size = slots``).

    python bench_synthesis_stream.py [--preset deepvoice3_ljspeech] [--slots 16] [--utterances 64] [--max-steps 200]

Random weights (seeded); text lengths are drawn in 20..190 tokens.  A random-weight model never raises its done flag on
its own, so every utterance would run to max_decoder_steps and hide the whole effect.  Assumption stated here: the done
head's bias is calibrated once (``spread_done_bias`` in tests/test_gpu_synthesis_stream.py) from one run of the done
pre-activations, set to minus the median of each utterance's largest pre-activation after min_decoder_steps; about
half the utterances then stop at their own steps and the rest at max_decoder_steps.  The spread of stop steps this
produced is reported.

Reports, for each arm: utterances/s, seconds of audio per second, per-stage time (each stage ends in a device
synchronise), and decoder row occupancy = useful decoder steps / row-steps executed (a chunk of tts_batch executes
rows x its steps rounded up to the check interval; tts_stream executes slots x its step-program replays).  The card's
name and power limit are read in the same run.  With ``--conv-math fp32`` it checks that both arms produced the same
outputs bit for bit; in the default tensor-core mode it reports how far the waveforms are apart.  Prints one JSON
line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="deepvoice3_ljspeech")
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--utterances", type=int, default=64)
    ap.add_argument("--max-steps", type=int, default=200)
    ap.add_argument("--min-steps", type=int, default=10)
    ap.add_argument("--conv-math", default="tc", choices=["tc", "fp32"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_synthesis_stream.py measures the GPU path; no GPU found")
    from bench_synthesis import StageTimer, card
    from test_gpu_models import preset_kwargs
    from test_gpu_synthesis_stream import spread_done_bias
    from deepvoice3_pytorch_b200 import audio, builder, incremental, ops
    from deepvoice3_pytorch_b200.synthesis import tts_batch, tts_stream
    ops.conv_math = a.conv_math
    bname, kw = preset_kwargs(a.preset)
    torch.manual_seed(1234)
    model = getattr(builder, bname)(dropout=0.0, **kw).cuda().eval()
    dec = model.seq2seq.decoder
    dec.max_decoder_steps, dec.min_decoder_steps = a.max_steps, a.min_steps
    rng = np.random.RandomState(1)
    lengths = rng.randint(20, 191, size=a.utterances)
    seqs = [rng.randint(2, 149, size=n).astype(np.int64) for n in lengths]
    spk = [int(x) for x in rng.randint(0, kw["n_speakers"], size=a.utterances)] if kw["n_speakers"] > 1 else None
    bias = spread_done_bias(model, seqs, spk)

    out = {"metric": "continuous-batching text-to-speech synthesis", "unit": "utterances/s", "preset": a.preset,
           "slots": a.slots, "utterances": a.utterances, "max_decoder_steps": a.max_steps,
           "min_decoder_steps": a.min_steps, "text_tokens": [int(lengths.min()), int(lengths.max())],
           "conv_math": a.conv_math, "done_bias": bias, "griffin_lim_iters": audio.hparams.griffin_lim_iters,
           "weights": "random (seeded), done bias calibrated", "card": card()}

    def report(timer, wall, wavs, executed, useful):
        audio_s = sum(w.size for w in wavs) / audio.hparams.sample_rate
        return {"utterances_per_s": a.utterances / wall, "audio_s_per_s": audio_s / wall, "wall_s": wall,
                "stage_s": {k: round(v, 4) for k, v in timer.t.items()},
                "decoder_row_steps": executed, "useful_steps": useful, "occupancy": useful / executed}

    # warm-up: module loads, both arms' graph capture paths, the allocator
    n_w = min(a.utterances, a.slots + 2)
    tts_batch(model, seqs[:n_w], speaker_ids=spk[:n_w] if spk else None, batch_size=a.slots)
    list(tts_stream(model, seqs[:n_w], speaker_ids=spk[:n_w] if spk else None, slots=a.slots, post_batch=a.slots))

    timer = StageTimer()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = tts_batch(model, seqs, speaker_ids=spk, batch_size=a.slots, stage_timer=timer)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    steps = [r[1].shape[0] for r in res]
    order = sorted(range(len(seqs)), key=lambda i: -seqs[i].size)      # tts_batch's chunks
    Tmax, chk = a.max_steps + 1, incremental.CHECK_EVERY
    executed = 0
    for c in range(0, len(order), a.slots):
        chunk = order[c:c + a.slots]
        n = max(steps[i] for i in chunk)
        executed += len(chunk) * min(-(-n // chk) * chk, Tmax)
    out["batched"] = report(timer, wall, [r[0] for r in res], executed, sum(steps))

    timer = StageTimer()
    stats = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = dict(tts_stream(model, seqs, speaker_ids=spk, slots=a.slots, post_batch=a.slots, stage_timer=timer,
                          stats=stats))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    stream = [got[i] for i in range(len(seqs))]
    out["stream"] = report(timer, wall, [r[0] for r in stream], stats["replays"] * a.slots, stats["useful_steps"])
    out["stream"]["refills"] = len(stats["refills"])
    out["value"] = out["stream"]["utterances_per_s"]
    out["speedup"] = out["batched"]["wall_s"] / out["stream"]["wall_s"]

    s = np.array(steps)
    out["stop_steps"] = {"min": int(s.min()), "median": float(np.median(s)), "max": int(s.max()),
                         "distinct": int(len(set(steps))), "at_max": int((s == a.max_steps + 1).sum())}
    same = [i for i in range(len(seqs)) if stream[i][1].shape[0] == steps[i]]
    out["utterances_with_other_steps"] = len(seqs) - len(same)
    out["max_waveform_diff_rel_peak"] = max(float(np.abs(stream[i][0] - res[i][0]).max() /
                                                  max(np.abs(res[i][0]).max(), 1e-12)) for i in same)
    if a.conv_math == "fp32":
        assert all(np.array_equal(x, y) for r, q in zip(stream, res) for x, y in zip(r, q)), "outputs differ"
        out["check"] = "every output bit-identical between the arms"
    else:
        # tensor-core mode: the two arms encode different groups, whose GEMMs may take other kernels, so an utterance
        # whose done flag grazes 0.5 can stop a step apart; the exact equality is the fp32-mode check
        out["check"] = "tensor-core mode: waveforms of equal length compared relative to their peak"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
