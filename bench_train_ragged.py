"""Training throughput on variable-length batches: eager steps vs. bucketed CUDA-graph steps.

    python bench_train_ragged.py [--preset deepvoice3_ljspeech] [--batches 64] [--batch-size 16] [--json out.json]

A seeded LJSpeech-like corpus goes through the data path of the package -- DistributedSimilarLengthSampler ->
collate (pinned) -> H2D -> TrainStep.step -- once in eager mode and once with TrainStep(use_graph=True), whose first
batch shape gets its own graph and every other shape a graph per bucket (data.bucket_shape).  Both modes see the same
batches in the same order; each runs one untimed pass (warm-up; graph mode captures its buckets there) and one timed
pass.  Batches are collated before the timed pass, so the timed pass covers H2D + step.

No real corpus is available offline, so lengths are drawn from a distribution shaped like LJSpeech (13,100 clips of
1.1-10.1 s, ~6.6 s mean, ~15 characters per second, 22050 Hz audio with hop 256) -- an assumption, not a measurement:
    duration ~ Normal(6.6 s, 2.2 s) clipped to [1.1 s, 10.1 s];  frames = round(duration * 22050 / 256)
    characters = round(duration * 15.5 * LogNormal(0, 0.1)) clipped to [5, 190]
Spectrogram and text content is random (the step's cost does not depend on it).

Reports steps/s and real frames/s (frames of the utterances themselves, no padding) per mode, the padding overhead
(padded / real linear frames), graphs captured, total capture time, peak device memory, and the card's name and
power limit read in the same run.  Prints one JSON line.
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from bench import PRESETS
from deepvoice3_pytorch_b200 import builder, data
from deepvoice3_pytorch_b200.train_step import TrainStep, to_device

SR, HOP, CHARS_PER_S = 22050, 256, 15.5
DUR_MEAN, DUR_SD, DUR_MIN, DUR_MAX = 6.6, 2.2, 1.1, 10.1


def corpus_lengths(n, seed):
    rng = np.random.RandomState(seed)
    dur = np.clip(rng.normal(DUR_MEAN, DUR_SD, n), DUR_MIN, DUR_MAX)
    frames = np.round(dur * SR / HOP).astype(np.int64)
    chars = np.clip(np.round(dur * CHARS_PER_S * rng.lognormal(0.0, 0.1, n)), 5, 190).astype(np.int64)
    return chars, frames


def make_batches(n_batches, B, linear_dim, n_speakers, seed, r=1, downsample_step=4):
    """Host batches (pinned) in sampler order."""
    n = n_batches * B
    chars, frames = corpus_lengths(n, seed)
    rng = np.random.RandomState(seed + 1)
    pool_t = int(frames.max())
    mel_pool = rng.rand(pool_t, 80).astype(np.float32)
    lin_pool = rng.rand(pool_t, linear_dim).astype(np.float32)
    sampler = data.DistributedSimilarLengthSampler(frames, batch_size=B, seed=seed)
    order = list(iter(sampler))
    batches = []
    for i in range(0, len(order), B):
        items = []
        for j in order[i:i + B]:
            item = (rng.randint(2, 149, chars[j]).astype(np.int32), mel_pool[:frames[j]], lin_pool[:frames[j]])
            items.append(item + (int(j) % n_speakers,) if n_speakers > 1 else item)
        batches.append(data.collate(items, r=r, downsample_step=downsample_step, pin=True))
    return batches


def run_mode(preset, batches, use_graph, seed):
    bname, kw, extra = PRESETS[preset]
    torch.manual_seed(seed)
    model = getattr(builder, bname)(**kw).cuda().train()
    step = TrainStep(model, use_graph=use_graph, guided_attention_sigma=extra["guided_attention_sigma"],
                     r=kw["r"], downsample_step=kw["downsample_step"])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for b in batches:                                   # warm-up pass (graph mode: captures every bucket)
        step.step(to_device(b, "cuda"))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in batches:
        loss = step.step(to_device(b, "cuda"))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    real = sum(int(b["target_lengths"].sum()) for b in batches)
    out = {"steps_per_s": len(batches) / dt, "real_frames_per_s": real / dt, "ms_per_step": 1e3 * dt / len(batches),
           "final_loss": float(loss), "peak_allocated_gb": torch.cuda.max_memory_allocated() / 1e9,
           "peak_reserved_gb": torch.cuda.max_memory_reserved() / 1e9}
    if use_graph:
        out.update(graphs_captured=step.graphs_captured, capture_seconds=step.capture_seconds)
    del step, model
    torch.cuda.empty_cache()
    return out


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (None, None)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="deepvoice3_ljspeech", choices=sorted(PRESETS))
    ap.add_argument("--batches", type=int, default=64)
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_ragged.py needs a CUDA device")
    bname, kw, _ = PRESETS[args.preset]
    batches = make_batches(args.batches, args.batch_size, kw["linear_dim"], kw.get("n_speakers", 1), args.seed,
                           kw["r"], kw["downsample_step"])
    real = sum(int(b["target_lengths"].sum()) for b in batches)
    collated = sum(b["y"].shape[0] * b["y"].shape[1] for b in batches)
    first = (batches[0]["x"].shape, batches[0]["y"].shape)
    bucketed = 0                        # graph mode runs the first shape exactly, every other one padded to its bucket
    for b in batches:
        _, bd = data.bucket_shape(b["x"].shape[1], b["done"].shape[1])
        T = b["y"].shape[1] if (b["x"].shape, b["y"].shape) == first else bd * kw["r"] * kw["downsample_step"]
        bucketed += b["y"].shape[0] * T
    res = {"preset": args.preset, "batches": len(batches), "batch_size": args.batch_size,
           "distinct_shapes": len({(b["x"].shape[1], b["done"].shape[1]) for b in batches}),
           "padding_collate": collated / real, "padding_bucketed": bucketed / real,
           "bucket_grid": [data.BUCKET_TEXT, data.BUCKET_DEC], **card()}
    res["eager"] = run_mode(args.preset, batches, False, args.seed)
    res["graph"] = run_mode(args.preset, batches, True, args.seed)
    res["speedup"] = res["graph"]["steps_per_s"] / res["eager"]["steps_per_s"]
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
