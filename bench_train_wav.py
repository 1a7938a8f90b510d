"""Training fed from wav files vs. from the preprocessed .npy corpus, end to end through a DataLoader.

    python bench_train_wav.py [--preset deepvoice3_ljspeech] [--clips 256] [--batch-size 16] [--workers 0,2,4]
                              [--json out.json]

A seeded synthetic corpus in LJSpeech layout (metadata.csv + wavs/*.wav, random 16-bit PCM with the length model of
bench_train_ragged.py) is written to a temporary directory and preprocessed with preprocess.build_from_path.  The same
DistributedSimilarLengthSampler order then runs through a DataLoader (pinned memory) into TrainStep(use_graph=True),
for conv_math "tc" and "tc1", once per worker count from each source, the two sources alternating in one process:

    npy   TrainTxtDataset -> collate -> to_device
    wav   WavDataset.from_ljspeech -> collate_wav -> wav_batch_to_device (targets on the GPU)

Each source's loader is iterated once untimed (worker start-up, page cache) and once timed.  Reported per arm: steps/s
and real frames/s (the utterances' own frames); per math mode: the device-resident step time of the same batches
(already on the GPU, so a loader that starves the step shows up as the gap); per source: host collate ms/batch (item
loading + collate on one thread), H2D bytes/step and disk bytes/clip; the targets kernel's time per batch (CUDA
events); the card's name and power limit read in the same run.  Prints one JSON line.
"""
import argparse
import functools
import json
import os
import shutil
import tempfile
import time

import numpy as np
import torch

from bench import PRESETS
from bench_train_ragged import SR, card, corpus_lengths
from deepvoice3_pytorch_b200 import audio, builder, data, ops, preprocess
from deepvoice3_pytorch_b200.train_step import TrainStep, to_device

LETTERS = "abcdefghijklmnopqrstuvwxyz ,."


def text_to_sequence(text):
    return [LETTERS.index(c) + 2 for c in text]


def write_corpus(root, n, seed):
    """n utterances: samples = frames * hop of the length model, text of its character count (at least min_text)."""
    from scipy.io import wavfile
    chars, frames = corpus_lengths(n, seed)
    rng = np.random.RandomState(seed + 1)
    os.makedirs(os.path.join(root, "wavs"))
    lines = []
    for i in range(n):
        n_samples = int(frames[i]) * audio.hparams.hop_size
        x = np.clip(rng.normal(0.0, 3000.0, n_samples), -32768, 32767).astype(np.int16)
        wavfile.write(os.path.join(root, "wavs", "LJ%05d.wav" % i), SR, x)
        text = "".join(rng.choice(list(LETTERS), max(int(chars[i]), audio.hparams.min_text)))
        lines.append("LJ%05d|%s|%s\n" % (i, text, text))
    with open(os.path.join(root, "metadata.csv"), "w", encoding="utf-8") as f:
        f.writelines(lines)


def dir_bytes(path, suffix):
    return sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path) if f.endswith(suffix))


def host_batch_bytes(b):
    return sum(v.numel() * v.element_size() for v in b.values() if torch.is_tensor(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="deepvoice3_ljspeech", choices=sorted(PRESETS))
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--workers", default="0,2,4")
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_wav.py needs a CUDA device")
    bname, kw, extra = PRESETS[args.preset]
    r, ds, B = kw["r"], kw["downsample_step"], args.batch_size
    workers = [int(w) for w in args.workers.split(",")]
    tmp = tempfile.mkdtemp(prefix="dv3_wavbench_")
    try:
        in_dir, out_dir = os.path.join(tmp, "in"), os.path.join(tmp, "out")
        os.makedirs(out_dir)
        write_corpus(in_dir, args.clips, args.seed)
        t0 = time.perf_counter()
        rows = preprocess.build_from_path(in_dir, out_dir, num_workers=4)
        preprocess.write_metadata(rows, out_dir)
        t_pre = time.perf_counter() - t0
        srcs = {"npy": (data.TrainTxtDataset(out_dir, text_to_sequence), data.collate),
                "wav": (data.WavDataset.from_ljspeech(in_dir, text_to_sequence), data.collate_wav)}
        assert srcs["npy"][0].frame_lengths == srcs["wav"][0].frame_lengths
        n_clips = len(srcs["npy"][0])
        sampler = data.DistributedSimilarLengthSampler(srcs["npy"][0].frame_lengths, batch_size=B, seed=args.seed)
        order = list(iter(sampler))
        batch_idx = [order[i:i + B] for i in range(0, len(order), B)]
        real = sum(srcs["npy"][0].frame_lengths[i] for i in order)

        def to_dev(name, hb):
            return to_device(hb, "cuda") if name == "npy" else data.wav_batch_to_device(hb, "cuda", r, ds)

        res = {"preset": args.preset, "clips": n_clips, "batch_size": B, "batches": len(batch_idx),
               "real_frames": real, "preprocess_seconds": t_pre,
               "host_cpus": len(os.sched_getaffinity(0)), **card()}
        per_src = {}
        for name, (dset, coll) in srcs.items():               # one thread: what one loader worker does per batch
            t0 = time.perf_counter()
            hbs = [coll([dset[i] for i in idx], r, ds) for idx in batch_idx]
            per_src[name] = {"host_collate_ms_per_batch": 1e3 * (time.perf_counter() - t0) / len(hbs),
                             "h2d_bytes_per_step": float(np.mean([host_batch_bytes(b) for b in hbs]))}
            if name == "npy":
                resident = [to_device(b, "cuda") for b in hbs]
            else:
                wav_hbs = hbs
        per_src["npy"]["disk_bytes_per_clip"] = dir_bytes(out_dir, ".npy") / n_clips
        per_src["wav"]["disk_bytes_per_clip"] = dir_bytes(os.path.join(in_dir, "wavs"), ".wav") / n_clips
        res["sources"] = per_src

        # targets kernel alone (waveforms already on the device), CUDA events over every batch
        dev_wavs = [(b["wav"].cuda(), b["wav_lengths"], b["wav_lengths"].cuda(),
                     data.max_target_length(b["target_lengths"].tolist(), r, ds)) for b in wav_hbs]
        for w, lh, ld, T in dev_wavs:
            audio.stft_mel_targets(w, lh, T, r, ds, lengths_dev=ld)
        ts = []
        for _ in range(5):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for w, lh, ld, T in dev_wavs:
                audio.stft_mel_targets(w, lh, T, r, ds, lengths_dev=ld)
            e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e) * 1e3 / len(dev_wavs))
        res["targets_kernel_us_per_batch"] = float(np.median(ts))

        res["modes"] = {}
        for math in ("tc", "tc1"):
            old = ops.conv_math
            ops.conv_math = math
            try:
                torch.manual_seed(args.seed)
                model = getattr(builder, bname)(**kw).cuda().train()
                step = TrainStep(model, use_graph=True, guided_attention_sigma=extra["guided_attention_sigma"],
                                 r=r, downsample_step=ds)
                for b in resident:                             # captures every bucket
                    step.step(b)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for b in resident:
                    step.step(b)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                mode = {"resident": {"steps_per_s": len(resident) / dt, "real_frames_per_s": real / dt,
                                     "ms_per_step": 1e3 * dt / len(resident)}}
                for w in workers:
                    for name in ("npy", "wav"):                # alternating sources
                        dset, coll = srcs[name]
                        loader = torch.utils.data.DataLoader(
                            dset, batch_size=B, sampler=sampler, drop_last=True, num_workers=w, pin_memory=True,
                            collate_fn=functools.partial(coll, r=r, downsample_step=ds), persistent_workers=w > 0)
                        for hb in loader:                      # untimed: worker start-up, page cache
                            step.step(to_dev(name, hb))
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        n = 0
                        for hb in loader:
                            step.step(to_dev(name, hb))
                            n += 1
                        torch.cuda.synchronize()
                        dt = time.perf_counter() - t0
                        del loader
                        mode["%s_w%d" % (name, w)] = {"steps_per_s": n / dt, "real_frames_per_s": real / dt,
                                                      "ms_per_step": 1e3 * dt / n}
                mode["graphs_captured"] = step.graphs_captured
                res["modes"][math] = mode
                del step, model
                torch.cuda.empty_cache()
            finally:
                ops.conv_math = old
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
