"""Training the multi-speaker preset from a VCTK tree: the preprocessed .npy corpus vs. the wav48 files with per-batch
GPU resampling of each trimmed segment, end to end through a DataLoader.

    python bench_train_vctk_wav.py [--utts 192] [--speakers 8] [--batch-size 16] [--workers 0,2,4] [--json out.json]

A seeded synthetic 48 kHz int16 VCTK tree (bench_preprocess_vctk.make_corpus: 1-8 s clips, a third with HTS labels) is
written to a temporary directory.  Three sources then feed TrainStep(use_graph=True) on the deepvoice3_vctk preset,
for conv_math "tc" and "tc1", in the same DistributedSimilarLengthSampler order, once per DataLoader worker count
(pinned memory), the sources alternating in one process:

    npy     build_vctk_from_path -> TrainTxtDataset -> collate -> to_device
    vctk    WavDataset.from_vctk -> collate_wav -> wav_batch_to_device (segments resampled on the GPU)
    wav48   WavDataset over the same files -> collate_wav -> wav_batch_to_device: HOST-resampled (audio.load_wav) and
            UNTRIMMED, so its targets are longer and differ; it shows what the plain wav path would cost here

Each loader runs once untimed (worker start-up, page cache), then once timed.  Reported: steps/s and real frames/s per
arm (the npy/vctk frames; wav48 trains on more frames per utterance and is reported with its own count), the resident
step rate of the same npy batches already on the device, host item+collate ms per batch on one thread, H2D bytes per
step, disk bytes per utterance, the segment resampler's and the targets kernel's time per batch (CUDA events around
many replays of a CUDA graph of each stage) with the resampler's fp64 FLOP/s and bytes/s computed from shapes, the
index pass cold and from its cache, and the card's name, power limit and max SM clock read in the same run.  Prints
one JSON line.
"""
import argparse
import functools
import json
import os
import shutil
import subprocess
import tempfile
import time

import numpy as np
import torch

from bench import PRESETS
from bench_preprocess_vctk import make_corpus
from bench_train_wav import dir_bytes, host_batch_bytes
from deepvoice3_pytorch_b200 import audio, builder, data, ops, preprocess
from deepvoice3_pytorch_b200.train_step import TrainStep, to_device

PRESET = "deepvoice3_vctk"


def text_to_sequence(text):
    return [ord(c) % 60 + 2 for c in text]


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    vals = (q.stdout.strip().split(", ") + ["?"] * 3)[:3] if q.returncode == 0 else [None] * 3
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi_name": vals[0], "power_limit": vals[1],
            "max_sm_clock": vals[2]}


def resampler_work(batches):
    """(fp64 FMAs, bytes moved) of the segment launches of these collate_wav batches: ntaps FMAs per output sample;
    the span read once, the bank once per CTA, the fp32 rows written (padding included)."""
    flops = nbytes = 0
    for b in batches:
        pitch_out = max(8, -(-max(b["wav_lengths"].tolist()) // 8) * 8)
        for (row, n_in, a, m, s0, n), sr in zip(b["src_desc"].tolist(), b["src_rates"].tolist()):
            up, down = audio.resample_ratio(sr)
            bank, _ = audio.resample_filter_bank(up, down)
            ntaps = bank.shape[0]
            flops += 2 * ntaps * n
            nbytes += m * b["wav"].element_size() + 4 * pitch_out + bank.nbytes * -(-pitch_out // 4096)
    return flops, nbytes


def graph_us(fn, reps):
    """Device time of fn's launches in us: captured once in a CUDA graph (so the host-side checks between launches do
    not show up as device idle time), then CUDA events around reps replays."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=192)
    ap.add_argument("--speakers", type=int, default=8)
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--workers", default="0,2,4")
    ap.add_argument("--reps", type=int, default=20, help="CUDA-event repetitions of the kernel timings")
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_vctk_wav.py needs a CUDA device")
    bname, kw, extra = PRESETS[PRESET]
    r, ds, B = kw["r"], kw["downsample_step"], args.batch_size
    workers = [int(w) for w in args.workers.split(",")]
    tmp = tempfile.mkdtemp(prefix="dv3_vctkwav_")
    try:
        in_dir, out_dir, idx = os.path.join(tmp, "in"), os.path.join(tmp, "out"), os.path.join(tmp, "index.npz")
        os.makedirs(out_dir)
        make_corpus(in_dir, args.utts, args.speakers, args.seed)
        t0 = time.perf_counter()
        preprocess.write_metadata(preprocess.build_vctk_from_path(in_dir, out_dir, num_workers=4), out_dir)
        t_pre = time.perf_counter() - t0
        t0 = time.perf_counter()
        vctk = data.WavDataset.from_vctk(in_dir, text_to_sequence, index_path=idx)
        t_cold = time.perf_counter() - t0
        t0 = time.perf_counter()
        data.WavDataset.from_vctk(in_dir, text_to_sequence, index_path=idx)
        t_cached = time.perf_counter() - t0
        npy = data.TrainTxtDataset(out_dir, text_to_sequence)
        assert npy.frame_lengths == vctk.frame_lengths
        wav48 = data.WavDataset(vctk.items, text_to_sequence)
        srcs = {"npy": (npy, data.collate), "vctk": (vctk, data.collate_wav), "wav48": (wav48, data.collate_wav)}
        n_utts = len(npy)
        sampler = data.DistributedSimilarLengthSampler(npy.frame_lengths, batch_size=B, seed=args.seed)
        order = list(iter(sampler))
        batch_idx = [order[i:i + B] for i in range(0, len(order), B)]
        real = {"npy": sum(npy.frame_lengths[i] for i in order)}
        real["vctk"], real["wav48"] = real["npy"], sum(wav48.frame_lengths[i] for i in order)

        def to_dev(name, hb):
            return to_device(hb, "cuda") if name == "npy" else data.wav_batch_to_device(hb, "cuda", r, ds)

        res = {"preset": PRESET, "utterances": n_utts, "batch_size": B, "batches": len(batch_idx),
               "real_frames": real, "preprocess_seconds": t_pre, "index_seconds_cold": t_cold,
               "index_seconds_cached": t_cached, "host_cpus": len(os.sched_getaffinity(0)), **card()}
        per_src, hbs = {}, {}
        for name, (dset, coll) in srcs.items():               # one thread: what one loader worker does per batch
            t0 = time.perf_counter()
            hbs[name] = [coll([dset[i] for i in b], r, ds) for b in batch_idx]
            per_src[name] = {"host_item_collate_ms_per_batch": 1e3 * (time.perf_counter() - t0) / len(batch_idx),
                             "h2d_bytes_per_step": float(np.mean([host_batch_bytes(b) for b in hbs[name]]))}
        per_src["npy"]["disk_bytes_per_utt"] = dir_bytes(out_dir, ".npy") / n_utts
        wav_bytes = sum(os.path.getsize(it[0]) for it in vctk.items) / n_utts
        per_src["vctk"]["disk_bytes_per_utt"] = per_src["wav48"]["disk_bytes_per_utt"] = wav_bytes
        res["sources"] = per_src

        # the device stages alone (inputs already on the device), CUDA events over every batch, many times
        staged = []
        for b in hbs["vctk"]:
            dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()}
            lens = b["wav_lengths"].tolist()
            out = torch.empty(len(lens), max(8, -(-max(lens) // 8) * 8), device="cuda")
            desc, rates = b["src_desc"].tolist(), b["src_rates"].tolist()
            groups = []
            for sr in sorted(set(rates)):
                rows = [i for i, x in enumerate(rates) if x == sr]
                groups.append(([desc[i] for i in rows], sr, dev["src_desc"][rows[0]:rows[-1] + 1]))
            T = data.max_target_length(b["target_lengths"].tolist(), r, ds)
            staged.append((dev, out, groups, lens, T))

        def resample_all():
            for dev, out, groups, _, _ in staged:
                for seg, sr, seg_dev in groups:
                    audio.resample_segments(dev["wav"], seg, sr, out, seg_dev=seg_dev)

        def targets_all():
            for dev, out, _, lens, T in staged:
                audio.stft_mel_targets(out, lens, T, r, ds, lengths_dev=dev["wav_lengths"])
        rs_us = graph_us(resample_all, args.reps) / len(staged)
        flops, nbytes = resampler_work(hbs["vctk"])
        res["resampler_us_per_batch"] = rs_us
        res["resampler_fp64_flop_per_s"] = flops / len(staged) / (rs_us * 1e-6)
        res["resampler_bytes_per_s"] = nbytes / len(staged) / (rs_us * 1e-6)
        res["targets_us_per_batch"] = graph_us(targets_all, args.reps) / len(staged)
        resident = [to_device(b, "cuda") for b in hbs["npy"]]
        del staged

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
                mode = {"resident": {"steps_per_s": len(resident) / dt, "real_frames_per_s": real["npy"] / dt,
                                     "ms_per_step": 1e3 * dt / len(resident)}}
                for w in workers:
                    for name in srcs:                          # alternating sources
                        dset, coll = srcs[name]
                        loader = torch.utils.data.DataLoader(
                            dset, batch_size=B, sampler=sampler, drop_last=True, num_workers=w, pin_memory=True,
                            collate_fn=functools.partial(coll, r=r, downsample_step=ds), persistent_workers=w > 0)
                        for hb in loader:                      # untimed: worker start-up, page cache, new buckets
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
                        mode["%s_w%d" % (name, w)] = {"steps_per_s": n / dt, "real_frames_per_s": real[name] / dt,
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
