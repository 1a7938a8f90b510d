"""VCTK preprocessing throughput: ``preprocess.build_vctk_from_path`` (GPU resampling, trim bounds and fused STFT)
against a host arm on the same batches -- ``audio.load_wav`` (scipy resample_poly), the numpy fp64 trim restatement
``audio.trim_bounds_reference`` and the same fused STFT (a restatement of the reference's per-clip work, not the
reference itself: librosa and nnmnkwii are not used).

The corpus is synthetic and seeded, written to a temporary directory in the VCTK-Corpus layout: 48 kHz int16 clips of
1-8 s with quiet heads and tails, several speakers, a third of the utterances with HTS labels.  Prints one JSON line:
utterances/s and audio-s/s of both arms, per-stage times of the GPU pipeline, CUDA-event kernel times of the
resampler and the trim kernel with achieved fp64 FLOP/s and HBM bytes/s against the H100 SXM data sheet (34 TFLOP/s
fp64 vector, 3.35 TB/s), and the card name and power limit read in the same run.

    python bench_preprocess_vctk.py --utts 256 --batch 64
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FP64_PEAK, HBM_PEAK = 34e12, 3.35e12


def make_corpus(root, n_utts, n_speakers, seed):
    from scipy.io import wavfile
    rng = np.random.RandomState(seed)
    sr = 48000
    for i in range(n_utts):
        spk = "p%d" % (225 + i % n_speakers)
        stem = "%s_%03d" % (spk, i // n_speakers + 1)
        for d in ("txt", "wav48", "lab"):
            os.makedirs(os.path.join(root, d, spk), exist_ok=True)
        secs = rng.uniform(1.0, 8.0)
        n = int(secs * sr)
        head, tail = rng.uniform(0.1, 0.6), rng.uniform(0.1, 0.6)
        a, b = int(head * sr), n - int(tail * sr)
        t = np.arange(b - a) / sr
        f0 = rng.uniform(90, 220)
        x = 3e-4 * rng.randn(n)
        x[a:b] += 0.25 * sum(np.sin(2 * np.pi * k * f0 * t) / k for k in range(1, 6)) * (0.5 + 0.5 * np.sin(3 * t))
        x[a:b] += 0.02 * rng.randn(b - a)
        wavfile.write(os.path.join(root, "wav48", spk, stem + ".wav"), sr, (np.clip(x, -1, 1) * 32767).astype(np.int16))
        with open(os.path.join(root, "txt", spk, stem + ".txt"), "w", encoding="utf-8") as f:
            f.write("synthetic utterance %d of speaker %s.\n" % (i, spk))
        if i % 3 == 0:
            s, e = int(0.8 * head * 1e7), int((secs - 0.8 * tail) * 1e7)
            with open(os.path.join(root, "lab", spk, stem + ".lab"), "w") as f:
                f.write("0 %d pau\n%d %d a\n%d %d pau\n" % (s, s, e, e, int(secs * 1e7)))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in out.split(",")]
        return name, power
    except Exception as ex:          # the card name still comes from torch
        import torch
        return torch.cuda.get_device_name(0), "unknown (%s)" % ex


def host_arm(items, out_dir, batch):
    """load_wav (scipy) -> numpy label cut -> fp64 trim restatement -> rescaling -> the fused STFT, per batch."""
    from deepvoice3_pytorch_b200 import audio, preprocess
    hp = audio.hparams
    n = 0
    for i in range(0, len(items), batch):
        wavs = []
        for idx, (wav_path, lab_path), _ in items[i:i + batch]:
            x = audio.load_wav(wav_path)
            top_db = preprocess.TOP_DB_UNLABELLED
            if lab_path:
                b, e = preprocess.label_cut(lab_path, hp.sample_rate)
                x, top_db = x[b:e], preprocess.TOP_DB_LABELLED
            s, e = audio.trim_bounds_reference(x, top_db)
            y = x[s:e]
            if len(y):
                wavs.append(y / np.abs(y).max() * hp.rescaling_max if hp.rescaling else y)
        for k, (lin, mel) in enumerate(preprocess.spectrograms_batch(wavs)):
            np.save(os.path.join(out_dir, "h-spec-%05d.npy" % (n + k)), lin, allow_pickle=False)
            np.save(os.path.join(out_dir, "h-mel-%05d.npy" % (n + k)), mel, allow_pickle=False)
        n += len(wavs)


def stages(items, out_dir, batch):
    """The GPU pipeline of one pass split at its stage boundaries (each stage synchronised, so the sum exceeds the
    overlapped end-to-end time)."""
    import torch
    from deepvoice3_pytorch_b200 import audio, preprocess
    T = dict.fromkeys(["decode", "h2d", "resample", "trim", "d2h", "stft", "save"], 0.0)

    def clock(key, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        T[key] += time.perf_counter() - t0
        return r

    for i in range(0, len(items), batch):
        clips = clock("decode", lambda: [preprocess._load_vctk(src) for _, src, _ in items[i:i + batch]])
        dev = clock("h2d", lambda: preprocess._host_buffer(clips).cuda())
        out, lens = clock("resample", lambda: audio.resample_batch(dev, [len(c[0]) for c in clips], 48000))
        cuts = []
        for (pcm, sr, cut), n in zip(clips, lens):
            b, e = (0, n) if cut is None else (min(cut[0], n), min(cut[1], n))
            cuts.append((b, max(0, e - b), 15 if cut is None else 25))
        bounds = clock("trim", lambda: audio.trim_bounds_batch(out, [c[1] for c in cuts], [c[2] for c in cuts],
                                                               [c[0] for c in cuts]))
        host, bh = clock("d2h", lambda: (out.cpu().numpy(), bounds.cpu().numpy()))
        segs = [host[k, c[0] + bh[k, 0]:c[0] + bh[k, 1]] for k, c in enumerate(cuts)]
        feats = clock("stft", lambda: preprocess.spectrograms_batch([s for s in segs if len(s)]))

        def save():
            for k, (lin, mel) in enumerate(feats):
                np.save(os.path.join(out_dir, "s-spec-%05d.npy" % (i + k)), lin, allow_pickle=False)
                np.save(os.path.join(out_dir, "s-mel-%05d.npy" % (i + k)), mel, allow_pickle=False)
        clock("save", save)
    return {k: round(v * 1e3, 2) for k, v in T.items()}


def kernel_times(items, batch, reps):
    """CUDA-event times of one batch's resampler and trim launches, with the work they do."""
    import torch
    from deepvoice3_pytorch_b200 import audio, preprocess
    clips = [preprocess._load_vctk(src) for _, src, _ in items[:batch]]
    dev = preprocess._host_buffer(clips).cuda()
    lens = [len(c[0]) for c in clips]
    out, olens = audio.resample_batch(dev, lens, 48000)
    _, ntaps, _ = audio._device_bank(dev.device, *audio.resample_ratio(48000))
    res = {}
    for name, fn, flops, nbytes in (
            ("resample", lambda: audio.resample_batch(dev, lens, 48000),
             2.0 * ntaps * sum(olens), 2.0 * sum(lens) + 4.0 * out.numel()),
            ("trim", lambda: audio.trim_bounds_batch(out, olens, 15),
             2 * 2.0 * 2048 * sum(n // 512 + 1 for n in olens), 4.0 * sum(olens))):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        s = e0.elapsed_time(e1) / reps * 1e-3
        bound = max(flops / FP64_PEAK, nbytes / HBM_PEAK)
        res[name] = {"us_per_call": round(s * 1e6, 1), "fp64_tflops": round(flops / s / 1e12, 3),
                     "hbm_gbs": round(nbytes / s / 1e9, 1),
                     "bound": "fp64" if flops / FP64_PEAK > nbytes / HBM_PEAK else "hbm",
                     "share_of_roof": round(bound / s, 3)}
    res["clips"], res["audio_s"] = len(clips), round(sum(lens) / 48000.0, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--speakers", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_preprocess_vctk.py needs a GPU")
    from deepvoice3_pytorch_b200 import data, preprocess
    name, power = card()
    with tempfile.TemporaryDirectory() as tmp:
        in_dir = os.path.join(tmp, "VCTK-Corpus")
        make_corpus(in_dir, args.utts, args.speakers, args.seed)
        items = preprocess.vctk_utterances(in_dir)
        audio_s = sum(data._wav_header(src[0])[1] for _, src, _ in items) / 48000.0
        warm = os.path.join(tmp, "warm")
        os.makedirs(warm)
        preprocess.build_vctk_from_path(in_dir, warm, batch_clips=args.batch,
                                        speakers=sorted({os.path.basename(os.path.dirname(s[0])) for _, s, _ in items[:2]}))
        arms = {}
        for arm in ("gpu", "host"):
            out = os.path.join(tmp, arm)
            os.makedirs(out)
            t0 = time.perf_counter()
            if arm == "gpu":
                rows = preprocess.build_vctk_from_path(in_dir, out, num_workers=args.workers, batch_clips=args.batch)
            else:
                host_arm(items, out, args.batch)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            arms[arm] = {"s": round(dt, 3), "utts_per_s": round(len(items) / dt, 1),
                         "audio_s_per_s": round(audio_s / dt, 1)}
        arms["gpu"]["rows"] = len(rows)
        st_dir = os.path.join(tmp, "stages")
        os.makedirs(st_dir)
        stage_ms = stages(items, st_dir, args.batch)
        kern = kernel_times(items, args.batch, args.reps)
    print(json.dumps({"bench": "preprocess_vctk", "card": name, "power_limit": power, "utts": len(items),
                      "audio_s": round(audio_s, 1), "batch_clips": args.batch, "workers": args.workers,
                      "gpu_pipeline": arms["gpu"], "host_restatement": arms["host"],
                      "speedup": round(arms["host"]["s"] / arms["gpu"]["s"], 2),
                      "stage_ms_single_thread": stage_ms, "kernels": kern}))


if __name__ == "__main__":
    main()
