"""Intelligibility (DESIGN.md section 2.20), four measurements:

  1. the STOI / ESTOI kernels on 512 seeded ragged pairs of 1-10 s at 22.05 kHz (a speech-like clip and a noisy copy):
     µs per stage with CUDA events over --iters calls after --warmup (resampling to 10 kHz, silence removal + overlap-add,
     band envelopes, segments + per-pair means), the whole ``intelligibility.stoi`` call and pairs/s, and for each stage
     the bytes and FLOPs computed from the shapes against the roof that binds it;
  2. the fp64 numpy oracle (tests/stoi_oracle.py) on the first --cpu-pairs pairs on the host CPU, extrapolated to all
     512 by samples;
  3. ``evaluate_vocoder`` (copy synthesis) on bench_vocoder.py's 16 clips for Griffin-Lim-60, LWS-30 and fast
     Griffin-Lim-20: mean STOI / ESTOI and seconds per call;
  4. ``evaluate_intelligibility`` on deepvoice3_ljspeech with random weights, 64 utterances: stage times.

Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing to the tree.

    python bench_stoi.py [--iters 20] [--warmup 3] [--cpu-pairs 4]
"""
import argparse
import contextlib
import json
import os
import sys
import time

import numpy as np
import torch

from bench import PRESETS
from bench_mcd import _cpu_name, _events
from bench_speaker_adapt import card
from deepvoice3_pytorch_b200 import audio, builder, intelligibility as I, ops
from deepvoice3_pytorch_b200._lib import lib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import stoi_oracle as SO  # noqa: E402
from test_stoi_host import voiced  # noqa: E402

HBM = 3.35e12
FP32_PEAK = 67e12
FP64_PEAK = 34e12                 # non-tensor fp64


def _pairs(n_pairs=512, seed=0):
    rng = np.random.RandomState(seed)
    sr = 22050
    clean, proc = [], []
    for k in range(n_pairs):
        n = int(rng.uniform(1.0, 10.0) * sr)
        x = voiced(n, sr, seed + k).astype(np.float64)
        snr = rng.uniform(-5, 20)
        y = x + rng.randn(n) * np.sqrt(np.mean(x ** 2) / 10 ** (snr / 10))
        clean.append(x.astype(np.float32))
        proc.append(y.astype(np.float32))
    return clean, proc


def _share(flops, nbytes, peak, us):
    t = us * 1e-6
    bound = max(flops / peak, nbytes / HBM)
    return {"flops": int(flops), "bytes": int(nbytes), "gflop_s": round(flops / t / 1e9, 1),
            "gb_s": round(nbytes / t / 1e9, 1), "binding": "compute" if flops / peak > nbytes / HBM else "hbm",
            "bound_us": round(bound * 1e6, 2), "roof_share": round(bound / t, 4)}


def kernels(clean, proc, iters, warmup):
    dev = torch.device("cuda")
    a, b = [torch.from_numpy(x).to(dev) for x in clean], [torch.from_numpy(x).to(dev) for x in proc]
    P = len(a)
    wavs = a + b
    lens = [int(w.numel()) for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True)
    an = I._Analysis(wavs, list(range(P)) * 2)
    x10, n10 = audio.resample_batch(pad, lens, audio.hparams.sample_rate, sr_to=I.FS)
    table, win64, bands = I._tables(dev)
    st = ops._stream()
    p = ops._p
    n = 2 * P
    F0 = an.F0
    cap = [(f - 1) * I.HOP + I.FRAME if f else 0 for f in F0]
    blocks = [(c, t0) for c in range(n) for t0 in range(0, max(F0[c] - 1, 0), I.BAND_WARPS)]
    blocks_d = torch.tensor(blocks, dtype=torch.int32).to(dev)
    caps = [max(f - 1, 0) for f in F0[:P]]
    seg_cap = [max(c - I.N_SEG + 1, 0) for c in caps]
    paths = [np.repeat(np.arange(c, dtype=np.int32)[:, None], 2, 1) for c in caps]
    path_off = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    seg_off = np.concatenate([[0], np.cumsum(seg_cap)[:-1]]).astype(np.int64)
    pr_d = torch.from_numpy(np.stack([np.arange(P), np.arange(P) + P, path_off, seg_off], 1).astype(np.int64)).to(dev)
    path_d = torch.from_numpy(np.concatenate(paths)).to(dev)
    sblocks = [(q, s0) for q in range(P) for s0 in range(0, seg_cap[q], I.SEG_WARPS)]
    sblocks_d = torch.tensor(sblocks, dtype=torch.int32).to(dev)
    seg = torch.empty(sum(seg_cap), 2, dtype=torch.float64, device=dev)
    res = torch.empty(P, 2, dtype=torch.float64, device=dev)
    counts = torch.empty(P, 2, dtype=torch.int32, device=dev)

    def silence_ola():
        lib.call("dv3_stoi_frames", p(x10), p(an.clips), n, p(win64), p(an.energy), p(an.keep), p(an.kept_idx),
                 p(an.kept), st)
        lib.call("dv3_stoi_overlap_add", p(x10), p(an.clips), n, max(cap), p(table), p(an.kept_idx), p(an.kept),
                 p(an.ola), p(an.frames), st)

    t = {"resample": _events(lambda: audio.resample_batch(pad, lens, audio.hparams.sample_rate, sr_to=I.FS), iters,
                             warmup),
         "silence_ola": _events(silence_ola, iters, warmup),
         "bands": _events(lambda: lib.call("dv3_stoi_bands", p(an.ola), p(an.clips), p(blocks_d), len(blocks),
                                           p(table), p(bands), p(an.frames), p(an.env), None, st), iters, warmup),
         "segments": _events(lambda: lib.call("dv3_stoi_segments", p(an.env), p(an.clips), p(pr_d), P, p(sblocks_d),
                                              len(sblocks), p(path_d), p(an.frames), p(an.kept), p(seg), p(res),
                                              p(counts), st), iters, warmup)}
    t_call = _events(lambda: I.stoi(a, b), max(3, iters // 4), 1)
    out = I.stoi(a, b)
    # work from the shapes
    up, down = audio.resample_ratio(audio.hparams.sample_rate, I.FS)
    ntaps = audio.resample_filter_bank(up, down)[0].shape[0]
    s_in, s_out = sum(lens), sum(n10)
    frames_all = sum(F0)
    kept = an.kept.cpu().numpy()
    K = int(kept[:P].sum()) * 2                                     # both sides use the clean mask
    F = int(an.frames.cpu().numpy().sum())
    J = int(out["segments"].sum())
    ola_samples = sum((int(k) - 1) * I.HOP + I.FRAME for k in np.concatenate([kept[:P], kept[:P]]) if k > 0)
    fft_flops = 5 * 256 * 8 + 10 * 256 + 2 * 256 + 3 * 220          # 4 radix-4 passes, split, window, band sums
    work = {"resample": _share(2 * ntaps * s_out, 4 * s_in + 4 * s_out, FP64_PEAK, t["resample"]),
            "silence_ola": _share(3 * 256 * frames_all + 3 * ola_samples,
                                  4 * s_out + 16 * frames_all + 12 * ola_samples, FP64_PEAK, t["silence_ola"]),
            "bands": _share(fft_flops * F, 4 * 256 * F + 4 * 15 * F, FP32_PEAK, t["bands"]),
            "segments": _share(24 * 450 * J, (2 * 450 * 4 + 30 * 8 + 16) * J, FP64_PEAK, t["segments"])}
    return {"pairs": P, "seconds_of_audio": round(s_in / audio.hparams.sample_rate, 1), "frames_10k": frames_all,
            "kept_frames": K, "envelope_frames": F, "segments": J,
            "us": {k: round(v, 1) for k, v in t.items()}, "stoi_call_us": round(t_call, 1),
            "pairs_per_s": round(P / (t_call * 1e-6), 1), "work": work,
            "mean_stoi": float(np.nanmean(out["stoi"])), "mean_estoi": float(np.nanmean(out["estoi"]))}


def cpu_oracle(clean, proc, n):
    t0 = time.perf_counter()
    for x, y in zip(clean[:n], proc[:n]):
        SO.stoi(x, y, 22050)
    s = time.perf_counter() - t0
    done, total = sum(x.size for x in clean[:n]), sum(x.size for x in clean)
    return {"cpu": _cpu_name(), "threads": torch.get_num_threads(), "pairs_timed": n, "s": round(s, 3),
            "all_pairs_s_extrapolated_by_samples": round(s * total / done, 1)}


def vocoders():
    """bench_vocoder.py's 16 clips, copy-synthesized by each phase-recovery method at its default iteration count."""
    from oracle import audio_oracle as A
    rng = np.random.RandomState(0)
    frames = [int(t) for t in rng.randint(2 * 22050 // 256, 10 * 22050 // 256, size=16)]
    wavs = [torch.from_numpy(A.synthetic_clip(100 + c, n=audio.inv_num_samples(t)).astype(np.float32)).cuda()
            for c, t in enumerate(frames)]
    hp = audio.hparams
    out = {}
    for method, iters in (("griffin_lim", hp.griffin_lim_iters), ("lws", hp.lws_iters),
                          ("fast_griffin_lim", hp.fast_griffin_lim_iters)):
        I.evaluate_vocoder(wavs, method)                               # warm-up
        ts = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = I.evaluate_vocoder(wavs, method)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        out[method] = {"iterations": iters, "mean_stoi": round(r["mean_stoi"], 4), "mean_estoi": round(r["mean_estoi"], 4),
                       "min_stoi": round(float(np.nanmin(r["stoi"])), 4), "s": [round(v, 3) for v in ts]}
    return out


def evaluation(n_utt=64, max_steps=200):
    bname, kw, _ = PRESETS["deepvoice3_ljspeech"]
    torch.manual_seed(0)
    model = getattr(builder, bname)(**kw).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = max_steps
    rng = np.random.RandomState(0)
    seqs = [rng.randint(2, 149, rng.randint(20, 80)) for _ in range(n_utt)]
    refs = [voiced(rng.randint(2, 6) * 22050, 22050, k) for k in range(n_utt)]
    times = {}

    @contextlib.contextmanager
    def timer(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    I.evaluate_intelligibility(model, seqs, refs, stage_timer=timer)             # warm-up
    times.clear()
    res = I.evaluate_intelligibility(model, seqs, refs, stage_timer=timer)
    return {"preset": "deepvoice3_ljspeech", "utterances": n_utt, "max_decoder_steps": max_steps,
            "ms": {k: round(t * 1e3, 2) for k, t in times.items()},
            "scored": int(np.isfinite(res["stoi"]).sum()), "mean_stoi": res["mean_stoi"],
            "mean_estoi": res["mean_estoi"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-pairs", type=int, default=4)
    ap.add_argument("--no-eval", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stoi.py needs a CUDA device")
    clean, proc = _pairs()
    out = {"card": card(), "stoi": kernels(clean, proc, args.iters, args.warmup),
           "cpu_oracle_fp64": cpu_oracle(clean, proc, args.cpu_pairs), "evaluate_vocoder": vocoders()}
    if not args.no_eval:
        out["evaluate_intelligibility"] = evaluation()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
