"""Pitch accuracy (DESIGN.md section 2.18), four measurements:

  1. the YIN kernel on 512 seeded clips of 200-900 frames (bench_mcd.py's a-side lengths, speech-like harmonic signals
     with noise): µs per call (the tracker and the gate launch) with CUDA events over --iters calls after --warmup,
     frames/s, and FLOP/s (3 flops per difference term: a subtract and an fma) against the FP32 data-sheet roof;
  2. bench_mcd.py's 512 cepstrum pairs: ``dtw_path``'s two kernels next to ``dtw``'s one, in alternation, the
     direction-buffer bytes, and the backtrace alone;
  3. the fp64 numpy oracle (tests/pitch_oracle.py) on the first --cpu-clips clips on the host CPU, extrapolated to all
     512 by frames;
  4. pitch.evaluate_pitch on deepvoice3_ljspeech with random weights, 64 utterances: stage times.

Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing to the tree.

    python bench_pitch.py [--iters 20] [--warmup 3] [--cpu-clips 4]
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
from bench_mcd import K, _cpu_name, _events, _pairs
from bench_speaker_adapt import card
from deepvoice3_pytorch_b200 import audio, builder, mcd, ops, pitch
from deepvoice3_pytorch_b200._lib import lib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import pitch_oracle as PO  # noqa: E402

FP32_PEAK = 67e12


def _clips(seed=0):
    """512 waveforms of bench_mcd.py's a-side frame counts: a harmonic tone with a slow glide, plus noise."""
    a_np, _ = _pairs(seed)
    rng = np.random.RandomState(seed + 1)
    sr, R = audio.hparams.sample_rate, audio.hparams.hop_size
    out = []
    for a in a_np:
        n = (a.shape[0] - 3) * R                            # num_frames(n) = a.shape[0] at N = 4 R
        t = np.arange(n) / sr
        f0 = rng.uniform(80, 300) * (1 + 0.1 * np.sin(2 * np.pi * rng.uniform(0.5, 3) * t))
        ph = 2 * np.pi * np.cumsum(f0) / sr
        x = sum(0.3 / h * np.sin(h * ph) for h in range(1, 6)) + 0.01 * rng.randn(n)
        out.append(x.astype(np.float32))
    return out


def yin_kernel(wavs, iters, warmup):
    dev = torch.device("cuda")
    clips = [torch.from_numpy(w).to(dev) for w in wavs]
    tau_min, tau_max, gate = pitch.yin_params()
    frames = pitch._check_wavs(clips)
    t = _events(lambda: pitch._yin(clips, frames, tau_min, tau_max, 0.1, gate), iters, warmup)
    F = int(sum(frames))
    W = audio.hparams.fft_size
    terms = F * W * tau_max
    flops = 3 * terms
    f0 = torch.cat([f for f, _ in pitch.yin_f0(clips)]).cpu().numpy()
    return {"clips": len(wavs), "frames": F, "W": W, "tau_range": [tau_min, tau_max], "us": round(t, 1),
            "frames_per_s": F / (t * 1e-6), "difference_terms": terms, "flops": flops,
            "tflops": round(flops / (t * 1e-6) / 1e12, 2), "fp32_roof_share": round(flops / FP32_PEAK / (t * 1e-6), 4),
            "fp32_bound_us": round(flops / FP32_PEAK * 1e6, 1), "voiced_fraction": float((f0 > 0).mean())}


def dtw_kernels(iters, warmup):
    dev = torch.device("cuda")
    a_np, b_np = _pairs()
    P = len(a_np)
    cep = mcd.mel_cepstra([torch.from_numpy(x).to(dev) for x in a_np + b_np], K)
    la, lb = [x.shape[0] for x in a_np], [x.shape[0] for x in b_np]
    a, b = cep[:P], cep[P:]
    t_dtw, t_path = [], []
    for _ in range(3):                                     # alternate the two calls
        t_dtw.append(_events(lambda: mcd.dtw(a, b), iters, warmup))
        t_path.append(_events(lambda: mcd.dtw_path(a, b), iters, warmup))
    # the raw launches of one chunk: dtw_path's recursion, then the backtrace alone
    rows = [0] + np.cumsum(la + lb)[:-1].tolist()
    flat = torch.cat([c.contiguous() for c in list(a) + list(b)])
    work, ws_floats = mcd._work_list(rows[:P], la, rows[P:], lb)
    words = [mcd._dir_words(int(w[2]), int(w[4])) for w in work]
    path_work = np.stack([np.concatenate([[0], np.cumsum(words)[:-1]]),
                          np.concatenate([[0], np.cumsum([int(w[2]) + int(w[4]) - 1 for w in work])[:-1]])], 1)
    work_d, pw_d = torch.from_numpy(work).to(dev), torch.from_numpy(path_work).to(dev)
    ws = torch.empty(ws_floats, device=dev)
    dirs = torch.empty(int(sum(words)), dtype=torch.int32, device=dev)
    cost, length = torch.empty(P, device=dev), torch.empty(P, dtype=torch.int32, device=dev)
    path = torch.empty(int(sum(la) + sum(lb)), 2, dtype=torch.int32, device=dev)
    path_rows = torch.empty(P, dtype=torch.int32, device=dev)
    p, st = ops._p, ops._stream
    t_rec_path = _events(lambda: lib.call("dv3_dtw_path", p(flat), K, p(work_d), p(pw_d), p(ws), p(dirs), p(cost),
                                          p(length), P, st()), iters, warmup)
    t_rec = _events(lambda: lib.call("dv3_dtw_mcd", p(flat), K, p(work_d), p(ws), p(cost), p(length), P, st()),
                    iters, warmup)
    t_bt = _events(lambda: lib.call("dv3_dtw_backtrace", p(work_d), p(pw_d), p(dirs), p(path), p(path_rows), P, st()),
                   iters, warmup)
    assert np.array_equal(path_rows.cpu().numpy(), length.cpu().numpy())       # finite costs: the walk has L cells
    return {"pairs": P, "K": K, "dtw_us": [round(x, 1) for x in t_dtw], "dtw_path_us": [round(x, 1) for x in t_path],
            "direction_bytes": 4 * int(sum(words)), "kernel_dtw_mcd_us": round(t_rec, 1),
            "kernel_dtw_path_us": round(t_rec_path, 1), "kernel_backtrace_us": round(t_bt, 1)}


def cpu_oracle(wavs, n):
    t0 = time.perf_counter()
    frames = 0
    for w in wavs[:n]:
        frames += len(PO.yin(w)["f0"])
    s = time.perf_counter() - t0
    total = sum(PO.num_frames(w.size) for w in wavs)
    return {"cpu": _cpu_name(), "threads": torch.get_num_threads(), "clips_timed": n, "s": round(s, 3),
            "frames_per_s": frames / s, "all_512_clips_s_extrapolated_by_frames": round(s * total / frames, 1)}


def evaluation(n_utt=64, max_steps=200):
    bname, kw, _ = PRESETS["deepvoice3_ljspeech"]
    torch.manual_seed(0)
    model = getattr(builder, bname)(**kw).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = max_steps
    rng = np.random.RandomState(0)
    seqs = [rng.randint(2, 149, rng.randint(20, 80)) for _ in range(n_utt)]
    refs = [(rng.randn(rng.randint(2, 6) * 22050) * 0.1).astype(np.float32) for _ in range(n_utt)]
    times = {}

    @contextlib.contextmanager
    def timer(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    pitch.evaluate_pitch(model, seqs, refs, stage_timer=timer)             # warm-up
    times.clear()
    res = pitch.evaluate_pitch(model, seqs, refs, stage_timer=timer)
    return {"preset": "deepvoice3_ljspeech", "utterances": n_utt, "max_decoder_steps": max_steps,
            "ms": {k: round(t * 1e3, 2) for k, t in times.items()},
            "frames_synth_total": int(res["frames"][:, 0].sum()), "frames_ref_total": int(res["frames"][:, 1].sum()),
            "mean_vde": res["mean_vde"], "mean_mcd": res["mean_mcd"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-clips", type=int, default=4)
    ap.add_argument("--no-eval", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pitch.py needs a CUDA device")
    wavs = _clips()
    out = {"card": card(), "yin": yin_kernel(wavs, args.iters, args.warmup),
           "dtw_path": dtw_kernels(args.iters, args.warmup), "cpu_oracle_fp64": cpu_oracle(wavs, args.cpu_clips)}
    if not args.no_eval:
        out["evaluate_pitch"] = evaluation()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
