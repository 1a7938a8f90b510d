#!/usr/bin/env python
"""Vocoder phase recovery: Griffin-Lim (``hparams.griffin_lim_iters`` = 60 iterations) against LWS (no-future
initialisation + ``hparams.lws_iters`` batch iterations, csrc/lws.cu) and fast Griffin-Lim (momentum
``hparams.griffin_lim_momentum``, ``hparams.fast_griffin_lim_iters`` iterations, DESIGN.md section 7.3) on 16
synthetic clips of mixed length (2-10 s at 22.05 kHz, seeded), run one clip at a time (batch 1) and as one ragged
batch (batch 16).

    python bench_vocoder.py [--clips 16] [--rounds 7] [--sweep 60] [--fgla-sweep 60]

Device-resident magnitudes in, waveforms out (the phase recovery and inverse STFT; no dB conversion or de-emphasis).
The three methods alternate within each round, in one process; times are CUDA events, median and [min, max] over the
rounds.  Also: the init scan and one batch iteration alone, one plain and one momentum Griffin-Lim iteration alone
(and their complex-STFT launches), the spectral convergence ||A - |STFT(x)||| / ||A|| of each method (numpy fp64 STFT
of the result, mean over clips), and the LWS and fast Griffin-Lim iteration counts that reach Griffin-Lim's (and, for
fast Griffin-Lim, LWS's) convergence.  Prints ONE JSON line.  Needs a GPU; writes nothing.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _device_info():
    info = {"name": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit_and_max_sm_clock"] = out[torch.cuda.current_device()] if out else "unknown"
    except Exception as ex:
        info["power_limit_and_max_sm_clock"] = "unknown (%s)" % ex
    return info


def _stats(ts):
    ts = sorted(ts)
    return {"median": float(np.median(ts)), "min": ts[0], "max": ts[-1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--sweep", type=int, default=60, help="largest LWS iteration count of the convergence sweep")
    ap.add_argument("--fgla-sweep", type=int, default=60,
                    help="largest fast Griffin-Lim iteration count of the convergence sweep")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocoder.py needs a CUDA device")
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    from oracle import audio_oracle as A

    hp = audio.hparams
    rng = np.random.RandomState(0)
    frames = [int(t) for t in rng.randint(2 * 22050 // 256, 10 * 22050 // 256, size=args.clips)]
    mags = [np.abs(A.lws_stft(A.synthetic_clip(100 + c, n=audio.inv_num_samples(t)))).astype(np.float32)
            for c, t in enumerate(frames)]
    T_max = max(frames)
    batch = torch.zeros(args.clips, T_max, 513, device="cuda")
    for c, a in enumerate(mags):
        batch[c, :a.shape[0]] = torch.from_numpy(a)
    singles = [batch[c:c + 1, :t].contiguous() for c, t in enumerate(frames)]
    audio_s = sum(audio.inv_num_samples(t) for t in frames) / float(hp.sample_rate)

    methods = {"griffin_lim": lambda m, f: audio.griffin_lim_batch(m, f, hp.griffin_lim_iters),
               "lws": lambda m, f: audio.lws_batch(m, f, hp.lws_iters),
               "fast_griffin_lim": lambda m, f: audio.griffin_lim_batch(m, f, hp.fast_griffin_lim_iters,
                                                                        momentum=hp.griffin_lim_momentum)}
    runs = {"batch16": lambda fn: fn(batch, frames),
            "batch1": lambda fn: [fn(singles[c], [t]) for c, t in enumerate(frames)]}

    def timed(fn):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) * 1e-3

    for run in runs.values():                            # warm every shape
        for fn in methods.values():
            run(fn)
    torch.cuda.synchronize()
    times = {(r, m): [] for r in runs for m in methods}
    for _ in range(args.rounds):
        for r, run in runs.items():
            for m, fn in methods.items():
                times[(r, m)].append(timed(lambda: run(fn)))

    # the LWS stages alone on the ragged batch
    w = audio._lws_weights(batch.device)
    frames_d = torch.tensor(frames, dtype=torch.int32, device="cuda")
    spec = torch.empty(args.clips, T_max, 513, 2, device="cuda")
    other = torch.empty_like(spec)
    st = torch.cuda.current_stream().cuda_stream
    vp = lambda t: ctypes.c_void_p(t.data_ptr())

    def init_scan():
        lib.call("dv3_lws_nofuture_batched", vp(batch), vp(spec), vp(w), vp(frames_d), T_max, args.clips, 1,
                 ctypes.c_void_p(st))

    def iterations(n=20):
        for i in range(n):
            a, b = (spec, other) if i % 2 == 0 else (other, spec)
            lib.call("dv3_lws_iterate_batched", vp(batch), vp(a), vp(b), vp(w), vp(frames_d), T_max, args.clips,
                     ctypes.c_void_p(st))
    init_scan(); iterations()
    t_init = [timed(init_scan) for _ in range(args.rounds)]
    t_iter = [timed(iterations) / 20 for _ in range(args.rounds)]
    bins = sum(frames) * 513
    it_med = float(np.median(t_iter))

    # one Griffin-Lim iteration alone on the ragged batch, plain and with momentum, alternating; and its STFT launch
    samples_d = torch.tensor([audio.inv_num_samples(t) for t in frames], dtype=torch.int32, device="cuda")
    n_max = max(audio.inv_num_samples(t) for t in frames)
    x = torch.zeros(args.clips, n_max, device="cuda")
    prev = torch.zeros_like(spec)
    beta = hp.griffin_lim_momentum / (1.0 + hp.griffin_lim_momentum)
    g = audio.check_geometry(mel=False)
    tab = audio._geometry_table(batch.device, g.n_fft, g.hop)

    def stft_plain():
        lib.call("dv3_stft_complex_geom", vp(x), vp(samples_d), n_max, vp(batch), vp(spec), vp(frames_d), T_max,
                 args.clips, vp(tab), g.n_fft, g.hop, ctypes.c_void_p(st))

    def stft_momentum():
        lib.call("dv3_stft_complex_momentum_geom", vp(x), vp(samples_d), n_max, vp(batch), vp(prev), vp(spec),
                 vp(frames_d), T_max, args.clips, beta, vp(tab), g.n_fft, g.hop, ctypes.c_void_p(st))

    def gl_iterations(stft, n=20):
        for _ in range(n):
            stft()
            x.zero_()
            lib.call("dv3_istft_geom", vp(spec), vp(x), vp(samples_d), n_max, vp(frames_d), T_max, args.clips,
                     vp(tab), g.n_fft, g.hop, ctypes.c_void_p(st))

    def stft_launches(stft, n=20):
        for _ in range(n):
            stft()
    gl_iterations(stft_plain); gl_iterations(stft_momentum)
    t_gl = {"plain": [], "momentum": []}
    t_stft = {"plain": [], "momentum": []}
    for _ in range(args.rounds):
        for name, fn in (("plain", stft_plain), ("momentum", stft_momentum)):
            t_gl[name].append(timed(lambda: gl_iterations(fn)) / 20)
            t_stft[name].append(timed(lambda: stft_launches(fn)) / 20)

    # quality
    def sc(wavs):
        w_ = wavs.cpu().numpy()
        out = []
        for c, a in enumerate(mags):
            S = np.abs(A.lws_stft(w_[c, :audio.inv_num_samples(frames[c])].astype(np.float64)))[:a.shape[0]]
            out.append(float(np.linalg.norm(a - S) / np.linalg.norm(a)))
        return float(np.mean(out)), out
    sc_gl, sc_gl_clips = sc(audio.griffin_lim_batch(batch, frames, hp.griffin_lim_iters))
    sweep = {}
    for n in sorted(set(list(range(0, 11)) + list(range(15, args.sweep + 1, 5)) + [hp.lws_iters])):
        sweep[n] = sc(audio.lws_batch(batch, frames, n))[0]
    reach = next((n for n in sorted(sweep) if sweep[n] <= sc_gl), None)
    sc_lws, sc_lws_clips = sc(audio.lws_batch(batch, frames, hp.lws_iters))
    fgla = lambda n: audio.griffin_lim_batch(batch, frames, n, momentum=hp.griffin_lim_momentum)
    sc_fgla, sc_fgla_clips = sc(fgla(hp.fast_griffin_lim_iters))
    fgla_sweep = {}
    for n in sorted(set(list(range(0, 11)) + list(range(15, args.fgla_sweep + 1, 5)) + [hp.fast_griffin_lim_iters])):
        fgla_sweep[n] = sc(fgla(n))[0]
    fgla_reach = {target: next((n for n in sorted(fgla_sweep) if fgla_sweep[n] <= v), None)
                  for target, v in (("griffin_lim", sc_gl), ("lws", sc_lws))}

    out = {"metric": "vocoder phase recovery: Griffin-Lim vs LWS", "device": _device_info(),
           "clips": args.clips, "frames": frames, "audio_seconds": audio_s, "rounds": args.rounds,
           "griffin_lim_iters": hp.griffin_lim_iters, "lws_iters": hp.lws_iters,
           "fast_griffin_lim_iters": hp.fast_griffin_lim_iters, "griffin_lim_momentum": hp.griffin_lim_momentum}
    for (r, m), ts in times.items():
        s = _stats(ts)
        out.setdefault(r, {})[m] = {"seconds": s, "clips_per_s": args.clips / s["median"],
                                    "audio_s_per_s": audio_s / s["median"]}
    out["lws_stages_batch16"] = {
        "init_scan_ms": {k: v * 1e3 for k, v in _stats(t_init).items()},
        "iteration_ms": {k: v * 1e3 for k, v in _stats(t_iter).items()},
        # per bin: 76 complex multiply-adds (608 flop) and >= 20 bytes (8 in, 4 magnitude, 8 out)
        "iteration_gflops": bins * 608 / it_med / 1e9, "iteration_gbs_min_traffic": bins * 20 / it_med / 1e9}
    ms = lambda ts: {k: v * 1e3 for k, v in _stats(ts).items()}
    gl_med = {k: float(np.median(v)) for k, v in t_gl.items()}
    stft_med = {k: float(np.median(v)) for k, v in t_stft.items()}
    out["griffin_lim_stages_batch16"] = {
        "plain_iteration_ms": ms(t_gl["plain"]), "momentum_iteration_ms": ms(t_gl["momentum"]),
        "momentum_over_plain_iteration": gl_med["momentum"] / gl_med["plain"],
        "plain_stft_ms": ms(t_stft["plain"]), "momentum_stft_ms": ms(t_stft["momentum"]),
        "momentum_over_plain_stft": stft_med["momentum"] / stft_med["plain"],
        # the momentum epilogue reads and writes prev: 16 more bytes per bin than the projected STFT
        "momentum_extra_bytes": bins * 16,
        "momentum_extra_bytes_min_us_at_3.35TBps": bins * 16 / 3.35e12 * 1e6}
    out["spectral_convergence"] = {"griffin_lim": sc_gl, "lws": sc_lws, "griffin_lim_clips": sc_gl_clips,
                                   "lws_clips": sc_lws_clips, "lws_sweep": sweep,
                                   "lws_iters_to_reach_griffin_lim": reach,
                                   "fast_griffin_lim": sc_fgla, "fast_griffin_lim_clips": sc_fgla_clips,
                                   "fast_griffin_lim_sweep": fgla_sweep,
                                   "fast_griffin_lim_iters_to_reach_griffin_lim": fgla_reach["griffin_lim"],
                                   "fast_griffin_lim_iters_to_reach_lws": fgla_reach["lws"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
