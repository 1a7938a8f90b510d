"""Audio path throughput at STFT frames other than 1024 / 256 (csrc/stft_any.cu, csrc/lws_any.cu).  Prints one JSON
line per geometry, then one for the 1024 / 256 A/B:

* forward (preemphasis -> STFT -> linear + mel dB, the preprocessing / training-target kernel) on 10 s synthetic clips at
  the geometry's sample rate, fp32 and int16 input: clips/s, kernel time from CUDA events, algorithmic bytes
  (samples in, (N/2+1 + n_mels) * T * 4 out) and FLOPs (5 (N/2) log2(N/2) for the complex FFT plus 2 per bin for the
  split and magnitude and 2 per non-zero mel weight) computed from shapes, achieved GB/s and the share of the
  3.35 TB/s HBM3 roof of the H100 SXM data sheet;
* Griffin-Lim (60 iterations) and LWS (no-future + 30 iterations) on a ragged batch of 16 clips of 2-10 s;
* at 1024 / 256 the specialised kernel (dv3_stft_mel) and the general one (dv3_stft_mel_geom) alternating in one process.
The card name and its power limit are read in the same run.

    python bench_stft_geometry.py [--clips 64] [--iters 10]
"""
import argparse
import ctypes
import json
import math
import subprocess

import numpy as np
import torch

from deepvoice3_pytorch_b200 import audio
from deepvoice3_pytorch_b200._lib import lib

GEOMS = [(16000, 256, 64), (16000, 512, 128), (16000, 800, 200), (22050, 1024, 512), (22050, 2048, 256),
         (24000, 1200, 300), (44100, 2048, 512), (48000, 2400, 600), (48000, 4096, 1024)]
HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                       # the number is still reported, with the reason the limit is missing
        pl = "unknown (%s)" % ex
    return name, pl


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def clips_at(sr, n, count, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.arange(n, device="cuda", dtype=torch.float32) / sr
    f = 200 + 3000 * torch.rand(count, 1, device="cuda", generator=g)
    x = 0.3 * torch.sin(2 * math.pi * f * t[None]) + 0.05 * torch.randn(count, n, device="cuda", generator=g)
    return x.contiguous()


def forward_row(sr, N, R, nclips, iters):
    audio.hparams.sample_rate, audio.hparams.fft_size, audio.hparams.hop_size = sr, N, R
    g = audio.check_geometry()
    n = 10 * sr
    n_pad = (n + 7) // 8 * 8
    x = torch.zeros(nclips, n_pad, device="cuda")
    x[:, :n] = clips_at(sr, n, nclips)
    x16 = (x * 32767).to(torch.int16)
    lens = [n] * nclips
    T = audio.num_frames(n)
    basis, start, length = audio._device_basis(x.device)
    nnz = int(length.sum())
    res = {}
    for name, wav in (("fp32", x), ("int16", x16)):
        ld = torch.tensor(lens, dtype=torch.int32, device="cuda")

        def fn():
            audio.stft_mel_targets(wav, lens, T + 1, 1, 1, lengths_dev=ld)
        s = timed(fn, iters)
        bytes_ = nclips * (n * wav.element_size() + (g.bins + audio.hparams.num_mels) * T * 4)
        M = N // 2
        flops = nclips * T * (5 * M * math.log2(M) + 2 * 3 * g.bins + 2 * nnz)
        res[name] = dict(clips_per_s=round(nclips / s, 1), ms=round(s * 1e3, 3), GBps=round(bytes_ / s / 1e9, 1),
                         hbm_share=round(bytes_ / s / HBM, 4), GFLOPs=round(flops / s / 1e9, 1))
    return res


def inverse_row(sr, N, R):
    audio.hparams.sample_rate, audio.hparams.fft_size, audio.hparams.hop_size = sr, N, R
    K = N // 2 + 1
    rng = np.random.RandomState(1)
    secs = rng.uniform(2, 10, 16)
    frames = [audio.num_frames(int(s * sr)) for s in secs]
    mag = torch.rand(16, max(frames), K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    gl = timed(lambda: audio.griffin_lim_batch(mag, frames, n_iter=60), 2)
    lw = timed(lambda: audio.lws_batch(mag, frames, n_iter=30), 2)
    return dict(griffin_lim60_ms=round(gl * 1e3, 1), lws30_ms=round(lw * 1e3, 1), audio_s=round(float(secs.sum()), 1))


def ab_default(nclips, iters, rounds=5):
    """dv3_stft_mel (specialised) and dv3_stft_mel_geom (general) at 1024 / 256, alternating."""
    audio.hparams.sample_rate, audio.hparams.fft_size, audio.hparams.hop_size = 22050, 1024, 256
    n = 220500
    x = clips_at(22050, n, nclips)
    ld = torch.full((nclips,), n, dtype=torch.int32, device="cuda")
    T = audio.num_frames(n)
    basis, start, length = audio._device_basis(x.device)
    lin = torch.empty(nclips, T, 513, device="cuda")
    mel = torch.empty(nclips, T, 80, device="cuda")
    tab = audio._geometry_table(x.device, 1024, 256)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    spec = lambda: lib.call("dv3_stft_mel", p(x), p(ld), p(basis), p(start), p(length), p(lin), p(mel), nclips, n, T,
                            80, 0.97, -100.0, 20.0, st)
    gen = lambda: lib.call("dv3_stft_mel_geom", p(x), 0, p(ld), None, 1.0, p(tab), p(basis), p(start), p(length),
                           p(lin), p(mel), nclips, n, T, 0, 1, 80, 1024, 256, 0.97, -100.0, 20.0, st)
    a, b = [], []
    for _ in range(rounds):
        a.append(timed(spec, iters))
        b.append(timed(gen, iters))
    bytes_ = nclips * (n * 4 + (513 + 80) * T * 4)
    return dict(specialised_ms=[round(v * 1e3, 3) for v in a], general_ms=[round(v * 1e3, 3) for v in b],
                specialised_hbm_share=round(bytes_ / min(a) / HBM, 4), general_hbm_share=round(bytes_ / min(b) / HBM, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--geoms", type=str, default="", help="comma-separated indices into GEOMS (default: all)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stft_geometry.py needs a GPU")
    name, pl = card()
    sel = [GEOMS[int(i)] for i in args.geoms.split(",")] if args.geoms else GEOMS
    for sr, N, R in sel:
        row = dict(bench="stft_geometry", gpu=name, power_limit=pl, sample_rate=sr, fft_size=N, hop_size=R,
                   clips=args.clips, forward=forward_row(sr, N, R, args.clips, args.iters), **inverse_row(sr, N, R))
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(bench="stft_geometry_ab_1024_256", gpu=name, power_limit=pl, clips=args.clips,
                          **ab_default(args.clips, args.iters))), flush=True)


if __name__ == "__main__":
    main()
