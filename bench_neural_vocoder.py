"""Neural vocoder benchmark (DESIGN.md section 2.23): the training step, the multi-resolution STFT loss kernels, inference
against the phase-recovery vocoders, and quality after a fixed training budget on synthetic clips.

  * step: B = 16 segments of S = 32 frames (8192 samples), graph-captured, in conv_math "tc" and "tc1", against the same
    network and loss in eager torch (cuDNN convs, torch.stft, TF32 off, torch.optim.Adam); ms/step (median, min, max
    over per-step device-event times) and native launches per step;
  * loss: forward (two complex STFTs + the reduction) and backward (per-bin gradient + inverse STFT) per resolution at
    the step's shape, timed as CUDA-graph replays, with the algorithmic bytes each moves against the 3.35 TB/s HBM
    roof;
  * inference: bench_vocoder.py's 16 synthetic clips of 2-10 s (seeds 100..115) vocoded at batch 16 and at batch 1,
    against Griffin-Lim-60, LWS-30 and fast Griffin-Lim-20 through audio.inv_spectrogram_batch; ms and audio s / s;
  * quality: --train-steps steps on synthetic clips with seeds from 1000 (disjoint from the evaluation clips), then the
    held-out MR-STFT loss on segments of the evaluation clips, spectral convergence at 1024 / 256 and STOI from
    intelligibility.evaluate_vocoder, next to the three phase-recovery methods.  Reported, not asserted.

Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM = 3.35e12


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
    return {"median": float(np.median(ts)), "min": float(ts[0]), "max": float(ts[-1])}


def _event_times(fn, n):
    out = []
    for _ in range(n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        out.append(s.elapsed_time(e))
    return out


def _wn(v, g):
    return g * v / v.pow(2).sum(tuple(range(1, v.dim())), keepdim=True).sqrt()


class EagerVocoder(torch.nn.Module):
    """The NeuralVocoder's network restated with torch ops (cuDNN convs) on copies of its parameters."""

    def __init__(self, voc):
        super().__init__()
        from deepvoice3_pytorch_b200 import conv as C, modules as Mo
        self.spec, params = [], torch.nn.ParameterList()
        for f in voc.layers:
            if isinstance(f, torch.nn.ReLU):
                self.spec.append(("relu", None, None))
                continue
            c = f.conv if isinstance(f, Mo.Conv1dGLU) else f
            kind = "glu" if isinstance(f, Mo.Conv1dGLU) else "convt" if isinstance(f, C.ConvTranspose1d) else "conv"
            i = len(params)
            for t in (c.weight_v, c.weight_g, c.bias):
                params.append(torch.nn.Parameter(t.detach().clone()))
            self.spec.append((kind, i, (c.kernel_size[0], getattr(c, "dilation", (1,))[0], getattr(c, "stride", (1,))[0])))
        self.params = params

    def forward(self, x):
        P = self.params
        for kind, i, cfg in self.spec:
            if kind == "relu":
                x = torch.relu(x)
                continue
            w, b = _wn(P[i], P[i + 1]), P[i + 2]
            k, d, s = cfg
            if kind == "convt":
                x = F.conv_transpose1d(x, w, b, stride=s)
            else:
                h = F.conv1d(x, w, b, padding=(k - 1) // 2 * d, dilation=d)
                if kind == "glu":
                    a, g = h.split(h.shape[1] // 2, dim=1)
                    h = (a * torch.sigmoid(g) + x) * 0.7071067811865476
                x = h
        return x.reshape(x.shape[0], -1)


def torch_stft_loss(y, x, resolutions):
    from oracle.audio_oracle import lws_window
    tot = 0.0
    n = y.shape[1]
    for N, R in resolutions:
        w = torch.from_numpy(lws_window(N, R)).float().to(y.device)
        nf = (n + N - 2 * R + R - 1) // R + 1
        L = (nf - 1) * R + N

        def spec(s):
            s = F.pad(s, (N - R, L - (N - R) - n))
            return torch.stft(s, N, R, window=w, center=False, return_complex=True)
        X, Y = spec(y), spec(x)
        a = torch.sqrt(torch.clamp_min(X.real ** 2 + X.imag ** 2, 1e-7))
        b = torch.sqrt(torch.clamp_min(Y.real ** 2 + Y.imag ** 2, 1e-7))
        sc = torch.linalg.norm((b - a).flatten(1), dim=1) / torch.linalg.norm(b.flatten(1), dim=1)
        mag = torch.mean(torch.abs(torch.log(b) - torch.log(a)).flatten(1), dim=1)
        tot = tot + (sc + mag).mean()
    return tot / len(resolutions)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=600)
    ap.add_argument("--clips", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_neural_vocoder.py needs a CUDA device")
    from deepvoice3_pytorch_b200 import audio, ops, vocoder
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.data import VocoderBatches
    from deepvoice3_pytorch_b200.intelligibility import evaluate_vocoder
    from oracle import audio_oracle as A

    hp = audio.hparams
    out = {"device": _device_info(), "B": 16, "seg_frames": 32}
    B, S = 16, 32
    train_wavs = [A.synthetic_clip(1000 + k, n=3 * 22050) for k in range(64)]
    batches = []
    vb = VocoderBatches(train_wavs, B, seg_frames=S, seed=0)
    epoch = 0
    while len(batches) < max(args.train_steps, args.steps + args.warmup):
        vb.set_epoch(epoch)
        batches += [vocoder.vocoder_batch(b, S) for b in vb]
        epoch += 1

    # ---- training step ----
    step_out = {}
    for mode in ("tc", "tc1"):
        ops.conv_math = mode
        torch.manual_seed(0)
        voc = vocoder.NeuralVocoder().cuda()
        st = vocoder.NeuralVocoderStep(voc, lr=1e-4, clip_thresh=1.0)
        for k in range(args.warmup):
            st.step(batches[k])
        ts = _event_times(lambda: st.step(batches[0]), args.steps)
        step_out[mode] = {"ms": _stats(ts), "launches_per_step": st.launches_per_step}
    ops.conv_math = "tc"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    eager = EagerVocoder(vocoder.NeuralVocoder()).cuda()
    opt = torch.optim.Adam(eager.parameters(), lr=1e-4)

    def eager_step():
        opt.zero_grad(set_to_none=True)
        loss = torch_stft_loss(eager(batches[0]["cond"]), batches[0]["target"], vocoder.DEFAULT_RESOLUTIONS)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(eager.parameters(), 1.0)
        opt.step()
    for _ in range(args.warmup):
        eager_step()
    step_out["eager_torch_fp32"] = {"ms": _stats(_event_times(eager_step, args.steps))}
    out["step"] = step_out

    # ---- loss kernels per resolution: each direction captured in a CUDA graph and replayed, so that the timed window
    # holds the device work of the launches alone (no Python, no allocator) ----
    y = torch.randn(B, S * hp.hop_size, device="cuda")
    x = torch.randn(B, S * hp.hop_size, device="cuda")
    n = y.shape[1]
    one = torch.ones(1, device="cuda")
    loss_out = {}

    def replay_us(fn, reps=50):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            keep = fn()                                  # warm the allocator and the kernels' attributes
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            keep = fn()
        g.replay()
        torch.cuda.synchronize()
        ts = _event_times(lambda: [g.replay() for _ in range(reps)], 5)
        del keep
        return float(np.median(ts)) * 1e3 / reps

    for N, R in vocoder.DEFAULT_RESOLUTIONS:
        res = ((N, R),)
        f_us = replay_us(lambda: vocoder._mrstft_forward(y, x, res, [n] * B))
        state = vocoder._mrstft_forward(y, x, res, [n] * B)[2]
        b_us = replay_us(lambda: vocoder._mrstft_backward(one, state, B, n, y.device))
        Fr = (n + N - 2 * R + R - 1) // R + 1
        spec = B * Fr * (N // 2 + 1) * 8
        fwd_bytes = 2 * (B * n * 4 + spec) + 2 * spec       # two STFTs write their spectra, the reduction reads both
        bwd_bytes = 3 * spec + spec + 2 * B * n * 4          # per-bin gradient: 2 in, 1 out; iSTFT: spectrum in, y rmw
        loss_out["%d/%d" % (N, R)] = {"fwd_us": float(f_us), "bwd_us": float(b_us), "fwd_bytes": fwd_bytes,
                                      "bwd_bytes": bwd_bytes, "fwd_hbm_roof_frac": fwd_bytes / HBM / (f_us * 1e-6),
                                      "bwd_hbm_roof_frac": bwd_bytes / HBM / (b_us * 1e-6)}
    out["loss_kernels"] = loss_out

    # ---- quality after a fixed training budget ----
    torch.manual_seed(0)
    voc = vocoder.NeuralVocoder().cuda()
    st = vocoder.NeuralVocoderStep(voc, lr=1e-3, clip_thresh=1.0)
    rng = np.random.RandomState(0)
    frames = [int(t) for t in rng.randint(2 * 22050 // 256, 10 * 22050 // 256, size=args.clips)]
    eval_wavs = [A.synthetic_clip(100 + c, n=audio.inv_num_samples(t)) for c, t in enumerate(frames)]
    held = [vocoder.vocoder_batch(b, S) for b in VocoderBatches(eval_wavs, B, seg_frames=S, seed=123)]

    def held_loss():
        with torch.no_grad():
            return float(np.mean([vocoder.stft_loss(voc(b["cond"]), b["target"]).item() for b in held]))
    before = held_loss()
    t0 = time.perf_counter()
    for k in range(args.train_steps):
        st.step(batches[k % len(batches)])
    torch.cuda.synchronize()
    out["train"] = {"steps": args.train_steps, "seconds": time.perf_counter() - t0, "lr": 1e-3,
                    "held_out_mrstft_before": before, "held_out_mrstft_after": held_loss()}

    # ---- inference and quality against phase recovery ----
    specs = [audio.spectrogram(w) for w in eval_wavs]
    audio_s = sum(w.size for w in eval_wavs) / float(hp.sample_rate)
    methods = {"neural": voc, "griffin_lim": "griffin_lim", "lws": "lws", "fast_griffin_lim": "fast_griffin_lim"}
    inf = {}
    for name, m in methods.items():
        runs = {"batch16": lambda: audio.inv_spectrogram_batch(specs, method=m),
                "batch1": lambda: [audio.inv_spectrogram_batch([s], method=m) for s in specs]}
        inf[name] = {}
        for r, fn in runs.items():
            fn()
            torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            inf[name][r] = {"ms": _stats([t * 1e3 for t in ts]), "audio_s_per_s": audio_s / float(np.median(ts))}
        rec = audio.inv_spectrogram_batch(specs, method=m)
        sc = []
        for w, r_ in zip(eval_wavs, rec):
            k = min(w.size, r_.size)
            ax, ay = np.abs(A.lws_stft(w[:k].astype(np.float64))), np.abs(A.lws_stft(r_[:k].astype(np.float64)))
            sc.append(float(np.linalg.norm(ax - ay) / np.linalg.norm(ax)))
        ev = evaluate_vocoder([torch.from_numpy(w).cuda() for w in eval_wavs], method=m)
        inf[name]["spectral_convergence_1024_256"] = float(np.mean(sc))
        inf[name]["mean_stoi"] = float(ev["mean_stoi"])
    out["inference"] = inf
    out["audio_seconds"] = audio_s
    print(json.dumps(out))


if __name__ == "__main__":
    main()
