"""Speaker-encoder training and cloning on the deepvoice3_vctk preset (DESIGN.md section 2.13), B = 16 speakers x N = 8
cloning samples x T_crop = 128 frames, for each conv_math in --maths:

  (a) SpeakerEncoderStep: one CUDA graph for forward, backward and the clip + Adam update;
  (b) the same encoder as eager PyTorch autograd on the GPU (cuDNN convolutions, cuBLAS GEMMs, TF32 off) with
      torch.optim.Adam -- ms/step of both, arms alternating over --rounds rounds (median, min, max);

the new kernels one launch at a time at the training shape (CUDA events), with the bytes / FLOPs each needs and the
bound that applies; the time to clone one voice from 10 full-length utterances with embed_batch, next to one
embedding-only adaptation step (TrainStep(adapt_speakers=...), graph mode, batch 16, as bench_speaker_adapt.py runs
it).  Prints one JSON line, with the card's name and power limit."""
import argparse
import ctypes
import json
import math
import time

import numpy as np
import torch
import torch.nn.functional as F

from bench_speaker_adapt import PRESET, PRESETS, T_MEL, T_TEXT, card
from deepvoice3_pytorch_b200 import builder, ops
from deepvoice3_pytorch_b200._lib import lib
from deepvoice3_pytorch_b200.speaker_encoder import _ATTN_PARAMS, SpeakerEncoder, SpeakerEncoderStep
from deepvoice3_pytorch_b200.train_step import TrainStep, make_synthetic_batch, to_device

B, N, T_CROP, HBM = 16, 8, 128, 3.35e12


def _model():
    _, kw, _ = PRESETS[PRESET]
    torch.manual_seed(0)
    return getattr(builder, PRESETS[PRESET][0])(**kw).cuda(), kw


def _batches(n_speakers, n=4):
    gen = torch.Generator().manual_seed(1)
    return [{"mels": torch.rand(B, N, T_CROP, 80, generator=gen).cuda(),
             "speaker_ids": torch.randperm(n_speakers, generator=gen)[:B].cuda()} for _ in range(n)]


class EagerEncoderStep:
    """(b): the encoder's arithmetic as plain torch autograd over a copy of its parameters."""

    def __init__(self, enc, model, lr=1e-3):
        self.p = {k: v.detach().clone().requires_grad_(True) for k, v in enc.state_dict().items()}
        self.heads, self.k, self.n_conv = enc.heads, enc.temporal[0].conv.kernel_size[0], len(enc.temporal)
        self.table = model.embed_speakers.weight.detach()
        self.opt = torch.optim.Adam(list(self.p.values()), lr=lr, betas=(0.9, 0.999), eps=1e-8)

    def _wn(self, pre):
        v, g = self.p[pre + "weight_v"], self.p[pre + "weight_g"]
        return g * v / v.pow(2).sum((1, 2), keepdim=True).sqrt()

    def step(self, b):
        p = self.p
        self.opt.zero_grad(set_to_none=False)
        Bb, Nn, T, M = b["mels"].shape
        x = b["mels"].view(Bb * Nn, T, M).transpose(1, 2)
        for i in (0, 2):
            x = torch.relu(F.conv1d(x, self._wn("spectral.%d." % i), p["spectral.%d.bias" % i]))
        for i in range(self.n_conv):
            pre = "temporal.%d.conv." % i
            y = F.conv1d(x, self._wn(pre), p[pre + "bias"], padding=(self.k - 1) // 2)
            a, gate = y.chunk(2, dim=1)
            x = (a * torch.sigmoid(gate) + x) * math.sqrt(0.5)
        h = x.mean(-1).view(Bb, Nn, -1)
        C = h.shape[-1]
        dh = C // self.heads

        def heads(t):
            return t.view(Bb, Nn, self.heads, dh).transpose(1, 2)
        q, k, v = (heads(F.linear(h, p["w_" + n], p["b_" + n])) for n in "qkv")
        o = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), -1) @ v
        o = o.transpose(1, 2).reshape(Bb, Nn, C)
        a = torch.softmax(o @ p["w_s"] + p["b_s"], dim=1)
        out = (a[..., None] * F.linear(h, p["w_e"], p["b_e"])).sum(1)
        loss = F.l1_loss(out, self.table[b["speaker_ids"]])
        loss.backward()
        self.opt.step()
        return loss


def time_steps(step, batches, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(batches[i % len(batches)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def _time_us(fn, iters=200):
    for _ in range(10):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def kernels(enc):
    """Each new kernel at the training shape: µs per launch, bytes, FLOPs, and the bound that applies."""
    dev = "cuda"
    R, C, S, H = B * N, enc.channels, enc.speaker_embed_dim, enc.heads
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())       # noqa: E731
    err = ops._err_flag(torch.device(dev))
    x = torch.rand(R, C, T_CROP, device=dev)
    lengths = torch.full((R,), T_CROP, dtype=torch.int32, device=dev)
    y = torch.empty(R, C, device=dev)
    dx = torch.empty_like(x)
    h = torch.rand(B, N, C, device=dev)
    counts = torch.full((B,), N, dtype=torch.int32, device=dev)
    params = [vp(getattr(enc, n)) for n in _ATTN_PARAMS]
    target = torch.rand(B, S, device=dev)
    out = torch.empty(B, S, device=dev)
    ws = torch.empty(B, lib.raw("dv3_spkenc_ws_floats")(N, C, S, H), device=dev)
    lp = torch.empty(B, device=dev)
    one = torch.ones((), device=dev)
    P = lib.raw("dv3_spkenc_param_floats")(C, S)
    part = torch.empty(B, P, device=dev)
    grad = torch.empty(P, device=dev)
    dh = torch.empty_like(h)
    attn_flops = B * (2 * 3 * N * C * C + 2 * 2 * N * N * C + 2 * N * C * S + 4 * N * C)
    runs = {
        "pool_fwd": (lambda: lib.call("dv3_spkenc_pool_fwd", vp(x), vp(lengths), vp(y), vp(err), R, C, T_CROP, st),
                     4 * R * C * (T_CROP + 1), R * C * T_CROP),
        "pool_bwd": (lambda: lib.call("dv3_spkenc_pool_bwd", vp(y), vp(lengths), vp(dx), vp(err), R, C, T_CROP, st),
                     4 * R * C * (T_CROP + 1), R * C * T_CROP),
        "attn_fwd": (lambda: lib.call("dv3_spkenc_attn_fwd", vp(h), vp(counts), *params, vp(target), vp(out), vp(ws),
                                      vp(lp), vp(err), B, N, C, S, H, st), 4 * (B * N * C + 3 * C * C), attn_flops),
        "attn_bwd": (lambda: lib.call("dv3_spkenc_attn_bwd", vp(h), vp(counts), *params, vp(target), None, vp(one),
                                      1.0 / (B * S), vp(ws), vp(dh), vp(part), vp(err), B, N, C, S, H, st),
                     4 * (2 * B * N * C + 3 * C * C + B * P), 2 * attn_flops),
        "reduce": (lambda: lib.call("dv3_spkenc_reduce", vp(part), P, vp(lp), 1.0, vp(grad), vp(one), B, st),
                   4 * (B * P + P), B * P),
    }
    res = {}
    for name, (fn, nbytes, flops) in runs.items():
        us = _time_us(fn)
        res[name] = {"us": round(us, 2), "bytes": int(nbytes), "flops": int(flops),
                     "hbm_floor_us": round(nbytes / HBM * 1e6, 2),
                     "bound": "latency (one CTA per speaker)" if name.startswith("attn") else "memory"}
    ops.check_index_errors()
    return res


def clone_time(enc, iters=20):
    rng = np.random.RandomState(0)
    utts = [rng.rand(rng.randint(200, 400), 80).astype(np.float32) for _ in range(10)]
    enc.embed_batch([utts])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        enc.embed_batch([utts])
    torch.cuda.synchronize()
    return {"ms": round((time.perf_counter() - t0) * 1e3 / iters, 3), "frames": [u.shape[0] for u in utts]}


def adapt_step_ms(steps=20):
    _, kw, extra = PRESETS[PRESET]
    torch.manual_seed(0)
    m = getattr(builder, PRESETS[PRESET][0])(**kw).cuda().train()
    new = m.add_speakers(1)[0]
    batches = []
    for i in range(4):
        hb = make_synthetic_batch(B=16, T_text=T_TEXT, T_mel=T_MEL, n_speakers=kw["n_speakers"], linear_dim=513, seed=i)
        hb["speaker_ids"] = torch.full((16,), new, dtype=torch.int64)
        batches.append(to_device(hb, "cuda"))
    st = TrainStep(m, adapt_speakers=[new], use_graph=True, **extra)
    time_steps(st.step, batches, 3)
    return round(time_steps(st.step, batches, steps), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maths", default="tc,tc1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speaker_encoder.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {"preset": PRESET, "card": card(), "B": B, "N": N, "T_crop": T_CROP, "runs": []}
    for m in args.maths.split(","):
        ops.conv_math = m
        model, kw = _model()
        batches = _batches(kw["n_speakers"])
        torch.manual_seed(1)
        enc_a = SpeakerEncoder().cuda()
        torch.manual_seed(1)
        enc_b = SpeakerEncoder().cuda()
        arms = {"a_graph": SpeakerEncoderStep(enc_a, model).step, "b_eager_torch": EagerEncoderStep(enc_b, model).step}
        for step in arms.values():
            time_steps(step, batches, args.warmup)
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, step in arms.items():
                ms[k].append(time_steps(step, batches, args.steps))
        run = {"math": m, "ms_per_step": {k: {"median": round(float(np.median(v)), 3), "min": round(min(v), 3),
                                              "max": round(max(v), 3)} for k, v in ms.items()},
               "launches_per_step": arms["a_graph"].__self__.launches_per_step,
               "kernels": kernels(enc_a), "clone_10_utterances": clone_time(enc_a)}
        run["speedup_a_vs_b"] = round(run["ms_per_step"]["b_eager_torch"]["median"] /
                                      run["ms_per_step"]["a_graph"]["median"], 2)
        res["runs"].append(run)
        del arms, model
        torch.cuda.empty_cache()
    ops.conv_math = args.maths.split(",")[0]
    res["adapt_step_ms_batch16"] = adapt_step_ms()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
