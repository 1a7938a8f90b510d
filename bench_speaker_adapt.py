"""Embedding-only speaker adaptation on the deepvoice3_vctk preset (108 speakers + 1 added): three arms on the same
batches, alternating, at batch 16 and batch 4, in "tc" and "tc1":

  (a) TrainStep(adapt_speakers=[108], use_graph=True): frozen network folded once, collapsed site gradients
      (csrc/spk_adapt.cu), clip + Adam over the one row;
  (b) the eager-autograd baseline a user would write today: requires_grad on embed_speakers.weight only, the model's
      forward + train_step.fused_training_loss + backward, clip_grad_norm_ + torch.optim.Adam on the table;
  (c) the full joint TrainStep(use_graph=True) on the same batches.

Reports ms/step (median and min-max over rounds), kernel launches per step, the device time per step of all site
kernels (torch.profiler, separate pass), and on the preset's largest site shape (C = 512, T_mel) the site kernel's
time, bytes and HBM share (bytes / time / 3.35 TB/s) against the timed autograd chain it replaces, with the card's
name and power limit read in the same run.  Prints one JSON line.
Writes nothing to the tree.

    python bench_speaker_adapt.py [--steps 20] [--rounds 3]
"""
import argparse
import ctypes
import json
import subprocess
import time

import numpy as np
import torch

from bench import PRESETS
from deepvoice3_pytorch_b200 import builder, ops
from deepvoice3_pytorch_b200._lib import lib
from deepvoice3_pytorch_b200.train_step import TrainStep, fused_training_loss, make_synthetic_batch, to_device

PRESET = "deepvoice3_vctk"
HBM = 3.35e12
T_TEXT, T_MEL = 128, 800


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    vals = (q.stdout.strip().split(", ") + ["?"] * 3)[:3] if q.returncode == 0 else [None] * 3
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi_name": vals[0], "power_limit": vals[1],
            "max_sm_clock": vals[2]}


def _model(kw, seed=0):
    torch.manual_seed(seed)
    m = getattr(builder, PRESETS[PRESET][0])(**kw).cuda().train()
    new = m.add_speakers(1)[0]
    return m, new


def _batches(B, new, kw, n=4):
    out = []
    for i in range(n):
        h = make_synthetic_batch(B=B, T_text=T_TEXT, T_mel=T_MEL, n_speakers=kw["n_speakers"], linear_dim=513, seed=i)
        h["speaker_ids"] = torch.full((B,), new, dtype=torch.int64)
        out.append(to_device(h, "cuda"))
    return out


class EagerBaseline:
    """(b): plain autograd with only the speaker table trainable (every row: what torch.optim.Adam does)."""

    def __init__(self, model, extra):
        self.model = model
        for p in model.parameters():
            p.requires_grad_(False)
        self.table = model.embed_speakers.weight
        self.table.requires_grad_(True)
        self.opt = torch.optim.Adam([self.table], lr=5e-4, betas=(0.5, 0.9), eps=1e-6)
        self.extra = extra

    def step(self, b):
        m = self.model
        self.opt.zero_grad(set_to_none=False)
        outs = m(b["x"], b["mel"], speaker_ids=b["speaker_ids"], text_positions=b["text_positions"],
                 frame_positions=b["frame_positions"], input_lengths=b["input_lengths_dev"])
        loss = fused_training_loss(outs, b, guided_attention_sigma=self.extra["guided_attention_sigma"])
        loss.backward()
        torch.nn.utils.clip_grad_norm_([self.table], 0.1)
        self.opt.step()
        return loss


def time_steps(step, batches, steps):
    torch.cuda.synchronize()
    n0 = lib.raw("dv3_launch_count")()
    t0 = time.perf_counter()
    for i in range(steps):
        step(batches[i % len(batches)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps, (lib.raw("dv3_launch_count")() - n0) / steps


def _time_us(fn, iters):
    for _ in range(10):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def site_kernel(B, npl, C=512, T=T_MEL, S=16, iters=100):
    """The largest site of the preset (a converter GLU block, C = 512 at T_mel frames): the collapsed kernel (site
    launch + its share of the reduce) against the autograd chain it replaces, both timed: the fp32 "a" half rebuilt
    from the planes and transposed, softsign backward, the projection's data gradient (frozen weights), the transpose
    back and the time sum of the expanded (B,T,S) gradient.  Bytes counted from shapes."""
    from deepvoice3_pytorch_b200.modules import Linear
    import torch.nn.functional as F
    dev = "cuda"
    planes = torch.randn(npl, B, T, 2 * C, device=dev).to(torch.bfloat16)
    y = torch.rand(B, C, T, device=dev) * 1.8 - 0.9
    w = torch.randn(C, S, device=dev)
    ns = lib.raw("dv3_spk_grad_splits")()
    part = torch.zeros(ns * B * S, device=dev)
    d_e = torch.zeros(B, S, device=dev)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())

    def collapsed():
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        lib.call("dv3_spk_grad_planes", vp(planes), npl, planes[0].numel(), 2 * C, vp(y), vp(w), vp(part), B, C, T, S,
                 None, 1, 0.05, None, 0, st)
        lib.call("dv3_spk_grad_reduce", vp(part), ns, vp(d_e), B, S, st)
    us = _time_us(collapsed, iters)

    proj = Linear(S, C).to(dev)
    for q in proj.parameters():
        q.requires_grad_(False)
    e_btc = torch.randn(B, T, S, device=dev, requires_grad=True)
    spk = F.softsign(proj.forward_bct(ops.transpose12(e_btc)))

    def chain():
        da = planes[0, :, :, :C].float()
        if npl == 2:
            da = da + planes[1, :, :, :C].float() * (1.0 / 2048.0)
        dspk = ops.transpose12(da.contiguous())
        (g,) = torch.autograd.grad(spk, e_btc, dspk, retain_graph=True)
        return g.sum(1)
    us_chain = _time_us(chain, iters)
    n = B * C * T
    nbytes = n * (2 * npl + 4) + B * C * S * 4 + ns * B * S * 8       # G planes (a half) + y once, W per block, partials
    chain_bytes = n * (2 * npl + 4 + 8 + 12 + 4) + B * T * S * 4 * 3
    return {"C": C, "T": T, "us": round(us, 2), "bytes": nbytes, "hbm_share": round(nbytes / (us * 1e-6) / HBM, 3),
            "chain_us": round(us_chain, 2), "chain_bytes": chain_bytes, "speedup_vs_chain": round(us_chain / us, 2)}


def site_time_per_step(step, batches, steps=5):
    """Device time per step of the collapsed site kernels and their reduce, from torch.profiler (a separate pass)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            step(batches[i % len(batches)])
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "spk_grad" in e.key)
    return round(us / steps, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch-sizes", default="16,4")
    ap.add_argument("--maths", default="tc,tc1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speaker_adapt.py needs a CUDA device")
    _, kw, extra = PRESETS[PRESET]
    res = {"preset": PRESET, "card": card(), "T_text": T_TEXT, "T_mel": T_MEL, "runs": []}
    for math in args.maths.split(","):
        ops.conv_math = math
        for B in [int(b) for b in args.batch_sizes.split(",")]:
            ma, new = _model(kw)
            mb, _ = _model(kw)
            mc, _ = _model(kw)
            batches = _batches(B, new, kw)
            arms = {"a_adapt_graph": TrainStep(ma, adapt_speakers=[new], use_graph=True, **extra).step,
                    "b_eager_autograd": EagerBaseline(mb, extra).step,
                    "c_joint_graph": TrainStep(mc, use_graph=True, **extra).step}
            for step in arms.values():
                time_steps(step, batches, args.warmup)
            ms = {k: [] for k in arms}
            launches = {}
            for _ in range(args.rounds):
                for k, step in arms.items():
                    t, n = time_steps(step, batches, args.steps)
                    ms[k].append(t)
                    launches[k] = n
            launches["a_adapt_graph"] = arms["a_adapt_graph"].__self__.launches_per_step
            launches["c_joint_graph"] = arms["c_joint_graph"].__self__.launches_per_step
            run = {"math": math, "B": B,
                   "ms_per_step": {k: {"median": round(float(np.median(v)), 3), "min": round(min(v), 3),
                                       "max": round(max(v), 3)} for k, v in ms.items()},
                   "launches_per_step": launches,
                   "site_kernel": site_kernel(B, 1 if math == "tc1" else 2),
                   "site_kernels_us_per_step": site_time_per_step(arms["a_adapt_graph"], batches)}
            run["speedup_a_vs_b"] = round(run["ms_per_step"]["b_eager_autograd"]["median"] /
                                          run["ms_per_step"]["a_adapt_graph"]["median"], 2)
            run["speedup_a_vs_c"] = round(run["ms_per_step"]["c_joint_graph"]["median"] /
                                          run["ms_per_step"]["a_adapt_graph"]["median"], 2)
            res["runs"].append(run)
            del ma, mb, mc, arms
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
