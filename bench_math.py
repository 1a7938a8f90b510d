#!/usr/bin/env python
"""Arithmetic modes of the tensor-core conv GEMMs side by side: "tc" (three MMAs per K-step on hi / lo operand pairs,
fp32-class results, the default) against "tc1" (one MMA on a single 16-bit plane per operand, TF32 / bf16-autocast
class; DESIGN.md section 2.7).

    python bench_math.py --steps 20 --warmup 5 --repeats 5

* Training step: the graph-captured TrainStep of bench.py (same presets, same synthetic B=16 / T_text=128 / T_mel=800
  batch), both modes built in one process and timed in alternation (CUDA events around K steps, repeated R times):
  ms/step, mel-frames/s and the spread (min / max) over the repeats.
* ConvBlock family: forward + data gradient of the 25 ConvBlocks of a deepvoice3_ljspeech step (5 shapes with their
  launch counts) and their weight gradients, per mode, operands prepared outside, L2 flushed between launches.
* Accuracy: relative L2 error of each model output against the fp64 CPU oracle, both modes (B=2: the oracle runs on the
  host).
Prints one JSON line per section, with the card's name and power limit.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import B, PRESETS, T_MEL, T_TEXT, _time_launch  # noqa: E402

MODES = ("tc", "tc1")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def train_steps(preset, steps, warmup, repeats):
    from deepvoice3_pytorch_b200 import builder, ops
    from deepvoice3_pytorch_b200.train_step import TrainStep, make_synthetic_batch, to_device
    dev = torch.device("cuda")
    bname, kw, extra = PRESETS[preset]
    batch = to_device(make_synthetic_batch(B, T_TEXT, T_MEL, n_speakers=kw["n_speakers"], seed=1234), dev)
    runs = {}
    for math in MODES:
        ops.conv_math = math
        torch.manual_seed(1234)
        ops.rng.manual_seed(1234, dev)
        st = TrainStep(getattr(builder, bname)(**kw).to(dev), use_graph=True, **extra)
        for _ in range(max(warmup, 3)):
            st.step(batch)
        runs[math] = st
    torch.cuda.synchronize()
    times = {m: [] for m in MODES}
    for _ in range(repeats):
        for math in MODES:
            ops.conv_math = math
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(steps):
                runs[math].step(batch)
            e.record()
            torch.cuda.synchronize()
            times[math].append(s.elapsed_time(e) / steps)
    ops.conv_math = "tc"
    out = {}
    for m in MODES:
        t = np.array(times[m])
        out[m] = {"ms_per_step": float(np.median(t)), "min_ms": float(t.min()), "max_ms": float(t.max()),
                  "mel_frames_per_s": B * T_MEL / (float(np.median(t)) * 1e-3)}
    out["speedup"] = out["tc"]["ms_per_step"] / out["tc1"]["ms_per_step"]
    del runs
    torch.cuda.empty_cache()
    return out


def conv_family():
    """Forward + data gradient + weight gradient of the deepvoice3_ljspeech ConvBlocks (B=16, k=3), per mode."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    dev = "cuda"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    shapes = [(512, 128, 10), (256, 200, 7), (256, 400, 2), (256, 800, 4), (512, 800, 2)]   # (C, T, blocks per step)
    Bc, k = 16, 3
    res = {}
    for math in MODES:
        npl = 1 if math == "tc1" else 2
        fam = {"fwd_dgrad_us": 0.0, "wgrad_us": 0.0, "shapes": []}
        for C, T, n in shapes:
            g = torch.Generator(device=dev).manual_seed(C + T)
            v = torch.randn(2 * C, C, k, device=dev, generator=g)
            gg = v.pow(2).sum((1, 2)).sqrt()
            bias = torch.zeros(2 * C, device=dev)
            x = torch.randn(Bc, C, T, device=dev, generator=g)
            y, sa, ss, dx = (torch.empty_like(x) for _ in range(4))
            inv, scale = torch.empty(2 * C, device=dev), torch.empty(2 * C, device=dev)
            wfwd = torch.empty(npl, k, 2 * C, C, device=dev, dtype=torch.float16)
            wbwd = torch.empty(npl, k, C, 2 * C, device=dev, dtype=torch.bfloat16)
            ops.lib.call("dv3_tc_weightnorm_fwd", ops._p(v), ops._p(gg), ops._p(inv), ops._p(scale), ops._p(wfwd), npl,
                         ops._p(wbwd), 2 * C, C, k, ops._stream())
            xs = torch.empty(npl, Bc, T, C, device=dev, dtype=torch.float16)
            xw = torch.empty(npl, Bc, T, C, device=dev, dtype=torch.bfloat16)
            ops.lib.call("dv3_tc_split_input", ops._p(x), ops._p(xs), npl, ops._p(xw), Bc, C, T, k, 1, 0, 0.0, None, 0,
                         ops._stream())
            dab = torch.empty(npl, Bc, T, 2 * C, device=dev, dtype=torch.bfloat16)
            ops.lib.call("dv3_tc_gate_bwd_split_npl", ops._p(x), ops._p(sa.normal_()), ops._p(ss.uniform_()), None,
                         ops._p(dab), npl, None, None, Bc, C, T, 0, 1, None, 1, ops._stream())
            nsplit = lib.raw("dv3_tc_wgrad_nsplit")(Bc, 2 * C, C, T, k)
            parts = torch.empty(nsplit, 2 * C * C * k, device=dev)

            def fwd():
                ops.lib.call("dv3_tc_convblock_fwd", ops._p(xs), ops._p(wfwd), npl, ops._p(bias), None, ops._p(x),
                             ops._p(y), ops._p(sa), ops._p(ss), Bc, C, T, k, 1, 0, 0, 1, None, ops._stream())

            def dgrad():
                ops.lib.call("dv3_tc_conv", ops._p(dab), ops._p(wbwd), npl, ops._p(dx), Bc, 2 * C, C, T, k, 1, 0, 1,
                             None, 0, 0.0, None, 0, 1, ops._p(y), None, 0.7071067811865476, None, ops._stream())

            def wgrad():
                ops.lib.call("dv3_tc_wgrad_mn_npl", ops._p(dab), ops._p(xw), npl, ops._p(parts), 2 * C * C * k, Bc,
                             2 * C, C, T, k, 1, 0, 2 * C, C, 0, 1, 2 * C * C, ops._stream())
            tf, tb, tw = (_time_launch(f, flush, reps=20) * 1e6 for f in (fwd, dgrad, wgrad))
            fam["shapes"].append({"C": C, "T": T, "blocks": n, "fwd_us": tf, "dgrad_us": tb, "wgrad_us": tw})
            fam["fwd_dgrad_us"] += n * (tf + tb)
            fam["wgrad_us"] += n * tw
        res[math] = fam
    res["fwd_dgrad_speedup"] = res["tc"]["fwd_dgrad_us"] / res["tc1"]["fwd_dgrad_us"]
    res["wgrad_speedup"] = res["tc"]["wgrad_us"] / res["tc1"]["wgrad_us"]
    return res


def accuracy(preset, Bs=2):
    """Relative L2 error of every model output against the fp64 oracle, per mode (dropout off, same weights)."""
    from deepvoice3_pytorch_b200 import builder, ops
    from oracle import dv3_oracle as O
    from oracle.specs import spec_from_builder
    bname, kw, _ = PRESETS[preset]
    kw = dict(kw, dropout=0.0)
    torch.manual_seed(11)
    model = getattr(builder, bname)(**kw)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    gen = torch.Generator().manual_seed(77)
    Td = T_MEL // 4
    text = torch.randint(2, 149, (Bs, T_TEXT), generator=gen)
    mel = torch.rand(Bs, Td, 80, generator=gen)
    tpos = torch.arange(1, T_TEXT + 1)[None].repeat(Bs, 1)
    fpos = torch.arange(1, Td + 1)[None].repeat(Bs, 1)
    lengths = np.full(Bs, T_TEXT)
    spk = torch.randint(0, kw["n_speakers"], (Bs,), generator=gen) if kw["n_speakers"] > 1 else None
    leaves = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad():
        truth = O.model_forward(leaves, spec_from_builder(bname, **kw), text, mel.double(), spk, tpos, fpos, lengths)
    model = model.cuda().eval()
    names = ("mel", "linear", "alignments", "done")
    out = {}
    for math in MODES:
        ops.conv_math = math
        with torch.no_grad():
            got = model(text.cuda(), mel.cuda(), speaker_ids=None if spk is None else spk.cuda(),
                        text_positions=tpos.cuda(), frame_positions=fpos.cuda(), input_lengths=lengths)
        out[math] = {n: float((g.double().cpu() - t).norm() / t.norm()) for n, g, t in zip(names, got, truth)}
    ops.conv_math = "tc"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--presets", default=",".join(PRESETS))
    ap.add_argument("--skip-accuracy", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_math.py needs a CUDA device")
    info = card()
    presets = a.presets.split(",")
    for p in presets:
        print(json.dumps(dict(info, section="train_step", preset=p, steps=a.steps, repeats=a.repeats,
                              **train_steps(p, a.steps, a.warmup, a.repeats))), flush=True)
    print(json.dumps(dict(info, section="convblock_family", **conv_family())), flush=True)
    if not a.skip_accuracy:
        for p in presets:
            print(json.dumps(dict(info, section="accuracy", preset=p, **accuracy(p))), flush=True)


if __name__ == "__main__":
    main()
