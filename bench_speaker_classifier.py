"""Speaker-classifier training, classification and cloned-voice evaluation on the deepvoice3_vctk shapes (DESIGN.md
section 2.15), K = 108 speaker classes, B = 16 speakers x N = 8 utterances x T_crop = 128 frames, for each conv_math in
--maths:

  (a) SpeakerClassifierStep: one CUDA graph for forward, backward and the clip + Adam update;
  (b) the same classifier as eager PyTorch autograd on the GPU (cuDNN convolutions, cuBLAS GEMMs, TF32 off,
      F.cross_entropy) with torch.optim.Adam -- ms/step of both, arms alternating over --rounds rounds (median, min,
      max);

launches per graph step; each new kernel at the training shape (B*N = 128 rows) and at the classification shapes
2 000 utterances x K = 108 and x K = 2 484 -- µs from torch.profiler in a child process with programmatic dependent
launch off (DV3_PDL=0: with it on, a kernel's recorded time includes its wait for the one before), the entry points'
µs from CUDA events with it on -- with the bytes / FLOPs each kernel needs from shapes, the roof that binds (HBM
bandwidth or FP32 CUDA-core rate) and the kernel's share of it; classification throughput in
utterances/s through SpeakerClassifier.classify (2 000 utterances of 128 frames, trunk included); and the stage times of
classify_cloned_voices (synthesis, mel, classification) on the preset model.  Prints one JSON line, with the card's name
and power limit.  Writes nothing to the tree.

    python bench_speaker_classifier.py [--steps 50] [--rounds 3] [--maths tc,tc1]
"""
import argparse
import contextlib
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

from bench_speaker_adapt import PRESET, PRESETS, card
from bench_speaker_verifier import EagerVerifierStep, _entry, _time_us, time_steps
from deepvoice3_pytorch_b200 import builder, ops
from deepvoice3_pytorch_b200._lib import lib
from deepvoice3_pytorch_b200.speaker_classifier import (SpeakerClassifier, SpeakerClassifierStep,
                                                        classify_cloned_voices)

K, B, N, T_CROP = 108, 16, 8, 128
N_CLS, K_LARGE = 2000, 2484


def _batches(n=4):
    gen = torch.Generator().manual_seed(1)
    return [{"mels": torch.rand(B, N, T_CROP, 80, generator=gen).cuda(),
             "speaker_ids": torch.randperm(K, generator=gen)[:B].cuda()} for _ in range(n)]


class EagerClassifierStep(EagerVerifierStep):
    """(b): the classifier's arithmetic as plain torch autograd over a copy of its parameters."""

    def step(self, b):
        p = self.p
        self.opt.zero_grad(set_to_none=False)
        h = self.trunk(b["mels"])
        Bb, Nn, C = h.shape
        logits = F.linear(h.reshape(Bb * Nn, C), p["w"], p["c"])
        loss = F.cross_entropy(logits, b["speaker_ids"].repeat_interleave(Nn))
        loss.backward()
        self.opt.step()
        return loss


def _cost(R, C, K_, labels):
    """(bytes, FLOPs) each kernel needs, from shapes."""
    f, z = 4, R * K_
    return {"spkcls_logits": (f * (R * C + K_ * C + K_ + z), 2 * z * C),
            "spkcls_rows": (f * (z + 2 * R + (R if labels else 0)) + (8 * R if labels else 0) + 4 * R, 4 * z),
            "spkcls_dh": (f * (z + K_ * C + R * C + R) + 8 * R, 2 * z * C + 4 * z),
            "spkcls_dw": (f * (z + R * C + K_ * C + K_ + R) + 8 * R, 2 * z * C + 4 * z)}


def kernels(C=128, iters=50):
    """The four kernels at the training shape (forward with labels, backward) and the forward at the classification
    shapes: µs per launch from a profiler pass, bytes and FLOPs from shapes, the binding roof; and µs per call of
    each entry point (CUDA events)."""
    dev = "cuda"
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())       # noqa: E731
    err = ops._err_flag(torch.device(dev))
    res = {}
    for name, R, K_, train in (("train_128x108", B * N, K, True), ("classify_2000x108", N_CLS, K, False),
                               ("classify_2000x2484", N_CLS, K_LARGE, False)):
        h = torch.rand(R, C, device=dev)
        w, c = torch.randn(K_, C, device=dev) / C ** 0.5, torch.zeros(K_, device=dev)
        lab = torch.randint(0, K_, (R,), device=dev) if train else None
        logits, lse = torch.empty(R, K_, device=dev), torch.empty(R, device=dev)
        pred, lp = torch.empty(R, dtype=torch.int32, device=dev), torch.empty(R, device=dev) if train else None
        d_h, d_w, d_c = torch.empty(R, C, device=dev), torch.empty(K_, C, device=dev), torch.empty(K_, device=dev)
        one = torch.ones((), device=dev)

        def fwd():
            lib.call("dv3_spkcls_fwd", vp(h), C, vp(w), vp(c), vp(lab), vp(logits), vp(lse), vp(pred), vp(lp),
                     vp(err), R, C, K_, st)

        def bwd():
            lib.call("dv3_spkcls_bwd", vp(h), C, vp(w), vp(logits), vp(lse), vp(lab), None, vp(one), 1.0 / R,
                     vp(d_h), vp(d_w), vp(d_c), vp(err), R, C, K_, st)

        def run():
            fwd()
            if train:
                bwd()
        for _ in range(10):
            run()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                run()
            torch.cuda.synchronize()
        us = {}
        for e in prof.key_averages():
            for k in ("spkcls_logits", "spkcls_rows", "spkcls_dh", "spkcls_dw"):
                if k + "_kernel" in e.key:
                    total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                    us[k] = total / max(1, e.count)
        cost = _cost(R, C, K_, train)
        res[name] = {k: _entry(t, *cost[k]) for k, t in sorted(us.items())}
        res[name]["dv3_spkcls_fwd_us"] = round(_time_us(fwd), 2)
        if train:
            res[name]["dv3_spkcls_bwd_us"] = round(_time_us(bwd), 2)
    ops.check_index_errors()
    return res


def classification_throughput(K_, n=N_CLS, T=128, iters=5):
    torch.manual_seed(1)
    cl = SpeakerClassifier(K_).cuda()
    rng = np.random.RandomState(0)
    utts = [rng.rand(T, 80).astype(np.float32) for _ in range(n)]
    cl.classify(utts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        cl.classify(utts)
    torch.cuda.synchronize()
    s = (time.perf_counter() - t0) / iters
    return {"K": K_, "utterances": n, "frames": T, "ms_per_call": round(s * 1e3, 2), "utterances_per_s": round(n / s)}


def evaluation_stages(cl, n_seq=16, max_steps=100):
    """classify_cloned_voices on the preset model (random weights, decoder capped at max_steps), every sequence in one
    of the model's own voices: seconds per stage."""
    _, kw, _ = PRESETS[PRESET]
    torch.manual_seed(0)
    model = getattr(builder, PRESETS[PRESET][0])(**kw).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = max_steps
    rng = np.random.RandomState(0)
    seqs = [rng.randint(2, 149, rng.randint(20, 60)) for _ in range(n_seq)]
    ids = [(7 * k) % K for k in range(n_seq)]
    times = {}

    @contextlib.contextmanager
    def timer(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    classify_cloned_voices(model, cl, ids, seqs, stage_timer=timer)           # warm-up
    times.clear()
    res = classify_cloned_voices(model, cl, ids, seqs, stage_timer=timer)
    return {"n_seq": n_seq, "max_decoder_steps": max_steps, "ms": {k: round(t * 1e3, 2) for k, t in times.items()},
            "accuracy": res["accuracy"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maths", default="tc,tc1")
    ap.add_argument("--kernels-only", action="store_true", help="print the kernel table alone (the child process)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speaker_classifier.py needs a CUDA device")
    if args.kernels_only:
        print(json.dumps(kernels()))
        return
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {"preset": PRESET, "card": card(), "K": K, "B": B, "N": N, "T_crop": T_CROP, "runs": []}
    for m in args.maths.split(","):
        ops.conv_math = m
        batches = _batches()
        torch.manual_seed(1)
        c_a = SpeakerClassifier(K).cuda()
        torch.manual_seed(1)
        c_b = SpeakerClassifier(K).cuda()
        arms = {"a_graph": SpeakerClassifierStep(c_a).step, "b_eager_torch": EagerClassifierStep(c_b).step}
        for step in arms.values():
            time_steps(step, batches, args.warmup)
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, step in arms.items():
                ms[k].append(time_steps(step, batches, args.steps))
        run = {"math": m, "ms_per_step": {k: {"median": round(float(np.median(t)), 3), "min": round(min(t), 3),
                                              "max": round(max(t), 3)} for k, t in ms.items()},
               "launches_per_step": arms["a_graph"].__self__.launches_per_step,
               "classification": [classification_throughput(K), classification_throughput(K_LARGE)]}
        run["speedup_a_vs_b"] = round(run["ms_per_step"]["b_eager_torch"]["median"] /
                                      run["ms_per_step"]["a_graph"]["median"], 2)
        res["runs"].append(run)
        del arms
        torch.cuda.empty_cache()
    res["kernels_pdl_on"] = kernels()
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernels-only"], capture_output=True,
                           text=True, check=True, env=dict(os.environ, DV3_PDL="0"))
    res["kernels_pdl_off"] = json.loads(child.stdout.strip().splitlines()[-1])
    ops.conv_math = args.maths.split(",")[0]
    torch.manual_seed(1)
    res["classify_cloned_voices"] = evaluation_stages(SpeakerClassifier(K).cuda())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
