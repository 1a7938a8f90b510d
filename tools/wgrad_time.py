#!/usr/bin/env python
"""Per-kernel time of every tensor-core weight-gradient shape of one deepvoice3_ljspeech training step.

The shapes and their launch counts are recorded from one eager forward + backward of the benchmark step (B=16,
T_text=128, T_mel=800): every dv3_tc_wgrad_mn_npl call with its layout.  Each shape is then launched alone on random
bf16 pair planes, CUDA events around the launch, L2 flushed before every launch, median of --reps runs.  Prints
TF/s algorithmic (2 * B * T * Mw * Nw * k per launch) next to the launches per step, and the launch-weighted totals
of the ConvBlock shapes (k > 1, Mw = 2 Nw) and of all shapes.

Runs with any build of the library: DV3_LIB=<path to libdv3b200.so> selects one, so that two builds can be timed
alternately in one session.  --fit (for the persistent kernel) adds calibration shapes and fits
    t = t0 + t_iter * (K-iterations of CTA 0) + t_unit * (units of CTA 0)
over all shapes, with CTA 0's share from the kernel's round-robin schedule; t_unit / t_iter is the per-unit cost of
the split rule in tc_gemm.cu (dv3_tc_wgrad_nsplit), in K-iterations.

    python tools/wgrad_time.py [--reps 50] [--fit] [--json out.json]
"""
import argparse
import collections
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from deepvoice3_pytorch_b200 import builder, ops  # noqa: E402
from deepvoice3_pytorch_b200._lib import lib  # noqa: E402
from deepvoice3_pytorch_b200.train_step import make_synthetic_batch, to_device  # noqa: E402

# (B, Mw, Nw, T, k, dilation): ConvBlock-like shapes of other batch sizes and lengths, for the --fit regression only
CALIB = [(4, 1024, 512, 128, 3, 1), (8, 1024, 512, 128, 3, 1), (32, 1024, 512, 128, 3, 1), (64, 1024, 512, 128, 3, 1),
         (2, 512, 256, 800, 3, 1), (4, 512, 256, 800, 3, 1), (8, 512, 256, 800, 3, 1), (16, 512, 256, 64, 3, 1)]


def step_shapes(preset):
    """{(B, Mw, Nw, T, k, dilation, causal, msplit, s_m, s_mh, s_n, s_j): launches per step} of one eager step."""
    bname, kw, _ = bench.PRESETS[preset]
    torch.manual_seed(1234)
    model = getattr(builder, bname)(**kw).cuda().train()
    b = to_device(make_synthetic_batch(bench.B, bench.T_TEXT, bench.T_MEL, n_speakers=kw["n_speakers"]), "cuda")
    seen = collections.Counter()
    call = lib.call

    def record(name, *args):
        if name == "dv3_tc_wgrad_mn_npl":
            seen[tuple(int(a) for a in args[5:17])] += 1
        return call(name, *args)

    lib.call = record
    try:
        spk = {"speaker_ids": b["speaker_ids"]} if "speaker_ids" in b else {}
        outs = model(b["x"], b["mel"], text_positions=b["text_positions"], frame_positions=b["frame_positions"],
                     input_lengths=b["input_lengths"], **spk)
        sum(o.float().sum() for o in outs if o is not None).backward()
        torch.cuda.synchronize()
    finally:
        lib.call = call
    return seen


def schedule(B, Mw, Nw, T, k, ns, sms):
    """(units, K-iterations) of CTA 0 in the persistent kernel's round-robin, longest-first schedule."""
    tk = -(-Mw // 128) * -(-Nw // 128) * k
    kb_n, bps = -(-T // 32), -(-B // ns)
    units = tk * ns
    its = [(min(B, (u // tk + 1) * bps) - (u // tk) * bps) * kb_n for u in range(0, units, min(units, sms))]
    return len(its), sum(its)


def time_shape(shape, reps, flush, npl):
    B, Mw, Nw, T, k, dil, causal, ms, s_m, s_mh, s_n, s_j = shape
    g = torch.Generator(device="cuda").manual_seed(Mw + Nw + T + k)
    p8 = lambda n: (n + 7) // 8 * 8  # noqa: E731
    dy = (torch.randn(npl, B, T, p8(Mw), device="cuda", generator=g) * 1e-3).to(torch.bfloat16)
    x = torch.randn(npl, B, T, p8(Nw), device="cuda", generator=g).to(torch.bfloat16)
    nsplit = lib.raw("dv3_tc_wgrad_nsplit")(B, Mw, Nw, T, k)
    numel = Mw * Nw * k
    parts = torch.empty(nsplit, numel, device="cuda")
    st = ops._stream()

    def launch():
        lib.call("dv3_tc_wgrad_mn_npl", ops._p(dy), ops._p(x), npl, ops._p(parts), numel, B, Mw, Nw, T, k, dil, causal,
                 ms, s_m, s_mh, s_n, s_j, st)

    for _ in range(3):
        launch()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    return float(np.median(ts)), nsplit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="deepvoice3_ljspeech")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--npl", type=int, default=2)
    ap.add_argument("--fit", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "wgrad_time.py times the GPU kernel: it needs a GPU"
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    print("%s, %d SMs, library %s" % (props.name, sms, os.environ.get("DV3_LIB") or "in-tree"))
    shapes = step_shapes(a.preset)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows, tot, tot_cb = [], 0.0, 0.0
    print("%4s %5s %5s %4s %2s %3s %7s %6s %9s %7s" % ("B", "Mw", "Nw", "T", "k", "dil", "layout", "nsplit", "us",
                                                       "TF/s") + "  launches/step")
    for shape, n in sorted(shapes.items(), key=lambda kv: -kv[0][1] * kv[0][2] * kv[0][3] * kv[0][4]):
        B, Mw, Nw, T, k, dil = shape[:6]
        us, ns = time_shape(shape, a.reps, flush, a.npl)
        tf = 2.0 * B * T * Mw * Nw * k / us / 1e6
        convblock = k > 1 and Mw == 2 * Nw
        tot += n * us
        tot_cb += n * us if convblock else 0.0
        print("%4d %5d %5d %4d %2d %3d %7s %6d %9.1f %7.1f  %d%s" % (B, Mw, Nw, T, k, dil,
              "tap" if shape[10] == 1 else "convT", ns, us, tf, n, "  ConvBlock" if convblock else ""), flush=True)
        rows.append(dict(shape=list(shape), launches=n, us=us, tflops=tf, nsplit=ns, convblock=convblock))
    print("launch-weighted per step: ConvBlock weight gradients %.1f us, all weight gradients %.1f us" % (tot_cb, tot))
    res = dict(gpu=props.name, sms=sms, lib=os.environ.get("DV3_LIB") or "in-tree", shapes=rows,
               convblock_us=tot_cb, total_us=tot)
    if a.fit:
        X, y = [], []
        extra = [(B, M, N, T, k, d, 0, M, N, 0, 1, M * N) for (B, M, N, T, k, d) in CALIB]
        for shape in [tuple(r["shape"]) for r in rows] + extra:
            us, ns = time_shape(shape, a.reps, flush, a.npl)
            units, its = schedule(*shape[:5], ns, sms)
            X.append([1.0, its, units])
            y.append(us)
        coef = np.linalg.lstsq(np.array(X), np.array(y), rcond=None)[0]
        resid = np.array(y) - np.array(X) @ coef
        print("fit: t = %.2f us + %.4f us x iterations + %.3f us x units (rms residual %.2f us); per-unit cost %.2f "
              "iterations" % (coef[0], coef[1], coef[2], float(np.sqrt((resid ** 2).mean())), coef[2] / coef[1]))
        res["fit"] = dict(t0_us=coef[0], iter_us=coef[1], unit_us=coef[2], unit_iters=coef[2] / coef[1])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
