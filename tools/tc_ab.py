#!/usr/bin/env python
"""A/B of two builds of the tensor-core conv kernel on the same seeded operands.

    python tools/tc_ab.py OLD.so NEW.so [OUT_DIR]

For each build (a child process with DV3_LIB pointing at it) the gated ConvBlock forward (dv3_tc_convblock_fwd), its
data gradient and a 1x1 forward conv (dv3_tc_conv) run at the five ConvBlock shapes of bench.py's roofline (B=16, k=3)
on operand planes drawn from a fixed seed; the outputs are compared element-wise (max |delta|, expected 0) and the
per-launch times (CUDA events, L2 flushed, mean of 20) are printed side by side.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(512, 128), (256, 200), (256, 400), (256, 800), (512, 800)]    # (C, T), B = 16, k = 3, dilation 1
B, K = 16, 3


def child(out_path):
    import torch
    sys.path.insert(0, ROOT)
    from deepvoice3_pytorch_b200 import ops
    dev = "cuda"
    bf, f16 = torch.bfloat16, torch.float16
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn, reps=20):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(reps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); fn(); e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e) * 1e3)
        return float(np.mean(ts))

    outs, times = {}, {}
    for C, T in SHAPES:
        g = torch.Generator().manual_seed(1000 * C + T)

        def rnd(*shape, scale=1.0, dtype=torch.float32):
            return (torch.randn(*shape, generator=g) * scale).to(dtype).to(dev)

        # gated forward: fp16 hi / lo planes of input and weight
        xs = torch.stack([rnd(B, T, C, dtype=f16), rnd(B, T, C, scale=0.5, dtype=f16)])
        wf = torch.stack([rnd(K, 2 * C, C, scale=(1.0 / (K * C)) ** 0.5, dtype=f16),
                          rnd(K, 2 * C, C, scale=0.5 * (1.0 / (K * C)) ** 0.5, dtype=f16)])
        bias, res = rnd(2 * C, scale=0.1), rnd(B, C, T)
        y, sa, ss = [torch.empty(B, C, T, device=dev) for _ in range(3)]
        # data gradient: bf16 planes of dAB (B,T,2C) and of the transposed weight (k, C, 2C)
        dab = torch.stack([rnd(B, T, 2 * C, dtype=bf), rnd(B, T, 2 * C, scale=0.5, dtype=bf)])
        wb = torch.stack([rnd(K, C, 2 * C, scale=(1.0 / (K * C)) ** 0.5, dtype=bf),
                          rnd(K, C, 2 * C, scale=0.5 * (1.0 / (K * C)) ** 0.5, dtype=bf)])
        e1, dx = rnd(B, C, T), torch.empty(B, C, T, device=dev)
        # 1x1 forward conv C -> C with bias and ReLU: fp16 planes
        w1 = torch.stack([rnd(1, C, C, scale=C ** -0.5, dtype=f16), rnd(1, C, C, scale=0.5 * C ** -0.5, dtype=f16)])
        yc = torch.empty(B, C, T, device=dev)

        def fwd():
            ops.lib.call("dv3_tc_convblock_fwd", ops._p(xs), ops._p(wf), 2, ops._p(bias), None, ops._p(res),
                         ops._p(y), ops._p(sa), ops._p(ss), B, C, T, K, 1, 0, 0, 1, None, ops._stream())

        def dgrad():
            ops.lib.call("dv3_tc_conv", ops._p(dab), ops._p(wb), 2, ops._p(dx), B, 2 * C, C, T, K, 1, 0, 1, None, 0,
                         0.0, None, 0, 1, ops._p(e1), None, 0.7071067811865476, None, ops._stream())

        def conv1():
            ops.lib.call("dv3_tc_conv", ops._p(xs), ops._p(w1), 2, ops._p(yc), B, C, C, T, 1, 1, 0, 0, ops._p(bias),
                         1, 0.0, None, 0, 0, None, None, 0.0, None, ops._stream())

        for name, fn, arrs in [("fwd", fwd, {"y": y, "a": sa, "s": ss}), ("dgrad", dgrad, {"dx": dx}),
                               ("conv1x1", conv1, {"y": yc})]:
            fn()
            torch.cuda.synchronize()
            for k, v in arrs.items():
                outs["%s_C%d_T%d_%s" % (name, C, T, k)] = v.cpu().numpy()
            times["%s C=%d T=%d" % (name, C, T)] = timed(fn)
    np.savez(out_path, **outs)
    print(json.dumps(times))


def main():
    old, new = sys.argv[1], sys.argv[2]
    out_dir = sys.argv[3] if len(sys.argv) > 3 else "/tmp"
    res = {}
    for tag, path in [("old", old), ("new", new)]:
        env = dict(os.environ, DV3_LIB=os.path.abspath(path))
        npz = os.path.join(out_dir, "tc_ab_%s.npz" % tag)
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", npz], env=env, check=True,
                             capture_output=True, text=True).stdout
        res[tag] = (np.load(npz), json.loads(out.strip().splitlines()[-1]))
    (a, ta), (b, tb) = res["old"], res["new"]
    worst = 0.0
    for k in a.files:
        d = float(np.abs(a[k].astype(np.float64) - b[k]).max())
        worst = max(worst, d)
        if d != 0.0:
            print("DIFF %-28s max|delta| %.3e (max|old| %.3e)" % (k, d, float(np.abs(a[k]).max())))
    print("outputs compared: %d, max |delta| over all: %.3e" % (len(a.files), worst))
    print("%-22s %10s %10s %7s" % ("launch", "old us", "new us", "ratio"))
    for k in ta:
        print("%-22s %10.1f %10.1f %7.3f" % (k, ta[k], tb[k], tb[k] / ta[k]))


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        child(sys.argv[2])
    else:
        main()
