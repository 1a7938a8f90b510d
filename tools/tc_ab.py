#!/usr/bin/env python
"""A/B of two builds of the tensor-core GEMM kernels on the same seeded operands.

    python tools/tc_ab.py OLD.so NEW.so [OUT_DIR]

For each build (a child process with DV3_LIB pointing at it) the gated ConvBlock forward (dv3_tc_convblock_fwd), its
data gradient and a 1x1 forward conv (dv3_tc_conv) run at the five ConvBlock shapes of bench.py's roofline (B=16, k=3),
with two operand planes and with one (npl1); the weight gradient (dv3_tc_wgrad_mn_npl) runs at the same five shapes
and at two more of tests/test_gpu_tc_wgrad.py, with two planes and with one:
  * the ConvBlock shapes in the tap-major layout; at (512, 800) every CTA walks three work units;
  * (B=37, 512 x 256, T=64, k=3, causal, dilation 27) in the tap-major layout: a short last batch split;
  * (B=77, 1024 x 512, T=40, k=1) in the ConvTranspose layout of ops._CONVT: a short last split.
All operand planes are drawn from a fixed seed; the outputs are compared element-wise (max |delta|, expected 0) and the
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
# weight-gradient shapes beyond the ConvBlock ones: (B, Mw, Nw, T, k, dilation, causal, ConvTranspose layout)
WG_EXTRA = [(37, 512, 256, 64, 3, 27, 1, False), (77, 1024, 512, 40, 1, 1, 0, True)]


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

        def fwd(npl):
            ops.lib.call("dv3_tc_convblock_fwd", ops._p(xs), ops._p(wf), npl, ops._p(bias), None, ops._p(res),
                         ops._p(y), ops._p(sa), ops._p(ss), B, C, T, K, 1, 0, 0, 1, None, ops._stream())

        def dgrad(npl):
            ops.lib.call("dv3_tc_conv", ops._p(dab), ops._p(wb), npl, ops._p(dx), B, 2 * C, C, T, K, 1, 0, 1, None, 0,
                         0.0, None, 0, 1, ops._p(e1), None, 0.7071067811865476, None, ops._stream())

        def conv1(npl):
            ops.lib.call("dv3_tc_conv", ops._p(xs), ops._p(w1), npl, ops._p(yc), B, C, C, T, 1, 1, 0, 0, ops._p(bias),
                         1, 0.0, None, 0, 0, None, None, 0.0, None, ops._stream())

        # with npl = 1 the launches read plane 0 of the same buffers
        for npl, tag in [(2, ""), (1, "_npl1")]:
            for name, fn, arrs in [("fwd", fwd, {"y": y, "a": sa, "s": ss}), ("dgrad", dgrad, {"dx": dx}),
                                   ("conv1x1", conv1, {"y": yc})]:
                fn(npl)
                torch.cuda.synchronize()
                for k, v in arrs.items():
                    outs["%s%s_C%d_T%d_%s" % (name, tag, C, T, k)] = v.cpu().numpy()
                times["%s%s C=%d T=%d" % (name, tag.replace("_", " "), C, T)] = timed(lambda: fn(npl))
    for Bw, Mw, Nw, T, k, dil, causal, convt in [(B, 2 * C, C, T, K, 1, 0, False) for C, T in SHAPES] + WG_EXTRA:
        g = torch.Generator().manual_seed(7 * Mw + 3 * Nw + T + Bw)
        p8 = lambda n: (n + 7) // 8 * 8  # noqa: E731
        dy = torch.stack([(torch.randn(Bw, T, p8(Mw), generator=g) * s).to(bf) for s in (1e-3, 5e-4)]).to(dev)
        xw = torch.stack([(torch.randn(Bw, T, p8(Nw), generator=g) * s).to(bf) for s in (1.0, 0.5)]).to(dev)
        if convt:       # ops._CONVT: m = (tap, co), Cout = Mw / 2, element (m % Cout) * 2 + m // Cout + n * Mw
            ms, s_m, s_mh, s_n, s_j = Mw // 2, 2, 1, Mw, 0
        else:           # tap-major
            ms, s_m, s_mh, s_n, s_j = Mw, Nw, 0, 1, Mw * Nw
        nsplit = ops.lib.raw("dv3_tc_wgrad_nsplit")(Bw, Mw, Nw, T, k)
        numel = Mw * Nw * k
        parts = torch.zeros(nsplit, numel, device=dev)

        def wgrad(npl):
            ops.lib.call("dv3_tc_wgrad_mn_npl", ops._p(dy), ops._p(xw), npl, ops._p(parts), numel, Bw, Mw, Nw, T, k,
                         dil, causal, ms, s_m, s_mh, s_n, s_j, ops._stream())

        shape = "B%d %dx%d T%d k%d%s%s" % (Bw, Mw, Nw, T, k, " d%d causal" % dil if causal else "",
                                          " convT" if convt else "")
        for npl in (2, 1):
            wgrad(npl)
            torch.cuda.synchronize()
            outs["wgrad_npl%d_%s" % (npl, shape.replace(" ", "_"))] = parts.cpu().numpy()
            times["wgrad npl%d %s" % (npl, shape)] = timed(lambda: wgrad(npl))
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
    w = max([22] + [len(k) for k in ta])
    print("%-*s %10s %10s %7s" % (w, "launch", "old us", "new us", "ratio"))
    for k in ta:
        print("%-*s %10.1f %10.1f %7.3f" % (w, k, ta[k], tb[k], tb[k] / ta[k]))


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        child(sys.argv[2])
    else:
        main()
