#!/usr/bin/env python
"""Systematic (scale) error of the tensor-core split-bf16 convolution against float64: the tensor core accumulates with
truncation, which shrinks every output by ~n_mma * 2^-25.  Prints, for a plain k-tap conv at a few contraction
lengths, bias = <(y - y64), y64> / <y64, y64> and the relative rms error.  DV3_TC_GAMMA (units of 2^-25 per MMA) sets the
epilogue compensation (read once per process)."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepvoice3_pytorch_b200 import ops  # noqa: E402

ops.conv_math = "tc"
torch.manual_seed(0)
for (B, Cin, Cout, T, k) in [(4, 256, 256, 800, 1), (4, 256, 256, 800, 3), (4, 512, 512, 800, 3), (4, 512, 512, 800, 5)]:
    x = torch.randn(B, Cin, T, device="cuda")
    v = torch.randn(Cout, Cin, k, device="cuda") * (1.0 / (k * Cin)) ** 0.5
    g = v.pow(2).sum((1, 2), keepdim=True).sqrt()
    bias = torch.zeros(Cout, device="cuda")
    with torch.no_grad():
        y = ops.conv1d(x, v, g, bias, k=k, dilation=1).double()
        y64 = F.conv1d(x.double(), v.double(), padding=(k - 1) // 2)
        ops.conv_math = "fp32"
        y32 = ops.conv1d(x, v, g, bias, k=k, dilation=1).double()
        ops.conv_math = "tc"
    for name, t in (("tc", y), ("fp32", y32)):
        e = t - y64
        print("Cin=%d k=%d n_mma=%d  %-5s bias=%+.3e  rel_rms=%.3e" % (
            Cin, k, Cin * k // 16, name, float((e * y64).sum() / (y64 * y64).sum()),
            float(e.pow(2).mean().sqrt() / y64.pow(2).mean().sqrt())), flush=True)
