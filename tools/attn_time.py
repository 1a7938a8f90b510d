#!/usr/bin/env python
"""Stand-alone timing of the tensor-core attention core at the deepvoice3_ljspeech training shape (B=16, E=256,
Td=200, Ts=128, padded keys masked, dropout 0.05, a non-null dprobs), L2 flushed before every launch:

  * forward and whole backward with CUDA events around the C-ABI calls (median of --reps);
  * every attention kernel separately (backward rows / cols) with its grid, from a torch.profiler pass of its own;
  * the card name and power limit, read in the same run.

    python tools/attn_time.py                              # the library the package loads (DV3_LIB or csrc/)
    python tools/attn_time.py --libs A.so B.so --rounds 3  # two builds alternately, each round a fresh process
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, E, TD, TS = 16, 256, 200, 128
P_DROP = 0.05


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(reps):
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    from deepvoice3_pytorch_b200._lib import LIB_PATH, lib

    torch.manual_seed(0)
    dev = "cuda"
    q = torch.randn(B, E, TD, device=dev)
    k = 0.3 * torch.randn(B, E, TS, device=dev)
    v = torch.randn(B, E, TS, device=dev)
    mask = torch.zeros(B, TS, dtype=torch.uint8, device=dev)
    mask[1, 100:] = 1
    mask[5, 60:] = 1
    dout = torch.randn(B, E, TD, device=dev)
    dprobs = 1e-3 * torch.randn(B, TD, TS, device=dev)
    seed = torch.tensor([1234], dtype=torch.int64, device=dev)
    probs = torch.empty(B, TD, TS, device=dev)
    out = torch.empty(B, E, TD, device=dev)
    ds = torch.empty(B, TD, TS, device=dev)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    scale = TS * (1.0 / TS) ** 0.5
    salt = 7

    def fwd():
        lib.call("dv3_tc_attn_fwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), probs.data_ptr(),
                 out.data_ptr(), B, E, TD, TS, scale, P_DROP, seed.data_ptr(), salt,
                 torch.cuda.current_stream().cuda_stream)

    def bwd():
        lib.call("dv3_tc_attn_bwd", dout.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), probs.data_ptr(),
                 dprobs.data_ptr(), ds.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, E, TD, TS, scale,
                 P_DROP, seed.data_ptr(), salt, torch.cuda.current_stream().cuda_stream)

    tf, tb = [], []
    for it in range(reps + 3):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        flush.zero_()
        ev[0].record(); fwd(); ev[1].record()
        flush.zero_()
        ev[2].record(); bwd(); ev[3].record()
        torch.cuda.synchronize()
        if it >= 3:
            tf.append(ev[0].elapsed_time(ev[1]) * 1e3)
            tb.append(ev[2].elapsed_time(ev[3]) * 1e3)

    # per-kernel durations and grids (a separate, traced pass)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            flush.zero_(); fwd()
            flush.zero_(); bwd()
        torch.cuda.synchronize()
    path = os.path.join(tempfile.mkdtemp(), "attn.json")
    prof.export_chrome_trace(path)
    durs, grids, order = collections.defaultdict(list), {}, []
    for e in json.load(open(path))["traceEvents"]:
        if e.get("cat") == "kernel" and "attn" in e["name"]:
            name = e["name"].replace("void ", "").split("(")[0]
            if name not in grids:
                order.append(name)
            durs[name].append(e["dur"])
            grids[name] = (e["args"].get("grid"), e["args"].get("block"), e["args"].get("shared memory"))
    kernels = [dict(name=n, us=float(np.median(durs[n])), grid=grids[n][0], block=grids[n][1], smem=grids[n][2])
               for n in order]
    return dict(lib=LIB_PATH, card=card(), fwd_us=float(np.median(tf)), bwd_us=float(np.median(tb)),
                fwd_spread_us=[float(min(tf)), float(max(tf))], bwd_spread_us=[float(min(tb)), float(max(tb))],
                kernels=kernels)


def report(r):
    print("%s  [%s]" % (r["lib"], r["card"]))
    print("  forward %.1f us (min %.1f, max %.1f)   backward %.1f us (min %.1f, max %.1f)" % (
        r["fwd_us"], *r["fwd_spread_us"], r["bwd_us"], *r["bwd_spread_us"]))
    for kk in r["kernels"]:
        print("    %-32s %7.1f us  grid %s block %s smem %s" % (kk["name"], kk["us"], kk["grid"], kk["block"],
                                                                 kk["smem"]))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=int(os.environ.get("ATTN_REPS", "50")))
    ap.add_argument("--libs", nargs="+", help="builds of libdv3b200.so to compare, run alternately via DV3_LIB")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", action="store_true", help="print one JSON line (used by the --libs driver)")
    a = ap.parse_args()
    if not a.libs:
        r = measure(a.reps)
        print(json.dumps(r)) if a.json else report(r)
        return
    res = collections.defaultdict(list)
    for rnd in range(a.rounds):
        for lib_path in a.libs:
            env = dict(os.environ, DV3_LIB=os.path.abspath(lib_path))
            outp = subprocess.run([sys.executable, os.path.abspath(__file__), "--json", "--reps", str(a.reps)],
                                  env=env, capture_output=True, text=True, check=True).stdout
            r = json.loads(outp.strip().splitlines()[-1])
            res[lib_path].append(r)
            print("round %d: " % rnd, end="")
            report(r)
    print("summary (median over rounds of per-round medians):")
    for lib_path in a.libs:
        rs = res[lib_path]
        f = sorted(x["fwd_us"] for x in rs)[len(rs) // 2]
        b = sorted(x["bwd_us"] for x in rs)[len(rs) // 2]
        print("  %-48s forward %.1f us  backward %.1f us" % (lib_path, f, b))


if __name__ == "__main__":
    main()
