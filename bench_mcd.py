"""MCD-DTW (DESIGN.md section 2.17), three workloads:

  1. 512 ragged pairs of 200-900 frames (seeded), M = 80 mel bins, K = 24 cepstra: the cepstra kernel and the DTW
     kernel timed separately with CUDA events over --iters launches after --warmup; µs per pair, DP cells/s, and
     achieved FLOP/s (2K + 4 flops per cell) against the FP32 data-sheet roof, next to the HBM bound of the cepstra;
  2. the same pairs through the fp64 numpy oracle (tests/mcd_oracle.py, DTW vectorised over anti-diagonals) on the host
     CPU, on the first --cpu-pairs pairs: the baseline a user has without the kernels;
  3. mcd.evaluate_synthesis on deepvoice3_ljspeech with random weights, 64 utterances: stage times.

Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing to the tree.

    python bench_mcd.py [--iters 20] [--warmup 3] [--cpu-pairs 8]
"""
import argparse
import contextlib
import json
import os
import platform
import sys
import time

import numpy as np
import torch

from bench import PRESETS
from bench_speaker_adapt import card
from deepvoice3_pytorch_b200 import builder, mcd
from deepvoice3_pytorch_b200._lib import lib
from deepvoice3_pytorch_b200.ops import _p, _stream

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import mcd_oracle as MO  # noqa: E402

P, LO, HI, M, K = 512, 200, 900, 80, 24
FP32_PEAK, HBM = 67e12, 3.35e12


def _pairs(seed=0):
    rng = np.random.RandomState(seed)
    la, lb = rng.randint(LO, HI + 1, P), rng.randint(LO, HI + 1, P)
    return [rng.rand(n, M).astype(np.float32) for n in la], [rng.rand(n, M).astype(np.float32) for n in lb]


def _events(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters                      # µs per launch


def kernels(a_np, b_np, iters, warmup):
    dev = torch.device("cuda")
    mels = [torch.from_numpy(x).to(dev) for x in a_np + b_np]
    la, lb = [x.shape[0] for x in a_np], [x.shape[0] for x in b_np]
    padded = torch.nn.utils.rnn.pad_sequence(mels, batch_first=True).contiguous()
    n, T_max = padded.shape[:2]
    lens = torch.tensor(la + lb, dtype=torch.int32, device=dev)
    basis = mcd._device_basis(dev, M, K)
    cep = torch.empty(n, T_max, K, device=dev)

    def cepstra():
        lib.call("dv3_mel_cepstra", _p(padded), _p(lens), _p(basis), _p(cep), n, T_max, M, K,
                 _stream())
    cepstra()
    rows = [q * T_max for q in range(n)]
    work, ws_floats = mcd._work_list(rows[:P], la, rows[P:], lb)
    work_d = torch.from_numpy(work).to(dev)
    ws = torch.empty(ws_floats, device=dev)
    cost = torch.empty(P, device=dev)
    path = torch.empty(P, dtype=torch.int32, device=dev)

    def dtw():
        lib.call("dv3_dtw_mcd", _p(cep), K, _p(work_d), _p(ws), _p(cost), _p(path), P,
                 _stream())
    t_cep = _events(cepstra, iters, warmup)
    t_dtw = _events(dtw, iters, warmup)
    res = mcd.mcd_dtw(mels[:P], mels[P:], K)                       # the public call, checked against the raw one
    assert np.array_equal(res["path_length"], path.cpu().numpy())
    cells = int(sum(x * y for x, y in zip(la, lb)))
    frames = sum(la) + sum(lb)
    cep_bytes = 4 * frames * (M + K) + 4 * K * M
    dtw_flops = cells * (2 * K + 4)
    dtw_bytes = 4 * K * sum(x + -(-x // 32) * y for x, y in zip(la, lb)) + 16 * sum(-(-x // 32) * y for x, y in zip(la, lb))
    longest = max(-(-x // 32) * (y + 31) for x, y in zip(la, lb))
    return {
        "pairs": P, "frames": [LO, HI], "M": M, "K": K, "dp_cells": cells,
        "cepstra": {"us": round(t_cep, 2), "us_per_pair": round(t_cep / P, 4), "bytes": cep_bytes,
                    "flops": 2 * frames * M * K,
                    "hbm_bound_us": round(cep_bytes / HBM * 1e6, 2), "fp32_bound_us": round(2 * frames * M * K / FP32_PEAK * 1e6, 2)},
        "dtw": {"us": round(t_dtw, 1), "us_per_pair": round(t_dtw / P, 3), "cells_per_s": cells / (t_dtw * 1e-6),
                "flops": dtw_flops, "tflops": round(dtw_flops / (t_dtw * 1e-6) / 1e12, 3),
                "fp32_roof_share": round(dtw_flops / FP32_PEAK / (t_dtw * 1e-6), 5),
                "fp32_bound_us": round(dtw_flops / FP32_PEAK * 1e6, 1),
                "bytes_min": 4 * K * frames, "hbm_bound_us": round(4 * K * frames / HBM * 1e6, 1),
                "bytes_read_incl_restaging": dtw_bytes,
                "longest_pair_serial_steps": longest,
                "ns_per_serial_step_of_longest": round(t_dtw * 1e3 / longest, 2)},
        "mean_mcd_random_mels": float(res["mcd"].mean()),
    }


def _cpu_name():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or platform.machine()


def cpu_oracle(a_np, b_np, n):
    t0 = time.perf_counter()
    cells = 0
    for a, b in zip(a_np[:n], b_np[:n]):
        MO.dtw(MO.cepstra(a, K), MO.cepstra(b, K))
        cells += a.shape[0] * b.shape[0]
    s = time.perf_counter() - t0
    total = sum(a.shape[0] * b.shape[0] for a, b in zip(a_np, b_np))
    return {"cpu": _cpu_name(), "threads": torch.get_num_threads(), "pairs_timed": n, "s": round(s, 3),
            "ms_per_pair": round(s / n * 1e3, 2), "cells_per_s": cells / s,
            "all_512_pairs_s_extrapolated_by_cells": round(s * total / cells, 2)}


def evaluation(n_utt=64, max_steps=200):
    bname, kw, _ = PRESETS["deepvoice3_ljspeech"]
    torch.manual_seed(0)
    model = getattr(builder, bname)(**kw).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = max_steps
    rng = np.random.RandomState(0)
    seqs = [rng.randint(2, 149, rng.randint(20, 80)) for _ in range(n_utt)]
    refs = [(rng.randn(rng.randint(2, 6) * 22050) * 0.1).astype(np.float32) for _ in range(n_utt)]
    times = {}

    @contextlib.contextmanager
    def timer(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    mcd.evaluate_synthesis(model, seqs, refs, stage_timer=timer)           # warm-up
    times.clear()
    res = mcd.evaluate_synthesis(model, seqs, refs, stage_timer=timer)
    return {"preset": "deepvoice3_ljspeech", "utterances": n_utt, "max_decoder_steps": max_steps,
            "ms": {k: round(t * 1e3, 2) for k, t in times.items()},
            "frames_synth_total": int(res["frames"][:, 0].sum()), "frames_ref_total": int(res["frames"][:, 1].sum()),
            "mean_mcd": res["mean_mcd"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-pairs", type=int, default=8)
    ap.add_argument("--no-eval", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mcd.py needs a CUDA device")
    a_np, b_np = _pairs()
    out = {"card": card(), "kernels": kernels(a_np, b_np, args.iters, args.warmup),
           "cpu_oracle_fp64": cpu_oracle(a_np, b_np, args.cpu_pairs)}
    if not args.no_eval:
        out["evaluate_synthesis"] = evaluation()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
