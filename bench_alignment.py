"""Attention alignments (DESIGN.md section 2.19), four measurements:

  1. the MAS kernels on a corpus-shaped ragged batch: 2 048 seeded alignments of 40-250 tokens x 150-1 000 decoder
     steps (softmax rows around a noisy diagonal): forward and backtrace µs with CUDA events over --iters calls after
     --warmup, cells/s, and the bytes the forward must read (every valid cell of A once) against the 3.35 TB/s HBM roof,
     next to the number of per-step barriers of the longest row (the forward's serial dependency);
  2. the fp64 numpy oracle (tests/alignment_oracle.py) on the first --cpu-rows rows on the host CPU, extrapolated to all
     2 048 by cells;
  3. alignment.evaluate_attention on deepvoice3_ljspeech with random weights, 64 utterances: stage times;
  4. alignment.teacher_forced_alignment on a B = 16 training-shaped batch of deepvoice3_ljspeech, next to one TrainStep
     step on the same batch for scale.

Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing to the tree.

    python bench_alignment.py [--iters 20] [--warmup 3] [--cpu-rows 4]
"""
import argparse
import contextlib
import json
import os
import sys
import time

import numpy as np
import torch

from bench import PRESETS
from bench_mcd import _cpu_name, _events
from bench_speaker_adapt import card
from deepvoice3_pytorch_b200 import alignment, builder, data, mcd, ops
from deepvoice3_pytorch_b200._lib import lib
from deepvoice3_pytorch_b200.train_step import TrainStep, to_device

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import alignment_oracle as AO  # noqa: E402

HBM_PEAK = 3.35e12


def corpus(B=2048, seed=0):
    """B alignments (N_b, L_b) padded into one (B, N, L) fp32 host array: softmax rows around a noisy diagonal."""
    rng = np.random.RandomState(seed)
    steps = rng.randint(150, 1001, B)
    tokens = np.array([rng.randint(40, min(250, n) + 1) for n in steps])       # every row has a path: N_b >= L_b
    A = np.zeros((B, steps.max(), tokens.max()), np.float32)
    for b in range(B):
        N, L = steps[b], tokens[b]
        c = np.linspace(0, L - 1, N)[:, None] + np.cumsum(rng.randn(N, 1) * 0.2, 0)
        x = -(np.arange(L)[None] - c) ** 2 / 4.0
        e = np.exp(x - x.max(1, keepdims=True))
        A[b, :N, :L] = e / e.sum(1, keepdims=True)
    return A, steps, tokens


def kernels(A_np, steps, tokens, iters, warmup):
    dev = torch.device("cuda")
    A = torch.from_numpy(A_np).to(dev)
    B, N, L = A.shape
    steps_l, tokens_l = alignment._check_alignments(A, steps, tokens)
    t_api = _events(lambda: alignment._mas(A, steps_l, tokens_l), iters, warmup)
    # the two launches alone, on buffers set up once
    words = [int(lib.raw("dv3_mas_dir_words")(n, l)) for n, l in zip(steps_l, tokens_l)]
    dir_off = torch.from_numpy(np.concatenate([[0], np.cumsum(words)[:-1]]).astype(np.int64)).to(dev)
    dirs = torch.empty(int(sum(words)), dtype=torch.int32, device=dev)
    s_d = torch.tensor(steps_l, dtype=torch.int32, device=dev)
    l_d = torch.tensor(tokens_l, dtype=torch.int32, device=dev)
    argmax, maxv = torch.empty(B, N, dtype=torch.int32, device=dev), torch.empty(B, N, device=dev)
    cov, score = torch.empty(B, L, device=dev), torch.empty(B, device=dev)
    dur = torch.empty(B, L, dtype=torch.int32, device=dev)
    p, st = ops._p, ops._stream
    fwd = lambda: lib.call("dv3_mas_forward", p(A), A.stride(0), A.stride(1), p(s_d), p(l_d), B, N, L, p(dir_off),
                           p(dirs), p(argmax), p(maxv), p(cov), p(score), st())
    bt = lambda: lib.call("dv3_mas_backtrace", p(s_d), p(l_d), B, L, p(dir_off), p(dirs), p(dur), st())
    t_fwd, t_bt = [], []
    for _ in range(3):
        t_fwd.append(_events(fwd, iters, warmup))
        t_bt.append(_events(bt, iters, warmup))
    cells = int(np.sum(steps.astype(np.int64) * tokens))
    fwd_bytes = 4 * cells + 4 * 2 * int(steps.sum()) + 4 * int(tokens.sum()) + 4 * int(sum(words))
    best = min(t_fwd)
    d = dur.cpu().numpy()
    assert all(d[b, :tokens[b]].sum() == steps[b] for b in range(B))
    return {"rows": B, "steps_range": [int(steps.min()), int(steps.max())],
            "tokens_range": [int(tokens.min()), int(tokens.max())], "cells": cells,
            "monotonic_alignment_device_us": round(t_api, 1), "forward_us": [round(x, 1) for x in t_fwd],
            "backtrace_us": [round(x, 1) for x in t_bt], "cells_per_s": cells / (best * 1e-6),
            "forward_bytes": fwd_bytes, "hbm_bound_us": round(fwd_bytes / HBM_PEAK * 1e6, 1),
            "hbm_roof_share": round(fwd_bytes / HBM_PEAK / (best * 1e-6), 4),
            "barriers_longest_row": int(steps.max()), "us_per_step_of_longest_row": round(best / steps.max(), 3),
            "direction_bytes": 4 * int(sum(words))}


def cpu_oracle(A_np, steps, tokens, n):
    t0 = time.perf_counter()
    cells = 0
    for b in range(n):
        a = A_np[b, :steps[b], :tokens[b]]
        AO.mas(a)
        AO.statistics(a)
        cells += a.size
    s = time.perf_counter() - t0
    total = int(np.sum(steps.astype(np.int64) * tokens))
    return {"cpu": _cpu_name(), "rows_timed": n, "s": round(s, 3), "cells_per_s": cells / s,
            "all_rows_s_extrapolated_by_cells": round(s * total / cells, 1)}


def _timer(times):
    @contextlib.contextmanager
    def timer(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    return timer


def evaluation(n_utt=64, max_steps=200):
    bname, kw, _ = PRESETS["deepvoice3_ljspeech"]
    torch.manual_seed(0)
    model = getattr(builder, bname)(**kw).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = max_steps
    rng = np.random.RandomState(0)
    seqs = [rng.randint(2, 149, rng.randint(20, 80)) for _ in range(n_utt)]
    times = {}
    alignment.evaluate_attention(model, seqs, stage_timer=_timer(times))          # warm-up
    times.clear()
    res = alignment.evaluate_attention(model, seqs, stage_timer=_timer(times))
    return {"preset": "deepvoice3_ljspeech", "utterances": n_utt, "max_decoder_steps": max_steps,
            "ms": {k: round(t * 1e3, 2) for k, t in times.items()}, "steps_total": int(res["steps"].sum()),
            "stop_failures": res["stop_failures"], "mean_focus_rate": res["mean_focus_rate"]}


def teacher_forcing(B=16, iters=10):
    bname, kw, extra = PRESETS["deepvoice3_ljspeech"]
    torch.manual_seed(0)
    model = getattr(builder, bname)(**kw).cuda()
    rng = np.random.RandomState(1)
    items = [(rng.randint(2, 149, rng.randint(60, 160)), rng.rand(n, 80).astype(np.float32),
              rng.rand(n, kw["linear_dim"]).astype(np.float32)) for n in rng.randint(400, 800, B)]
    batch = to_device(data.collate(items, r=kw["r"], downsample_step=kw["downsample_step"]), "cuda")
    step = TrainStep(model, **extra)
    for _ in range(3):
        step.step(batch)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        step.step(batch)
    torch.cuda.synchronize()
    t_step = (time.perf_counter() - t0) / iters
    model.eval()
    for _ in range(3):
        alignment.teacher_forced_alignment(model, batch)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        res = alignment.teacher_forced_alignment(model, batch)
    torch.cuda.synchronize()
    t_tf = (time.perf_counter() - t0) / iters
    return {"preset": "deepvoice3_ljspeech", "B": B, "T_dec": int(batch["frame_positions"].size(1)),
            "teacher_forced_alignment_ms": round(t_tf * 1e3, 2), "train_step_ms": round(t_step * 1e3, 2),
            "frames_per_step": res["frames_per_step"], "mean_score_per_step": float(np.mean(res["score_per_step"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-rows", type=int, default=4)
    ap.add_argument("--no-eval", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_alignment.py needs a CUDA device")
    A, steps, tokens = corpus()
    out = {"card": card(), "mas": kernels(A, steps, tokens, args.iters, args.warmup),
           "cpu_oracle_fp64": cpu_oracle(A, steps, tokens, args.cpu_rows)}
    if not args.no_eval:
        out["evaluate_attention"] = evaluation()
        out["teacher_forced_alignment"] = teacher_forcing()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
