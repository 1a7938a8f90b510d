"""Cost of the deterministic training mode (ops.deterministic, DESIGN.md section 2.10), measured in one process with
the mode off and on alternating.

    python bench_deterministic.py [--rounds 5] [--steps 30] [--micro-iters 200]

Steps: the CUDA-graph training step of the three presets at the benchmark shape (B = 16, T_text = 128, T_mel = 800) in
conv_math "tc" and "tc1": ms/step as median [min, max] over the rounds, and kernel launches per step.
Kernels: every replaced kernel against its atomic form at the preset shapes, CUDA events around many launches; bytes are
computed from the shapes and include the scratch traffic.
The card's name and power limit are read in the same run and belong beside every number quoted from it.  Writes
nothing; prints one JSON line at the end."""
import argparse
import ctypes
import json
import subprocess

import numpy as np
import torch

B, T_TEXT, T_MEL = 16, 128, 800


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:          # the numbers stay usable, but say that the limit is unknown
        return {"name": torch.cuda.get_device_name(), "power_limit": "unknown (%s)" % type(ex).__name__}


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def time_ms(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_steps(rounds, steps):
    from bench import PRESETS
    from deepvoice3_pytorch_b200 import builder, ops
    from deepvoice3_pytorch_b200.train_step import TrainStep, make_synthetic_batch, to_device
    rows = []
    old = ops.conv_math
    try:
        for preset in ("deepvoice3_ljspeech", "nyanko_ljspeech", "deepvoice3_vctk"):
            bname, kw, extra = PRESETS[preset]
            batch = to_device(make_synthetic_batch(B, T_TEXT, T_MEL, n_speakers=kw["n_speakers"]), "cuda")
            for math in ("tc", "tc1"):
                ops.conv_math = math
                arms = {}
                for det in (False, True):
                    torch.manual_seed(1234)
                    arms[det] = TrainStep(getattr(builder, bname)(**kw).cuda(), use_graph=True, deterministic=det, **extra)
                    for _ in range(5):
                        arms[det].step(batch)
                torch.cuda.synchronize()
                ms = {False: [], True: []}
                for _ in range(rounds):
                    for det in (False, True):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(steps):
                            arms[det].step(batch)
                        e1.record()
                        torch.cuda.synchronize()
                        ms[det].append(e0.elapsed_time(e1) / steps)
                row = {"preset": preset, "conv_math": math}
                for det, tag in ((False, "off"), (True, "on")):
                    row[tag] = {"ms_median": float(np.median(ms[det])), "ms_min": min(ms[det]), "ms_max": max(ms[det]),
                                "launches": arms[det].launches_per_step}
                row["on_over_off"] = row["on"]["ms_median"] / row["off"]["ms_median"]
                print("step %-20s %-3s  off %.3f [%.3f, %.3f] ms, %d launches   on %.3f [%.3f, %.3f] ms, %d launches   "
                      "on/off %.4f" % (preset, math, row["off"]["ms_median"], row["off"]["ms_min"], row["off"]["ms_max"],
                                       row["off"]["launches"], row["on"]["ms_median"], row["on"]["ms_min"],
                                       row["on"]["ms_max"], row["on"]["launches"], row["on_over_off"]), flush=True)
                rows.append(row)
                del arms
    finally:
        ops.conv_math = old
    return rows


def bench_kernels(iters):
    """-> rows {kernel, shape, atomic_us, det_us, atomic_GBps, det_GBps}; bytes: tensors read + written once, plus for
    the deterministic form the scratch written and read back."""
    from deepvoice3_pytorch_b200._lib import lib
    lib.load()
    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    rows = []

    def add(kernel, shape, atomic, det, nbytes, scratch_bytes):
        ta, td = time_ms(atomic, iters), time_ms(det, iters)
        row = {"kernel": kernel, "shape": shape, "atomic_us": ta * 1e3, "det_us": td * 1e3,
               "atomic_GBps": nbytes / ta / 1e6, "det_GBps": (nbytes + scratch_bytes) / td / 1e6}
        print("kernel %-22s %-28s atomic %8.2f us %7.1f GB/s   deterministic %8.2f us %7.1f GB/s" %
              (kernel, shape, row["atomic_us"], row["atomic_GBps"], row["det_us"], row["det_GBps"]), flush=True)
        rows.append(row)

    lscr = torch.zeros(lib.raw("dv3_loss_det_scratch_floats")(), device="cuda")
    loss, terms = torch.zeros(1, device="cuda"), torch.zeros(2, device="cuda")
    lens = torch.full((B,), T_MEL, dtype=torch.int64, device="cuda")
    for name, T, D in (("spec_loss mel", T_MEL // 4, 80), ("spec_loss linear", T_MEL, 513)):
        yh, y = torch.rand(B, T, D, device="cuda", generator=g) * 0.98 + 0.01, torch.rand(B, T, D, device="cuda", generator=g)
        grad = torch.empty_like(yh)
        add(name, "B%d T%d D%d" % (B, T, D),
            lambda: lib.call("dv3_spec_loss_terms", _p(yh), _p(y), _p(lens), None, _p(grad), _p(loss), _p(terms), B, T, D,
                             1, 0.5, 0.1, 0, 0.0, _st()),
            lambda: lib.call("dv3_spec_loss_det", _p(yh), _p(y), _p(lens), None, _p(grad), _p(loss), _p(terms), _p(lscr),
                             B, T, D, 1, 0.5, 0.1, 0, 0.0, _st()),
            12 * B * T * D, 2 * 4 * 3 * min((B * T * D + 255) // 256, 132 * 8))
    A, Td = 4, T_MEL // 4
    dh, dn = torch.rand(B, Td, device="cuda", generator=g) * 0.98 + 0.01, torch.zeros(B, Td, device="cuda")
    attn = torch.softmax(rn(A, B, Td, T_TEXT), -1)
    gd, ga = torch.empty_like(dh), torch.empty_like(attn)
    il, dl = torch.full((B,), T_TEXT, dtype=torch.int64, device="cuda"), torch.full((B,), Td, dtype=torch.int64, device="cuda")
    add("aux_loss", "A%d B%d Td%d Ts%d" % (A, B, Td, T_TEXT),
        lambda: lib.call("dv3_aux_loss_terms", _p(dh), _p(dn), _p(gd), B * Td, _p(attn), _p(ga), _p(il), _p(dl), None, A,
                         B, Td, T_TEXT, 0.2, 1, _p(loss), _p(terms), _st()),
        lambda: lib.call("dv3_aux_loss_det", _p(dh), _p(dn), _p(gd), B * Td, _p(attn), _p(ga), _p(il), _p(dl), None, A, B,
                         Td, T_TEXT, 0.2, 1, _p(loss), _p(terms), _p(lscr), _st()),
        8 * attn.numel() + 12 * B * Td, 2 * 4 * 3 * 264)

    fl = lib.raw("dv3_bias_det_scratch_floats")
    for C, T in ((256, T_MEL // 4), (256, T_MEL), (512, T_TEXT)):
        dy, a, x, s = rn(B, C, T), rn(B, C, T), rn(B, C, T), torch.rand(B, C, T, device="cuda", generator=g)
        db, pl = torch.zeros(2 * C, device="cuda"), torch.empty(2, B, T, 2 * C, device="cuda", dtype=torch.bfloat16)
        n = fl(B, 2 * C, T, 1)
        scr = torch.empty(n, device="cuda")
        add("tc_gate_bwd_split", "B%d C%d T%d" % (B, C, T),
            lambda: lib.call("dv3_tc_gate_bwd_split_npl", _p(dy), _p(a), _p(s), _p(x), _p(pl), 2, None, _p(db), B, C, T,
                             0, 1, None, 1, _st()),
            lambda: lib.call("dv3_tc_gate_bwd_split_det", _p(dy), _p(a), _p(s), _p(x), _p(pl), 2, _p(db), _p(scr), n, B,
                             C, T, 0, 1, None, 1, _st()),
            12 * B * C * T + 2 * pl.numel(), 8 * n)
        db1, pl1 = torch.zeros(C, device="cuda"), torch.empty(2, B, T, C, device="cuda", dtype=torch.bfloat16)
        n1 = fl(B, C, T, 1)
        add("tc_grad_split", "B%d C%d T%d" % (B, C, T),
            lambda: lib.call("dv3_tc_grad_split_npl", _p(dy), None, _p(pl1), 2, None, _p(db1), B, C, T, 0, None, 1, _st()),
            lambda: lib.call("dv3_tc_grad_split_det", _p(dy), None, _p(pl1), 2, _p(db1), _p(scr), n1, B, C, T, 0, None, 1,
                             _st()),
            4 * B * C * T + 2 * pl1.numel(), 8 * n1)
    C, T = 513, T_MEL                               # exact-fp32 kernels: the odd-width layers tensor cores do not take
    dy, a, x, s = rn(B, C, T), rn(B, C, T), rn(B, C, T), torch.rand(B, C, T, device="cuda", generator=g)
    dab, db, n = torch.empty(B, 2 * C, T, device="cuda"), torch.zeros(2 * C, device="cuda"), fl(B, 2 * C, T, 0)
    scr = torch.empty(n, device="cuda")
    add("convblock_gate_bwd", "B%d C%d T%d" % (B, C, T),
        lambda: lib.call("dv3_convblock_gate_bwd", _p(dy), _p(a), _p(s), _p(x), _p(dab), _p(db), B, C, T, 0, 1, _st()),
        lambda: lib.call("dv3_convblock_gate_bwd_det", _p(dy), _p(a), _p(s), _p(x), _p(dab), _p(db), _p(scr), n, B, C, T,
                         0, 1, _st()),
        20 * B * C * T, 8 * n)
    add("bias_act_bwd", "B%d C%d T%d" % (B, C, T),
        lambda: lib.call("dv3_bias_act_bwd", _p(dy), None, None, _p(db), B, C, T, 0, _st()),
        lambda: lib.call("dv3_bias_act_bwd_det", _p(dy), None, None, _p(db), _p(scr), n // 2, B, C, T, 0, _st()),
        4 * B * C * T, 8 * (n // 2))

    for name, V, D, N in (("embedding_bwd text", 149, 256, B * T_TEXT), ("embedding_bwd speaker", 108, 16, B)):
        ids, dy, dt = torch.randint(1, V, (N,), device="cuda", generator=g), rn(N, D), torch.zeros(V, D, device="cuda")
        add(name, "V%d D%d N%d" % (V, D, N),
            lambda: lib.call("dv3_embedding_bwd", _p(ids), _p(dy), _p(dt), N, D, V, 0, _st()),
            lambda: lib.call("dv3_embedding_bwd_det", _p(ids), _p(dy), _p(dt), N, D, V, 0, _st()),
            8 * N + 4 * N * D + 8 * V * D, 0)
    for name, P, D, T in (("sinusoid_bwd text", 512, 256, T_TEXT), ("sinusoid_bwd frames", 512, 256, T_MEL // 4)):
        pos = torch.arange(1, T + 1, device="cuda")[None].repeat(B, 1).contiguous()
        table, w, dy, dt = rn(P, D), torch.ones(1, device="cuda"), rn(B, T, D), torch.zeros(P, D, device="cuda")
        add(name, "P%d D%d B%d T%d" % (P, D, B, T),
            lambda: lib.call("dv3_sinusoid_bwd", _p(pos), _p(table), _p(w), 1, _p(dy), _p(dt), None, B, T, D, P, _st()),
            lambda: lib.call("dv3_sinusoid_bwd_det", _p(pos), _p(table), _p(w), 1, _p(dy), _p(dt), None, B, T, D, P, _st()),
            8 * B * T + 4 * B * T * D + 12 * P * D, 0)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--micro-iters", type=int, default=200)
    ap.add_argument("--skip-steps", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py needs a GPU")
    c = card()
    print("card: %s, power limit %s" % (c["name"], c["power_limit"]), flush=True)
    result = {"card": c, "shape": {"B": B, "T_text": T_TEXT, "T_mel": T_MEL}}
    result["kernels"] = bench_kernels(args.micro_iters)
    if not args.skip_steps:
        result["steps"] = bench_steps(args.rounds, args.steps)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
