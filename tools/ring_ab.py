#!/usr/bin/env python
"""A/B of two builds of tc_gemm.cu over every tensor-core GEMM shape of one training step.

    python tools/ring_ab.py build [--rev HEAD] [--dir build/ring_ab]       # no GPU needed
    python tools/ring_ab.py run [--dir build/ring_ab] [--reps 50] [--rounds 3] [--json OUT.json]

`build` compiles two copies of the library: `old` with tc_gemm.cu as committed at --rev (default HEAD, the parent of
uncommitted work) and `new` with the working tree's; every other source is the working tree's and is compiled once.

`run` needs a GPU.  Each round runs one child process per build (DV3_LIB selects it), alternating which goes first.
A child records every dv3_tc_convblock_fwd / dv3_tc_conv / dv3_tc_wgrad_mn_npl call of one eager forward + backward
of the preset (B=16, T_text=128, T_mel=800: the 25 ConvBlock forward / data-gradient shapes, the 1x1 / projection /
upsampler convs, every weight gradient) with its launch count, then launches each distinct call on seeded random
operands, two planes as the step does and one plane ("tc1"), L2 flushed before every launch, CUDA events, median of
--reps.  The outputs of round 0 are compared element for element between the builds (expected: identical).  Prints
the card, its power limit and SM clock, the per-shape medians over the rounds (min-max) and the launch-weighted
totals per step.
"""
import argparse
import collections
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc")
BUILDS = ("old", "new")


# ---- build (host) ---------------------------------------------------------------------------------------------------
def build(a):
    sys.path.insert(0, ROOT)
    from deepvoice3_pytorch_b200 import _build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f for f in _build.NVCC_FLAGS if not f.startswith("--use_fast_math")] + ["-I", CSRC]
    common = os.path.join(a.dir, "common")
    os.makedirs(common, exist_ok=True)
    srcs = {}
    for tag in BUILDS:
        d = os.path.join(a.dir, tag)
        os.makedirs(d, exist_ok=True)
        srcs[tag] = os.path.join(d, "tc_gemm.cu")
    with open(srcs["old"], "wb") as f:
        f.write(subprocess.check_output(["git", "-C", ROOT, "show",
                                         "%s:deepvoice3_pytorch_b200/csrc/tc_gemm.cu" % a.rev]))
    shutil.copyfile(os.path.join(CSRC, "tc_gemm.cu"), srcs["new"])
    jobs = [(s, os.path.join(common, os.path.basename(s)[:-3] + ".o")) for s in _build.sources()
            if os.path.basename(s) != "tc_gemm.cu"]
    jobs += [(srcs[t], srcs[t][:-3] + ".o") for t in BUILDS]
    procs = [(s, subprocess.Popen([nvcc] + flags + ["-c", s, "-o", o], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT)) for s, o in jobs]
    for s, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode:
            raise SystemExit("nvcc failed on %s:\n%s" % (s, out))
    objs = [o for s, o in jobs[:-2]]
    for t in BUILDS:
        lib = os.path.join(a.dir, t, "libdv3b200.so")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", lib,
                               srcs[t][:-3] + ".o"] + objs)
        print(lib)


# ---- child (GPU): record the step's GEMM calls, time and dump them -------------------------------------------------
def record_calls(preset):
    """{call key: launches per step} of one eager forward + backward."""
    import torch
    import bench
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200.train_step import make_synthetic_batch, to_device
    bname, kw, _ = bench.PRESETS[preset]
    torch.manual_seed(1234)
    model = getattr(builder, bname)(**kw).cuda().train()
    b = to_device(make_synthetic_batch(bench.B, bench.T_TEXT, bench.T_MEL, n_speakers=kw["n_speakers"]), "cuda")
    seen = collections.Counter()
    call = lib.call
    nn = lambda v: int(v is not None)  # noqa: E731

    def rec(name, *x):
        if name == "dv3_tc_convblock_fwd":       # xd w npl bias spk res y a s | B C T k dil causal mode residual
            seen[("fwd", nn(x[3]), nn(x[4]), nn(x[5]), nn(x[7]), nn(x[8])) + tuple(int(v) for v in x[9:17])] += 1
        elif name == "dv3_tc_conv":              # a w npl out | B Kc Nc T k dil causal tt | bias relu p seed salt
            seen[("conv",) + tuple(int(v) for v in x[4:12]) +   # addmode e1 e2 alpha
                 (nn(x[12]), int(x[13]), float(x[14]), nn(x[15]), int(x[16]), int(x[17]), nn(x[18]), nn(x[19]),
                  float(x[20]))] += 1
        elif name == "dv3_tc_wgrad_mn_npl":      # dy xd npl parts stride | B Mw Nw T k dil causal ms s_m s_mh s_n s_j
            seen[("wgrad",) + tuple(int(v) for v in x[5:17])] += 1
        return call(name, *x)

    lib.call = rec
    try:
        spk = {"speaker_ids": b["speaker_ids"]} if "speaker_ids" in b else {}
        outs = model(b["x"], b["mel"], text_positions=b["text_positions"], frame_positions=b["frame_positions"],
                     input_lengths=b["input_lengths"], **spk)
        sum(o.float().sum() for o in outs if o is not None).backward()
        torch.cuda.synchronize()
    finally:
        lib.call = call
    return seen


def label(key):
    if key[0] == "fwd":
        B, C, T, k, dil, causal, mode, res = key[6:]
        return "fwd B%d C%d T%d k%d d%d%s%s" % (B, C, T, k, dil, " causal" if causal else "", " spk" if key[2] else "")
    if key[0] == "conv":
        B, Kc, Nc, T, k, dil, causal, tt = key[1:9]
        bias, relu, p, seed, salt, addmode = key[9:15]
        return "%s B%d %d->%d T%d k%d d%d%s%s%s" % ("dgrad" if tt else "conv", B, Kc, Nc, T, k, dil,
                                                    " causal" if causal else "", " drop" if p > 0 else "",
                                                    " add%d" % addmode if addmode else "")
    B, Mw, Nw, T, k, dil, causal, ms, s_m, s_mh, s_n, s_j = key[1:]
    return "wgrad B%d %dx%d T%d k%d d%d%s%s" % (B, Mw, Nw, T, k, dil, " causal" if causal else "",
                                               "" if s_n == 1 else " convT")


def family(key):
    if key[0] == "fwd" or (key[0] == "conv" and key[8] and key[5] > 1):
        return "convblock"           # gated forward, k-tap data gradients
    return "wgrad" if key[0] == "wgrad" else "conv"


def child(a, out_npz, out_json):
    import torch
    sys.path.insert(0, ROOT)
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    dev = "cuda"
    calls = record_calls(a.preset)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    seed = torch.tensor([20240607], dtype=torch.int64, device=dev)
    st = ops._stream()
    p8 = lambda n: (n + 7) // 8 * 8  # noqa: E731

    def timed(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(a.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        return float(np.median(ts))

    outs, rows = {}, []
    for idx, (key, n) in enumerate(sorted(calls.items(), key=lambda kv: (label(kv[0]), str(kv[0])))):
        g = torch.Generator().manual_seed(1000 + idx)

        def rnd(*shape, scale=1.0, dtype=torch.float32):
            return (torch.randn(*shape, generator=g) * scale).to(dtype).to(dev)

        def planes(*shape, scale=1.0, dtype=torch.float16):
            return torch.stack([rnd(*shape, scale=scale, dtype=dtype), rnd(*shape, scale=scale * 2 ** -11, dtype=dtype)])

        if key[0] == "fwd":
            has_bias, has_spk, has_res, has_a, has_s = key[1:6]
            B, C, T, k, dil, causal, mode, resid = key[6:]
            xs, w = planes(B, T, C), planes(k, 2 * C, C, scale=(1.0 / (k * C)) ** 0.5)
            bias = rnd(2 * C, scale=0.1) if has_bias else None
            spk = rnd(B, C, T, scale=0.1) if has_spk else None
            res = rnd(B, C, T) if has_res else None
            res_out = {"y": torch.empty(B, C, T, device=dev)}
            if has_a:
                res_out["a"] = torch.empty(B, C, T, device=dev)
            if has_s:
                res_out["s"] = torch.empty(B, C, T, device=dev)

            def fn(npl):
                lib.call("dv3_tc_convblock_fwd", ops._p(xs), ops._p(w), npl, ops._p(bias), ops._p(spk), ops._p(res),
                         ops._p(res_out["y"]), ops._p(res_out.get("a")), ops._p(res_out.get("s")), B, C, T, k, dil,
                         causal, mode, resid, None, st)
        elif key[0] == "conv":
            B, Kc, Nc, T, k, dil, causal, tt, has_bias, relu, p, has_seed, salt, addmode, has_e1, has_e2, alpha = key[1:]
            dt = torch.bfloat16 if tt else torch.float16
            x, w = planes(B, T, p8(Kc), dtype=dt), planes(k, Nc, p8(Kc), scale=(1.0 / (k * Kc)) ** 0.5, dtype=dt)
            bias = rnd(Nc, scale=0.1) if has_bias else None
            e1 = rnd(B, Nc, T) if has_e1 else None
            e2 = torch.rand(B, Nc, T, generator=g).to(dev) if has_e2 else None
            res_out = {"out": torch.empty(B, Nc, T, device=dev)}

            def fn(npl):
                lib.call("dv3_tc_conv", ops._p(x), ops._p(w), npl, ops._p(res_out["out"]), B, Kc, Nc, T, k, dil,
                         causal, tt, ops._p(bias), relu, p, ops._p(seed) if has_seed else None, salt, addmode,
                         ops._p(e1), ops._p(e2), alpha, None, st)
        else:
            B, Mw, Nw, T, k, dil, causal, ms, s_m, s_mh, s_n, s_j = key[1:]
            dy = planes(B, T, p8(Mw), scale=1e-3, dtype=torch.bfloat16)
            xw = planes(B, T, p8(Nw), dtype=torch.bfloat16)
            nsplit = lib.raw("dv3_tc_wgrad_nsplit")(B, Mw, Nw, T, k)
            numel = Mw * Nw * k
            res_out = {"dw": torch.zeros(nsplit, numel, device=dev)}

            def fn(npl):
                lib.call("dv3_tc_wgrad_mn_npl", ops._p(dy), ops._p(xw), npl, ops._p(res_out["dw"]), numel, B, Mw, Nw,
                         T, k, dil, causal, ms, s_m, s_mh, s_n, s_j, st)
        row = dict(key=list(key), label=label(key), family=family(key), launches=n)
        for npl in (2, 1):
            for v in res_out.values():
                v.fill_(float("nan"))
            fn(npl)
            torch.cuda.synchronize()
            if out_npz:
                for name, v in res_out.items():
                    outs["%03d_npl%d_%s" % (idx, npl, name)] = v.cpu().numpy()
            row["us_npl%d" % npl] = timed(lambda: fn(npl))
        rows.append(row)
    if out_npz:
        np.savez(out_npz, **outs)
    with open(out_json, "w") as f:
        json.dump(rows, f)


# ---- run (GPU) ------------------------------------------------------------------------------------------------------
def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as ex:
        return "nvidia-smi unavailable (%s)" % ex


def run(a):
    tmp = tempfile.mkdtemp(prefix="ring_ab_")
    print("card (name, power limit, SM clock, max SM clock): %s" % card(), flush=True)
    times = {t: [] for t in BUILDS}
    for r in range(a.rounds):
        for t in (BUILDS if r % 2 == 0 else BUILDS[::-1]):
            lib = os.path.abspath(os.path.join(a.dir, t, "libdv3b200.so"))
            npz = os.path.join(tmp, "%s.npz" % t) if r == 0 else ""
            js = os.path.join(tmp, "%s_%d.json" % (t, r))
            cmd = [sys.executable, os.path.abspath(__file__), "child", "--preset", a.preset, "--reps", str(a.reps),
                   "--npz", npz, "--json", js]
            subprocess.run(cmd, env=dict(os.environ, DV3_LIB=lib), check=True, cwd=ROOT)
            times[t].append(json.load(open(js)))
        print("round %d done; card now: %s" % (r, card()), flush=True)
    # bit-for-bit comparison of round 0's outputs
    A, Bn = np.load(os.path.join(tmp, "old.npz")), np.load(os.path.join(tmp, "new.npz"))
    assert sorted(A.files) == sorted(Bn.files), "the builds recorded different calls"
    ndiff = 0
    for k in A.files:
        x, y = A[k], Bn[k]
        if x.tobytes() != y.tobytes():
            ndiff += 1
            d = np.nanmax(np.abs(x.astype(np.float64) - y))
            print("DIFF %s: max |delta| %.3e, %d elements differ" % (k, d, int((x.view(np.uint32) != y.view(np.uint32)).sum())))
    print("outputs compared bit for bit: %d arrays, %d differ" % (len(A.files), ndiff))
    rows0 = times["old"][0]
    res = dict(card=card(), identical=ndiff == 0, arrays=len(A.files), rows=[])
    tot = collections.defaultdict(lambda: np.zeros((2, a.rounds)))
    w = max(len(r["label"]) for r in rows0)
    for npl in (2, 1):
        print("\n%-*s %4s %22s %22s %7s   (npl=%d, us per launch: median of rounds [min-max])"
              % (w, "call", "n", "old", "new", "ratio", npl))
        for i, r in enumerate(rows0):
            ts = [[times[t][k][i]["us_npl%d" % npl] for k in range(a.rounds)] for t in BUILDS]
            mo, mn = float(np.median(ts[0])), float(np.median(ts[1]))
            print("%-*s %4d %8.1f [%5.1f-%5.1f] %8.1f [%5.1f-%5.1f] %7.3f" % (
                w, r["label"], r["launches"], mo, min(ts[0]), max(ts[0]), mn, min(ts[1]), max(ts[1]), mn / mo))
            for fam in (r["family"], "all"):
                tot[(npl, fam)] += r["launches"] * np.array(ts)
            res["rows"].append(dict(label=r["label"], key=r["key"], npl=npl, launches=r["launches"],
                                    old_us=ts[0], new_us=ts[1]))
    print("\nlaunch-weighted us per step (per round; old -> new):")
    for (npl, fam), v in sorted(tot.items()):
        print("  npl=%d %-10s %s -> %s  (median %.1f -> %.1f, %+.2f %%)" % (
            npl, fam, " ".join("%.1f" % x for x in v[0]), " ".join("%.1f" % x for x in v[1]), np.median(v[0]),
            np.median(v[1]), 100.0 * (np.median(v[1]) / np.median(v[0]) - 1.0)))
    res["totals"] = {"npl%d_%s" % k: dict(old=v[0].tolist(), new=v[1].tolist()) for k, v in tot.items()}
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    shutil.rmtree(tmp, ignore_errors=True)
    if ndiff:
        raise SystemExit("outputs differ between the builds")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("cmd", choices=["build", "run", "child"])
    ap.add_argument("--dir", default=os.path.join(ROOT, "build", "ring_ab"))
    ap.add_argument("--rev", default="HEAD")
    ap.add_argument("--preset", default="deepvoice3_ljspeech")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--npz", default="")
    ap.add_argument("--json", default="", help="run: write the table here; child: its timings")
    a = ap.parse_args()
    if a.cmd == "build":
        build(a)
    elif a.cmd == "run":
        run(a)
    else:
        child(a, a.npz, a.json)


if __name__ == "__main__":
    main()
