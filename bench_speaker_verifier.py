"""Speaker-verifier training, scoring and cloned-voice evaluation on the deepvoice3_vctk shapes (DESIGN.md section 2.14),
B = 16 speakers x N = 9 samples (8 enrollment + 1 test) x T_crop = 128 frames, for each conv_math in --maths:

  (a) SpeakerVerifierStep: one CUDA graph for forward, backward and the clip + Adam update;
  (b) the same verifier as eager PyTorch autograd on the GPU (cuDNN convolutions, cuBLAS GEMMs, TF32 off) with
      torch.optim.Adam -- ms/step of both, arms alternating over --rounds rounds (median, min, max);

launches per graph step; the new kernels one launch at a time (CUDA events) at the training shape and at the scoring
shape, with the bytes / FLOPs each needs from shapes, the roof that binds (HBM bandwidth or FP32 CUDA-core rate) and
the kernel's share of it; scoring throughput in trials/s for 108 enrollment sets x 2 000 test utterances (embeddings
given); and the stage times of verify_cloned_voices (synthesis, mel, scoring) on the preset model.  Prints one JSON line,
with the card's name and power limit."""
import argparse
import contextlib
import ctypes
import json
import math
import time

import numpy as np
import torch
import torch.nn.functional as F

from bench_speaker_adapt import PRESET, PRESETS, card
from deepvoice3_pytorch_b200 import builder, ops
from deepvoice3_pytorch_b200._lib import lib
from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier, SpeakerVerifierStep, verify_cloned_voices

B, N, T_CROP = 16, 9, 128
N_ENR, N_TEST = 108, 2000
HBM, FP32 = 3.35e12, 67e12          # H100 SXM data sheet: HBM3 bytes/s, dense FP32 FLOP/s


def _batches(n=4):
    gen = torch.Generator().manual_seed(1)
    return [{"mels": torch.rand(B, N, T_CROP, 80, generator=gen).cuda(),
             "speaker_ids": torch.randperm(108, generator=gen)[:B].cuda()} for _ in range(n)]


class EagerVerifierStep:
    """(b): the verifier's arithmetic as plain torch autograd over a copy of its parameters."""

    def __init__(self, v, lr=1e-3):
        self.p = {k: t.detach().clone().requires_grad_(True) for k, t in v.state_dict().items()}
        self.k, self.n_conv = v.temporal[0].conv.kernel_size[0], len(v.temporal)
        self.opt = torch.optim.Adam(list(self.p.values()), lr=lr, betas=(0.9, 0.999), eps=1e-8)

    def _wn(self, pre):
        v, g = self.p[pre + "weight_v"], self.p[pre + "weight_g"]
        return g * v / v.pow(2).sum((1, 2), keepdim=True).sqrt()

    def trunk(self, mels):
        """mels (B, N, T, M) -> pooled features (B, N, C): the speaker encoder's trunk in eager torch."""
        p = self.p
        Bb, Nn, T, M = mels.shape
        x = mels.view(Bb * Nn, T, M).transpose(1, 2)
        for i in (0, 2):
            x = torch.relu(F.conv1d(x, self._wn("spectral.%d." % i), p["spectral.%d.bias" % i]))
        for i in range(self.n_conv):
            pre = "temporal.%d.conv." % i
            y = F.conv1d(x, self._wn(pre), p[pre + "bias"], padding=(self.k - 1) // 2)
            a, gate = y.chunk(2, dim=1)
            x = (a * torch.sigmoid(gate) + x) * math.sqrt(0.5)
        return x.mean(-1).view(Bb, Nn, -1)

    def step(self, b):
        p = self.p
        self.opt.zero_grad(set_to_none=False)
        h = self.trunk(b["mels"])
        e = F.linear(h[:, :-1].mean(1), p["w"], p["c"])
        t = F.linear(h[:, -1], p["w"], p["c"])
        S = p["S"]
        L = e @ t.T - ((e @ S) * e).sum(1)[:, None] - ((t @ S) * t).sum(1)[None, :] + p["b"]
        ids = b["speaker_ids"]
        same = ids[:, None] == ids[None, :]
        loss = 0.5 * F.softplus(-L[same]).mean() + 0.5 * F.softplus(L[~same]).mean()
        loss.backward()
        self.opt.step()
        return loss


def time_steps(step, batches, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(batches[i % len(batches)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def _time_us(fn, iters=200):
    for _ in range(10):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def _entry(us, nbytes, flops):
    t_mem, t_fp = nbytes / HBM * 1e6, flops / FP32 * 1e6
    roof = "HBM 3.35 TB/s" if t_mem >= t_fp else "FP32 67 TFLOP/s"
    return {"us": round(us, 2), "bytes": int(nbytes), "flops": int(flops), "roof": roof,
            "roof_us": round(max(t_mem, t_fp), 3), "share_of_roof": round(max(t_mem, t_fp) / us, 4)}


def kernels(v):
    """Each new kernel at the training shape (enrollment embed over B x (N-1) rows; score + loss over B x B pairs) and
    the score forward at the scoring shape: µs per launch, bytes and FLOPs from shapes, the binding roof."""
    dev = "cuda"
    C, D = v.channels, v.embed_dim
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())       # noqa: E731
    err = ops._err_flag(torch.device(dev))
    h = torch.rand(B, N, C, device=dev)
    n_e = torch.full((B,), N - 1, dtype=torch.int32, device=dev)
    hbar, x, dx = torch.empty(B, C, device=dev), torch.rand(B, D, device=dev) * 0.1, torch.rand(B, D, device=dev)
    d_h = torch.empty_like(h)
    part_e = torch.empty(B, D * C + D, device=dev)
    ids = torch.arange(B, device=dev)
    y = torch.rand(B, D, device=dev) * 0.1
    q, scores = torch.empty(2 * B, device=dev), torch.empty(B, B, device=dev)
    lp = torch.empty(lib.raw("dv3_spkver_loss_floats")(B, B), device=dev)
    dxx, dyy = torch.empty_like(x), torch.empty_like(y)
    part_s = torch.empty(2 * B, D * D + 1, device=dev)
    one = torch.ones((), device=dev)
    E, Y = torch.rand(N_ENR, D, device=dev) * 0.1, torch.rand(N_TEST, D, device=dev) * 0.1
    q2, s2 = torch.empty(N_ENR + N_TEST, device=dev), torch.empty(N_ENR, N_TEST, device=dev)
    Be, Bt = N_ENR, N_TEST
    runs = {
        "embed_fwd": (lambda: lib.call("dv3_spkver_embed_fwd", vp(h), N * C, vp(n_e), vp(v.w), vp(v.c), vp(hbar),
                                       vp(x), vp(err), B, N - 1, C, D, st),
                      4 * (B * (N - 1) * C + D * C + D + B * (C + D)), 2 * B * D * C + B * (N - 1) * C),
        "embed_bwd": (lambda: lib.call("dv3_spkver_embed_bwd", vp(dx), vp(hbar), vp(n_e), vp(v.w), vp(d_h), N * C,
                                       vp(part_e), vp(err), B, N - 1, C, D, st),
                      4 * (B * D + B * C + D * C + B * (N - 1) * C + B * (D * C + D)), 2 * B * D * C + B * D * C),
        "score_fwd_loss": (lambda: lib.call("dv3_spkver_score_fwd", vp(x), vp(y), vp(v.S), vp(v.b), vp(ids), vp(ids),
                                            vp(q), vp(q[B:]), vp(scores), vp(lp), B, B, D, st),
                           4 * (2 * B * D + D * D + B * B) + 16 * B, 2 * B * B * D + 2 * 2 * B * D * D),
        "score_bwd": (lambda: lib.call("dv3_spkver_score_bwd", vp(x), vp(y), vp(v.S), vp(scores), vp(ids), vp(ids),
                                       None, vp(one), vp(dxx), vp(dyy), vp(part_s), B, B, D, st),
                      4 * (2 * B * D + D * D + B * B + 2 * B * D + 2 * B * (D * D + 1)),
                      2 * 2 * B * B * D + 2 * 2 * B * 2 * D * D + 2 * B * D * D),
        "score_fwd_108x2000": (lambda: lib.call("dv3_spkver_score_fwd", vp(E), vp(Y), vp(v.S), vp(v.b), None, None,
                                                vp(q2), vp(q2[Be:]), vp(s2), None, Be, Bt, D, st),
                               4 * ((Be + Bt) * D + D * D + Be * Bt), 2 * Be * Bt * D + 2 * (Be + Bt) * D * D),
    }
    res = {name: _entry(_time_us(fn), nbytes, flops) for name, (fn, nbytes, flops) in runs.items()}
    ops.check_index_errors()
    return res


def scoring_throughput(v, iters=100):
    E = torch.rand(N_ENR, v.embed_dim, device="cuda") * 0.1
    Y = torch.rand(N_TEST, v.embed_dim, device="cuda") * 0.1
    us = _time_us(lambda: v.score(E, Y), iters)
    return {"trials": N_ENR * N_TEST, "us_per_call": round(us, 2), "trials_per_s": round(N_ENR * N_TEST / us * 1e6)}


def evaluation_stages(v, n_seq=16, max_steps=100):
    """verify_cloned_voices on the preset model (random weights, decoder capped at max_steps) with 4 enrolled speakers
    of 8 random utterances each: seconds per stage."""
    _, kw, _ = PRESETS[PRESET]
    torch.manual_seed(0)
    model = getattr(builder, PRESETS[PRESET][0])(**kw).cuda().eval()
    model.seq2seq.decoder.max_decoder_steps = max_steps
    rng = np.random.RandomState(0)
    enroll = {s: [rng.rand(rng.randint(150, 300), 80).astype(np.float32) for _ in range(8)] for s in range(4)}
    seqs = [rng.randint(2, 149, rng.randint(20, 60)) for _ in range(n_seq)]
    ids = [k % 4 for k in range(n_seq)]
    times = {}

    @contextlib.contextmanager
    def timer(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    verify_cloned_voices(model, v, ids, enroll, seqs, stage_timer=timer)          # warm-up
    times.clear()
    res = verify_cloned_voices(model, v, ids, enroll, seqs, stage_timer=timer)
    return {"n_seq": n_seq, "max_decoder_steps": max_steps, "enrolled": 4,
            "ms": {k: round(t * 1e3, 2) for k, t in times.items()}, "eer": round(res["eer"], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maths", default="tc,tc1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speaker_verifier.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {"preset": PRESET, "card": card(), "B": B, "N": N, "T_crop": T_CROP, "runs": []}
    for m in args.maths.split(","):
        ops.conv_math = m
        batches = _batches()
        torch.manual_seed(1)
        v_a = SpeakerVerifier().cuda()
        torch.manual_seed(1)
        v_b = SpeakerVerifier().cuda()
        arms = {"a_graph": SpeakerVerifierStep(v_a).step, "b_eager_torch": EagerVerifierStep(v_b).step}
        for step in arms.values():
            time_steps(step, batches, args.warmup)
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, step in arms.items():
                ms[k].append(time_steps(step, batches, args.steps))
        run = {"math": m, "ms_per_step": {k: {"median": round(float(np.median(t)), 3), "min": round(min(t), 3),
                                              "max": round(max(t), 3)} for k, t in ms.items()},
               "launches_per_step": arms["a_graph"].__self__.launches_per_step,
               "kernels": kernels(v_a), "scoring": scoring_throughput(v_a)}
        run["speedup_a_vs_b"] = round(run["ms_per_step"]["b_eager_torch"]["median"] /
                                      run["ms_per_step"]["a_graph"]["median"], 2)
        res["runs"].append(run)
        del arms
        torch.cuda.empty_cache()
    ops.conv_math = args.maths.split(",")[0]
    torch.manual_seed(1)
    res["verify_cloned_voices"] = evaluation_stages(SpeakerVerifier().cuda())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
