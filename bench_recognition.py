"""Token recognizer training, the CTC kernels, greedy decoding, edit distance and evaluate_recognition (DESIGN.md section
2.21).  Measures:

  (a) TokenRecognizerStep on B = 16, T = 800 frames, L = 200 tokens, V = 149, one CUDA graph, for each conv_math in
      --maths, against (b) the same recognizer in eager torch (cuDNN convolutions, CUDA F.ctc_loss, TF32 off) with
      torch.optim.Adam -- ms/step, arms alternating over --rounds rounds (median, min, max);
  the CTC forward and backward entry points on 512 ragged rows (T 200-900, L 40-250): µs per call (CUDA events), alpha
  cells per second and ns per frame step of the longest row; greedy decoding and edit distance in pairs/s; the fp64
  numpy oracle on a few rows, extrapolated to the 512; the stage times of evaluate_recognition on the
  deepvoice3_ljspeech preset with 64 utterances (random weights, so the error rates mean nothing).  Prints one JSON
  line, with the card's name and power limit.  Writes nothing to the tree.

    python bench_recognition.py [--steps 30] [--rounds 3] [--maths tc,tc1]
"""
import argparse
import contextlib
import ctypes
import json
import math
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
from bench_speaker_adapt import card                                            # noqa: E402
from bench_speaker_verifier import _time_us                                     # noqa: E402
from deepvoice3_pytorch_b200 import ops, recognition as R                       # noqa: E402
from deepvoice3_pytorch_b200._lib import lib                                    # noqa: E402

V, B, T, L = 149, 16, 800, 200


def _batches(n=3):
    gen = torch.Generator().manual_seed(1)
    out = []
    for _ in range(n):
        tl = torch.randint(L // 2, L + 1, (B,), generator=gen)
        out.append({"mels": torch.rand(B, T, 80, generator=gen), "mel_lengths": torch.randint(T // 2, T + 1, (B,),
                                                                                              generator=gen),
                    "tokens": torch.randint(2, V, (B, L), generator=gen), "token_lengths": tl})
    return out


class EagerStep:
    """(b): the recognizer's arithmetic as plain torch autograd over a copy of its parameters."""

    def __init__(self, rec, lr=1e-3):
        self.p = {k: t.detach().clone().requires_grad_(True) for k, t in rec.state_dict().items()}
        self.k = rec.temporal[0].conv.kernel_size[0]
        self.dil = [m.conv.dilation[0] for m in rec.temporal]
        self.opt = torch.optim.Adam(list(self.p.values()), lr=lr)

    def _wn(self, pre):
        v, g = self.p[pre + "weight_v"], self.p[pre + "weight_g"]
        return g * v / v.pow(2).sum((1, 2), keepdim=True).sqrt()

    def step(self, b):
        p = self.p
        self.opt.zero_grad(set_to_none=False)
        x = b["mels"].transpose(1, 2)
        for i in (0, 2):
            x = torch.relu(F.conv1d(x, self._wn("spectral.%d." % i), p["spectral.%d.bias" % i]))
        for i, d in enumerate(self.dil):
            pre = "temporal.%d.conv." % i
            y = F.conv1d(x, self._wn(pre), p[pre + "bias"], padding=(self.k - 1) // 2 * d, dilation=d)
            a, gate = y.chunk(2, dim=1)
            x = (a * torch.sigmoid(gate) + x) * math.sqrt(0.5)
        z = F.conv1d(x, self._wn("out.0."), p["out.0.bias"])
        loss = F.ctc_loss(F.log_softmax(z, 1).permute(2, 0, 1), b["tokens"], b["mel_lengths"], b["token_lengths"],
                          zero_infinity=True)
        loss.backward()
        self.opt.step()
        return loss


def training(maths, steps, rounds):
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {}
    host = _batches()
    for m in maths:
        ops.conv_math = m
        torch.manual_seed(0)
        rec = R.TokenRecognizer(V).cuda()
        st = R.TokenRecognizerStep(rec, use_graph=True)
        eager = EagerStep(rec)
        dev_b = []
        for h in host:
            tok, n = rec.strip_batch(h["tokens"], h["token_lengths"])
            dev_b.append({"mels": h["mels"].cuda(), "mel_lengths": h["mel_lengths"].cuda(),
                          "tokens": torch.from_numpy(tok).long().cuda(), "token_lengths": torch.from_numpy(n).cuda()})
        for i in range(3):
            st.step(host[i % 3])
            eager.step(dev_b[i % 3])
        arms = {"graph": [], "eager": []}
        for _ in range(rounds):
            for name, fn, bs in (("graph", st.step, host), ("eager", eager.step, dev_b)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(steps):
                    fn(bs[i % 3])
                torch.cuda.synchronize()
                arms[name].append((time.perf_counter() - t0) * 1e3 / steps)
        out[m] = {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
                  for k, v in arms.items()}
        out[m]["launches_per_step"] = st.launches_per_step
    ops.conv_math = "tc"
    return out


def ctc_kernels(iters=20):
    rng = np.random.RandomState(0)
    n, Vk = 512, V
    fr = rng.randint(200, 901, n).astype(np.int32)
    tl = np.minimum(rng.randint(40, 251, n), fr // 2).astype(np.int32)
    Tm, Lm = int(fr.max()), int(tl.max())
    tg = rng.randint(2, Vk, (n, Lm)).astype(np.int32)
    z = torch.randn(n, Vk, Tm, device="cuda") * 2
    dev = z.device
    frd, tgd, tld = (torch.from_numpy(a).to(dev) for a in (fr, tg, tl))
    ws = torch.empty(int(lib.raw("dv3_ctc_ws_bytes")(n, Tm, Lm)), dtype=torch.uint8, device=dev)
    nll, part = torch.empty(n, device=dev), torch.empty(n, device=dev)
    inf = torch.empty(n, dtype=torch.int32, device=dev)
    one = torch.ones(1, device=dev)
    dz = torch.empty(n, Vk, Tm, device=dev)
    p, s = ops._p, ops._stream

    def fwd():
        lib.call("dv3_ctc_fwd", p(z), z.stride(0), z.stride(1), p(frd), p(tgd), Lm, p(tld), n, Vk, Tm, Lm, p(ws),
                 p(nll), p(part), p(inf), p(ops._err_flag(dev)), s())

    def bwd():
        lib.call("dv3_ctc_bwd", p(z), z.stride(0), z.stride(1), p(frd), p(tgd), Lm, p(tld), n, Vk, Tm, Lm, p(ws), p(one),
                 1.0 / n, p(dz), s())
    fwd()
    t_f, t_b = _time_us(fwd, iters), _time_us(bwd, iters)
    cells = float(np.sum(fr.astype(np.int64) * (2 * tl + 1)))
    hyps = torch.empty(n, Tm, dtype=torch.int32, device=dev)
    hl = torch.empty(n, dtype=torch.int32, device=dev)
    t_g = _time_us(lambda: lib.call("dv3_ctc_greedy", p(z), z.stride(0), z.stride(1), p(frd), n, Vk, Tm, p(hyps),
                                    p(hl), p(ops._err_flag(dev)), s()), iters)
    hy = R.greedy_decode(z, fr)
    refs = [tg[b, :tl[b]] for b in range(n)]
    R.edit_distance(hy, refs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    R.edit_distance(hy, refs)
    t_e = (time.perf_counter() - t0) * 1e6
    import ctc_oracle as CO
    zc = z[:2].cpu().numpy()
    t0 = time.perf_counter()
    for b in range(2):
        CO.ctc(zc[b, :, :fr[b]], tg[b, :tl[b]])
    t_o = (time.perf_counter() - t0) / 2 * n
    ops.check_index_errors()
    return {"rows": n, "T_max": Tm, "L_max": Lm, "alpha_cells": cells, "fwd_us": t_f, "bwd_us": t_b,
            "fwd_cells_per_s": cells / (t_f * 1e-6), "bwd_cells_per_s": cells / (t_b * 1e-6),
            "fwd_ns_per_frame_step": t_f * 1e3 / Tm, "bwd_ns_per_frame_step": t_b * 1e3 / Tm,
            "greedy_us": t_g, "greedy_pairs_per_s": n / (t_g * 1e-6),
            "edit_distance_call_us": t_e, "edit_pairs_per_s": n / (t_e * 1e-6),
            "edit_mean_hyp_tokens": float(np.mean([h.size for h in hy])),
            "oracle_fp64_numpy_s_extrapolated": t_o}


def evaluation(n_utt=64):
    from deepvoice3_pytorch_b200 import builder
    from test_gpu_synthesis import preset_kwargs
    bname, kw = preset_kwargs("deepvoice3_ljspeech")
    torch.manual_seed(7)
    model = getattr(builder, bname)(dropout=0.0, **kw).cuda().eval()
    rng = np.random.RandomState(3)
    seqs = [rng.randint(2, 149, rng.randint(20, 120)).astype(np.int64) for _ in range(n_utt)]
    torch.manual_seed(0)
    rec = R.TokenRecognizer(149).cuda()
    times = {}

    @contextlib.contextmanager
    def stage(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        times[name] = times.get(name, 0.0) + time.perf_counter() - t0
    res = R.evaluate_recognition(model, rec, seqs, stage_timer=stage)
    return {"utterances": n_utt, "stage_s": times, "corpus_ter_random_weights": res["corpus_ter"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maths", default="tc,tc1")
    a = ap.parse_args()
    out = {"card": card(), "training": training(a.maths.split(","), a.steps, a.rounds), "ctc": ctc_kernels(),
           "evaluate_recognition": evaluation()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
