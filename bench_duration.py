"""Duration-guided synthesis (DESIGN.md section 2.22).  Measures:

  (a) DurationPredictorStep on B = 16, L = 200 tokens, E = C = 256, three GLU blocks, one CUDA graph, for each
      conv_math in --maths, against (b) the same predictor in eager torch (cuDNN convolutions, TF32 off) with
      torch.optim.Adam -- ms/step, arms alternating over --rounds rounds (median, min, max);
  (c) tts_batch and tts_stream on deepvoice3_ljspeech with random weights, free-running against guided (durations
      drawn from 1-4 steps per token), on --utts sentences of 20-80 tokens: utterances/s of the whole call and decoder
      steps/s of its decoder stage (the guided attention step is the ROWS step with its centre read from a table);
  (d) the loss entry points on B = 16, L = 200: µs per call (CUDA events).
Prints one JSON line, with the card's name and power limit.  Writes nothing to the tree.

    python bench_duration.py [--steps 30] [--rounds 3] [--maths tc,tc1] [--utts 32]
"""
import argparse
import collections
import contextlib
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
from bench_speaker_adapt import card                                            # noqa: E402
from bench_speaker_verifier import _time_us                                     # noqa: E402
from deepvoice3_pytorch_b200 import builder, ops, synthesis                     # noqa: E402
from deepvoice3_pytorch_b200 import duration as D                               # noqa: E402
from deepvoice3_pytorch_b200._lib import lib                                    # noqa: E402
from test_gpu_models import preset_kwargs                                       # noqa: E402

B, L, E, C = 16, 200, 256, 256


def _batches(n=3):
    gen = torch.Generator().manual_seed(1)
    out = []
    for _ in range(n):
        tl = torch.randint(L // 2, L + 1, (B,), generator=gen).to(torch.int32)
        out.append({"values": torch.randn(B, L, E, generator=gen), "durations":
                    torch.randint(1, 12, (B, L), generator=gen).to(torch.int32), "token_lengths": tl})
    return out


class EagerStep:
    """(b): the predictor's arithmetic as plain torch autograd over a copy of its parameters."""

    def __init__(self, pred, lr=1e-3):
        self.p = {k: t.detach().clone().requires_grad_(True) for k, t in pred.state_dict().items()}
        self.n = len(pred.blocks)
        self.opt = torch.optim.Adam(list(self.p.values()), lr=lr)

    def _w(self, pre):
        v, g = self.p[pre + "weight_v"], self.p[pre + "weight_g"]
        return g * v / v.pow(2).sum((1, 2), keepdim=True).sqrt()

    def step(self, batch):
        x, d, n = batch["values"], batch["durations"], batch["token_lengths"]
        mask = (torch.arange(L, device=x.device)[None] < n[:, None]).float()
        h = F.relu(F.conv1d(x.transpose(1, 2), self._w("proj.0."), self.p["proj.0.bias"]))
        for i in range(self.n):
            h = h * mask[:, None]
            a, b = F.conv1d(h, self._w("blocks.%d.conv." % i), self.p["blocks.%d.conv.bias" % i], padding=1).chunk(2, 1)
            h = (a * torch.sigmoid(b) + h) * 0.5 ** 0.5
        y = F.conv1d(h, self._w("out.0."), self.p["out.0.bias"]).squeeze(1)
        loss = (((y - torch.log(d.float())) ** 2 * mask).sum(1) / n.float()).mean()
        self.opt.zero_grad(set_to_none=False)
        loss.backward()
        self.opt.step()
        return loss


def _ms(fn, batches, steps):
    for b in batches:
        fn(b)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(steps):
        fn(batches[k % len(batches)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(min(xs)), "max": float(max(xs))}


def bench_step(maths, steps, rounds):
    host = _batches()
    dev = [{k: v.cuda() for k, v in b.items()} for b in host]
    arms = {}
    for m in maths:
        ops.conv_math = m
        torch.manual_seed(0)
        st = D.DurationPredictorStep(D.DurationPredictor(E, channels=C).cuda(), use_graph=True)
        arms[m] = (m, lambda b, st=st: st.step(b))
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    eager = EagerStep(D.DurationPredictor(E, channels=C).cuda())
    arms["eager"] = ("fp32", eager.step)
    times = collections.defaultdict(list)
    for _ in range(rounds):
        for name, (m, fn) in arms.items():
            ops.conv_math = m
            times[name].append(_ms(fn, dev, steps))
    return {k: _stats(v) for k, v in times.items()}


def bench_synthesis(n_utts):
    bname, kw = preset_kwargs("deepvoice3_ljspeech")
    torch.manual_seed(7)
    model = getattr(builder, bname)(dropout=0.0, **kw).cuda().eval()
    rng = np.random.RandomState(3)
    seqs = [rng.randint(2, 149, size=n).astype(np.int64) for n in rng.randint(20, 81, n_utts)]
    durs = [rng.randint(1, 5, s.size).astype(np.int64) for s in seqs]
    ops.conv_math = "tc"
    out = {}
    for api in ("tts_batch", "tts_stream"):
        for mode, kw_ in (("free", {}), ("guided", {"durations": durs})):
            stage_t = collections.defaultdict(float)

            @contextlib.contextmanager
            def stage(name):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                yield
                torch.cuda.synchronize()
                stage_t[name] += time.perf_counter() - t0

            def run(timer=None):
                if api == "tts_batch":
                    return synthesis.tts_batch(model, seqs, batch_size=16, stage_timer=timer, **kw_)
                return [r for _, r in synthesis.tts_stream(model, seqs, slots=16, stage_timer=timer, **kw_)]
            run()                                                            # warm-up: graphs, allocator
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = run()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            run(stage)
            steps = sum(r[1].shape[0] for r in res)
            out["%s_%s" % (api, mode)] = {"utts_per_s": n_utts / wall, "decoder_steps": steps,
                                          "decoder_s": stage_t["decoder"],
                                          "decoder_steps_per_s": steps / stage_t["decoder"]}
    return out


def bench_loss():
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randn(B, L, device="cuda", generator=g)
    d = torch.randint(1, 12, (B, L), device="cuda", generator=g).to(torch.int32)
    n = torch.randint(L // 2, L + 1, (B,), device="cuda", generator=g).to(torch.int32)
    row = torch.empty(B, dtype=torch.float64, device="cuda")
    loss = torch.empty((), device="cuda")
    one = torch.ones((), device="cuda")
    dy = torch.empty(B, L, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = ops._p
    fwd = _time_us(lambda: lib.call("dv3_duration_loss_fwd", p(y), L, p(d), L, p(n), B, L, p(row), p(loss),
                                    p(ops._err_flag(y.device)), st))
    bwd = _time_us(lambda: lib.call("dv3_duration_loss_bwd", p(y), L, p(d), L, p(n), B, L, p(one), p(dy), st))
    return {"fwd_us": fwd, "bwd_us": bwd}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maths", default="tc,tc1")
    ap.add_argument("--utts", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_duration.py needs a CUDA device")
    res = {"card": card(), "step_ms": bench_step(a.maths.split(","), a.steps, a.rounds),
           "synthesis": bench_synthesis(a.utts), "loss": bench_loss()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
