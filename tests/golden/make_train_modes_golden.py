#!/usr/bin/env python
"""Golden vectors for the seq2seq-only and postnet-only losses of the reference's ``train()`` (train.py:655-776),
produced by EXECUTING that file (unchanged, through oracle/ref_harness.py) -- the partial-mode counterpart of
make_train_golden.py's ``step*`` cases, which stay as they are.

    python tests/golden/make_train_modes_golden.py    (build container: needs /root/reference)

Writes tests/golden/train_modes.npz.  ``train(..., train_seq2seq, train_postnet)`` runs one step on a stand-in model
whose ``seq2seq`` / ``postnet`` return fixed leaf tensors, so every scalar train() logs ("loss", "mel loss",
"mel_l1_loss", "mel_binary_div_loss", "done_loss", "linear_loss", "linear_l1_loss", "linear_binary_div_loss",
"attn_loss"; stored with spaces as "_") and d(loss)/d(outputs) are the reference's own (clip_thresh = 0, lr = 0).
Cases: ``s2s*`` seq2seq-only, ``post*`` postnet-only, ``joint*`` both (for the per-term slots of the joint step).
"""
import os
import sys
import warnings

import numpy as np
import torch
from torch import nn

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_harness as H  # noqa: E402
import golden_util as G  # noqa: E402

OUT = {}


def put(case, group, name, value):
    OUT["%s|%s|%s" % (case, group, name)] = value.detach().cpu().numpy() if torch.is_tensor(value) else np.asarray(value)


class _Leaves(nn.Module):
    def __init__(self, **leaves):
        super().__init__()
        for k, v in leaves.items():
            setattr(self, k, nn.Parameter(v))


class FixedSeq2Seq(_Leaves):
    """model.seq2seq stand-in: (mel (B, T_dec, mel_dim*r), attn, done, decoder states) of stored leaves."""

    def forward(self, x, mel, text_positions=None, frame_positions=None, input_lengths=None):
        return self.mel, self.attn, self.done, None


class FixedPostnet(_Leaves):
    def forward(self, mel, speaker_embed=None):
        return self.lin


class FixedModel(nn.Module):
    """Stand-in for the whole model: model(...), model.seq2seq(...) and model.postnet(...) all return stored leaves,
    so d(loss)/d(outputs) lands in their .grad."""

    def __init__(self, mel, lin, attn, done, linear_dim):
        super().__init__()
        self.seq2seq = FixedSeq2Seq(mel=mel, attn=attn, done=done)
        self.postnet = FixedPostnet(lin=lin)
        self.linear_dim = linear_dim

    def get_trainable_parameters(self):
        return self.parameters()

    def forward(self, x, mel, speaker_ids=None, text_positions=None, frame_positions=None, input_lengths=None):
        return self.seq2seq.mel, self.postnet.lin, self.seq2seq.attn, self.seq2seq.done


def main():
    tr = H.load_train("reference")
    hp = tr.hparams
    gen = torch.Generator().manual_seed(0)
    cases = (("s2s0", True, False, 0.5, 0.1, 0.0, True), ("s2s1", True, False, 0.0, 0.2, 0.0, False),
             ("post0", False, True, 0.5, 0.1, 0.25, True), ("post1", False, True, 0.0, 0.0, 0.5, True),
             ("joint0", True, True, 0.5, 0.1, 0.25, True))
    for name, s2s, post, w, bw, pw, guided in cases:
        H.apply_preset(tr, "deepvoice3_ljspeech", masked_loss_weight=w, binary_divergence_weight=bw,
                       priority_freq_weight=pw, use_guided_attention=guided, eval_interval=10 ** 9)
        r, ds = hp.outputs_per_step, hp.downsample_step
        utts = H.synthetic_utterances(3, seed=31, min_text=9, max_text=20, min_frames=24, max_frames=45)
        batch = tr.collate_fn(utts)
        x, ilen, mel, y, (tpos, fpos), done, tlen, spk = batch
        B, T_lin, T_dec, Ts = x.size(0), y.size(1), y.size(1) // ds // r, x.size(1)
        outs = (torch.rand(B, T_dec, 80, generator=gen).clamp(1e-3, 1 - 1e-3),
                torch.rand(B, T_lin, 513, generator=gen).clamp(1e-3, 1 - 1e-3),
                torch.softmax(2 * torch.randn(2, B, T_dec, Ts, generator=gen), -1),
                torch.rand(B, T_dec, 1, generator=gen).clamp(1e-3, 1 - 1e-3))
        model = FixedModel(*outs, linear_dim=513)
        writer = H.ScalarLog()
        opt = torch.optim.SGD(model.parameters(), lr=0.0)
        tr.global_step, tr.global_epoch = 0, 0
        tr.train(torch.device("cpu"), model, [batch], opt, writer, init_lr=0.0, checkpoint_dir="/tmp",
                 checkpoint_interval=10 ** 9, nepochs=1, clip_thresh=0, train_seq2seq=s2s, train_postnet=post)
        put(name, "meta", "cfg", np.array([w, bw, pw, float(guided), hp.priority_freq, hp.sample_rate,
                                           hp.guided_attention_sigma, r, ds, float(s2s), float(post)],
                                          dtype=np.float64))
        for k, v in (("x", x), ("input_lengths", ilen), ("mel", mel), ("y", y), ("done", done),
                     ("target_lengths", tlen)):
            put(name, "in", k, v)
        for k, v in zip(("mel_out", "lin_out", "attn", "done_hat"), outs):
            put(name, "in", k, v)
        for tag, vals in writer.scalars.items():
            if tag != "learning rate":
                put(name, "out", tag.replace(" ", "_"), np.float64(vals[0][1]))
        for k, p in (("mel_out", model.seq2seq.mel), ("lin_out", model.postnet.lin), ("attn", model.seq2seq.attn),
                     ("done_hat", model.seq2seq.done)):
            put(name, "out", "grad_" + k, p.grad if p.grad is not None else torch.zeros_like(p))

    G.save("train_modes.npz", OUT)
    print("wrote train_modes.npz: %d arrays" % len(OUT))


if __name__ == "__main__":
    main()
