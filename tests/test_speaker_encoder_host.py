"""No GPU: the speaker encoder's fp64 restatement (tests/speaker_encoder_oracle.py) -- its hand-written pool and attention
+ L1 backward against torch autograd (gradcheck) --, the C ABI and ptxas report of csrc/spk_enc.cu, the training-batch
sampler, and the refusals of the encoder, its step and the cloning API before any library call."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import speaker_encoder_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _params(C, S, gen):
    p = {"w_q": torch.randn(C, C, generator=gen) / C ** 0.5, "w_k": torch.randn(C, C, generator=gen) / C ** 0.5,
         "w_v": torch.randn(C, C, generator=gen) / C ** 0.5, "b_q": torch.randn(C, generator=gen) * 0.1,
         "b_k": torch.randn(C, generator=gen) * 0.1, "b_v": torch.randn(C, generator=gen) * 0.1,
         "w_s": torch.randn(C, generator=gen) / C ** 0.5, "b_s": torch.randn(1, generator=gen) * 0.1,
         "w_e": torch.randn(S, C, generator=gen) / C ** 0.5, "b_e": torch.randn(S, generator=gen) * 0.1}
    return {k: v.double() for k, v in p.items()}


def test_pool_backward_gradcheck():
    gen = torch.Generator().manual_seed(0)
    lengths = torch.tensor([5, 1, 7, 3])

    class Pool(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x):
            ctx.T = x.shape[2]
            return SO.pool_fwd(x, lengths)

        @staticmethod
        def backward(ctx, dy):
            return SO.pool_bwd(dy, lengths, ctx.T)

    x = torch.randn(4, 3, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(Pool.apply, (x,))
    want = torch.stack([x[r, :, :int(lengths[r])].mean(-1) for r in range(4)])
    torch.testing.assert_close(SO.pool_fwd(x, lengths), want, rtol=1e-14, atol=1e-14)


@pytest.mark.parametrize("counts,heads", [([3, 5, 1], 2), ([5, 5, 2], 4)])
def test_attention_l1_backward_gradcheck(counts, heads):
    """The hand-derived backward (what the kernel computes) equals torch autograd of the fp64 forward."""
    gen = torch.Generator().manual_seed(1)
    B, N, C, S = 3, 5, 8, 3
    p = _params(C, S, gen)
    names = list(p)
    h = torch.randn(B, N, C, generator=gen, dtype=torch.float64)
    target = torch.randn(B, S, generator=gen, dtype=torch.float64)
    d_out_ext = torch.randn(B, S, generator=gen, dtype=torch.float64)

    class Attn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, h, *vals):
            pp = dict(zip(names, vals))
            out, loss, saved = SO.attn_fwd(h, counts, pp, heads, target)
            ctx.keep = (h, pp, saved)
            return out, loss

        @staticmethod
        def backward(ctx, d_out, d_loss):
            h, pp, saved = ctx.keep
            d_h, g = SO.attn_bwd(h, counts, pp, heads, saved, target, d_out, d_loss)
            return (d_h,) + tuple(g[k] for k in names)

    def f(h, *vals):
        out, loss = Attn.apply(h, *vals)
        return loss + (out * d_out_ext).sum()

    leaves = [h.clone().requires_grad_(True)] + [v.clone().requires_grad_(True) for v in p.values()]
    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-5)
    d_h, _ = SO.attn_bwd(h, counts, p, heads, SO.attn_fwd(h, counts, p, heads, target)[2], target,
                         d_out_ext, torch.tensor(1.0, dtype=torch.float64))
    for b, n in enumerate(counts):
        assert torch.all(d_h[b, n:] == 0)


def test_c_abi_declares_the_encoder_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {name: [a for _, a in d[name][1]] for name in d if name.startswith("dv3_spkenc_")}
    assert args["dv3_spkenc_pool_fwd"] == ["x", "lengths", "y", "err_flag", "R", "C", "T", "stream"]
    assert args["dv3_spkenc_pool_bwd"] == ["dy", "lengths", "dx", "err_flag", "R", "C", "T", "stream"]
    assert args["dv3_spkenc_attn_fwd"][:2] == ["h", "counts"]
    assert args["dv3_spkenc_attn_fwd"][12:] == ["target", "out", "ws", "loss_partials", "err_flag", "B", "N", "C",
                                                "S", "heads", "stream"]
    assert args["dv3_spkenc_attn_bwd"][12:] == ["target", "d_out", "d_loss", "loss_scale", "ws", "d_h", "partials",
                                                "err_flag", "B", "N", "C", "S", "heads", "stream"]
    assert args["dv3_spkenc_reduce"] == ["partials", "P", "loss_partials", "loss_scale", "grad", "loss", "B", "stream"]
    assert args["dv3_spkenc_param_floats"] == ["C", "S"]
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in args:
            assert re.search(r"\bT %s\b" % name, nm), name


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "spk_enc.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 5, rep
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


# ---- SpeakerSampleBatches -------------------------------------------------------------------------------------------
def _corpus(tmp_path, frames_by_speaker, M=4):
    rows = []
    for spk, frames in frames_by_speaker.items():
        for j, T in enumerate(frames):
            name = "mel-%d-%d.npy" % (spk, j)
            np.save(tmp_path / name, np.full((T, M), spk * 100 + j, dtype=np.float32) +
                    np.arange(T, dtype=np.float32)[:, None] / 1000)
            rows.append("lin-%d-%d.npy|%s|%d|text|%d" % (spk, j, name, T, spk))
    (tmp_path / "train.txt").write_text("\n".join(rows) + "\n")
    from deepvoice3_pytorch_b200.data import TrainTxtDataset
    return TrainTxtDataset(str(tmp_path), lambda s: [1, 2])


def test_sample_batches_deterministic_eligible_distinct_in_bounds(tmp_path):
    from deepvoice3_pytorch_b200.data import SpeakerSampleBatches
    ds = _corpus(tmp_path, {0: [20, 30, 12, 25], 1: [40, 9, 16], 2: [15, 15, 15, 15], 3: [50, 5, 5], 4: [18, 17, 16]})
    sb = SpeakerSampleBatches(ds, B=2, N=3, T_crop=15, seed=7)
    assert sb.speakers == [0, 2, 4]                  # 1 and 3 have fewer than 3 utterances of >= 15 frames
    assert len(sb) == 1
    a, b = list(sb), list(SpeakerSampleBatches(ds, 2, 3, 15, seed=7))
    assert all(torch.equal(x[k], y[k]) for x, y in zip(a, b) for k in x)
    seen = set()
    for epoch in range(6):
        sb.set_epoch(epoch)
        for batch in sb:
            ids = batch["speaker_ids"].tolist()
            assert batch["mels"].shape == (2, 3, 15, 4) and len(set(ids)) == 2
            for bi, spk in enumerate(ids):
                items = batch["items"][bi].tolist()
                assert len(set(items)) == 3
                for j, i in enumerate(items):
                    assert int(ds.rows[i][4]) == spk and ds.frame_lengths[i] >= 15
                    o = int(batch["offsets"][bi, j])
                    assert 0 <= o <= ds.frame_lengths[i] - 15
                    full = np.load(os.path.join(str(tmp_path), ds.rows[i][1]))
                    assert np.array_equal(batch["mels"][bi, j].numpy(), full[o:o + 15])
                seen.add(spk)
    assert seen == {0, 2, 4}
    sb.set_epoch(0)
    other = list(SpeakerSampleBatches(ds, 2, 3, 15, seed=8))
    assert any(not torch.equal(x["offsets"], y["offsets"]) for x, y in zip(a, other)) or \
        any(not torch.equal(x["speaker_ids"], y["speaker_ids"]) for x, y in zip(a, other))


def test_sample_batches_refuse_too_few_speakers(tmp_path):
    from deepvoice3_pytorch_b200.data import SpeakerSampleBatches
    ds = _corpus(tmp_path, {0: [20, 30], 1: [40, 41], 2: [10, 50]})
    with pytest.raises(ValueError):
        SpeakerSampleBatches(ds, B=3, N=2, T_crop=15, seed=0)
    assert len(SpeakerSampleBatches(ds, B=2, N=2, T_crop=15, seed=0)) == 1


# ---- refusals before any library call ---------------------------------------------------------------------------------
@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


def _ms_model(S=16, n_speakers=4):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    return builder.deepvoice3_multispeaker(n_vocab=40, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4,
                                           kernel_size=3, encoder_channels=16, decoder_channels=16,
                                           converter_channels=16, max_positions=64, n_speakers=n_speakers,
                                           speaker_embed_dim=S, speaker_embedding_weight_std=0.2)


@pytest.mark.parametrize("kw", [dict(channels=512), dict(max_samples=33), dict(heads=3), dict(kernel_size=4),
                                dict(speaker_embed_dim=65), dict(heads=16, channels=256)])
def test_encoder_refuses_unsupported_shapes(kw):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder
    with pytest.raises(ValueError):
        SpeakerEncoder(**kw)


def test_embed_batch_and_clone_refusals(no_lib):
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoder, clone_voices
    enc = SpeakerEncoder(mel_dim=8, speaker_embed_dim=16, channels=16, max_samples=3)
    ok = np.zeros((5, 8), np.float32)
    for bad in ([], [[]], [[ok] * 4], [[np.zeros((5, 7), np.float32)]], [[np.zeros((0, 8), np.float32)]],
                [[np.zeros(8, np.float32)]], "x"):
        with pytest.raises(ValueError):
            enc.embed_batch(bad)
    model = _ms_model()
    before = model.embed_speakers.weight.detach().clone()
    with pytest.raises(ValueError):
        clone_voices(model, SpeakerEncoder(mel_dim=8, speaker_embed_dim=8, channels=16), [[ok]])
    with pytest.raises(ValueError):
        clone_voices(model, enc, [[ok] * 4])
    from deepvoice3_pytorch_b200 import builder
    single = builder.deepvoice3(n_vocab=40, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4,
                                kernel_size=3, encoder_channels=16, decoder_channels=16, converter_channels=16,
                                max_positions=64)
    with pytest.raises(ValueError):
        clone_voices(single, enc, [[ok]])
    assert model.n_speakers == 4 and torch.equal(model.embed_speakers.weight.detach(), before)
    assert no_lib == []


def test_encoder_step_refusals(no_lib, monkeypatch):
    from deepvoice3_pytorch_b200 import speaker_encoder as SE
    from deepvoice3_pytorch_b200 import builder
    enc = SE.SpeakerEncoder(mel_dim=8, speaker_embed_dim=16, channels=16)
    with pytest.raises(ValueError):
        SE.SpeakerEncoderStep(enc, _ms_model(S=8))
    single = builder.deepvoice3(n_vocab=40, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4,
                                kernel_size=3, encoder_channels=16, decoder_channels=16, converter_channels=16,
                                max_positions=64)
    with pytest.raises(ValueError):
        SE.SpeakerEncoderStep(enc, single)
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda: 2)
    with pytest.raises(ValueError):
        SE.SpeakerEncoderStep(enc, _ms_model())
    assert no_lib == []


def test_encoder_step_refuses_bad_batches(no_lib):
    from deepvoice3_pytorch_b200 import speaker_encoder as SE
    enc = SE.SpeakerEncoder(mel_dim=8, speaker_embed_dim=16, channels=16, max_samples=4)
    step = SE.SpeakerEncoderStep(enc, _ms_model(), use_graph=False)
    ids = torch.zeros(2, dtype=torch.int64)
    for mels, i in ((torch.zeros(2, 5, 10, 8), ids), (torch.zeros(2, 3, 10, 7), ids), (torch.zeros(2, 3, 10), ids),
                    (torch.zeros(2, 3, 10, 8), torch.zeros(3, dtype=torch.int64)),
                    (torch.zeros(2, 3, 10, 8).double(), ids)):
        with pytest.raises(ValueError):
            step.step({"mels": mels, "speaker_ids": i})
    assert no_lib == []
