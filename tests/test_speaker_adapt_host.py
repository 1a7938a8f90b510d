"""No GPU: growing the speaker table (MultiSpeakerTTSModel.add_speakers), the collapsed speaker-site gradient
restated in fp64 against torch autograd of the uncollapsed chain, the adaptation step's argument checks, the C ABI of
csrc/spk_adapt.cu and its ptxas report."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import dropout_mask as DM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(n_vocab=40, embed_dim=16, mel_dim=8, linear_dim=9, r=1, downsample_step=4, kernel_size=3,
          encoder_channels=16, decoder_channels=16, converter_channels=16, max_positions=64, n_speakers=5,
          speaker_embed_dim=8, speaker_embedding_weight_std=0.2)


def _model(**over):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    return builder.deepvoice3_multispeaker(**dict(KW, **over))


def test_add_speakers_mean_keeps_rows_and_loads_strictly():
    m = _model()
    old = m.embed_speakers.weight.detach().clone()
    keys = list(m.state_dict())
    ids = m.add_speakers(2)
    assert ids == [5, 6] and m.n_speakers == 7
    w = m.embed_speakers.weight.detach()
    assert torch.equal(w[:5], old)
    mean = old.double().mean(0).float()
    assert torch.equal(w[5], mean) and torch.equal(w[6], mean)
    assert list(m.state_dict()) == keys
    ref = _model(n_speakers=7)
    ref.load_state_dict(m.state_dict(), strict=True)
    assert torch.equal(ref.embed_speakers.weight.detach(), w)


def test_add_speakers_normal_and_tensor_init():
    m = _model()
    torch.manual_seed(9)
    m.add_speakers(3, init="normal")
    torch.manual_seed(9)
    want = torch.empty(3, 8).normal_(0, 0.2)
    assert torch.equal(m.embed_speakers.weight.detach()[5:], want)
    rows = torch.randn(1, 8)
    assert m.add_speakers(1, init=rows) == [8]
    assert torch.equal(m.embed_speakers.weight.detach()[8:], rows)


@pytest.mark.parametrize("n,init", [(0, "mean"), (-1, "mean"), (1.5, "mean"), (True, "mean"), (1, "zeros"),
                                    (2, torch.zeros(1, 8)), (1, torch.zeros(1, 7)), (1, torch.zeros(1, 8).double())])
def test_add_speakers_refusals_change_nothing(n, init):
    m = _model()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(ValueError):
        m.add_speakers(n, init=init)
    assert m.n_speakers == 5
    after = m.state_dict()
    assert all(torch.equal(after[k], v) for k, v in before.items())


def test_add_speakers_refuses_single_speaker_models():
    from deepvoice3_pytorch_b200 import builder
    kw = {k: v for k, v in KW.items() if k not in ("n_speakers", "speaker_embedding_weight_std")}
    for fn in (builder.deepvoice3, builder.nyanko):
        m = fn(**{k: v for k, v in kw.items() if k != "speaker_embed_dim"})
        with pytest.raises(ValueError):
            m.add_speakers(1)


def test_adapt_speaker_id_checks():
    from deepvoice3_pytorch_b200.speaker_adapt import check_adapt_speakers
    m = _model()
    assert check_adapt_speakers(m, [3, 4]) == [3, 4]
    assert check_adapt_speakers(m, 4) == [4]
    for bad in ([], [2, 2], [5], [-1], [4, 3], [1, 3]):
        with pytest.raises(ValueError):
            check_adapt_speakers(m, bad)
    from deepvoice3_pytorch_b200 import builder
    single = builder.deepvoice3(**{k: v for k, v in KW.items() if k not in ("n_speakers", "speaker_embed_dim",
                                                                             "speaker_embedding_weight_std")})
    with pytest.raises(ValueError):
        check_adapt_speakers(single, [0])


@pytest.mark.parametrize("p", [0.0, 0.25])
def test_collapsed_gradient_equals_autograd_of_the_chain(p):
    """sum_t m/(1-p) sum_c W G (1-|y|)^2 == d/de of sum(G * softsign(Linear(dropout(expand(e))))) in fp64."""
    gen = torch.Generator().manual_seed(1)
    B, T, Sd, C = 3, 29, 8, 12
    e = torch.randn(B, Sd, generator=gen, dtype=torch.float64, requires_grad=True)
    W = torch.randn(C, Sd, generator=gen, dtype=torch.float64)
    bias = torch.randn(C, generator=gen, dtype=torch.float64)
    G = torch.randn(B, C, T, generator=gen, dtype=torch.float64)
    mask = torch.as_tensor(DM.mask(0xABCDEF12345, 3, p, (B, T, Sd)), dtype=torch.float64)
    et = e[:, None, :].expand(B, T, Sd) * mask
    z = torch.einsum("bts,cs->bct", et, W) + bias[None, :, None]
    (G * torch.nn.functional.softsign(z)).sum().backward()
    y = torch.nn.functional.softsign(z).detach()
    H = G * (1 - y.abs()) ** 2
    collapsed = (mask * torch.einsum("bct,cs->bts", H, W)).sum(1)
    np.testing.assert_allclose(collapsed.numpy(), e.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_c_abi_declares_the_site_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    for name in ("dv3_spk_grad_planes", "dv3_spk_grad_bct", "dv3_spk_grad_btc", "dv3_spk_grad_reduce",
                 "dv3_spk_grad_splits", "dv3_spk_rows_grad"):
        assert name in d, name
    assert [a for _, a in d["dv3_spk_grad_planes"][1]][:4] == ["g_planes", "npl", "plane_stride", "ldg"]
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in ("dv3_spk_grad_planes", "dv3_spk_grad_bct", "dv3_spk_grad_btc", "dv3_spk_rows_grad"):
            assert re.search(r"\bT %s\b" % name, nm), name


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "spk_adapt.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 4, rep
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)
