"""No GPU: the speaker classifier's fp64 restatement (tests/speaker_classifier_oracle.py) -- its hand-written head
backward against torch autograd (gradcheck) and its loss against torch's cross-entropy --, the C ABI and ptxas report of
csrc/spk_cls.cu, top-k accuracy against a brute-force ranking, and the refusals of the classifier, its step and the
evaluation API before any library call."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import speaker_classifier_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("R,C,K,with_labels,with_ext", [(5, 4, 3, True, True), (7, 3, 2, True, False),
                                                         (4, 5, 6, False, True)])
def test_head_backward_gradcheck(R, C, K, with_labels, with_ext):
    """The hand-derived backward (what the kernels compute) equals torch autograd of the fp64 forward."""
    gen = torch.Generator().manual_seed(R * 100 + K)
    labels = torch.randint(0, K, (R,), generator=gen) if with_labels else None
    d_ext = torch.randn(R, K, generator=gen, dtype=torch.float64) if with_ext else None

    class Head(torch.autograd.Function):
        @staticmethod
        def forward(ctx, h, w, c):
            z, lse, loss = CO.head_fwd(h, w, c, labels)
            ctx.save_for_backward(h, w, z, lse)
            return z, (loss if loss is not None else torch.zeros((), dtype=h.dtype))

        @staticmethod
        def backward(ctx, d_z, d_loss):
            h, w, z, lse = ctx.saved_tensors
            return CO.head_bwd(h, w, z, lse, labels, d_z if with_ext else None, d_loss if with_labels else None)

    def f(*a):
        z, loss = Head.apply(*a)
        return loss + ((z * d_ext).sum() if with_ext else 0.0)

    leaves = (torch.randn(R, C, generator=gen, dtype=torch.float64, requires_grad=True),
              torch.randn(K, C, generator=gen, dtype=torch.float64, requires_grad=True),
              torch.randn(K, generator=gen, dtype=torch.float64, requires_grad=True))
    assert torch.autograd.gradcheck(f, leaves)


def test_oracle_loss_is_the_mean_cross_entropy_and_a_bad_label_adds_zero():
    gen = torch.Generator().manual_seed(1)
    h, w, c = (torch.randn(6, 4, generator=gen, dtype=torch.float64), torch.randn(5, 4, generator=gen,
                                                                                  dtype=torch.float64),
               torch.randn(5, generator=gen, dtype=torch.float64))
    labels = torch.tensor([0, 4, 2, 2, 1, 3])
    z, lse, loss = CO.head_fwd(h, w, c, labels)
    assert float(loss) == pytest.approx(float(torch.nn.functional.cross_entropy(z, labels)), rel=1e-12)
    assert torch.allclose(lse, torch.logsumexp(z, 1))
    bad = labels.clone()
    bad[1] = 5
    _, _, loss_bad = CO.head_fwd(h, w, c, bad)
    want = (torch.nn.functional.cross_entropy(z, labels, reduction="none") * (torch.arange(6) != 1)).mean()
    assert float(loss_bad) == pytest.approx(float(want), rel=1e-12)
    G = CO.grad_logits(z, lse, bad, None, torch.tensor(1.0, dtype=torch.float64))
    assert torch.allclose(G[1], torch.softmax(z[1], 0) / 6)                 # no onehot on the bad row


# ---- C ABI and ptxas ------------------------------------------------------------------------------------------------
def test_c_abi_declares_the_classifier_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {name: [a for _, a in d[name][1]] for name in d if name.startswith("dv3_spkcls_")}
    assert args["dv3_spkcls_fwd"] == ["h", "ld", "w", "bias", "labels", "logits", "lse", "pred", "loss_partials",
                                      "err_flag", "R", "C", "K", "stream"]
    assert args["dv3_spkcls_bwd"] == ["h", "ld", "w", "logits", "lse", "labels", "d_logits", "d_loss", "loss_scale",
                                      "d_h", "d_w", "d_bias", "err_flag", "R", "C", "K", "stream"]
    import ctypes
    types = {name: [t for t, _ in d[name][1]] for name in args}
    P, LL, I, F = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float
    assert types["dv3_spkcls_fwd"] == [P, LL, P, P, P, P, P, P, P, P, I, I, I, P]
    assert types["dv3_spkcls_bwd"] == [P, LL, P, P, P, P, P, P, F, P, P, P, P, I, I, I, P]
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
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "spk_cls.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 4, rep
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


# ---- top-k accuracy -------------------------------------------------------------------------------------------------
def _rank_brute(row, t):
    """Position of class t when the classes are sorted by decreasing logit, ties by increasing index."""
    order = sorted(range(len(row)), key=lambda k: (-row[k], k))
    return order.index(t)


@pytest.mark.parametrize("seed", range(6))
def test_top_k_accuracy_matches_a_brute_force_ranking(seed):
    from deepvoice3_pytorch_b200.speaker_classifier import top_k_accuracy
    rng = np.random.RandomState(seed)
    n, K = rng.randint(5, 40), rng.randint(2, 12)
    z = rng.randn(n, K).astype(np.float32)
    if seed % 2:
        z = np.round(z * 2) / 2                          # ties, also at the target's logit
    t = rng.randint(0, K, n)
    ks = (1, 2, 3, 5, K)
    got = top_k_accuracy(torch.from_numpy(z), torch.from_numpy(t), ks)
    ranks = [_rank_brute(list(map(float, z[i])), int(t[i])) for i in range(n)]
    for k in ks:
        assert got[k] == pytest.approx(np.mean([r < k for r in ranks]), abs=1e-15), k
    assert got[K] == 1.0
    # rank 0 is the first class of largest logit, the kernels' prediction
    pred = np.array([min(range(K), key=lambda k: (-z[i, k], k)) for i in range(n)])
    assert top_k_accuracy(z, pred, (1,))[1] == 1.0


def test_top_k_accuracy_ties_and_refusals():
    from deepvoice3_pytorch_b200.speaker_classifier import top_k_accuracy
    z = np.array([[1.0, 1.0, 0.0], [0.0, 2.0, 2.0], [3.0, 3.0, 3.0]])
    assert top_k_accuracy(z, [0, 2, 2], (1, 2, 3)) == {1: pytest.approx(1 / 3), 2: pytest.approx(2 / 3), 3: 1.0}
    for lg, t, ks in ((np.zeros(3), [0], (1,)), (np.zeros((2, 3)), [0], (1,)), (np.zeros((2, 3)), [0, 3], (1,)),
                      (np.zeros((2, 3)), [0, -1], (1,)), (np.zeros((2, 3)), [0.0, 1.0], (1,)),
                      (np.array([[0.0, np.nan]]), [0], (1,)), (np.zeros((2, 3)), [0, 1], (0,)),
                      (np.zeros((0, 3)), np.zeros(0, int), (1,))):
        with pytest.raises(ValueError):
            top_k_accuracy(lg, np.array(t), ks)


# ---- refusals before any library call ---------------------------------------------------------------------------------
@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


@pytest.mark.parametrize("kw", [dict(n_classes=1), dict(n_classes=8193), dict(n_classes=4, channels=257),
                                dict(n_classes=4, channels=0), dict(n_classes=4, kernel_size=4),
                                dict(n_classes=4, n_conv=-1)])
def test_classifier_refuses_unsupported_shapes(kw):
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifier
    with pytest.raises(ValueError):
        SpeakerClassifier(**kw)


def test_head_refusals(no_lib):
    from deepvoice3_pytorch_b200 import speaker_classifier as SC
    for R, C, K in ((4, 257, 10), (4, 0, 10), (4, 128, 1), (4, 128, 8193), (2 ** 20, 128, 2048), (0, 128, 4)):
        with pytest.raises(ValueError):
            SC.check_head(R, C, K)
    SC.check_head(2 ** 20, 256, 2047)
    meta = dict(device="meta")
    for h, w in ((torch.empty(4, 257, **meta), torch.empty(10, 257, **meta)),
                 (torch.empty(4, 128, **meta), torch.empty(1, 128, **meta)),
                 (torch.empty(4, 128, **meta), torch.empty(8193, 128, **meta)),
                 (torch.empty(2 ** 20, 128, **meta), torch.empty(2048, 128, **meta)),
                 (torch.empty(4, 128, **meta), torch.empty(10, 64, **meta)),
                 (torch.empty(128, 4, **meta).T, torch.empty(10, 128, **meta))):
        with pytest.raises(ValueError):
            SC.logits_forward(h, w, torch.empty(w.shape[0], **meta))
        with pytest.raises(ValueError):
            SC.logits_backward(h, w, torch.empty(h.shape[0], w.shape[0], **meta), torch.empty(h.shape[0], **meta))
    assert no_lib == []


def test_forward_and_classify_refusals(no_lib):
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifier
    cl = SpeakerClassifier(5, mel_dim=8, channels=16)
    for bad in ([], [np.zeros((5, 7), np.float32)], [np.zeros(8, np.float32)], [np.zeros((0, 8), np.float32)], "x"):
        with pytest.raises(ValueError):
            cl.classify(bad)
    for ids in (torch.tensor([1, 2, 3]), torch.tensor([1, 2], dtype=torch.int32), torch.tensor([[1, 2]])):
        with pytest.raises(ValueError):
            cl(torch.zeros(2, 3, 10, 8), ids)
    big = SpeakerClassifier(8192, mel_dim=8, channels=16)
    with pytest.raises(ValueError):                       # R*K = 2^18 * 2^13 rows x classes
        big(torch.zeros(2 ** 12, 64, 1, 8, device="meta"), torch.zeros(2 ** 12, dtype=torch.int64))
    assert no_lib == []


def test_step_refusals(no_lib, monkeypatch):
    from deepvoice3_pytorch_b200 import speaker_encoder as SE
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifier, SpeakerClassifierStep
    cl = SpeakerClassifier(5, mel_dim=8, channels=16)
    step = SpeakerClassifierStep(cl, use_graph=False)
    ids = torch.tensor([0, 4], dtype=torch.int64)
    for mels, i in ((torch.zeros(2, 3, 10, 7), ids), (torch.zeros(2, 3, 10), ids),
                    (torch.zeros(2, 3, 10, 8), torch.zeros(3, dtype=torch.int64)),
                    (torch.zeros(2, 3, 10, 8).double(), ids), (torch.zeros(2, 3, 10, 8), ids.int()),
                    (torch.zeros(2, 3, 10, 8), torch.tensor([0, 5])), (torch.zeros(2, 3, 10, 8), torch.tensor([-1, 2])),
                    (torch.zeros(2, 0, 10, 8), ids)):
        with pytest.raises(ValueError):
            step.step({"mels": mels, "speaker_ids": i})
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda: 2)
    with pytest.raises(ValueError):
        SpeakerClassifierStep(cl)
    assert no_lib == []


def _ms_model(n_speakers=4):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    return builder.deepvoice3_multispeaker(n_vocab=40, embed_dim=16, mel_dim=80, linear_dim=9, r=1, downsample_step=4,
                                           kernel_size=3, encoder_channels=16, decoder_channels=16,
                                           converter_channels=16, max_positions=64, n_speakers=n_speakers,
                                           speaker_embed_dim=16, speaker_embedding_weight_std=0.2)


def test_classify_cloned_voices_refusals(no_lib):
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifier, classify_cloned_voices
    cl = SpeakerClassifier(3, channels=16)
    model = _ms_model().eval()
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    single = builder.deepvoice3(n_vocab=40, embed_dim=16, mel_dim=80, linear_dim=9, r=1, downsample_step=4,
                                kernel_size=3, encoder_channels=16, decoder_channels=16, converter_channels=16,
                                max_positions=64).eval()
    bad_calls = [
        (single, cl, [0, 2], seqs, None, {}),                                # single-speaker model
        (model, cl, [0, 4], seqs, [0, 1], {}),                               # id out of the model's range
        (model, cl, [0, -1], seqs, [0, 1], {}),
        (model, cl, [0, 3], seqs, None, {}),                                 # default target 3 outside [0, 3)
        (model, cl, [0, 1], seqs, [0, 3], {}),                               # explicit target outside [0, 3)
        (model, cl, [0, 1], seqs, [0, -1], {}),
        (model, cl, [0], seqs, None, {}),                                    # mismatched lengths
        (model, cl, [0, 1], seqs, [0], {}),
        (model, cl, [0, 1], [np.array([3, 4])], [0], {}),
        (model, SpeakerClassifier(3, mel_dim=40, channels=16), [0, 1], seqs, None, {}),
        (model, cl, [0, 1], seqs, None, {"vocoder": "wavenet"}),
        (model, cl, [0, 1], [np.array([3, 4]), np.array([], np.int64)], None, {}),
    ]
    for m, c, ids, sq, tg, kw in bad_calls:
        with pytest.raises(ValueError):
            classify_cloned_voices(m, c, ids, sq, targets=tg, **kw)
    assert no_lib == []
