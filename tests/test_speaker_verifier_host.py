"""No GPU: the speaker verifier's fp64 restatement (tests/speaker_verifier_oracle.py) -- its hand-written embed, score
and balanced-BCE backward against torch autograd (gradcheck) --, the C ABI and ptxas report of csrc/spk_ver.cu, the
equal error rate against a brute-force sweep, and the refusals of the verifier, its step and the evaluation API before
any library call."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import speaker_verifier_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_embed_backward_gradcheck():
    gen = torch.Generator().manual_seed(0)
    B, N, C, D = 4, 5, 6, 3
    counts = [5, 1, 3, 2]

    class Embed(torch.autograd.Function):
        @staticmethod
        def forward(ctx, h, w, c):
            out, hbar = VO.embed_fwd(h, counts, w, c)
            ctx.save_for_backward(hbar, w)
            return out

        @staticmethod
        def backward(ctx, d_out):
            hbar, w = ctx.saved_tensors
            return VO.embed_bwd(d_out, hbar, counts, w, N)

    leaves = (torch.randn(B, N, C, generator=gen, dtype=torch.float64, requires_grad=True),
              torch.randn(D, C, generator=gen, dtype=torch.float64, requires_grad=True),
              torch.randn(D, generator=gen, dtype=torch.float64, requires_grad=True))
    assert torch.autograd.gradcheck(Embed.apply, leaves)
    d_h, _, _ = VO.embed_bwd(torch.randn(B, D, dtype=torch.float64), VO.embed_fwd(*leaves[:1], counts, *leaves[1:])[1],
                             counts, leaves[1].detach(), N)
    for b, n in enumerate(counts):
        assert torch.all(d_h[b, n:] == 0)


@pytest.mark.parametrize("ids_e,ids_t", [([0, 1, 2], [0, 1, 2]), ([3, 1, 3, 0], [1, 3]), ([5, 6], [5, 5, 6, 7, 6])])
def test_score_and_balanced_bce_backward_gradcheck(ids_e, ids_t):
    """The hand-derived backward (what the kernels compute) equals torch autograd of the fp64 forward."""
    gen = torch.Generator().manual_seed(len(ids_e) * 10 + len(ids_t))
    D = 4
    d_ext = torch.randn(len(ids_e), len(ids_t), generator=gen, dtype=torch.float64)

    class Score(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, y, S, b):
            L, loss = VO.score_fwd(x, y, S, b, ids_e, ids_t)
            ctx.save_for_backward(x, y, S, L)
            return L, loss

        @staticmethod
        def backward(ctx, d_scores, d_loss):
            x, y, S, L = ctx.saved_tensors
            return VO.score_bwd(x, y, S, L, ids_e, ids_t, d_scores, d_loss)

    def f(*a):
        L, loss = Score.apply(*a)
        return loss + (L * d_ext).sum()

    leaves = (torch.randn(len(ids_e), D, generator=gen, dtype=torch.float64, requires_grad=True),
              torch.randn(len(ids_t), D, generator=gen, dtype=torch.float64, requires_grad=True),
              (0.3 * torch.randn(D, D, generator=gen, dtype=torch.float64)).requires_grad_(True),
              torch.randn(1, generator=gen, dtype=torch.float64, requires_grad=True))
    assert torch.autograd.gradcheck(f, leaves)


def test_oracle_loss_is_the_balanced_bce():
    L = torch.tensor([[2.0, -1.0], [0.5, 3.0]], dtype=torch.float64)
    x, y = torch.zeros(2, 3, dtype=torch.float64), torch.zeros(2, 3, dtype=torch.float64)
    _, loss = VO.score_fwd(x, y, torch.zeros(3, 3, dtype=torch.float64), 0.0, [0, 1], [0, 1])
    assert float(loss) == pytest.approx(np.log(2))              # every score 0: softplus(0) on both sides
    same = torch.tensor([[True, False], [False, True]])
    want = 0.5 * torch.nn.functional.softplus(-L[same]).mean() + 0.5 * torch.nn.functional.softplus(L[~same]).mean()
    assert float(want) == pytest.approx(0.5 * (np.log1p(np.exp(-2)) + np.log1p(np.exp(-3))) / 2 +
                                        0.5 * (np.log1p(np.exp(-1)) + np.log1p(np.exp(0.5))) / 2)


# ---- C ABI and ptxas ------------------------------------------------------------------------------------------------
def test_c_abi_declares_the_verifier_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {name: [a for _, a in d[name][1]] for name in d if name.startswith("dv3_spkver_")}
    assert args["dv3_spkver_embed_fwd"] == ["h", "ld", "counts", "w", "c", "hbar", "out", "err_flag", "B", "N", "C",
                                            "D", "stream"]
    assert args["dv3_spkver_embed_bwd"] == ["d_out", "hbar", "counts", "w", "d_h", "ld", "partials", "err_flag", "B",
                                            "N", "C", "D", "stream"]
    assert args["dv3_spkver_score_fwd"] == ["x", "y", "S", "bias", "ids_e", "ids_t", "qx", "qy", "scores",
                                            "loss_partials", "B_e", "B_t", "D", "stream"]
    assert args["dv3_spkver_score_bwd"] == ["x", "y", "S", "scores", "ids_e", "ids_t", "d_scores", "d_loss", "dx",
                                            "dy", "partials", "B_e", "B_t", "D", "stream"]
    assert args["dv3_spkver_loss_floats"] == ["B_e", "B_t"]
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
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "spk_ver.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    assert len(frames) == 5, rep
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


# ---- equal error rate -----------------------------------------------------------------------------------------------
def _eer_brute(scores, labels):
    """Every distinct threshold (and one above the largest score), FAR / FRR counted trial by trial; the crossing
    interpolated linearly between the last threshold with FRR < FAR and the first with FRR >= FAR."""
    s, y = list(map(float, np.ravel(scores))), list(map(bool, np.ravel(labels)))
    thr = sorted(set(s)) + [np.nextafter(max(s), np.inf)]
    pts = []
    for t in thr:
        fa = sum(1 for v, lab in zip(s, y) if not lab and v >= t) / sum(1 for lab in y if not lab)
        fr = sum(1 for v, lab in zip(s, y) if lab and v < t) / sum(1 for lab in y if lab)
        pts.append((t, fa, fr))
    for (t0, fa0, fr0), (t1, fa1, fr1) in zip(pts, pts[1:]):
        if fr0 < fa0 and fr1 >= fa1:
            a = (fa0 - fr0) / ((fa0 - fr0) - (fa1 - fr1))
            return fa0 + a * (fa1 - fa0), t0 + a * (t1 - t0)
    raise AssertionError("no crossing")


@pytest.mark.parametrize("seed", range(6))
def test_eer_matches_a_brute_force_sweep(seed):
    from deepvoice3_pytorch_b200.speaker_verifier import equal_error_rate
    rng = np.random.RandomState(seed)
    n = rng.randint(10, 80)
    labels = rng.rand(n) < 0.3
    labels[:2] = [True, False]
    scores = rng.randn(n) + 1.5 * labels
    if seed % 2:
        scores = np.round(scores * 2) / 2                # ties, also across the classes
    eer, thr = equal_error_rate(scores, labels)
    want_eer, want_thr = _eer_brute(scores, labels)
    assert eer == pytest.approx(want_eer, abs=1e-12) and thr == pytest.approx(want_thr, abs=1e-12)
    assert 0.0 <= eer <= 1.0


def test_eer_extremes_and_refusals():
    from deepvoice3_pytorch_b200.speaker_verifier import equal_error_rate
    labels = np.array([[1, 0, 0], [0, 1, 0]], dtype=bool)
    eer, thr = equal_error_rate(np.array([[3.0, -1.0, 0.5], [0.0, 2.0, 1.0]]), labels)
    assert eer == 0.0 and 1.0 < thr <= 2.0                           # separated: any threshold in (1, 2] is perfect
    eer, _ = equal_error_rate(np.full((2, 3), 0.7), labels)
    assert eer == pytest.approx(0.5)                                 # identical scores: chance
    eer, _ = equal_error_rate(np.array([[-3.0, 1.0, 0.5], [2.0, -2.0, 1.5]]), labels)
    assert eer == pytest.approx(1.0)                                 # reversed
    for s, lab in ((np.zeros(3), np.ones(3, bool)), (np.zeros(3), np.zeros(3, bool)), (np.zeros(3), np.ones(2, bool)),
                   (np.array([0.0, np.nan]), np.array([True, False]))):
        with pytest.raises(ValueError):
            equal_error_rate(s, lab)


# ---- refusals before any library call ---------------------------------------------------------------------------------
@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


@pytest.mark.parametrize("kw", [dict(channels=512), dict(channels=257), dict(max_enroll=33), dict(embed_dim=129),
                                dict(kernel_size=4), dict(n_conv=-1)])
def test_verifier_refuses_unsupported_shapes(kw):
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier
    with pytest.raises(ValueError):
        SpeakerVerifier(**kw)


def test_embed_and_loss_refusals(no_lib):
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier
    v = SpeakerVerifier(mel_dim=8, channels=16, embed_dim=8, max_enroll=3)
    ok = np.zeros((5, 8), np.float32)
    for bad in ([], [[]], [[ok] * 4], [[np.zeros((5, 7), np.float32)]], [[np.zeros((0, 8), np.float32)]], "x"):
        with pytest.raises(ValueError):
            v.embed_enrollment(bad)
    for bad in ([], [np.zeros((5, 7), np.float32)], [np.zeros(8, np.float32)], "x"):
        with pytest.raises(ValueError):
            v.embed_tests(bad)
    for ids in (torch.tensor([3, 3, 3]), torch.tensor([1])):
        with pytest.raises(ValueError):
            v.loss(torch.zeros(len(ids), 3, 10, 8), ids)
    assert no_lib == []


def test_step_refusals(no_lib, monkeypatch):
    from deepvoice3_pytorch_b200 import speaker_encoder as SE
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier, SpeakerVerifierStep
    v = SpeakerVerifier(mel_dim=8, channels=16, embed_dim=8, max_enroll=3)
    step = SpeakerVerifierStep(v, use_graph=False)
    ids = torch.tensor([0, 1], dtype=torch.int64)
    for mels, i in ((torch.zeros(2, 5, 10, 8), ids), (torch.zeros(2, 1, 10, 8), ids), (torch.zeros(2, 3, 10, 7), ids),
                    (torch.zeros(2, 3, 10), ids), (torch.zeros(2, 3, 10, 8), torch.zeros(3, dtype=torch.int64)),
                    (torch.zeros(2, 3, 10, 8).double(), ids), (torch.zeros(2, 3, 10, 8), ids.int()),
                    (torch.zeros(2, 3, 10, 8), torch.tensor([4, 4])), (torch.zeros(1, 3, 10, 8), ids[:1])):
        with pytest.raises(ValueError):
            step.step({"mels": mels, "speaker_ids": i})
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda: 2)
    with pytest.raises(ValueError):
        SpeakerVerifierStep(v)
    assert no_lib == []


def _ms_model(n_speakers=4):
    from deepvoice3_pytorch_b200 import builder
    torch.manual_seed(0)
    return builder.deepvoice3_multispeaker(n_vocab=40, embed_dim=16, mel_dim=80, linear_dim=9, r=1, downsample_step=4,
                                           kernel_size=3, encoder_channels=16, decoder_channels=16,
                                           converter_channels=16, max_positions=64, n_speakers=n_speakers,
                                           speaker_embed_dim=16, speaker_embedding_weight_std=0.2)


def test_verify_cloned_voices_refusals(no_lib):
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifier, verify_cloned_voices
    v = SpeakerVerifier(channels=16, embed_dim=8, max_enroll=3)
    model = _ms_model().eval()
    utt = np.zeros((20, 80), np.float32)
    enroll = {0: [utt], 2: [utt, utt]}
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    single = builder.deepvoice3(n_vocab=40, embed_dim=16, mel_dim=80, linear_dim=9, r=1, downsample_step=4,
                                kernel_size=3, encoder_channels=16, decoder_channels=16, converter_channels=16,
                                max_positions=64).eval()
    bad_calls = [
        (single, v, [0, 2], enroll, seqs, {}),                               # single-speaker model
        (model, v, [0, 4], enroll, seqs, {}),                                # id out of range
        (model, v, [0, -1], enroll, seqs, {}),
        (model, v, [0], enroll, seqs, {}),                                   # mismatched lengths
        (model, v, [0, 1], enroll, seqs, {}),                                # speaker 1 not enrolled
        (model, v, [0, 0], {0: [utt]}, seqs, {}),                            # one enrolled speaker: no impostor trial
        (model, v, [0, 2], {0: [utt], 2: [utt] * 4}, seqs, {}),              # more than max_enroll
        (model, v, [0, 2], {0: [utt], 2: [np.zeros((20, 79), np.float32)]}, seqs, {}),
        (model, SpeakerVerifier(mel_dim=40, channels=16, embed_dim=8), [0, 2], enroll, seqs, {}),
        (model, v, [0, 2], enroll, seqs, {"vocoder": "wavenet"}),
    ]
    for m, ver, ids, en, sq, kw in bad_calls:
        with pytest.raises(ValueError):
            verify_cloned_voices(m, ver, ids, en, sq, **kw)
    assert no_lib == []
