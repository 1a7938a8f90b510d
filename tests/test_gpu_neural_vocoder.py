"""GPU: the neural vocoder (deepvoice3_pytorch_b200/vocoder.py, csrc/vocoder.cu) against the fp64 oracle of
tests/vocoder_oracle.py: the loss kernels, the stride-s interleave and k = s transposed conv, the segment gather, the
generator, ragged-batch vocoding, the training step and the synthesis / evaluation entry points."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

import vocoder_oracle as VO

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RES = ((512, 128), (1024, 256), (2048, 512))


@contextlib.contextmanager
def _mode(conv_math="fp32", deterministic=None):
    from deepvoice3_pytorch_b200 import ops
    old = ops.conv_math, ops.deterministic
    ops.conv_math = conv_math
    if deterministic is not None:
        ops.deterministic = deterministic
    try:
        yield
    finally:
        ops.conv_math, ops.deterministic = old


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _pair(seed, B, n, noise=0.3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, n, generator=g) * 0.3
    y = x + noise * torch.randn(B, n, generator=g)
    return y.cuda(), x.cuda()


# ---- loss kernels --------------------------------------------------------------------------------------------------
def test_loss_and_spectrum_gradient_on_given_spectra_against_fp64():
    from deepvoice3_pytorch_b200._lib import lib
    from deepvoice3_pytorch_b200 import ops
    N, R, B, n = 1024, 256, 3, 5000
    lengths = [5000, 3100, 1]
    F = VO.num_frames(n, N, R)
    K = N // 2 + 1
    g = torch.Generator().manual_seed(1)
    sy = torch.randn(B, F, K, 2, generator=g)
    sx = sy + 0.5 * torch.randn(B, F, K, 2, generator=g)
    sy[0, 3, :40] = 0.0                                     # the clamp is active there
    dev = "cuda"
    lens = torch.tensor(lengths, dtype=torch.int32, device=dev)
    ws = torch.empty(lib.raw("dv3_mrstft_ws_doubles")(B, F), dtype=torch.float64, device=dev)
    stats = torch.empty(1, B, 4, dtype=torch.float64, device=dev)
    syd, sxd = sy.cuda(), sx.cuda()
    lib.call("dv3_mrstft_loss_fwd", _p(syd), _p(sxd), _p(lens), n, B, F, N, R, _p(ws), _p(stats[0]),
             _p(ops._err_flag(torch.device(dev))), _st())
    loss = torch.empty((), device=dev)
    clip = torch.empty(B, dtype=torch.float64, device=dev)
    lib.call("dv3_mrstft_loss_total", _p(stats), 1, B, _p(clip), _p(loss), _st())
    d_loss = torch.tensor([1.7], device=dev)
    dspec = torch.empty_like(syd)
    lib.call("dv3_mrstft_loss_bwd", _p(syd), _p(sxd), _p(stats[0]), B, F, N, R, 1, _p(d_loss), 0, _p(dspec), _st())
    ops.check_index_errors()
    Xs = sy.double().numpy()
    Ys = sx.double().numpy()
    ref_clip, ref_grad = [], np.zeros((B, F, K), np.complex128)
    for c, L in enumerate(lengths):
        f = VO.num_frames(L, N, R)
        X = Xs[c, :f, :, 0] + 1j * Xs[c, :f, :, 1]
        Y = Ys[c, :f, :, 0] + 1j * Ys[c, :f, :, 1]
        ref_clip.append(sum(VO.clip_terms(X, Y)))
        ref_grad[c, :f] = VO.grad_spec(X, Y, 1.7 / B)
    np.testing.assert_allclose(clip.cpu().numpy(), ref_clip, rtol=1e-13)
    ref = np.mean(ref_clip)
    assert abs(loss.item() - ref) <= 2 * U * ref
    got = dspec.cpu().double().numpy()
    got = got[..., 0] + 1j * got[..., 1]
    err = np.abs(got - ref_grad)
    assert np.all(err <= 2 * U * np.abs(ref_grad) + 1e-37), err.max()
    assert np.all(got[0, 3, :40] == 0) and np.all(got[2, VO.num_frames(1, N, R):] == 0)


def test_waveform_gradient_end_to_end_against_fp64():
    from deepvoice3_pytorch_b200 import vocoder, ops
    y, x = _pair(2, 2, 6000)
    yg = y.clone().requires_grad_(True)
    L = vocoder.stft_loss(yg, x, RES)
    L.backward()
    ops.check_index_errors()
    yn, xn = y.cpu().double().numpy(), x.cpu().double().numpy()
    ref = VO.loss(list(yn), list(xn), RES)
    # fp32 spectra: each magnitude carries a relative error of a few units of 2^-24 times log2 N
    assert abs(L.item() - ref) <= 1e-5 * ref
    want = VO.grad_wave(list(yn), list(xn), RES)
    got = yg.grad.cpu().double().numpy()
    for g, w in zip(got, want):
        scale = np.abs(w).max()
        assert np.abs(g - w).max() <= 1e-3 * scale
        assert np.linalg.norm(g - w) <= 1e-4 * np.linalg.norm(w)


@pytest.mark.parametrize("N,R", RES)
def test_adjoint_identity_on_the_cuda_path(N, R):
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    n, B = 3 * N + 11, 1
    F = VO.num_frames(n, N, R)
    x, _ = _pair(5, 1, n)
    g = torch.Generator().manual_seed(N)
    G = torch.randn(F, N // 2 + 1, 2, generator=g).double().numpy()
    Gc = G[..., 0] + 1j * G[..., 1]
    dev = x.device
    lens = torch.tensor([n], dtype=torch.int32, device=dev)
    frames = torch.tensor([F], dtype=torch.int32, device=dev)
    tab = audio._geometry_table(dev, N, R)
    spec = torch.empty(1, F, N // 2 + 1, 2, device=dev)
    lib.call("dv3_stft_complex_geom", _p(x), _p(lens), n, None, _p(spec), _p(frames), F, B, _p(tab), N, R, _st())
    S = VO.adjoint_spectrum(Gc, N)
    Sd = torch.from_numpy(np.stack([S.real, S.imag], -1).astype(np.float32)).cuda().contiguous()
    adj = torch.zeros(1, n, device=dev)
    lib.call("dv3_istft_geom", _p(Sd), _p(adj), _p(lens), n, _p(frames), F, B, _p(tab), N, R, _st())
    X = spec[0].cpu().double().numpy()
    lhs = np.sum(X[..., 0] * G[..., 0] + X[..., 1] * G[..., 1])
    rhs = np.dot(x[0].cpu().double().numpy(), adj[0].cpu().double().numpy())
    mass = np.sum(np.abs(X[..., 0] * G[..., 0]) + np.abs(X[..., 1] * G[..., 1]))
    assert abs(lhs - rhs) <= 1e-5 * mass
    np.testing.assert_allclose(adj[0].cpu().double().numpy(), VO.stft_adjoint(Gc, N, R, n), rtol=0,
                               atol=1e-5 * np.abs(VO.stft_adjoint(Gc, N, R, n)).max())


def test_clip_alone_equals_clip_in_batch_and_reruns_bit_identical():
    from deepvoice3_pytorch_b200 import vocoder
    y, x = _pair(7, 3, 7000)
    lengths = [7000, 4321, 2600]
    res = RES

    def run(yy, xx, lens, d):
        yg = yy.clone().requires_grad_(True)
        L = vocoder.stft_loss(yg, xx, res, lengths=lens)
        L.backward(torch.tensor(float(d), device="cuda"))
        return vocoder.clip_stft_losses(yy, xx, res, lengths=lens).cpu().numpy(), yg.grad.cpu().numpy(), L.item()
    cb, gb, lb = run(y, x, lengths, len(lengths))
    cb2, gb2, lb2 = run(y, x, lengths, len(lengths))
    assert np.array_equal(cb, cb2) and np.array_equal(gb, gb2) and lb == lb2
    for c, n in enumerate(lengths):
        ca, ga, _ = run(y[c:c + 1, :n].contiguous(), x[c:c + 1, :n].contiguous(), [n], 1)
        assert ca[0] == cb[c]
        assert np.array_equal(ga[0], gb[c, :n]) and not gb[c, n:].any()


def test_error_flag_on_bad_input():
    from deepvoice3_pytorch_b200 import vocoder, ops
    from deepvoice3_pytorch_b200._lib import lib
    ops.check_index_errors()
    y, x = _pair(9, 2, 4096)
    y[1, 100] = float("nan")
    vocoder.stft_loss(y, x, RES)
    with pytest.raises(IndexError):
        ops.check_index_errors()
    # a segment start past the utterance, handed to the kernel directly
    lin = torch.zeros(1, 20, 513, device="cuda")
    ints = torch.tensor([5000, 20, 15], dtype=torch.int32, device="cuda")
    cond, target = torch.empty(1, 513, 8, device="cuda"), torch.empty(1, 8 * 256, device="cuda")
    wav = torch.ones(1, 5000, device="cuda")
    lib.call("dv3_vocoder_gather", _p(lin), 20, _p(ints[1:2]), _p(wav), 5000, _p(ints[0:1]), _p(ints[2:3]), 1, 8,
             1024, 256, 0.97, _p(cond), _p(target), _p(ops._err_flag(torch.device("cuda"))), _st())
    with pytest.raises(IndexError):
        ops.check_index_errors()
    assert not target.any() and not cond.any()


# ---- building blocks -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", range(2, 9))
def test_interleave_is_an_exact_permutation(s):
    from deepvoice3_pytorch_b200 import ops
    B, C, T = 2, 5, 37
    x = torch.randn(B, s * C, T, device="cuda")
    y = ops.interleave(x, s)
    want = x.view(B, s, C, T).permute(0, 2, 3, 1).reshape(B, C, s * T)
    assert torch.equal(y, want)
    assert torch.equal(ops.interleave(y, s, 1), x)


@pytest.mark.parametrize("mode", ["fp32", "tc"])
@pytest.mark.parametrize("s", [3, 4, 8])
def test_conv_transpose_k_equals_s_against_fp64(mode, s):
    from deepvoice3_pytorch_b200 import modules
    torch.manual_seed(s)
    m = modules.ConvTranspose1d(128, 128, s, stride=s).cuda()
    with torch.no_grad():
        m.bias.normal_()
    x = torch.randn(4, 128, 160, device="cuda", requires_grad=True)
    dy = torch.randn(4, 128, 160 * s, device="cuda")
    with _mode(mode):
        y = m(x)
        y.backward(dy)
    v, g, b = (t.detach().cpu().double().requires_grad_(True) for t in (m.weight_v, m.weight_g, m.bias))
    xr = x.detach().cpu().double().requires_grad_(True)
    yr = torch.nn.functional.conv_transpose1d(xr, VO._wn(v, g), b, stride=s)
    yr.backward(dy.cpu().double())
    rtol, atol = (1e-5, 1e-6) if mode == "fp32" else (1e-3, 1e-4)
    for got, want in ((y, yr), (x.grad, xr.grad), (m.weight_v.grad, v.grad), (m.weight_g.grad, g.grad),
                      (m.bias.grad, b.grad)):
        w = want.detach().numpy()
        np.testing.assert_allclose(got.detach().cpu().numpy(), w, rtol=rtol, atol=atol * max(1.0, np.abs(w).max()))


def test_segment_gather_against_spectrogram_and_fp64_preemphasis():
    from deepvoice3_pytorch_b200 import audio, vocoder
    from deepvoice3_pytorch_b200.data import VocoderBatches
    from oracle.audio_oracle import synthetic_clip
    wavs = [synthetic_clip(s, n=n) for s, n in ((11, 30000), (12, 9000), (13, 52000))]
    vb = VocoderBatches(wavs, 3, seg_frames=16, seed=1)
    batch = next(iter(vb))
    out = vocoder.vocoder_batch(batch, 16)
    cond, target = out["cond"].cpu().numpy(), out["target"].cpu().numpy()
    off = (1024 - 256) // 2
    for row, (i, f0) in enumerate(zip(batch["items"].tolist(), batch["starts"].tolist())):
        spec = audio.spectrogram(wavs[i])
        assert np.array_equal(cond[row], spec[:, f0:f0 + 16])
        x = wavs[i].astype(np.float64)
        pe = np.concatenate([[x[0]], x[1:] - 0.97 * x[:-1]])
        p = f0 * 256 - off + np.arange(16 * 256)
        want = np.where((p >= 0) & (p < x.size), pe[np.clip(p, 0, x.size - 1)], 0.0).astype(np.float32)
        assert np.array_equal(target[row], want)


# ---- generator and inference ---------------------------------------------------------------------------------------
def _small_vocoder(seed=0):
    from deepvoice3_pytorch_b200 import vocoder
    torch.manual_seed(seed)
    voc = vocoder.NeuralVocoder(channels=128, upsample_channels=128, upsample=(4, 4, 4, 4),
                                frame_dilations=(1,), stage_dilations=(1, 3)).cuda()
    with torch.no_grad():
        for name, p in voc.named_parameters():
            if name.endswith("bias"):
                p.normal_(0, 0.1)
    return voc


@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_generator_forward_and_parameter_gradients_against_fp64(mode):
    voc = _small_vocoder(1)
    g = torch.Generator().manual_seed(2)
    cond = torch.rand(2, 513, 40, generator=g).cuda()
    dy = torch.randn(2, 40 * 256, generator=g).cuda()
    with _mode(mode):
        y = voc(cond)
        y.backward(dy)
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in voc.state_dict().items()}
    yr = VO.vocoder_forward(sd, voc, cond.cpu().double())
    yr.backward(dy.cpu().double())
    rtol, atol = (1e-4, 1e-5) if mode == "fp32" else (1e-3, 1e-4)
    w = yr.detach().numpy()
    np.testing.assert_allclose(y.detach().cpu().numpy(), w, rtol=rtol, atol=atol * max(1.0, np.abs(w).max()))
    for name, p in voc.named_parameters():
        w = sd[name].grad.numpy()
        np.testing.assert_allclose(p.grad.cpu().numpy(), w, rtol=rtol, atol=atol * max(1.0, np.abs(w).max()),
                                   err_msg=name)


@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_vocode_ragged_rows_equal_each_clip_alone(mode):
    from deepvoice3_pytorch_b200 import audio
    voc = _small_vocoder(3)
    rng = np.random.default_rng(4)
    specs = [rng.random((513, t), dtype=np.float32) for t in (61, 9, 130, 40)]
    with _mode(mode):
        got = voc.vocode(specs)
        alone = [voc.vocode([s])[0] for s in specs]
        via_audio = audio.inv_spectrogram_batch(specs, method=voc)
    for s, a, b, c in zip(specs, got, alone, via_audio):
        assert a.shape == b.shape == (audio.inv_num_samples(s.shape[1]),) and a.dtype == np.float32
        assert np.array_equal(a, c)
        if mode == "fp32":
            assert np.array_equal(a, b)
        else:
            np.testing.assert_allclose(a, b, rtol=1e-3, atol=1e-4 * max(1.0, np.abs(b).max()))


# ---- training step -------------------------------------------------------------------------------------------------
def _batches(n_batches, B=4, S=8, seed=0, first_seed=100):
    from deepvoice3_pytorch_b200 import vocoder
    from deepvoice3_pytorch_b200.data import VocoderBatches
    from oracle.audio_oracle import synthetic_clip
    wavs = [synthetic_clip(first_seed + k, n=22050) for k in range(B * 2)]
    vb = VocoderBatches(wavs, B, seg_frames=S, seed=seed)
    out, epoch = [], 0
    while len(out) < n_batches:
        vb.set_epoch(epoch)
        out += [vocoder.vocoder_batch(b, S) for b in vb]
        epoch += 1
    return out[:n_batches]


def _train(mode, det, use_graph, batches, ckpt_at=None, resume=None, seed=5):
    from deepvoice3_pytorch_b200.vocoder import NeuralVocoderStep
    with _mode(mode, det):
        voc = _small_vocoder(seed)
        step = NeuralVocoderStep(voc, lr=1e-3, clip_thresh=1.0, use_graph=use_graph)
        if resume is not None:
            step.load_state_dict(resume)
        losses, ckpt = [], None
        for k, b in enumerate(batches):
            if k == ckpt_at:
                ckpt = step.state_dict()
            losses.append(step.step(b).item())
        return losses, {k: v.detach().cpu() for k, v in voc.state_dict().items()}, ckpt, step


def test_graph_and_eager_steps_agree():
    batches = _batches(4)
    lg, sg, _, st = _train("tc", True, True, batches)
    le, se, _, _ = _train("tc", True, False, batches)
    assert st.graphs_captured == 1 and st.launches_per_step > 0
    assert lg == le
    for k in sg:
        assert torch.equal(sg[k], se[k]), k


def test_deterministic_runs_bit_identical_and_resume_bit_exact():
    batches = _batches(6)
    l1, s1, ck, _ = _train("tc", True, True, batches, ckpt_at=3)
    l2, s2, _, _ = _train("tc", True, True, batches)
    assert l1 == l2 and all(torch.equal(s1[k], s2[k]) for k in s1)
    l3, s3, _, _ = _train("tc", True, True, batches[3:], resume=ck)
    assert l3 == l1[3:] and all(torch.equal(s1[k], s3[k]) for k in s1)


def test_tc1_step_runs():
    losses, _, _, _ = _train("tc1", False, True, _batches(3))
    assert all(np.isfinite(losses))


LEARN_STEPS = 300
LEARN_FRACTION = 0.5      # measured 0.295 on an H100 (DESIGN.md section 2.23); the margin is set from that run


def test_learning_check_on_synthetic_clips():
    """A fixed budget of steps brings the held-out MR-STFT loss below LEARN_FRACTION of its initial value."""
    from deepvoice3_pytorch_b200 import vocoder
    from deepvoice3_pytorch_b200.vocoder import NeuralVocoderStep
    train = _batches(LEARN_STEPS, B=8, S=16, seed=0, first_seed=200)
    held = _batches(2, B=8, S=16, seed=9, first_seed=400)
    with _mode("tc", False):
        voc = _small_vocoder(6)

        def held_loss():
            with torch.no_grad():
                return float(np.mean([vocoder.stft_loss(voc(b["cond"]), b["target"]).item() for b in held]))
        before = held_loss()
        step = NeuralVocoderStep(voc, lr=1e-3, clip_thresh=1.0)
        for b in train:
            step.step(b)
        after = held_loss()
    print("held-out MR-STFT loss %.4f -> %.4f (ratio %.3f) after %d steps" % (before, after, after / before, LEARN_STEPS))
    assert after < LEARN_FRACTION * before


# ---- integration ---------------------------------------------------------------------------------------------------
def test_tts_batch_and_stream_with_the_neural_vocoder():
    from deepvoice3_pytorch_b200.synthesis import tts_batch, tts_stream
    from test_gpu_synthesis import _model, _sequences
    model = _model("deepvoice3_ljspeech", max_steps=30)
    seqs = _sequences([23, 7, 40])
    voc = _small_vocoder(8)
    with _mode("fp32"):
        got = tts_batch(model, seqs, vocoder=voc)
        streamed = dict(tts_stream(model, seqs, slots=2, post_batch=2, vocoder=voc))
        for k, (wav, _, _, _) in enumerate(got):
            with torch.no_grad():
                seq = torch.from_numpy(seqs[k]).unsqueeze(0).cuda()
                pos = torch.arange(1, seq.size(-1) + 1).unsqueeze(0).cuda()
                lin = model(seq, text_positions=pos)[1][0].cpu().numpy()
            alone = voc.vocode([lin.T])[0]
            assert np.array_equal(wav, alone), k
            assert np.array_equal(streamed[k][0], wav), k


def test_evaluate_vocoder_with_the_neural_vocoder():
    from deepvoice3_pytorch_b200.intelligibility import evaluate_vocoder
    from oracle.audio_oracle import synthetic_clip
    voc = _small_vocoder(10)
    wavs = [torch.from_numpy(synthetic_clip(s, n=n)).cuda() for s, n in ((1, 30000), (2, 44100))]
    out = evaluate_vocoder(wavs, method=voc)
    assert all(np.isfinite(out["stoi"])) and np.isfinite(out["mean_stoi"])
