"""GPU: training on batches padded to a bucket shape (data.pad_to_bucket, ops.extent_scope, TrainStep's per-bucket
CUDA graphs).  The padding must be invisible: loss, gradients and updates of the unpadded batch."""
import numpy as np
import pytest
import torch

N_VOCAB, LIN = 149, 129
TEXT_LENS, FRAME_LENS = (23, 17, 9), (70, 51, 33)


def _build(topo, dropout):
    from deepvoice3_pytorch_b200 import builder
    common = dict(n_vocab=N_VOCAB, embed_dim=64, mel_dim=80, linear_dim=LIN, r=1, downsample_step=4, kernel_size=3,
                  encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256,
                  dropout=dropout)
    if topo == "deepvoice3":
        return builder.deepvoice3(use_memory_mask=True, key_projection=True, value_projection=True, **common)
    if topo == "nyanko":
        return builder.nyanko(use_memory_mask=False, **common)
    return builder.deepvoice3_multispeaker(n_speakers=5, use_memory_mask=False, **common)


def _utterances(topo, text_lens=TEXT_LENS, frame_lens=FRAME_LENS, seed=0):
    rng = np.random.RandomState(seed)
    items = []
    for i, (n, t) in enumerate(zip(text_lens, frame_lens)):
        item = (rng.randint(2, N_VOCAB, n).astype(np.int32), (0.05 + 0.9 * rng.rand(t, 80)).astype(np.float32),
                (0.05 + 0.9 * rng.rand(t, LIN)).astype(np.float32))
        items.append(item + (i % 5,) if topo == "multispeaker" else item)
    return items


def _batches(topo, extra_text=13, extra_dec=5, **kw):
    """-> (unpadded device batch, the same padded to a larger bucket)."""
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    host = data.collate(_utterances(topo, **kw))
    ext = data.batch_extents(host)
    padded = data.pad_to_bucket(host, ext[1] + extra_text, ext[0] + extra_dec)
    return to_device(host, "cuda"), to_device(padded, "cuda")


def _train(topo, batches, math, dropout=0.0, graph=False):
    """Adam steps over ``batches`` -> (losses, gradient arena and grad norm after the first step, final parameters,
    the TrainStep)."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    old = ops.conv_math
    ops.conv_math = math
    try:
        torch.manual_seed(0)
        ops.rng.manual_seed(77, torch.device("cuda"))
        step = TrainStep(_build(topo, dropout).cuda().train(), use_graph=graph)
        losses, grad0, norm0 = [], None, None
        for b in batches:
            losses.append(float(step.step(b)))
            if grad0 is None:
                grad0, norm0 = step.arena.grad.clone(), float(step.opt.grad_norm())
        torch.cuda.synchronize()
        return np.array(losses), grad0, norm0, step.arena.flat.clone(), step
    finally:
        ops.conv_math = old


def _excess(got, want, rtol, atol):
    """max |got - want| / (atol + rtol |want|): <= 1 inside the tolerance."""
    got, want = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(want, dtype=torch.float64)
    return float(((got - want).abs() / (atol + rtol * want.abs())).max())


TOL = {"fp32": (1e-5, 1e-7), "tc": (2e-5, 1e-6)}


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tc"])
@pytest.mark.parametrize("topo", ["deepvoice3", "nyanko", "multispeaker"])
def test_padding_to_a_bucket_is_invisible(topo, math):
    """Eager steps on a batch padded to a larger bucket (with its extents) == eager steps on the unpadded batch: loss,
    the whole gradient arena, grad norm, parameters after 4 Adam steps.  Control: the padded batch with its padded sizes
    passed as the logical extents misses the tolerance by >= 10x."""
    rtol, atol = TOL[math]
    plain, padded = _batches(topo)
    l_ref, g_ref, n_ref, p_ref, _ = _train(topo, [plain] * 4, math)
    l_pad, g_pad, n_pad, p_pad, _ = _train(topo, [padded] * 4, math)
    assert float(g_ref.abs().max()) > 0
    assert _excess(l_pad, l_ref, rtol, atol) <= 1, (l_pad, l_ref)
    assert _excess(n_pad, n_ref, rtol, atol) <= 1, (n_pad, n_ref)
    torch.testing.assert_close(g_pad, g_ref, rtol=rtol, atol=atol)
    torch.testing.assert_close(p_pad, p_ref, rtol=rtol, atol=atol)
    # negative control 1: the padding declared logical
    wrong = dict(padded)
    wrong["extents"] = torch.tensor([padded["done"].shape[1], padded["x"].shape[1], padded["mel"].shape[1],
                                     padded["y"].shape[1]], dtype=torch.int64, device="cuda")
    l_bad, g_bad, _, _, _ = _train(topo, [wrong], math)
    assert max(_excess(l_bad, l_ref[:1], rtol, atol), _excess(g_bad, g_ref, rtol, atol)) >= 10


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tc"])
@pytest.mark.parametrize("topo", ["deepvoice3", "nyanko", "multispeaker"])
def test_padding_is_visible_without_the_time_mask(topo, math, monkeypatch):
    """Negative control 2: the correct extents, but the conv stacks told nothing (no time mask of the encoder and
    converter inputs or gradients): loss and gradients miss the unpadded batch's by >= 10x the tolerance, so the
    equality above rests on the masking, not only on the loss denominators."""
    from deepvoice3_pytorch_b200 import ops
    rtol, atol = TOL[math]
    plain, padded = _batches(topo)
    l_ref, g_ref, _, _, _ = _train(topo, [plain], math)
    monkeypatch.setattr(ops, "extent_frames", lambda x: None)
    l_bad, g_bad, _, _, _ = _train(topo, [padded], math)
    assert max(_excess(l_bad, l_ref, rtol, atol), _excess(g_bad, g_ref, rtol, atol)) >= 10


@pytest.mark.gpu
def test_bucket_graphs_equal_eager_steps_in_any_replay_order():
    """Shapes A, B, A, C, B through TrainStep(use_graph=True), dropout on: A runs the exact graph of the first shape,
    B and C are padded to their buckets and replay lazily captured graphs out of capture order.  Against eager steps on
    the same (padded) batches: same losses, final parameters and last gradient arena, three graphs.  (Not bitwise: the embedding and bias
    gradients are atomic reductions whose order differs between runs.)"""
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    a, _ = _batches("deepvoice3")
    b, _ = _batches("deepvoice3", text_lens=(31, 12, 20), frame_lens=(90, 40, 61), seed=1)
    c, _ = _batches("deepvoice3", text_lens=(8, 5, 7), frame_lens=(24, 30, 17), seed=2)
    seq = [a, b, a, c, b]
    l_graph, _, _, p_graph, step = _train("deepvoice3", seq, "tc", dropout=0.05, graph=True)
    g_graph = step.arena.grad.clone()
    assert step.graphs_captured == 3

    def padded(x):
        if x is a:
            return a
        ext = data.batch_extents(x)
        host = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in x.items()}
        return to_device(data.pad_to_bucket(host, *data.bucket_shape(ext[1], ext[0])), "cuda")
    l_eager, _, _, p_eager, eager = _train("deepvoice3", [padded(x) for x in seq], "tc", dropout=0.05)
    np.testing.assert_allclose(l_graph, l_eager, rtol=2e-5)
    torch.testing.assert_close(p_graph, p_eager, rtol=2e-5, atol=1e-6)
    assert float(g_graph.abs().max()) > 0
    torch.testing.assert_close(g_graph, eager.arena.grad, rtol=2e-5, atol=1e-6)      # the last step's gradients


@pytest.mark.gpu
def test_extent_loss_kernels_equal_the_torch_loss_on_the_unpadded_batch():
    """fused_training_loss on padded outputs + a padded batch == training_loss on the unpadded ones, value and
    gradients; the gradients outside the logical extents are exactly 0."""
    from deepvoice3_pytorch_b200.train_step import fused_training_loss, training_loss
    plain, padded = _batches("deepvoice3")
    B, Td, Tt = padded["done"].shape[0], padded["done"].shape[1], padded["x"].shape[1]
    td, tt = plain["done"].shape[1], plain["x"].shape[1]
    gen = torch.Generator().manual_seed(3)
    outs = [torch.rand(B, Td, 80, generator=gen), torch.rand(B, 4 * Td, LIN, generator=gen),
            torch.softmax(torch.randn(2, B, Td, Tt, generator=gen), -1), torch.rand(B, Td, 1, generator=gen)]
    outs = [o.cuda().requires_grad_(True) for o in outs]
    cut = [o[:, :td] for o in outs[:1]] + [outs[1][:, :4 * td]] + [outs[2][:, :, :td, :tt]] + [outs[3][:, :td]]
    cut = [o.detach().clone().requires_grad_(True) for o in cut]
    want = training_loss(tuple(cut), plain)
    want.backward()
    got = fused_training_loss(tuple(outs), padded)
    got.backward()
    np.testing.assert_allclose(float(got), float(want), rtol=1e-5)
    for o, c in zip(outs, cut):
        sl = tuple(slice(0, n) for n in c.shape)
        torch.testing.assert_close(o.grad[sl], c.grad, rtol=2e-4, atol=1e-9)
        rest = o.grad.clone()
        rest[sl] = 0
        assert not rest.any(), "gradient outside the logical extents"


@pytest.mark.gpu
def test_fixed_shape_graph_never_enters_the_extent_path(monkeypatch):
    """A run whose batches all have one shape captures one graph at that exact shape and never touches the extent
    machinery; the graph records exactly the kernels of a steady-state eager step (launches_per_step) and gives its
    losses, gradients and parameters."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib

    def refuse(self):
        raise AssertionError("extent scope entered on a fixed-shape run")
    monkeypatch.setattr(ops.extent_scope, "__enter__", refuse)
    plain, _ = _batches("deepvoice3")
    l_graph, _, _, p_graph, step = _train("deepvoice3", [plain] * 4, "tc", dropout=0.05, graph=True)
    assert step.graphs_captured == 1 and not step._buckets
    l_eager, _, _, p_eager, eager = _train("deepvoice3", [plain] * 3, "tc", dropout=0.05)
    n0 = lib.raw("dv3_launch_count")()
    l_eager = np.append(l_eager, float(eager.step(plain)))
    assert step.launches_per_step == int(lib.raw("dv3_launch_count")() - n0)
    np.testing.assert_allclose(l_graph, l_eager, rtol=2e-5)
    torch.testing.assert_close(step.arena.grad, eager.arena.grad, rtol=2e-5, atol=1e-6)
    torch.testing.assert_close(p_graph, eager.arena.flat, rtol=2e-5, atol=1e-6)


@pytest.mark.gpu
def test_graph_mode_refuses_shape_changes_it_cannot_bucket():
    from deepvoice3_pytorch_b200 import builder
    from deepvoice3_pytorch_b200.train_step import TrainStep
    a, _ = _batches("deepvoice3")
    b, _ = _batches("deepvoice3", text_lens=(31, 12, 20), frame_lens=(90, 40, 61), seed=1)
    torch.manual_seed(0)
    step = TrainStep(_build("deepvoice3", 0.0).cuda().train(), use_graph=True, fused_loss=False)
    step.step(a)
    with pytest.raises(ValueError, match="fused_loss=False"):
        step.step(b)
