"""GPU: TrainStep's training modes and optimizer settings against torch.optim.Adam and the torch-ops losses -- the
weight-decay / AMSGrad update kernel, the per-term loss slots, seq2seq-only and postnet-only steps (eager, exact-shape
graph and bucketed graph) and resuming a joint run from a partial checkpoint."""
import copy
import ctypes

import numpy as np
import pytest
import torch

N_VOCAB, LIN = 149, 129


def _utterances(text_lens=(23, 17, 9), frame_lens=(70, 51, 33), seed=0):
    rng = np.random.RandomState(seed)
    return [(rng.randint(2, N_VOCAB, n).astype(np.int32), (0.05 + 0.9 * rng.rand(t, 80)).astype(np.float32),
             (0.05 + 0.9 * rng.rand(t, LIN)).astype(np.float32)) for n, t in zip(text_lens, frame_lens)]


def _build(topo="deepvoice3", dropout=0.0):
    from deepvoice3_pytorch_b200 import builder
    common = dict(n_vocab=N_VOCAB, embed_dim=64, mel_dim=80, linear_dim=LIN, r=1, downsample_step=4, kernel_size=3,
                  encoder_channels=128, decoder_channels=128, converter_channels=128, max_positions=256,
                  dropout=dropout)
    torch.manual_seed(0)
    if topo == "deepvoice3":
        return builder.deepvoice3(use_memory_mask=True, key_projection=True, value_projection=True,
                                  use_decoder_state_for_postnet_input=False, **common).cuda().train()
    return builder.nyanko(use_memory_mask=False, **common).cuda().train()


def _batch(seed=0, **kw):
    from deepvoice3_pytorch_b200 import data
    from deepvoice3_pytorch_b200.train_step import to_device
    return to_device(data.collate(_utterances(seed=seed, **kw)), "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("wd,ams", [(0.0, False), (1e-2, False), (0.0, True), (1e-2, True)])
def test_adam_clip_opts_matches_torch_adam(wd, ams):
    """dv3_adam_clip_opts == clip_grad_norm_ + torch.optim.Adam(weight_decay, amsgrad) over 4 steps; with both options
    off it is bit-identical to dv3_adam_clip."""
    from deepvoice3_pytorch_b200._lib import lib
    n = 100003
    torch.manual_seed(0)
    p = torch.randn(n, device="cuda")
    m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    p2, m2, v2 = p.clone(), m.clone(), v.clone()
    ref = torch.nn.Parameter(p.clone())
    opt = torch.optim.Adam([ref], lr=1e-3, betas=(0.5, 0.9), eps=1e-6, weight_decay=wd, amsgrad=ams)
    hyper, sumsq = torch.zeros(4, device="cuda"), torch.zeros(1, device="cuda")
    scratch = torch.zeros(lib.raw("dv3_sumsq_scratch_floats")(), device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    for t in range(1, 5):
        g = torch.randn(n, device="cuda") * (0.5 if t % 2 else 3e-4)      # clipped and unclipped steps
        hyper.copy_(torch.tensor([1e-3, 1 - 0.5 ** t, 1 - 0.9 ** t, 1.0]))
        lib.call("dv3_sumsq", vp(g), n, vp(sumsq), vp(scratch), st)
        lib.call("dv3_adam_clip_opts", vp(p), vp(g), vp(m), vp(v), vp(vmax) if ams else None, n, vp(hyper),
                 vp(sumsq), 0.5, 0.9, 1e-6, 0.1, wd, st)
        if not wd and not ams:
            lib.call("dv3_adam_clip", vp(p2), vp(g), vp(m2), vp(v2), n, vp(hyper), vp(sumsq), 0.5, 0.9, 1e-6, 0.1, st)
            assert torch.equal(p, p2) and torch.equal(m, m2) and torch.equal(v, v2)
        ref.grad = g.clone()
        torch.nn.utils.clip_grad_norm_([ref], 0.1)
        opt.step()
    torch.testing.assert_close(p, ref.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m, opt.state[ref]["exp_avg"], rtol=1e-5, atol=1e-7)
    if ams:
        torch.testing.assert_close(vmax, opt.state[ref]["max_exp_avg_sq"], rtol=1e-5, atol=1e-10)


@pytest.mark.gpu
@pytest.mark.parametrize("pw", [0.0, 0.5])
def test_loss_terms_match_torch_losses(pw):
    """The *_terms kernels: every slot equals the torch-ops term (reference spec_loss / BCE / guided attention), their
    weighted sum equals the returned total, and total and gradients are bit-identical to the call without terms."""
    import torch.nn.functional as F
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200.train_step import (fused_training_loss, guided_attention_mask, priority_bin_of,
                                                    sequence_mask, spec_loss)
    b = _batch()
    B, Td = b["done"].shape[:2]
    gen = torch.Generator(device="cuda").manual_seed(1)
    outs = [torch.rand(B, Td, 80, device="cuda", generator=gen) * 0.9 + 0.05,
            torch.rand(B, Td * 4, LIN, device="cuda", generator=gen) * 0.9 + 0.05,
            torch.softmax(torch.randn(2, B, Td, b["x"].shape[1], device="cuda", generator=gen), -1),
            torch.rand(B, Td, 1, device="cuda", generator=gen) * 0.9 + 0.05]
    outs = [o.requires_grad_() for o in outs]
    kw = dict(priority_freq_weight=pw, sample_rate=22050, priority_freq=3000)
    terms = torch.zeros(ops.TERM_COUNT, device="cuda")
    total = fused_training_loss(outs, b, terms=terms, **kw)
    grads = torch.autograd.grad(total, outs)
    total0 = fused_training_loss(outs, b, **kw)
    grads0 = torch.autograd.grad(total0, outs)
    assert torch.equal(total, total0) or abs(float(total) - float(total0)) <= 1e-6 * abs(float(total0))
    for g, g0 in zip(grads, grads0):
        assert torch.equal(g, g0)
    tl = b["target_lengths"]
    dec_mask = sequence_mask(tl // 4, Td).unsqueeze(-1)[:, 1:]
    tgt_mask = sequence_mask(tl, Td * 4).unsqueeze(-1)[:, 1:]
    with torch.no_grad():
        ml1, mbd = spec_loss(outs[0][:, :-1], b["mel"][:, 1:], dec_mask, 0.5, 0.1)
        ll1, lbd = spec_loss(outs[1][:, :-1], b["y"][:, 1:], tgt_mask, 0.5, 0.1,
                             priority_bin=priority_bin_of(3000, 22050, LIN), priority_w=pw)
        done = F.binary_cross_entropy(outs[3], b["done"])
        W = guided_attention_mask(b["input_lengths_dev"], tl // 4, Td, b["x"].shape[1], 0.2)
        attn = (outs[2] * W).mean()
    want = {ops.TERM_MEL_L1: ml1, ops.TERM_MEL_BD: mbd, ops.TERM_LIN_L1: ll1, ops.TERM_LIN_BD: lbd,
            ops.TERM_DONE: done, ops.TERM_ATTN: attn}
    for slot, w in want.items():
        np.testing.assert_allclose(float(terms[slot]), float(w), rtol=2e-5, err_msg=str(slot))
    t = terms.double()
    summed = 0.9 * (t[0] + t[2]) + 0.1 * (t[1] + t[3]) + t[4] + t[5]
    np.testing.assert_allclose(float(summed), float(total), rtol=1e-5)


def _harness():
    from oracle import ref_harness as H
    if H.ref_root() is None:
        pytest.skip("oracle/_ref not built (python oracle/make_ref.py in the build container)")
    return H


REF_CASES = [("deepvoice3_ljspeech", "seq2seq", {}), ("nyanko_ljspeech", "seq2seq", {}),
             ("deepvoice3_ljspeech", "postnet", dict(use_decoder_state_for_postnet_input=False)),
             ("deepvoice3_ljspeech", "joint", dict(weight_decay=1e-6, amsgrad=True)),
             ("deepvoice3_ljspeech", "joint", dict(lr_schedule="cyclic_cosine_annealing"))]


@pytest.mark.gpu
@pytest.mark.parametrize("preset,mode,over", REF_CASES)
def test_train_step_matches_reference_train(preset, mode, over, tmp_path):
    """The reference's own train() (train.py, run unchanged from oracle/_ref on the reference package, eager, TF32 off,
    dropout 0, torch.optim.Adam) vs TrainStep on this package: same seed, utterances and order, 4 steps of 4.  Every
    tag train() logs agrees at rtol 2e-4 on step 0 and 5e-3 over the 4 steps, TrainStep reports exactly the tags of
    the mode, and the parameters of the part that is not trained keep their bits."""
    H = _harness()
    from torch.utils.data import DataLoader
    from deepvoice3_pytorch_b200 import data, hparams
    from deepvoice3_pytorch_b200.train_step import TrainStep, to_device
    s2s, post = mode != "postnet", mode != "seq2seq"
    over = dict(over)
    schedule = over.pop("lr_schedule", None)
    utts = H.synthetic_utterances(16, seed=3, min_text=40, max_text=100, min_frames=200, max_frames=400)

    def configure(tr):
        hp = H.apply_preset(tr, preset, dropout=0.0, eval_interval=10 ** 9, **over)
        if schedule is not None:
            hp.lr_schedule = schedule
            hp.lr_schedule_kwargs = dict(T=8, M=2)
        return hp

    old_tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        tr = H.load_train("reference")
        hp = configure(tr)
        torch.manual_seed(0)
        model = tr.build_model().to("cuda")
        opt = torch.optim.Adam(model.get_trainable_parameters(), lr=hp.initial_learning_rate,
                               betas=(hp.adam_beta1, hp.adam_beta2), eps=hp.adam_eps, weight_decay=hp.weight_decay,
                               amsgrad=hp.amsgrad)
        loader = DataLoader(utts, batch_size=4, collate_fn=tr.collate_fn, shuffle=False)
        writer = H.ScalarLog()
        tr.global_step, tr.global_epoch = 0, 0
        tr.train(torch.device("cuda"), model, loader, opt, writer, init_lr=hp.initial_learning_rate,
                 checkpoint_dir=str(tmp_path), checkpoint_interval=10 ** 9, nepochs=1, clip_thresh=hp.clip_thresh,
                 train_seq2seq=s2s, train_postnet=post)
        ref = {k: np.array([v for _, v in vals]) for k, vals in writer.scalars.items()}
        hpd = dict(hp.values())
        del model, opt
        torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32 = old_tf32

    trb = H.load_train("b200")
    configure(trb)
    torch.manual_seed(0)
    model = trb.build_model().to("cuda")
    before = {k: v.clone() for k, v in model.state_dict().items()}
    step = TrainStep(model, train_seq2seq=s2s, train_postnet=post, **hparams.train_step_kwargs(hpd))
    got = {}
    for i in range(0, len(utts), 4):
        b = data.collate(utts[i:i + 4], r=hpd["outputs_per_step"], downsample_step=hpd["downsample_step"])
        got.setdefault("loss", []).append(float(step.step(to_device(b, "cuda"))))
        for k, v in step.loss_terms().items():
            got.setdefault(k, []).append(float(v))
    assert set(got) == set(ref) - {"learning rate", "loss (per epoch)"}
    for tag, vals in got.items():
        vals = np.array(vals)
        assert len(vals) == 4 and len(ref[tag]) == 4, tag
        np.testing.assert_allclose(vals[0], ref[tag][0], rtol=2e-4, err_msg=tag + " (first step: identical weights)")
        np.testing.assert_allclose(vals, ref[tag], rtol=5e-3, err_msg=tag)
    untouched = {"seq2seq": "postnet.", "postnet": "seq2seq.", "joint": None}[mode]
    after = model.state_dict()
    for k, v in before.items():
        if untouched and k.startswith(untouched):
            assert torch.equal(after[k], v), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["seq2seq", "postnet"])
def test_partial_graph_steps_equal_eager(mode):
    """Exact-shape graph and bucket graphs replayed out of capture order (dropout on) == eager steps on the same padded
    batches, in each partial mode."""
    from deepvoice3_pytorch_b200 import data, ops
    from deepvoice3_pytorch_b200.train_step import TrainStep
    shapes = [dict(), dict(text_lens=(11, 7, 5), frame_lens=(40, 33, 21)), dict(text_lens=(30, 20, 9),
                                                                             frame_lens=(90, 61, 40))]
    base = [_batch(seed=s, **kw) for s, kw in enumerate(shapes)]
    order = [0, 1, 2, 1, 0, 2]
    kw = dict(train_seq2seq=mode == "seq2seq", train_postnet=mode == "postnet")
    results = []
    for graph in (False, True):
        torch.manual_seed(0)
        ops.rng.manual_seed(5, torch.device("cuda"))
        step = TrainStep(_build(dropout=0.1), use_graph=graph, **kw)
        losses = []
        for i in order:
            b = step._mode_batch(base[i])
            if i and not graph:       # the batch the graph step replays: padded to its bucket
                ext = data.batch_extents(b)
                b = data.pad_to_bucket(b, *data.bucket_shape(ext[1], ext[0]))
            losses.append(float(step.step(b)))
        torch.cuda.synchronize()
        results.append((np.array(losses), step.arena.flat.clone(), step.graphs_captured))
    (eager, p_eager, _), (graph, p_graph, n_graphs) = results
    assert n_graphs == 3
    np.testing.assert_allclose(graph, eager, rtol=2e-5, atol=1e-6)
    torch.testing.assert_close(p_graph, p_eager, rtol=2e-5, atol=1e-6)


@pytest.mark.gpu
def test_joint_resume_from_seq2seq_checkpoint_matches_torch_adam():
    """A seq2seq-only run's checkpoint (model.seq2seq.state_dict() + Adam state over all trainable parameters) resumes a
    joint TrainStep exactly as it resumes torch.optim.Adam: seq2seq moments at their step, postnet from step 0."""
    from deepvoice3_pytorch_b200.train_step import TrainStep
    batches = [_batch(seed=s) for s in range(4)]
    first = TrainStep(_build(), train_postnet=False)
    for b in batches[:2]:
        first.step(b)
    ckpt = copy.deepcopy(first.state_dict())
    assert set(ckpt["state_dict"]) == set(first.model.seq2seq.state_dict())
    n_post = len(list(first.model.postnet.parameters()))
    assert len(ckpt["optimizer"]["state"]) == len(list(first.model.get_trainable_parameters())) - n_post

    joint = TrainStep(_build())
    joint.load_state_dict(ckpt)
    assert joint.global_step == 2 and sorted(set(joint.opt.part_t)) == [0, 2]
    got = np.array([float(joint.step(b)) for b in batches[2:]])

    ref_model = _build()
    ref_model.seq2seq.load_state_dict(ckpt["state_dict"])
    opt = torch.optim.Adam(ref_model.get_trainable_parameters(), lr=5e-4, betas=(0.5, 0.9), eps=1e-6)
    opt.load_state_dict(ckpt["optimizer"])
    from deepvoice3_pytorch_b200.train_step import noam_learning_rate_decay, training_loss
    want = []
    for s, b in enumerate(batches[2:], start=2):
        for g in opt.param_groups:
            g["lr"] = noam_learning_rate_decay(5e-4, s)
        opt.zero_grad()
        outs = ref_model(b["x"], b["mel"], text_positions=b["text_positions"], frame_positions=b["frame_positions"],
                         input_lengths=b["input_lengths_dev"])
        loss = training_loss(outs, b)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(ref_model.get_trainable_parameters(), 0.1)
        opt.step()
        want.append(float(loss))
    np.testing.assert_allclose(got, want, rtol=5e-3)
    # graph mode: a graph captured while all clocks agreed is dropped by the load that splits them
    torch.manual_seed(7)
    graphed = TrainStep(_build(), use_graph=True)
    graphed.step(batches[0])
    assert graphed.graphs_captured == 1 and not graphed.opt.split_update()
    graphed.load_state_dict(copy.deepcopy(ckpt))
    assert graphed.graphs_captured == 0 and graphed.opt.split_update()
    got_graph = np.array([float(graphed.step(b)) for b in batches[2:]])
    np.testing.assert_allclose(got_graph, got, rtol=1e-4)
    sd = joint.opt.state_dict()
    ref_sd = opt.state_dict()
    for i, st in ref_sd["state"].items():
        assert float(sd["state"][i]["step"]) == float(st["step"]), i
    for k, v in ref_model.state_dict().items():
        torch.testing.assert_close(joint.model.state_dict()[k], v, rtol=5e-3, atol=1e-5)
