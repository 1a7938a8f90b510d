"""No GPU: duration-guided synthesis on the host -- the speaking-rate rule and the guided token path against their
restatements in tests/duration_oracle.py, the loss oracle against torch fp64 autograd, the C ABI and ptxas report of the
guided step kernels and csrc/duration.cu, and the refusals of the API before any library call."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import duration_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- speaking rate and path ---------------------------------------------------------------------------------------------
def _durations(seed, n=40):
    rng = np.random.RandomState(seed)
    return [rng.randint(1, 9, rng.randint(1, 60)).astype(np.int64) for _ in range(n)]


@pytest.mark.parametrize("speed", [0.5, 0.77, 1.0, 1.3, 2.0, 3.7])
def test_scale_durations_matches_the_rule(speed):
    from deepvoice3_pytorch_b200.duration import scale_durations
    ds = _durations(1) + [np.array([1]), np.array([1, 1, 1, 1]), np.array([2, 3, 2, 3, 2])]
    got = scale_durations(ds, speed)
    for d, g in zip(ds, got):
        assert g.dtype == np.int64 and g.shape == d.shape
        assert np.array_equal(g, DO.scale_durations(d, speed)), (d, g)
        assert g.min() >= 1
        if speed == 1.0:
            assert np.array_equal(g, d)


@pytest.mark.parametrize("speed", [0.5, 1.3, 2.0])
def test_scale_durations_totals(speed):
    """Where consecutive targets C_j / speed lie at least 1.5 apart (every d_j >= 3, speed <= 2) the floor of one step
    never binds, so the total is rint(C_L / speed) exactly; it is never below it."""
    from deepvoice3_pytorch_b200.duration import scale_durations
    for d in _durations(2):
        total = int(scale_durations([d], speed)[0].sum())
        want = int(np.rint(d.sum() / speed))
        assert total >= want
        d3 = d + 2
        assert int(scale_durations([d3], speed)[0].sum()) == int(np.rint(d3.sum() / speed))


def test_path_table_matches_its_definition():
    from deepvoice3_pytorch_b200.incremental import path_table
    ds = _durations(3, 12) + [np.array([1]), np.array([5])]
    path, totals = path_table(ds)
    assert totals == [int(d.sum()) for d in ds]
    assert path.dtype == np.int64 and path.shape == (len(ds), max(totals))
    assert np.array_equal(path, DO.path(ds, max(totals)))
    wide, _ = path_table(ds, max(totals) + 7)
    assert np.array_equal(wide, DO.path(ds, max(totals) + 7))
    for b, d in enumerate(ds):
        starts = np.concatenate([[0], np.cumsum(d)[:-1]])
        assert np.array_equal(path[b, starts], np.arange(d.size))


# ---- loss oracle ---------------------------------------------------------------------------------------------------------
def test_loss_oracle_matches_torch_fp64_autograd():
    rng = np.random.RandomState(4)
    B, L = 7, 23
    lens = np.array([23, 1, 5, 17, 2, 23, 9])
    y = rng.randn(B, L) * 2
    d = rng.randint(1, 40, (B, L))
    want, grad = DO.loss(y, d, lens)
    yt = torch.tensor(y, requires_grad=True)
    mask = torch.arange(L)[None] < torch.tensor(lens)[:, None]
    sq = (yt - torch.log(torch.tensor(d, dtype=torch.float64))) ** 2
    ref = ((sq * mask).sum(1) / torch.tensor(lens, dtype=torch.float64)).mean()
    ref.backward()
    assert want == pytest.approx(ref.item(), rel=1e-13)
    np.testing.assert_allclose(grad, yt.grad.numpy(), rtol=1e-12, atol=0)
    assert (grad[~mask.numpy()] == 0).all()


# ---- C ABI and ptxas -----------------------------------------------------------------------------------------------------
NEW = ("dv3_inc_attn_step_path", "dv3_inc_attn_step_slots_path", "dv3_inc_stop_rows_total", "dv3_duration_max_tokens",
       "dv3_duration_loss_fwd", "dv3_duration_loss_bwd")
PARENT = {"dv3_inc_conv_step": ["step", "stream"], "dv3_inc_conv_step_slots": ["step", "stream"],
          "dv3_inc_attn_step": ["attn", "stream"], "dv3_inc_attn_step_rows": ["attn", "text_len", "stream"],
          "dv3_inc_attn_step_slots": ["attn", "text_len", "stream"], "dv3_inc_advance": ["t_ptr", "stream"],
          "dv3_inc_stop_rows": ["done", "done_ld", "t", "stop", "B", "min_steps", "max_steps", "stream"],
          "dv3_inc_advance_rows": ["t", "stop", "B", "stream"],
          "dv3_inc_refill": ["table", "n_entries", "slots", "n_slots", "stream"]}


def test_c_abi_declares_and_exports_the_new_entry_points_and_keeps_the_old_ones():
    from deepvoice3_pytorch_b200._lib import parse_header
    d = parse_header()
    args = {n: [a for _, a in d[n][1]] for n in NEW + tuple(PARENT)}
    for name, want in PARENT.items():
        assert args[name] == want, name
    assert args["dv3_inc_attn_step_path"] == ["attn", "text_len", "path", "path_ld", "stream"]
    assert args["dv3_inc_attn_step_slots_path"] == ["attn", "text_len", "path", "path_ld", "stream"]
    assert args["dv3_inc_stop_rows_total"] == ["t", "stop", "total", "B", "stream"]
    assert args["dv3_duration_loss_fwd"] == ["y", "y_ld", "durations", "d_ld", "lengths", "B", "L", "row_loss", "loss",
                                             "err_flag", "stream"]
    assert args["dv3_duration_loss_bwd"] == ["y", "y_ld", "durations", "d_ld", "lengths", "B", "L", "d_loss", "dy",
                                             "stream"]
    P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    assert [t for t, _ in d["dv3_inc_attn_step_path"][1]] == [P, P, P, LL, P]
    assert [t for t, _ in d["dv3_inc_stop_rows_total"][1]] == [P, P, P, I, P]
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in NEW + tuple(PARENT):
            assert re.search(r"\bT %s\b" % name, nm), name
        assert ctypes.CDLL(so).dv3_duration_max_tokens() == 1024


def _ptxas(src):
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", src), "-o",
                        os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    return re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", rep, flags=re.S)


def test_ptxas_no_spills_zero_stack():
    frames = _ptxas("incremental.cu") + _ptxas("duration.cu")
    names = [n for n, *_ in frames]
    # the guided instantiations <ROWS, SLOTS, PATH> = <1, 0, 1> and <1, 1, 1>, the total stop rule, the loss kernels
    for want in ("inc_attn_step_kernelILb1ELb0ELb1E", "inc_attn_step_kernelILb1ELb1ELb1E", "inc_stop_rows_total_kernel",
                 "dur_loss_rows_kernel", "dur_loss_reduce_kernel", "dur_loss_grad_kernel"):
        assert any(want in n for n in names), want
    for name, stack, st, ld in frames:
        if "inc_attn_step" in name or "stop_rows" in name or "dur_loss" in name:
            assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


# ---- refusals before any library call ------------------------------------------------------------------------------------
@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


def test_scale_and_check_refusals(no_lib):
    from deepvoice3_pytorch_b200.duration import scale_durations
    from deepvoice3_pytorch_b200.incremental import check_durations
    d = [np.array([1, 2, 3])]
    for speed in (0, -1.0, float("nan"), float("inf"), True, "1", None):
        with pytest.raises(ValueError):
            scale_durations(d, speed)
    for bad in ([np.array([1, 0, 3])], [np.array([1.0, 2.0])], [np.array([[1, 2]])], np.array([1, 2]),
                [np.array([-2, 4])]):
        with pytest.raises(ValueError):
            scale_durations(bad, 1.0)
    for bad, lens in (([np.array([1, 2])], [3]), ([np.array([1, 2])], [2, 2]), ([np.array([2, 0])], [2])):
        with pytest.raises(ValueError):
            check_durations(bad, lens)
    assert [x.tolist() for x in check_durations([torch.tensor([2, 1])], [2])] == [[2, 1]]
    assert no_lib == []


def test_loss_and_predictor_refusals(no_lib):
    from deepvoice3_pytorch_b200.duration import DurationPredictor, _check_host_values, duration_loss
    y = torch.zeros(2, 4)                                      # a CPU tensor: refused
    with pytest.raises(ValueError):
        duration_loss(y, np.ones((2, 4), np.int64), np.array([4, 4]))
    d = np.ones((2, 4), np.int64)
    for dd, ll in ((d, np.array([0, 4])), (d, np.array([5, 4])), (np.array([[1, 1, 0, 1], [1, 1, 1, 1]]),
                                                                    np.array([4, 4]))):
        with pytest.raises(ValueError):
            _check_host_values(dd, ll, 4)
    _check_host_values(np.array([[1, 1, 0, 0], [1, 1, 1, 1]]), np.array([2, 4]), 4)     # past a row's length: free
    for kw in ({"in_dim": 0}, {"in_dim": 8, "kernel_size": 4}, {"in_dim": 8, "channels": 0},
               {"in_dim": 8, "n_blocks": -1}):
        with pytest.raises(ValueError):
            DurationPredictor(**kw)
    with pytest.raises(TypeError):
        DurationPredictor(8, dropout=0.1)                      # no dropout: the blocks run with p = 0
    pred = DurationPredictor(8, channels=16, n_blocks=1)
    values = torch.zeros(2, 5, 8)
    for lens in (torch.tensor([5, 3], dtype=torch.int32), torch.tensor([5, 3]), torch.tensor([5]), [5, 3],
                 np.array([5, 3])):
        with pytest.raises(ValueError, match="lengths"):       # int32, CPU, wrong shape, not a tensor
            pred(values, lens)
    with pytest.raises(ValueError):
        pred(torch.zeros(2, 5, 7), torch.tensor([5, 3]))
    assert no_lib == []


def test_synthesis_refusals(no_lib):
    from deepvoice3_pytorch_b200 import incremental
    from deepvoice3_pytorch_b200.alignment import evaluate_attention
    from deepvoice3_pytorch_b200.duration import predict_durations, DurationPredictor
    from deepvoice3_pytorch_b200.synthesis import tts_batch, tts_stream
    from test_mcd_host import _models
    single, multi = _models()
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    good = [np.array([2, 2, 2]), np.array([1, 3])]
    most = incremental.query_steps(single.seq2seq.decoder)
    bad = [dict(speed=2.0), dict(durations=good[:1]), dict(durations=[good[0], np.array([1, 2, 3])]),
           dict(durations=[good[0], np.array([0, 3])]), dict(durations=good, speed=0.0),
           dict(durations=good, speed=float("nan")), dict(durations=[good[0], np.array([1, most])]),
           dict(durations=[good[0], np.array([1.0, 2.0])]), dict(durations=good, speed=2.0 / most)]
    for kw in bad:
        for fn in (tts_batch, lambda *a, **k: next(iter(tts_stream(*a, **k))), evaluate_attention):
            with pytest.raises(ValueError):
                fn(single, seqs, **kw)
    keys = torch.zeros(2, 3, 16)
    tpos = torch.tensor([[1, 2, 3], [1, 2, 0]])
    dec = single.seq2seq.decoder
    for durs in ([np.array([1, 1, 1]), np.array([1, 1, 1])], [np.array([1, 1, 1])],
                 [np.array([1, 1, 1]), np.array([most, 1])]):
        with pytest.raises(ValueError):
            incremental.decode_ragged(dec, (keys, keys), tpos, [3, 2], durations=durs)
    with pytest.raises(ValueError):
        incremental.decode_ragged(dec, (keys, keys), tpos, [3, 2], test_inputs=torch.zeros(2, 4, 80),
                                  durations=good)
    pred = DurationPredictor(16, channels=16, n_blocks=1)
    for args in ((single, []), (single, [np.array([3.0])]), (multi, seqs)):
        with pytest.raises(ValueError):
            predict_durations(pred, *args)
    assert no_lib == []
