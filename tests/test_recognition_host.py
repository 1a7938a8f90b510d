"""No GPU: the fp64 CTC oracle (tests/ctc_oracle.py) against torch's CPU ``F.ctc_loss`` in fp64 and against brute force
over every alignment, the edit-distance oracle against brute force and on hand cases of the S/D/I tie rule, the WER
word mapping, the C ABI and ptxas report of csrc/ctc.cu, the batch keys of every ArenaGraphStep, RecognizerBatches,
and the refusals of the API before any library call."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ctc_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the CTC oracle ---------------------------------------------------------------------------------------------------
def _torch_ctc(z, frames, targets, tlen):
    z64 = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    lp = F.log_softmax(z64, 1).permute(2, 0, 1)
    w = F.ctc_loss(lp, torch.tensor(targets), torch.tensor(frames), torch.tensor(tlen), blank=0, reduction="none",
                   zero_infinity=True)
    (w / torch.tensor(tlen, dtype=torch.float64).clamp(min=1)).mean().backward()
    return w.detach().numpy(), z64.grad.numpy()


def test_ctc_oracle_matches_torch_fp64():
    rng = np.random.RandomState(0)
    V, T = 7, 24
    rows = [(24, [1, 2, 3]), (24, []), (1, []), (6, [2, 2, 2, 4]), (5, [2, 2, 2, 4]), (24, [1, 1, 1, 1]),
            (6, [1, 1, 1, 1]), (8, [1, 1, 1, 1]), (13, list(rng.randint(1, V, 9))), (24, list(rng.randint(1, 3, 12))),
            (3, [5, 6]), (2, [5, 5])]
    B, L = len(rows), 12
    z = rng.randn(B, V, T) * 3
    frames = np.array([r[0] for r in rows])
    tg = np.zeros((B, L), np.int64)
    for b, (_, t) in enumerate(rows):
        tg[b, :len(t)] = t
    tl = np.array([len(r[1]) for r in rows])
    nll, mean, dz, inf = CO.ctc_batch(z, frames, tg, tl)
    w, g = _torch_ctc(z, frames, tg, tl)
    assert inf.tolist() == [False, False, False, False, True, False, True, False, False, inf[9], False, True]
    np.testing.assert_allclose(nll, w, rtol=1e-10, atol=0)
    np.testing.assert_allclose(dz, g, rtol=1e-10, atol=1e-14)
    assert mean == pytest.approx(float(np.mean(w / np.maximum(tl, 1))), rel=1e-12)
    assert (dz[inf] == 0).all() and (nll[inf] == 0).all()


@pytest.mark.parametrize("T", range(1, 7))
def test_ctc_oracle_matches_brute_force(T):
    rng = np.random.RandomState(T)
    for V in (2, 3, 4):
        for L in range(0, min(T, 3) + 1):
            for _ in range(2):
                labels = list(rng.randint(1, V, L))
                z = rng.randn(V, T)
                nll, dz, infeasible = CO.ctc(z, labels)
                if infeasible:
                    assert not CO.feasible(T, labels)
                    continue
                assert nll == pytest.approx(CO.brute_force_nll(z, labels), rel=1e-12)
                eps = 1e-6                                   # the gradient by central differences
                k = (rng.randint(V), rng.randint(T))
                zp, zm = z.copy(), z.copy()
                zp[k] += eps
                zm[k] -= eps
                num = (CO.brute_force_nll(zp, labels) - CO.brute_force_nll(zm, labels)) / (2 * eps)
                assert dz[k] == pytest.approx(num, rel=1e-5, abs=1e-8)


def test_greedy_oracle():
    z = np.full((1, 4, 8), -1.0)
    for t, v in enumerate([1, 1, 0, 1, 2, 2, 0, 0]):
        z[0, v, t] = 1.0
    z[0, 3, 3] = 1.0                                          # a tie at t = 3: the lower class, 1, wins
    assert CO.greedy(z, [8])[0].tolist() == [1, 1, 2]
    assert CO.greedy(z, [2])[0].tolist() == [1]


# ---- the edit-distance oracle -----------------------------------------------------------------------------------------
def test_edit_oracle_matches_brute_force():
    rng = np.random.RandomState(1)
    for _ in range(300):
        h, r = rng.randint(1, 4, rng.randint(0, 7)), rng.randint(1, 4, rng.randint(0, 7))
        d, s, dl, ins = CO.edit(h, r)
        assert d == CO.brute_force_distance(h, r)
        assert s + dl + ins == d and dl - ins == len(r) - len(h) and min(s, dl, ins) >= 0


def test_edit_tie_rule_hand_cases():
    # (hyp, ref) -> (distance, S, D, I) under the rule: diagonal, then deletion, then insertion
    cases = {((1, 2), (2, 1)): (2, 2, 0, 0),      # two substitutions beat a deletion plus an insertion
             ((1,), (2, 3)): (2, 1, 1, 0),        # (1 -> 2) then 3 missing: the diagonal first
             ((2, 3), (1,)): (2, 1, 0, 1),
             ((), (4, 5)): (2, 0, 2, 0), ((4, 5), ()): (2, 0, 0, 2), ((), ()): (0, 0, 0, 0),
             ((1, 2, 3), (1, 2, 3)): (0, 0, 0, 0),
             ((5, 6, 7), (6,)): (2, 0, 0, 2),
             ((1, 3), (1, 2, 3)): (1, 0, 1, 0)}
    for (h, r), want in cases.items():
        assert CO.edit(h, r) == want, (h, r)


def test_word_mapping():
    from deepvoice3_pytorch_b200.recognition import word_ids, words
    assert words([5, 6, 2, 7, 2, 2, 8], 2) == [(5, 6), (7,), (8,)]
    assert words([2, 2], 2) == [] and words([], 2) == []
    h, r = word_ids([np.array([5, 6, 2, 9]), np.array([7])], [np.array([5, 6, 2, 7]), np.array([7, 2, 5, 6])], 2)
    assert [x.tolist() for x in r] == [[0, 1], [1, 0]] and [x.tolist() for x in h] == [[0, 2], [1]]


# ---- C ABI and ptxas ----------------------------------------------------------------------------------------------------
NAMES = ("dv3_ctc_max_vocab", "dv3_ctc_ws_bytes", "dv3_ctc_fwd", "dv3_ctc_bwd", "dv3_ctc_greedy", "dv3_edit_ws_ints",
         "dv3_edit_distance")


def test_c_abi_declares_and_exports_the_recognition_kernels():
    from deepvoice3_pytorch_b200._lib import parse_header
    from deepvoice3_pytorch_b200.recognition import ctc_ws_bytes
    d = parse_header()
    args = {n: [a for _, a in d[n][1]] for n in NAMES}
    assert args["dv3_ctc_fwd"] == ["z", "stride_b", "stride_v", "frames", "targets", "tgt_stride", "target_lengths", "B",
                                   "V", "T", "L", "ws", "nll", "partials", "infeasible", "err_flag", "stream"]
    assert args["dv3_ctc_bwd"] == ["z", "stride_b", "stride_v", "frames", "targets", "tgt_stride", "target_lengths", "B",
                                   "V", "T", "L", "ws", "d_loss", "scale", "dz", "stream"]
    assert args["dv3_edit_distance"] == ["hyp", "hyp_stride", "hyp_len", "ref", "ref_stride", "ref_len", "P", "M_max",
                                         "N_max", "ws", "out", "err_flag", "stream"]
    P, I, LL, Fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
    assert [t for t, _ in d["dv3_ctc_bwd"][1]] == [P, LL, LL, P, P, LL, P, I, I, I, I, P, P, Fl, P, P]
    assert d["dv3_ctc_ws_bytes"][0] == LL and d["dv3_edit_ws_ints"][0] == LL
    so = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "libdv3b200.so")
    if os.path.exists(so):
        nm = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        for name in NAMES:
            assert re.search(r"\bT %s\b" % name, nm), name
        lib = ctypes.CDLL(so)
        lib.dv3_ctc_ws_bytes.restype = ctypes.c_longlong
        assert lib.dv3_ctc_max_vocab() == 1024
        for B, T, L in ((1, 1, 1), (16, 800, 200), (3, 7, 1024)):
            assert lib.dv3_ctc_ws_bytes(B, T, L) == ctc_ws_bytes(B, T, L)
        assert lib.dv3_ctc_ws_bytes(1, 1, 1025) == 0 and lib.dv3_ctc_ws_bytes(0, 1, 1) == 0


def test_ptxas_no_spills_zero_stack():
    nvcc = next((c for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc"))
                 if c and os.path.isfile(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "ctc.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rep = r.stdout + r.stderr
    frames = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", rep, flags=re.S)
    kernels = sorted(re.sub(r"^_ZN3dv3\d+(\w+?)E.*$", r"\1", n) for n, *_ in frames)
    assert kernels == ["ctc_alpha_kernel", "ctc_argmax_kernel", "ctc_beta_grad_kernel", "ctc_collapse_kernel",
                       "ctc_lse_kernel", "edit_distance_kernel"], rep
    for name, stack, st, ld in frames:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, stack, st, ld)


# ---- ArenaGraphStep batch keys -----------------------------------------------------------------------------------------
def test_arena_graph_steps_read_their_keys():
    from deepvoice3_pytorch_b200.recognition import TokenRecognizerStep
    from deepvoice3_pytorch_b200.speaker_classifier import SpeakerClassifierStep
    from deepvoice3_pytorch_b200.speaker_encoder import SpeakerEncoderStep
    from deepvoice3_pytorch_b200.train_step import ArenaGraphStep
    from deepvoice3_pytorch_b200.speaker_verifier import SpeakerVerifierStep
    assert ArenaGraphStep._batch_keys == ("mels", "speaker_ids")
    for cls in (SpeakerEncoderStep, SpeakerVerifierStep, SpeakerClassifierStep):
        assert cls._batch_keys == ("mels", "speaker_ids"), cls
    assert TokenRecognizerStep._batch_keys == ("mels", "mel_lengths", "tokens", "token_lengths")


# ---- RecognizerBatches -------------------------------------------------------------------------------------------------
class _Items(torch.utils.data.Dataset):
    def __init__(self, n, seed=0):
        rng = np.random.RandomState(seed)
        self.items = [(rng.randint(1, 30, rng.randint(0, 12)).astype(np.int32),
                       rng.rand(rng.randint(1, 70), 4).astype(np.float32)) for _ in range(n)]

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        return self.items[i]


def test_recognizer_batches():
    from deepvoice3_pytorch_b200.data import RecognizerBatches
    ds = _Items(60)
    rb = RecognizerBatches(ds, 4, 50, 10, seed=3)
    ok = [i for i, (t, m) in enumerate(ds.items) if m.shape[0] <= 50 and t.size <= 10]
    assert rb.eligible == ok and len(rb) == len(ok) // 4
    batches = list(rb)
    assert len(batches) == len(rb)
    seen = []
    for b in batches:
        assert b["mels"].shape == (4, 50, 4) and b["tokens"].shape == (4, 10)
        assert b["mel_lengths"].dtype == torch.int32 and b["token_lengths"].dtype == torch.int32
        for k, i in enumerate(b["items"].tolist()):
            t, m = ds.items[i]
            n = m.shape[0]
            assert int(b["mel_lengths"][k]) == n and int(b["token_lengths"][k]) == t.size
            assert np.array_equal(b["mels"][k, :n].numpy(), m) and (b["mels"][k, n:] == 0).all()
            assert b["tokens"][k, :t.size].tolist() == t.tolist() and (b["tokens"][k, t.size:] == 0).all()
            seen.append(i)
    assert len(set(seen)) == len(seen)
    again = [b["items"].tolist() for b in RecognizerBatches(ds, 4, 50, 10, seed=3)]
    assert again == [b["items"].tolist() for b in batches]
    rb.set_epoch(1)
    assert [b["items"].tolist() for b in rb] != again
    with pytest.raises(ValueError):
        RecognizerBatches(ds, 100, 50, 10)
    with pytest.raises(ValueError):
        RecognizerBatches(ds, 0, 50, 10)


# ---- refusals before any library call ---------------------------------------------------------------------------------
@pytest.fixture
def no_lib(monkeypatch):
    from deepvoice3_pytorch_b200._lib import lib
    calls = []
    monkeypatch.setattr(lib, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(lib, "raw", lambda name: calls.append(name))
    return calls


def test_ctc_refusals(no_lib):
    from deepvoice3_pytorch_b200.recognition import check_ctc, ctc_loss, greedy_decode
    for args in ((0, 5, 10, 3), (2, 1, 10, 3), (2, 1025, 10, 3), (2, 5, 10, 1025), (2, 5, 0, 3), (1024, 1024, 2048, 1),
                 (64, 100, 3000, 1024)):
        with pytest.raises(ValueError):
            check_ctc(*args)
    check_ctc(16, 149, 800, 200)
    z = torch.zeros(2, 5, 10)                     # a CPU tensor: refused
    bad = [(z, [10, 10], np.ones((2, 3), np.int64), [3, 3]), (z.double(), [10, 10], np.ones((2, 3)), [3, 3]),
           (torch.zeros(5, 10), [10], np.ones((1, 3), np.int64), [3])]
    for a in bad:
        with pytest.raises(ValueError):
            ctc_loss(*a)
        with pytest.raises(ValueError):
            greedy_decode(a[0], a[1])
    assert no_lib == []


def test_ctc_value_refusals_on_host_inputs(no_lib, monkeypatch):
    from deepvoice3_pytorch_b200 import recognition as R
    monkeypatch.setattr(R, "_check_logits", lambda z: tuple(z.shape))
    z = torch.zeros(2, 5, 10)
    tg = np.array([[1, 2, 3], [4, 4, 0]])
    bad = [([10, 11], tg, [3, 2]), ([0, 10], tg, [3, 2]), ([10, 10], tg, [4, 2]), ([10, 10], tg, [3, -1]),
           ([10, 10], np.array([[1, 2, 5], [4, 4, 0]]), [3, 2]), ([10, 10], np.array([[0, 2, 3], [4, 4, 0]]), [3, 2]),
           ([10], tg, [3, 2]), ([10, 10], tg.astype(float), [3, 2]), ([10.0, 10.0], tg, [3, 2]),
           ([10, 10], tg[:1], [3])]
    for fr, t, tl in bad:
        with pytest.raises(ValueError):
            R._check_ctc_inputs(z, fr, t, tl)
    assert R._check_ctc_inputs(z, [10, 10], tg, [3, 2]) == (2, 5, 10, 3)
    assert no_lib == []


def test_edit_distance_refusals(no_lib):
    from deepvoice3_pytorch_b200.recognition import edit_distance
    a = np.array([1, 2])
    bad = [([], []), ([a], []), ([a], [a, a]), ([a.astype(float)], [a]), ([a[:, None]], [a]),
           ([np.zeros(65536, np.int64)], [a]), ([a], [np.zeros(1025, np.int64)]),
           ([np.array([2 ** 40])], [a])]
    for h, r in bad:
        with pytest.raises(ValueError):
            edit_distance(h, r)
    assert no_lib == []


def test_recognizer_refusals(no_lib):
    from deepvoice3_pytorch_b200.recognition import TokenRecognizer, token_error_rates
    for kw in ({"n_vocab": 1}, {"n_vocab": 1025}, {"n_vocab": 30, "kernel_size": 4}, {"n_vocab": 30, "channels": 0},
               {"n_vocab": 30, "dilations": (1, 0)}, {"n_vocab": 30, "strip_ids": (0,)},
               {"n_vocab": 30, "strip_ids": (30,)}):
        with pytest.raises(ValueError):
            TokenRecognizer(**kw)
    rec = TokenRecognizer(30, channels=16, dilations=(1,))
    tok, n = rec.strip_batch(np.array([[3, 1, 4, 0], [1, 1, 0, 0]]), np.array([3, 2]))
    assert tok.tolist() == [[3, 4, 0, 0], [0, 0, 0, 0]] and n.tolist() == [2, 0]
    for t, l in ((np.array([[3, 30, 0]]), [2]), (np.array([[3, 0, 0]]), [2]), (np.array([[3, 4]]), [3]),
                 (np.array([3, 4]), [2])):
        with pytest.raises(ValueError):
            rec.strip_batch(t, np.array(l))
    for mels in ([], [np.zeros((5, 79))], [np.zeros((0, 80))], np.zeros((5, 80))):
        with pytest.raises(ValueError):
            rec.recognize(mels)
    m = [np.zeros((5, 80), np.float32)]
    for args in ((m, []), (m, [np.array([1, 2]), np.array([3])]), (m, [np.array([1.5])]),
                 (m, [np.arange(2, 1100)]), (m, [np.array([2, 3])], 0.5)):
        with pytest.raises(ValueError):
            token_error_rates(rec, *args)
    assert no_lib == []


def test_evaluate_recognition_refusals(no_lib):
    from deepvoice3_pytorch_b200.recognition import TokenRecognizer, evaluate_recognition
    from test_mcd_host import _models
    single, multi = _models()
    rec = TokenRecognizer(149, channels=16, dilations=(1,))
    seqs = [np.array([3, 4, 5]), np.array([6, 7])]
    bad_calls = [(single, rec, seqs, [0, 1], {}), (multi, rec, seqs, None, {}), (single, rec, [], None, {}),
                 (single, rec, [np.array([3.0])], None, {}), (single, rec, seqs, None, {"batch_size": 0}),
                 (single, TokenRecognizer(5, channels=16, dilations=(1,)), seqs, None, {}),
                 (single, TokenRecognizer(149, mel_dim=40, channels=16, dilations=(1,)), seqs, None, {}),
                 (single, rec, seqs, None, {"vocoder": "wavenet"})]
    for model, r, sq, ids, kw in bad_calls:
        with pytest.raises(ValueError):
            evaluate_recognition(model, r, sq, speaker_ids=ids, **kw)
    assert no_lib == []
