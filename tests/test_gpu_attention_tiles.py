"""GPU: tile edges of the query-tiled tensor-core attention kernels (csrc/tc_attn.cu: 64-row query tiles in the rows
kernels, 64-channel tiles in the key/value-gradient kernel), against the fp64 references and elementwise bounds of
test_gpu_attention.py (dropout off) and test_gpu_dropout.py (dropout on):

  * Td around the 64-row tile (1, 63, 64, 65, 128, 200, 257), Ts around the 64-key slabs (1, 64, 100, 128),
    E = 16 / 80 / 256 (one partial or two full channel tiles), B = 1 / 16; keys masked or not, dropout on or off;
  * every output in a sentinel-guarded buffer: nothing written outside it, every element inside written;
  * two launches bit-identical; row b of a batched launch bit-identical to row b launched alone;
  * the _ext entry points with a logical key count below Ts.
"""
import math

import pytest
import torch

import test_gpu_attention as A
import test_gpu_dropout as D
from oracle import dropout_mask as DM

pytestmark = pytest.mark.gpu

SENT = -3.0e38
GUARD = 4096
TDS, TSS, ES, BS = (1, 63, 64, 65, 128, 200, 257), (1, 64, 100, 128), (16, 80, 256), (1, 16)


def _guarded(shape):
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), SENT, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(*shape)


def run(q, k, v, mask, dout, dprobs, p=0.0, seed=0, salt=0, ts_log=None):
    """Forward and backward on guarded outputs -> {name: tensor}; asserts every output is written exactly in place."""
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import lib
    B, E, Td = q.shape
    Ts = k.shape[2]
    sc = A._scale(Ts)
    shapes = {"probs": (B, Td, Ts), "out": (B, E, Td), "ds": (B, Td, Ts), "dq": (B, E, Td), "dk": (B, E, Ts),
              "dv": (B, E, Ts)}
    g = {n: _guarded(s) for n, s in shapes.items()}
    t = {n: view for n, (_, view) in g.items()}
    m8 = None if mask is None else mask.to(torch.uint8).contiguous()
    seed_t = torch.tensor([seed], dtype=torch.int64, device="cuda") if p > 0 else None
    tl = None if ts_log is None else torch.tensor([ts_log], dtype=torch.int64, device="cuda")
    P = ops._p
    if tl is None:
        lib.call("dv3_tc_attn_fwd", P(q), P(k), P(v), P(m8), P(t["probs"]), P(t["out"]), B, E, Td, Ts, sc, p,
                 P(seed_t), salt, ops._stream())
        lib.call("dv3_tc_attn_bwd", P(dout), P(q), P(k), P(v), P(t["probs"]), P(dprobs), P(t["ds"]), P(t["dq"]),
                 P(t["dk"]), P(t["dv"]), B, E, Td, Ts, sc, p, P(seed_t), salt, ops._stream())
    else:
        lib.call("dv3_tc_attn_fwd_ext", P(q), P(k), P(v), P(m8), P(t["probs"]), P(t["out"]), B, E, Td, Ts, P(tl), p,
                 P(seed_t), salt, ops._stream())
        lib.call("dv3_tc_attn_bwd_ext", P(dout), P(q), P(k), P(v), P(t["probs"]), P(dprobs), P(t["ds"]), P(t["dq"]),
                 P(t["dk"]), P(t["dv"]), B, E, Td, Ts, P(tl), p, P(seed_t), salt, ops._stream())
    torch.cuda.synchronize()
    for n, (buf, view) in g.items():
        assert bool((buf[:GUARD] == SENT).all()) and bool((buf[GUARD + view.numel():] == SENT).all()), \
            "%s: written outside the tensor" % n
        assert not bool((view == SENT).any()), "%s: %d elements not written" % (n, int((view == SENT).sum()))
    return t


def _cases():
    """Every (Td, Ts) pair; E, B, key mask, dropout and dprobs rotate so that each takes every value."""
    out = []
    for i, (Td, Ts) in enumerate((a, b) for a in TDS for b in TSS):
        out.append((BS[(i // 3) % 2], ES[i % 3], Td, Ts, i % 2 == 0, (i // 2) % 2 == 1, i % 5 != 0))
    return out


@pytest.mark.parametrize("B,E,Td,Ts,masked,drop,use_dp", _cases())
def test_attention_tile_edges(B, E, Td, Ts, masked, drop, use_dp):
    i = TDS.index(Td) * len(TSS) + TSS.index(Ts)
    q, k, v, dout, dprobs, mask = A.inputs(B, E, Td, Ts, 500 + i, A.mask_lengths(B, Ts, i) if masked else None)
    dp = dprobs if use_dp else None
    p, seed, salt = (0.25, 77 + i, 3) if drop else (0.0, 0, 0)
    got = run(q, k, v, mask, dout, dp, p, seed, salt)
    what = "B=%d E=%d Td=%d Ts=%d mask=%s p=%g dprobs=%s" % (B, E, Td, Ts, masked, p, use_dp)
    dmask = torch.from_numpy(DM.mask(seed, salt, p, (B, Td, Ts))).cuda().double() if drop else None
    P, out, bP, bout = A.ref_forward(q.double(), k.double(), v.double(), mask, dmask)
    r = A.check_forward(got["probs"], got["out"], P, out, bP, bout, mask, what)
    if not drop:
        ref = A.ref_backward(q.double(), k.double(), v.double(), got["probs"].double(), dout.double(),
                             None if dp is None else dp.double())
        r.update(A.check_backward(got, ref, what))
    else:
        ref = D._attn_ref(q, k, v, mask, dmask, dout, dp)
        ex = {n: D.excess(got[n], ref[n], grad=True) for n in ("dq", "dk", "dv")}
        assert max(ex.values()) <= 1, "%s: error / tolerance %s" % (what, ex)
        r.update(ex)
    print("%s: %s" % (what, " ".join("%s %.3g" % kv for kv in sorted(r.items()))))


def test_attention_tiles_repeat_bit_identical():
    B, E, Td, Ts = 16, 256, 200, 128
    q, k, v, dout, dprobs, mask = A.inputs(B, E, Td, Ts, 7, A.mask_lengths(B, Ts, 3))
    a = run(q, k, v, mask, dout, 1e-3 * dprobs, 0.05, 1234, 5)
    b = run(q, k, v, mask, dout, 1e-3 * dprobs, 0.05, 1234, 5)
    diff = [n for n in a if not torch.equal(a[n], b[n])]
    assert not diff, "two launches differ in %s" % diff


def test_attention_tiles_row_alone_bit_identical():
    """Row b of a batched launch is computed exactly as if launched alone (no dropout: its mask index depends on b)."""
    B, E, Td, Ts = 16, 80, 200, 100
    q, k, v, dout, dprobs, mask = A.inputs(B, E, Td, Ts, 8, A.mask_lengths(B, Ts, 1))
    full = run(q, k, v, mask, dout, dprobs)
    for b in range(B):
        one = run(*[t[b:b + 1].contiguous() for t in (q, k, v, mask, dout, dprobs)])
        diff = [n for n in one if not torch.equal(one[n][0], full[n][b])]
        assert not diff, "row %d alone differs in %s" % (b, diff)


@pytest.mark.parametrize("B,E,Td,Ts,ts_log", [(16, 256, 200, 128, 100), (3, 80, 65, 64, 1), (1, 16, 257, 100, 63)])
def test_attention_tiles_ext_ts_log(B, E, Td, Ts, ts_log):
    """The _ext entry points scale the context by the logical key count ts_log < Ts (a batch padded to a bucket)."""
    q, k, v, dout, dprobs, mask = A.inputs(B, E, Td, Ts, 9 + Ts, A.mask_lengths(B, Ts, 2))
    got = run(q, k, v, mask, dout, dprobs, ts_log=ts_log)
    f = A._scale(ts_log) / A._scale(Ts)
    what = "ext B=%d E=%d Td=%d Ts=%d ts_log=%d" % (B, E, Td, Ts, ts_log)
    P, out, bP, bout = A.ref_forward(q.double(), k.double(), v.double(), mask)
    r = A.check_forward(got["probs"], got["out"], P, f * out, bP, f * bout, mask, what)
    # scale(ts_log) dO.V == scale(Ts) (f dO).V: the fp64 backward of A.ref_backward with dO scaled by f
    ref = A.ref_backward(q.double(), k.double(), v.double(), got["probs"].double(), f * dout.double(), dprobs.double())
    r.update(A.check_backward(got, ref, what))
    print("%s: %s" % (what, " ".join("%s %.3g" % kv for kv in sorted(r.items()))))
