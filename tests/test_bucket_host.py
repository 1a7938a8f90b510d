"""CPU: bucket rounding and padding of a collated batch (data.bucket_shape / pad_to_bucket), and the C ABI of the
extent variants of the kernels."""
import ctypes

import numpy as np
import pytest
import torch

from deepvoice3_pytorch_b200 import data, ops


def _collated(multi=False):
    rng = np.random.RandomState(0)
    items = []
    for i, (n, t) in enumerate([(23, 70), (17, 51), (9, 33)]):
        item = (rng.randint(2, 149, n).astype(np.int32), rng.rand(t, 80).astype(np.float32),
                rng.rand(t, 129).astype(np.float32))
        items.append(item + (i,) if multi else item)
    return data.collate(items, r=1, downsample_step=4)


def test_bucket_shape_rounds_up_to_the_grid():
    assert data.bucket_shape(1, 1) == (data.BUCKET_TEXT, data.BUCKET_DEC)
    assert data.bucket_shape(data.BUCKET_TEXT, data.BUCKET_DEC) == (data.BUCKET_TEXT, data.BUCKET_DEC)
    assert data.bucket_shape(data.BUCKET_TEXT + 1, 2 * data.BUCKET_DEC - 1) == (2 * data.BUCKET_TEXT,
                                                                                 2 * data.BUCKET_DEC)
    for t in range(1, 300):
        bt, bd = data.bucket_shape(t, t)
        assert bt >= t and bd >= t and bt - t < data.BUCKET_TEXT and bd - t < data.BUCKET_DEC
        assert bt % 4 == 0 and bd % 4 == 0


@pytest.mark.parametrize("multi", [False, True])
def test_pad_to_bucket_content_and_extents(multi):
    b = _collated(multi)
    ext = data.batch_extents(b)
    T_dec, T_text = ext[0], ext[1]
    assert ext == (b["done"].shape[1], b["x"].shape[1], T_dec, 4 * T_dec)
    p = data.pad_to_bucket(b, T_text + 9, T_dec + 6)
    assert p["extents"].dtype == torch.int64 and p["extents"].tolist() == list(ext)
    assert data.batch_extents(p) == (T_dec + 6, T_text + 9, T_dec + 6, 4 * (T_dec + 6))
    for k, T in (("x", T_text), ("text_positions", T_text), ("frame_positions", T_dec), ("mel", T_dec),
                 ("y", 4 * T_dec), ("done", T_dec)):
        assert torch.equal(p[k][:, :T], b[k]), k
        assert not p[k][:, T:].any(), k                  # zeros (frame positions 0) past the logical extent
    assert int(p["frame_positions"].max()) == T_dec      # never past the logical positions: max_positions holds
    for k in ("target_lengths", "input_lengths_dev") + (("speaker_ids",) if multi else ()):
        assert torch.equal(p[k], b[k])
    assert np.array_equal(p["input_lengths"], b["input_lengths"])
    # in place into an existing bucket: same result
    q = {k: (torch.full_like(v, 7) if torch.is_tensor(v) else v) for k, v in p.items()}
    data.pad_to_bucket(b, T_text + 9, T_dec + 6, out=q)
    for k, v in p.items():
        assert (torch.equal(q[k], v) if torch.is_tensor(v) else np.array_equal(q[k], v)), k


def test_pad_to_bucket_refusals():
    b = _collated()
    ext = data.batch_extents(b)
    with pytest.raises(ValueError):
        data.pad_to_bucket(b, ext[1] - 1, ext[0])        # bucket smaller than the batch
    with pytest.raises(ValueError):
        data.pad_to_bucket(b, ext[1], ext[0] - 1)
    with pytest.raises(ValueError):
        data.pad_to_bucket(b, ext[1], ext[0], r=2)       # shapes of another r
    with pytest.raises(ValueError):
        data.pad_to_bucket(data.pad_to_bucket(b, ext[1], ext[0]), ext[1], ext[0])    # already padded


def test_extent_scope_refusals_and_training_loss_refuses_extents():
    from deepvoice3_pytorch_b200._lib import Dv3Error
    from deepvoice3_pytorch_b200.train_step import training_loss
    with pytest.raises(Dv3Error):
        with ops.extent_scope(torch.zeros(4, dtype=torch.int64), (1, 1, 1, 1)):      # not on the device
            pass
    assert ops._extent is None
    with ops.extent_axis(ops.EXT_TEXT):                  # no scope: a no-op
        x = torch.zeros(1, 2, 3)
        assert ops.mask_time(x) is x
    with pytest.raises(ValueError, match="extents"):
        training_loss(None, {"extents": torch.zeros(4, dtype=torch.int64)})


def test_extent_entry_points_match_the_header():
    """The new entry points are declared in include/dv3b200.h with the argument types the Python side passes and are
    exported by the library."""
    from deepvoice3_pytorch_b200 import _build
    from deepvoice3_pytorch_b200._lib import parse_header, LIB_PATH
    _build.build()
    decls = parse_header()
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    LL, U = ctypes.c_longlong, ctypes.c_uint
    want = {
        "dv3_mask_frames": [P, P, P, I, I, I, I, P],
        "dv3_spec_loss_ext": [P, P, P, P, P, P, I, I, I, I, F, F, I, F, P],
        "dv3_aux_loss_ext": [P, P, P, P, P, P, P, P, I, I, I, I, F, I, P, P],
        "dv3_tc_attn_fwd_ext": [P, P, P, P, P, P, I, I, I, I, P, F, P, U, P],
        "dv3_tc_attn_bwd_ext": [P] * 10 + [I, I, I, I, P, F, P, U, P],
        "dv3_bgemm_ctx_scale": [P, LL, LL, LL, P, LL, LL, LL, P, LL, I, I, I, I, I, P, I, P],
        "dv3_tc_split_input_ext": [P, P, I, P, I, I, I, F, P, U, P, I, P],
        "dv3_tc_gate_bwd_split_ext": [P, P, P, P, P, P, P, I, I, I, I, I, P, I, P],
        "dv3_tc_grad_split_ext": [P, P, P, P, P, I, I, I, I, P, I, P],
    }
    dll = ctypes.CDLL(LIB_PATH)
    for name, args in want.items():
        assert name in decls, name
        assert [t for t, _ in decls[name][1]] == args, name
        assert hasattr(dll, name), name
