"""Loader (and writer) of the golden vectors of tests/golden/make_golden.py and make_train_golden.py.

A fixture set "<stem>.npz" is one compressed file tests/golden/<stem>.npz when it fits in SHARD_BYTES, else the
directory tests/golden/<stem>/ with one .npz per case, or per (case, group) where a whole case would not fit; array
keys are "case|group|name" in every layout.
"""
import glob
import io
import os
from collections import defaultdict

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHARD_BYTES = 900 * 1024          # keeps every stored file well under 1 MB
_cache = {}


def _npz_bytes(arrays):
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    return buf.getvalue()


def save(fname, arrays):
    """Write {"case|group|name": array} as the fixture set fname (see the module docstring)."""
    stem = os.path.join(GOLDEN, os.path.splitext(fname)[0])
    for old in glob.glob(os.path.join(stem, "*.npz")) + glob.glob(stem + ".npz"):
        os.remove(old)
    data = _npz_bytes(arrays)
    if len(data) <= SHARD_BYTES:
        with open(stem + ".npz", "wb") as f:
            f.write(data)
        return
    os.makedirs(stem, exist_ok=True)
    cases = defaultdict(dict)
    for key, v in arrays.items():
        cases[key.split("|")[0]][key] = v
    for case, d in cases.items():
        data = _npz_bytes(d)
        if len(data) <= SHARD_BYTES:
            shards = {case: data}
        else:
            groups = defaultdict(dict)
            for key, v in d.items():
                groups[key.split("|")[1]][key] = v
            shards = {"%s.%s" % (case, g): _npz_bytes(gd) for g, gd in groups.items()}
        for name, data in shards.items():
            assert len(data) <= SHARD_BYTES, "golden shard %s/%s is %d bytes" % (stem, name, len(data))
            with open(os.path.join(stem, name + ".npz"), "wb") as f:
                f.write(data)


def load(fname):
    """-> {case: {group: {name: np.ndarray}}}"""
    if fname not in _cache:
        stem = os.path.join(GOLDEN, os.path.splitext(fname)[0])
        paths = sorted(glob.glob(os.path.join(stem, "*.npz"))) or [os.path.join(GOLDEN, fname)]
        out = defaultdict(lambda: defaultdict(dict))
        for path in paths:
            z = np.load(path, allow_pickle=False)
            for key in z.files:
                case, group, name = key.split("|")
                out[case][group][name] = z[key]
        _cache[fname] = out
    return _cache[fname]


def tensors(d, device="cpu", dtype=None):
    out = {}
    for k, v in d.items():
        t = torch.from_numpy(np.ascontiguousarray(v))
        if dtype is not None and t.is_floating_point():
            t = t.to(dtype)
        out[k] = t.to(device)
    return out


def loss_weights(shape, i, device="cpu", dtype=torch.float32):
    """Same projection tensor as make_golden.loss_weights."""
    n = int(np.prod(shape))
    return torch.cos(torch.arange(n, dtype=torch.float64) * 0.37 + i).to(torch.float32) \
        .reshape(shape).to(device=device, dtype=dtype)


def meta_scalar(case, name):
    return case["meta"][name].item()


def kwargs_of(case):
    kw = {}
    for k, v in case["kw"].items():
        if v.dtype.kind in "US":
            kw[k] = str(v)
        elif v.dtype.kind == "b":
            kw[k] = bool(v)
        elif v.dtype.kind in "iu":
            kw[k] = int(v)
        else:
            kw[k] = float(v)
    return kw
