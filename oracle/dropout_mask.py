"""TEST INFRASTRUCTURE ONLY.  numpy restatement of the package's counter-based dropout mask.

The kernels never store a mask: every site that applies one, or rebuilds it in a backward pass, evaluates
(deepvoice3_pytorch_b200/csrc/common.cuh ``mix32`` / ``make_drop`` / ``drop_scale``)

    s0 = mix32(lo32(seed) ^ (salt * 0x9E3779B1))        s1 = mix32(hi32(seed) + salt + 0x85ebca6b)
    keep(i) = mix32(mix32(i ^ s0) + s1) >= thresh,       thresh = (uint32)(double(float(p)) * 2^32), clamped
    scale   = 1.f / (1.f - p)                            (float32 arithmetic)

with ``seed`` the 8-byte step seed in device memory (``ops.rng.seed``, an int64 tensor read as uint64), ``salt``
the call site's number in the forward (``ops.rng.next_salt``) and ``i`` the flat element index cast to uint32.
This is the package's own contract -- nothing here restates the reference model -- and tests/test_gpu_dropout.py
pins it to the device bit for bit.  Tensors of more than 2^32 elements (where the uint32 index wraps) are out of
scope.
"""
import numpy as np

M32 = 0xFFFFFFFF
M64 = 0xFFFFFFFFFFFFFFFF


def mix32(x):
    """The 32-bit finaliser of common.cuh on a uint64 array holding uint32 values (products taken mod 2^32)."""
    x = np.asarray(x, dtype=np.uint64)
    x = x ^ (x >> np.uint64(16))
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x = x ^ (x >> np.uint64(15))
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    return x ^ (x >> np.uint64(16))


def _mix32_int(x):
    return int(mix32(np.uint64(x & M32)))


def seed_u64(seed):
    """The device's view of a step seed: an int64 (possibly negative after ``advance()`` wrapped it), a python int
    or a one-element int64 tensor -> its unsigned 64-bit pattern."""
    if hasattr(seed, "item"):
        seed = seed.item()
    return int(seed) & M64


def threshold(p):
    """Drop iff hash < threshold: (uint32)(double(float(p)) * 2^32), clamped to 0xFFFFFFFF as make_drop does."""
    t = float(np.float32(p)) * 4294967296.0
    return M32 if t >= 4294967295.0 else int(t)


def scale(p):
    """The float32 1.f / (1.f - p) of a kept element."""
    one = np.float32(1.0)
    return np.float32(one / (one - np.float32(p)))


def mask(seed, salt, p, shape):
    """float32 array of ``shape``: 0 where the device drops element i (flat index), 1/(1-p) where it keeps it;
    all ones when dropout is off (p <= 0)."""
    shape = (int(shape),) if np.isscalar(shape) else tuple(int(n) for n in shape)
    n = int(np.prod(shape, dtype=np.int64))
    if not np.float32(p) > 0:
        return np.ones(shape, dtype=np.float32)
    s = seed_u64(seed)
    salt = int(salt) & M32
    s0 = _mix32_int((s & M32) ^ ((salt * 0x9E3779B1) & M32))
    s1 = _mix32_int(((s >> 32) + salt + 0x85EBCA6B) & M32)
    idx = np.arange(n, dtype=np.uint64) & np.uint64(M32)
    h = mix32((mix32(idx ^ np.uint64(s0)) + np.uint64(s1)) & np.uint64(M32))
    keep = h >= np.uint64(threshold(p))
    return np.where(keep, scale(p), np.float32(0.0)).astype(np.float32).reshape(shape)
