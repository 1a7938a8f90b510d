"""Compile-time guard of the tensor-core attention kernels (no GPU needed): attn_rows_kernel<0/1> and attn_cols_kernel
must keep their wgmma chains pipelined (no ptxas C7511 "wgmma.mma_async instructions are serialized"), must not spill
and must use no local memory at all (0-byte stack frame)."""
import os
import re
import subprocess

import pytest

from test_tc_ptxas import _nvcc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "tc_attn.cu")
KERNELS = ("attn_rows_kernel", "attn_cols_kernel")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas") / "tc_attn.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", SRC, "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _attn_kernels(report):
    """-> {mangled name: (stack frame bytes, spill store bytes, spill load bytes)} of every attention kernel."""
    kernels, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            kernels[cur] = (int(m.group(1)), int(m.group(2)), int(m.group(3)))
            cur = None
    return kernels


def test_attn_kernels_present(ptxas_report):
    names = _attn_kernels(ptxas_report)
    assert len(names) == 3, "expected attn_rows_kernel<0>, <1> and attn_cols_kernel, got %s" % sorted(names)


def test_attn_wgmma_not_serialized(ptxas_report):
    bad = [l for l in ptxas_report.splitlines() if "C7511" in l and any(k in l for k in KERNELS)]
    assert not bad, "ptxas serialises the wgmma chain:\n" + "\n".join(bad)


def test_attn_no_spills_no_stack_frame(ptxas_report):
    kernels = _attn_kernels(ptxas_report)
    assert kernels, "no attention kernel in the ptxas report"
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, "attention kernels use local memory (stack frame, spill store, spill load bytes): %s" % bad
