"""Compile-time guard of the tensor-core conv kernel (no GPU needed): every tc_conv_kernel instantiation must keep its
wgmma chain pipelined (no ptxas C7511 "wgmma.mma_async instructions are serialized"), must not spill and must use no
local memory at all (0-byte stack frame)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc", "tc_gemm.cu")


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas") / "tc_gemm.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", SRC, "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _conv_kernels(report):
    """-> {mangled name: (stack frame bytes, spill store bytes, spill load bytes)} of every tc_conv_kernel
    instantiation."""
    kernels, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "tc_conv_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            kernels[cur] = (int(m.group(1)), int(m.group(2)), int(m.group(3)))
            cur = None
    return kernels


def test_tc_conv_kernel_wgmma_not_serialized(ptxas_report):
    assert _conv_kernels(ptxas_report), "no tc_conv_kernel instantiation in the ptxas report"
    bad = [l for l in ptxas_report.splitlines() if "C7511" in l and "tc_conv_kernel" in l]
    assert not bad, "ptxas serialises the wgmma chain:\n" + "\n".join(bad)


def test_tc_conv_kernel_no_spills(ptxas_report):
    kernels = _conv_kernels(ptxas_report)
    assert kernels, "no tc_conv_kernel instantiation in the ptxas report"
    spilling = {k: v[1:] for k, v in kernels.items() if v[1:] != (0, 0)}
    assert not spilling, "tc_conv_kernel spills (store, load bytes): %s" % spilling


def test_tc_conv_kernel_no_stack_frame(ptxas_report):
    kernels = _conv_kernels(ptxas_report)
    assert kernels, "no tc_conv_kernel instantiation in the ptxas report"
    framed = {k: v[0] for k, v in kernels.items() if v[0] != 0}
    assert not framed, "tc_conv_kernel uses local memory (stack frame bytes): %s" % framed
