"""Compile-time guard of the single-pass (NPL = 1) tensor-core kernels (no GPU needed): every NPL = 1 instantiation of
tc_conv_kernel and tc_wgrad_mn_kernel keeps its wgmma chain pipelined (no ptxas C7511), does not spill and uses no local
memory (0-byte stack frame)."""
import os
import re
import subprocess

import pytest

from test_tc_ptxas import SRC, _nvcc


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas1") / "tc_gemm.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", SRC, "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _single_pass(name):
    """tc_conv_kernel<MODE, NBOX, BR, BK, BF16, 1> / tc_wgrad_mn_kernel<1> (Itanium mangling)"""
    return ("tc_conv_kernel" in name and name.split("EEEv")[0].endswith("ELi1")) or "tc_wgrad_mn_kernelILi1EE" in name


def _kernels(report):
    kernels, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if _single_pass(m.group(1)) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            kernels[cur] = (int(m.group(1)), int(m.group(2)), int(m.group(3)))
            cur = None
    return kernels


def test_every_single_pass_instantiation_is_compiled_gated_fp16_only(report):
    names = list(_kernels(report))
    # gated forward (fp16 operands only: it is always a forward GEMM) + 4 conv configurations, each for fp16 and bf16
    # operands; one weight-gradient kernel
    assert sum("tc_conv_kernel" in n for n in names) == 9, names
    gated = [n for n in names if "tc_conv_kernelILi0E" in n]      # MODE = TC_GATED
    assert len(gated) == 1 and "ELb0ELi1E" in gated[0], gated     # BF16 = false
    assert sum("tc_wgrad_mn_kernel" in n for n in names) == 1, names


def test_single_pass_wgmma_not_serialized(report):
    bad = [l for l in report.splitlines() if "C7511" in l]
    assert not bad, "ptxas serialises a wgmma chain:\n" + "\n".join(bad)


def test_single_pass_no_spills_no_stack_frame(report):
    kernels = _kernels(report)
    assert kernels
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, "single-pass kernels with stack frame / spill stores / spill loads: %s" % bad
