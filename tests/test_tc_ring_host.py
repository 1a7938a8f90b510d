"""Host part of the ring-depth checks (no GPU needed).

* A probe compiled from csrc/tc_ring.cuh alone with the host C++ compiler prints the ring depth, stage bytes and total
  shared memory of every tc_conv_kernel configuration and of both weight-gradient rings: each fits the 227 KB opt-in
  limit and has the depth tests/test_gpu_tc_ring.py walks.
* `-Xptxas -v` of tc_gemm.cu: every tc_conv_kernel and tc_wgrad_mn_kernel instantiation with 0 spill bytes, a 0-byte
  stack frame and no C7511 (serialised wgmma chain).
"""
import os
import re
import shutil
import subprocess

import pytest

from test_gpu_tc_ring import CONV_STAGES, WGRAD_STAGES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc")
SMEM_LIMIT = 227 * 1024

PROBE = r"""
#include <cstdio>
#include "tc_ring.cuh"
using namespace dv3;
template <class C> void row(const char* name) {
    std::printf("%s %d %d %d %d\n", name, C::STAGES, C::STAGE, C::SMEM, C::MAX_STAGES);
}
#define CONV(NBOX, BK, BR, NPL) row<TcCfg<NBOX, BK, BR, NPL>>("conv," #NBOX "," #BR "," #BK "," #NPL)
int main() {
    CONV(2, 32, 64, 2); CONV(1, 32, 128, 2); CONV(1, 64, 64, 2); CONV(1, 32, 64, 2);
    CONV(2, 64, 64, 1); CONV(1, 64, 128, 1); CONV(1, 32, 128, 1); CONV(1, 64, 64, 1); CONV(1, 32, 64, 1);
    row<WgCfg<2>>("wgrad,2"); row<WgCfg<1>>("wgrad,1");
    std::printf("limit %d\n", SMEM_LIMIT);
}
"""


def _tool(*names):
    for cand in names:
        path = cand if cand and os.path.isabs(cand) else shutil.which(cand or "")
        if path and os.path.isfile(path) and os.access(path, os.X_OK):
            return path
    return None


@pytest.fixture(scope="module")
def ring_table(tmp_path_factory):
    cxx = _tool(os.environ.get("CXX"), "g++", "c++", "clang++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("ring_probe")
    (d / "probe.cpp").write_text(PROBE)
    r = subprocess.run([cxx, "-std=c++17", "-I", CSRC, str(d / "probe.cpp"), "-o", str(d / "probe")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = subprocess.run([str(d / "probe")], capture_output=True, text=True, check=True).stdout
    rows = {}
    for line in out.splitlines():
        name, *vals = line.split()
        rows[name] = tuple(int(v) for v in vals)
    return rows


def test_probe_limit_is_227_kb(ring_table):
    assert ring_table["limit"] == (SMEM_LIMIT,)


def test_every_ring_fits_and_has_its_depth(ring_table):
    want = {"conv,%d,%d,%d,%d" % k: v for k, v in CONV_STAGES.items()}
    want.update({"wgrad,%d" % k: v for k, v in WGRAD_STAGES.items()})
    got = {k: v for k, v in ring_table.items() if k != "limit"}
    assert set(got) == set(want)
    for name, (stages, stage, smem, max_stages) in got.items():
        print("%-14s %d x %6d B stages, %6d B of %d" % (name, stages, stage, smem, SMEM_LIMIT))
        assert stages == want[name], name
        assert 2 <= stages <= max_stages and smem <= SMEM_LIMIT, name
        assert stage % 1024 == 0, name


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _tool(os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas") / "tc_gemm.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, "tc_gemm.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def test_pipeline_kernels_keep_no_spills_no_stack_no_serialisation(ptxas_report):
    kernels, cur = {}, None
    for line in ptxas_report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if ("tc_conv_kernel" in m.group(1) or "tc_wgrad_mn_kernel" in m.group(1)) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            kernels[cur] = tuple(int(v) for v in m.groups())
            cur = None
    assert sum("tc_conv_kernel" in k for k in kernels) == 16 and sum("tc_wgrad_mn_kernel" in k for k in kernels) == 2
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert not bad, "stack frame / spill store / spill load bytes: %s" % bad
    serial = [l for l in ptxas_report.splitlines() if "C7511" in l]
    assert not serial, "ptxas serialises a wgmma chain:\n" + "\n".join(serial)
