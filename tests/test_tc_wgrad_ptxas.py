"""Compile-time guard of the persistent tensor-core weight gradient (no GPU needed): both tc_wgrad_mn_kernel
instantiations (NPL = 1, 2) keep their wgmma chain pipelined (no ptxas C7511), do not spill and use no local memory
(0-byte stack frame)."""
import re

from test_tc_ptxas import ptxas_report  # noqa: F401  (module-scoped fixture: one compile of tc_gemm.cu)


def _wgrad_kernels(report):
    """-> {mangled name: (stack frame bytes, spill store bytes, spill load bytes)} of every tc_wgrad_mn_kernel."""
    kernels, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "tc_wgrad_mn_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            kernels[cur] = (int(m.group(1)), int(m.group(2)), int(m.group(3)))
            cur = None
    return kernels


def test_tc_wgrad_both_plane_counts(ptxas_report):  # noqa: F811
    names = sorted(_wgrad_kernels(ptxas_report))
    assert len(names) == 2 and any("ILi1E" in n for n in names) and any("ILi2E" in n for n in names), names


def test_tc_wgrad_wgmma_not_serialized(ptxas_report):  # noqa: F811
    bad = [l for l in ptxas_report.splitlines() if "C7511" in l and "tc_wgrad_mn_kernel" in l]
    assert not bad, "ptxas serialises the wgmma chain:\n" + "\n".join(bad)


def test_tc_wgrad_no_spills_no_stack(ptxas_report):  # noqa: F811
    kernels = _wgrad_kernels(ptxas_report)
    bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
    assert kernels and not bad, "tc_wgrad_mn_kernel stack frame / spill bytes: %s" % bad
