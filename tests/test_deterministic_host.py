"""No GPU: the deterministic training mode's C ABI, its switch, a source guard over every float atomicAdd of the
library, and the ptxas report of the new kernels (DESIGN.md section 2.10)."""
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepvoice3_pytorch_b200", "csrc")

DET_SYMBOLS = ["dv3_loss_det_scratch_floats", "dv3_spec_loss_det", "dv3_aux_loss_det", "dv3_bias_det_scratch_floats",
               "dv3_convblock_gate_bwd_det", "dv3_bias_act_bwd_det", "dv3_tc_gate_bwd_split_det",
               "dv3_tc_grad_split_det", "dv3_embedding_bwd_det", "dv3_sinusoid_bwd_det"]


def test_symbols_in_header_library_and_binding():
    from deepvoice3_pytorch_b200._lib import lib, parse_header
    decls = parse_header()
    lib.load()
    for name in DET_SYMBOLS:
        assert name in decls, name
        assert callable(lib.raw(name)), name
    assert lib.raw("dv3_loss_det_scratch_floats")() == 3 * 132 * 8 + 1
    fn = lib.raw("dv3_bias_det_scratch_floats")
    assert fn(16, 1024, 800, 1) == 16 * 13 * 1024 and fn(16, 1024, 800, 0) == 16 * 1024
    # the twins take their atomic form's arguments plus the scratch: no existing declaration changed its arity
    assert len(decls["dv3_spec_loss_det"][1]) == len(decls["dv3_spec_loss_terms"][1]) + 1
    assert len(decls["dv3_aux_loss_det"][1]) == len(decls["dv3_aux_loss_terms"][1]) + 1
    assert len(decls["dv3_embedding_bwd_det"][1]) == len(decls["dv3_embedding_bwd"][1])
    assert len(decls["dv3_sinusoid_bwd_det"][1]) == len(decls["dv3_sinusoid_bwd"][1])


def test_switch_parses(monkeypatch):
    from deepvoice3_pytorch_b200 import ops
    from deepvoice3_pytorch_b200._lib import Dv3Error
    assert os.environ.get("DV3_DETERMINISTIC", "0") != "0" or ops.is_deterministic() is False
    for value, want in (("0", False), ("1", True), (False, False), (True, True)):
        monkeypatch.setattr(ops, "deterministic", value)
        assert ops.is_deterministic() is want
    for bad in ("yes", "2", "", None):
        monkeypatch.setattr(ops, "deterministic", bad)
        with pytest.raises(Dv3Error):
            ops.is_deterministic()


def test_train_step_and_loss_take_the_switch():
    import inspect
    from deepvoice3_pytorch_b200.train_step import TrainStep, fused_training_loss
    assert inspect.signature(TrainStep.__init__).parameters["deterministic"].default is None
    assert inspect.signature(fused_training_loss).parameters["deterministic"].default is None


# ---- source guard ---------------------------------------------------------------------------------------------------
# Every function of csrc/*.cu that contains a float atomicAdd, with the deterministic form that replaces it.  A new
# atomic in any other function fails this test: it would silently break ops.deterministic.
HAS_DETERMINISTIC_TWIN = {
    ("loss.cu", "spec_loss_body"): "spec_loss_det_kernel (DET branch of the same body)",
    ("loss.cu", "aux_loss_body"): "aux_loss_det_kernel (DET branch of the same body)",
    ("conv.cu", "gate_bwd_kernel"): "gate_bwd_kernel<true> + bias_reduce_kernel",
    ("conv.cu", "bias_act_bwd_kernel"): "bias_act_bwd_kernel<true> + bias_reduce_kernel",
    ("tc_split.cu", "plane_split_kernel"): "plane_split_kernel<KIND, NPL, true> + bias_reduce_kernel",
    ("elementwise.cu", "embedding_bwd_kernel"): "table_bwd_det_kernel<false>",
    ("elementwise.cu", "sinusoid_bwd_kernel"): "table_bwd_det_kernel<true>",
}
# integer tickets (order-free): the last-block pattern itself
INTEGER_ATOMICS = {("optim.cu", "sumsq_kernel"), ("loss.cu", "det_loss_tail")}


def _float_atomics():
    """-> {(file, enclosing function)} of every atomicAdd whose value is not an unsigned literal ticket."""
    found, ints = set(), set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        fn = None
        for line in open(path):
            code = re.sub(r"__launch_bounds__\([^)]*\)", "", line.split("//")[0])
            m = re.search(r"__(?:global|device)__[^;(]*?\b(\w+)\s*\(", code)
            if m and "asm" not in code:
                fn = m.group(1)
            if "atomicAdd" in code:
                key = (os.path.basename(path), fn)
                (ints if re.search(r"atomicAdd\(\s*ticket\s*,\s*1u\)", code) else found).add(key)
    return found, ints


def test_every_float_atomic_has_a_deterministic_twin():
    found, ints = _float_atomics()
    assert found, "the guard found no atomicAdd at all: its parser is broken"
    unknown = found - set(HAS_DETERMINISTIC_TWIN)
    assert not unknown, "float atomicAdd without a deterministic form (add one, then list it here): %s" % sorted(unknown)
    assert set(HAS_DETERMINISTIC_TWIN) == found, "stale entries: %s" % sorted(set(HAS_DETERMINISTIC_TWIN) - found)
    assert ints == INTEGER_ATOMICS, ints


def test_guard_parser_sees_a_planted_atomic(tmp_path, monkeypatch):
    src = tmp_path / "planted.cu"
    src.write_text("__global__ void planted_kernel(float* x) {\n    atomicAdd(&x[0], 1.f);\n}\n")
    monkeypatch.setitem(globals(), "CSRC", str(tmp_path))
    found, _ = _float_atomics()
    assert found == {("planted.cu", "planted_kernel")}


# ---- ptxas ----------------------------------------------------------------------------------------------------------
def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


@pytest.fixture(scope="module")
def reports(tmp_path_factory):
    """-> {file: {mangled kernel name: (registers, spill store bytes, spill load bytes)}}"""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = {}
    tmp = tmp_path_factory.mktemp("ptxas_det")
    procs = {f: subprocess.Popen([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler",
                                  "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, f), "-o", str(tmp / (f + ".o"))],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for f in ("loss.cu", "conv.cu", "tc_split.cu", "elementwise.cu")}
    for f, p in procs.items():
        text = p.communicate()[0]
        assert p.returncode == 0, text
        kernels, cur, spills = {}, None, None
        for line in text.splitlines():
            m = re.search(r"Compiling entry function '(\w+)'", line)
            if m:
                cur = m.group(1)
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                spills = (int(m.group(1)), int(m.group(2)))
            m = re.search(r"Used (\d+) registers", line)
            if m and cur:
                kernels[cur] = (int(m.group(1)),) + spills
                cur = None
        out[f] = kernels
    return out


@pytest.mark.parametrize("src,pattern,count", [
    ("loss.cu", "spec_loss_det_kernel", 2), ("loss.cu", "aux_loss_det_kernel", 2),
    ("conv.cu", "gate_bwd_kernelILb1E", 1), ("conv.cu", "bias_act_bwd_kernelILb1E", 1), ("conv.cu", "bias_reduce_kernel", 1),
    ("elementwise.cu", "table_bwd_det_kernel", 2),
])
def test_new_kernels_do_not_spill(reports, src, pattern, count):
    ks = {k: v for k, v in reports[src].items() if pattern in k}
    assert len(ks) == count, (pattern, sorted(reports[src]))
    assert all(v[1:] == (0, 0) for v in ks.values()), ks


def test_split_kernel_keeps_six_ctas_per_sm(reports):
    """plane_split_kernel<KIND, NPL, DET>: the deterministic instantiations fit the 6-CTA register budget (65536 / (6 *
    256) -> 40) without spills, and the default ones keep the register counts they had before the mode existed."""
    ks = {k: v for k, v in reports["tc_split.cu"].items() if "plane_split_kernel" in k}
    assert len(ks) == 10, sorted(ks)                  # 3 kinds x 2 plane counts + 2 x 2 deterministic
    assert all(v[0] <= 40 and v[1:] == (0, 0) for v in ks.values()), ks
    want = {("0", "1"): 32, ("0", "2"): 40, ("1", "1"): 40, ("1", "2"): 40, ("2", "1"): 29, ("2", "2"): 36}
    for (kind, npl), regs in want.items():
        name = [k for k in ks if "ILi%sELi%sELb0E" % (kind, npl) in k]
        assert len(name) == 1 and ks[name[0]][0] == regs, (kind, npl, name, ks)
    assert len([k for k in ks if "ELb1E" in k]) == 4
