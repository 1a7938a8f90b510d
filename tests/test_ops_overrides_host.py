"""No GPU: ``ops.overrides`` sets and restores the execution-state attributes of ``ops`` (nested, on exception, and
refusing unknown names before setting anything), ``ops.py`` is the only module of the package that assigns them, and
the ctypes launch helpers are defined in ``ops.py`` alone."""
import ast
import glob
import os
import re

import pytest
import torch

from deepvoice3_pytorch_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PACKAGE = os.path.join(ROOT, "deepvoice3_pytorch_b200")
STATE = ("conv_math", "deterministic", "det_scratch", "grad_sink", "weight_bank", "grad_boundary_cb",
         "frozen_weights", "speaker_adapt")


def _state():
    return {k: getattr(ops, k) for k in STATE}


def _same(a, b):
    return a.keys() == b.keys() and all(a[k] is b[k] for k in a)


def test_overrides_names_the_whole_state():
    assert set(ops._STATE) == set(STATE)


def test_nested_overrides_restore_the_outer_values(monkeypatch):
    monkeypatch.setattr(ops, "conv_math", "tc")          # set directly, as callers of the module may
    outer = _state()
    bank, adapt, scratch = object(), object(), ops.DetScratch()
    with ops.overrides(conv_math="fp32", grad_sink=True, weight_bank=bank):
        assert (ops.conv_math, ops.grad_sink, ops.weight_bank) == ("fp32", True, bank)
        mid = _state()
        with ops.overrides(conv_math="tc1", weight_bank=None, speaker_adapt=adapt, deterministic=True,
                           det_scratch=scratch):
            assert (ops.conv_math, ops.grad_sink, ops.weight_bank, ops.speaker_adapt) == ("tc1", True, None, adapt)
            assert ops.is_deterministic() and ops.det_scratch is scratch
        assert _same(_state(), mid)
    assert _same(_state(), outer)


def test_overrides_restore_after_an_exception():
    outer = _state()
    cb, frozen = (lambda tag: None), ops.FrozenWeights()
    with pytest.raises(RuntimeError, match="inside"):
        with ops.overrides(grad_boundary_cb=cb, frozen_weights=frozen, deterministic="1", conv_math="fp32"):
            assert ops.grad_boundary_cb is cb and ops.frozen_weights is frozen
            raise RuntimeError("inside")
    assert _same(_state(), outer)


def test_overrides_refuse_an_unknown_name_before_setting_anything():
    outer = _state()
    with pytest.raises(ValueError, match="grad_snk"):
        with ops.overrides(conv_math="fp32", grad_snk=True):
            pytest.fail("the body ran")
    assert _same(_state(), outer)


def _ops_state_writes(path):
    """(line, attribute) of every assignment to ``ops.<state>`` (plain, augmented or by setattr) in a source file."""
    tree = ast.parse(open(path).read(), path)
    hits = []

    def targets(t):
        if isinstance(t, (ast.Tuple, ast.List)):
            for e in t.elts:
                yield from targets(e)
        elif isinstance(t, ast.Starred):
            yield from targets(t.value)
        else:
            yield t

    for node in ast.walk(tree):
        if isinstance(node, ast.Assign):
            tgts = [x for t in node.targets for x in targets(t)]
        elif isinstance(node, (ast.AugAssign, ast.AnnAssign)):
            tgts = list(targets(node.target))
        elif isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "setattr" and \
                node.args and isinstance(node.args[0], ast.Name) and node.args[0].id == "ops":
            hits.append((node.lineno, ast.unparse(node.args[1]) if len(node.args) > 1 else "?"))
            continue
        else:
            continue
        for t in tgts:
            if isinstance(t, ast.Attribute) and t.attr in STATE and isinstance(t.value, ast.Name) and \
                    t.value.id == "ops":
                hits.append((t.lineno, t.attr))
    return hits


def test_only_ops_assigns_the_execution_state():
    files = sorted(glob.glob(os.path.join(PACKAGE, "*.py")))
    assert len(files) > 20
    found = {os.path.basename(f): _ops_state_writes(f) for f in files if os.path.basename(f) != "ops.py"}
    assert {f: h for f, h in found.items() if h} == {}


def test_launch_helpers_are_defined_in_ops_only():
    # the stream helper takes no argument: synthesis._stream(model, ...) is the streaming-synthesis generator
    pattern = re.compile(r"^\s*def (_p|_cp|_stream(?=\(\)))\(", re.M)
    defs = {os.path.basename(f): sorted(pattern.findall(open(f).read()))
            for f in sorted(glob.glob(os.path.join(PACKAGE, "*.py")))}
    assert {f: d for f, d in defs.items() if d} == {"ops.py": ["_p", "_stream"]}


def test_pointer_helper_takes_an_element_offset():
    t = torch.zeros(8)
    assert ops._p(None) is None
    assert ops._p(t).value == t.data_ptr()
    assert ops._p(t, 3).value == t.data_ptr() + 12
