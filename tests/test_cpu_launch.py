"""CPU: kernels.launch, the one path from the package to the C-ABI library's launching entry points.  The library loads
without a GPU, and its argument checks refuse bad input before any CUDA call, so the error path runs here."""
import os
import re

import pytest

from dynamicpdb_b200 import kernels

PKG = os.path.dirname(os.path.abspath(kernels.__file__))


def test_launch_raises_the_library_error_and_counts_nothing(monkeypatch):
    monkeypatch.setattr(kernels, "_stream", lambda: None)
    before = kernels.LAUNCH_COUNT
    with pytest.raises(RuntimeError) as err:
        kernels.launch("dfold_quat_to_rot_fwd", None, None, 0)
    msg = str(err.value)
    assert msg.startswith("dfold_quat_to_rot_fwd:") and "empty input" in msg, msg
    assert kernels.LAUNCH_COUNT == before


def test_only_kernels_py_calls_the_library_directly():
    direct = re.compile(r"\blib\(\)|\b_check\(|\b_stream\(")
    offenders = []
    for root, _, files in os.walk(PKG):
        for f in files:
            path = os.path.join(root, f)
            if f.endswith(".py") and path != os.path.join(PKG, "kernels.py"):
                with open(path) as fh:
                    offenders += [f"{os.path.relpath(path, PKG)}:{i}" for i, line in enumerate(fh, 1) if direct.search(line)]
    assert not offenders, offenders
