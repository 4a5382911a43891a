"""The actor-step kernels keep their accumulators in registers: ptxas -v reports no stack frame and no spills for the
five policy_phase_kernel instantiations, and their SASS in the shipped library has no local-memory traffic."""
import os
import re
import shutil
import subprocess

import pytest

from test_cpu_sass_gemm import CSRC, ROOT, _functions, _ops

KERNEL = "policy_phase_kernel"


def test_policy_step_kernels_do_not_spill():
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.isfile("/usr/local/cuda/bin/nvcc") else None)
    if not nvcc:
        pytest.skip("nvcc unavailable")
    res = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", os.path.join(CSRC, "policy.cu"),
                          "-o", os.devnull], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    found = 0
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", res.stderr):
        if KERNEL in m.group(1):
            found += 1
            assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert found == 5, res.stderr[-2000:]


def test_policy_step_sass_has_no_local_memory():
    from r2d2_b200 import native
    sass = subprocess.run(["cuobjdump", "-sass", native.LIB_PATH], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    funcs = _functions(sass, KERNEL)
    assert len(funcs) == 5, sorted(funcs)
    for name, body in funcs.items():
        ops = [op for op, _ in _ops(body)]
        assert not [op for op in ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
        assert any(op.startswith("FFMA") for op in ops), name
