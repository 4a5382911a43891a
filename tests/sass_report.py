"""What the compiler says about our kernels: ptxas -v's resource lines for one CUDA source compiled for sm_90a, and the
SASS of the built library split per function."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorch-r2d2-dpg_b200", "csrc")

# groups: function, stack frame, spill stores, spill loads, registers (None when ptxas printed no register line)
_PTXAS = re.compile(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                    r"(\d+) bytes spill loads(?:\n[^\n]*Used (\d+) registers)?")


def ptxas_report(source):
    """ptxas -v of csrc/<source> at sm_90a: (one match of the resource lines per function, the whole report).  Skips
    the test without nvcc."""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.isfile("/usr/local/cuda/bin/nvcc") else None)
    if not nvcc:
        pytest.skip("nvcc unavailable")
    res = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", os.path.join(CSRC, source),
                          "-o", os.devnull], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    return list(_PTXAS.finditer(res.stderr)), res.stderr


def library_sass():
    """cuobjdump -sass of the built library.  Skips the test without cuobjdump."""
    from r2d2_b200 import native
    sass = subprocess.run(["cuobjdump", "-sass", native.LIB_PATH], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    return sass


def functions(sass, key):
    """{function name: SASS body} of every function whose name contains key."""
    out = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name = block.split("\n", 1)[0].strip()
        if key in name:
            out[name] = block
    return out


def ops(body):
    """[(opcode, operands)] of a function body, predicates dropped."""
    return [(m.group(1), m.group(2).strip()) for m in
            re.finditer(r"/\*[0-9a-f]{4,}\*/\s*(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);", body)]
