"""The wgmma GEMM keeps the tensor pipe fed across k tiles: in the SASS of every gemm_packed_kernel instantiation the
first wait after a k tile's wgmmas is WARPGROUP.DEPBAR.LE gsb0, 0x1 (that k tile stays in flight while the stage of the
one before is released), and the kernel has no local-memory traffic.  ptxas -v must report no spills for these kernels
and at most 112 registers, so that two 288-thread CTAs fit on one SM."""
import os
import re
import shutil
import subprocess

import pytest

KERNEL = "gemm_packed_kernel"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorch-r2d2-dpg_b200", "csrc")


def _functions(sass, key):
    out = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name = block.split("\n", 1)[0].strip()
        if key in name:
            out[name] = block
    return out


def _ops(body):
    return [(m.group(1), m.group(2).strip()) for m in
            re.finditer(r"/\*[0-9a-f]{4,}\*/\s*(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);", body)]


def test_gemm_main_loop_keeps_one_k_tile_in_flight():
    from r2d2_b200 import native
    sass = subprocess.run(["cuobjdump", "-sass", native.LIB_PATH], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    funcs = _functions(sass, KERNEL)
    assert len(funcs) == 3, f"expected the NT, NN and TN instantiations of {KERNEL}, found {sorted(funcs)}"
    for name, body in funcs.items():
        ops = _ops(body)
        mma = [i for i, (op, _) in enumerate(ops) if op.startswith("HGMMA")]
        assert mma, f"no HGMMA in {name}"
        waits = [args for op, args in ops[mma[0]:] if op == "WARPGROUP.DEPBAR.LE"]
        assert waits and waits[0] == "gsb0, 0x1", f"{name}: first wait after the k tile's wgmmas is {waits[:1]}"
        assert not [op for op, _ in ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"


def test_gemm_kernels_do_not_spill_and_fit_two_ctas_per_sm():
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.isfile("/usr/local/cuda/bin/nvcc") else None)
    if not nvcc:
        pytest.skip("nvcc unavailable")
    res = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", os.path.join(CSRC, "gemm_tc.cu"),
                          "-o", os.devnull], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    found = 0
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", res.stderr):
        if KERNEL in m.group(1):
            found += 1
            assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
            assert int(m.group(5)) <= 112, m.group(0)
    assert found == 3, res.stderr[-2000:]
