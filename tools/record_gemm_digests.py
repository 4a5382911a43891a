"""Record the SHA-256 digests that tests/test_gpu_gemm_digests.py compares against (dev tool, needs a GPU).

  R2D2_B200_LIB=/path/to/libr2d2_b200.so python tools/record_gemm_digests.py tests/golden/gemm_digests.json

runs every case of that test on the library R2D2_B200_LIB points at (default: the in-tree build) and writes the JSON.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"), os.path.join(ROOT, "tests")]

from r2d2_b200 import native  # noqa: E402
import test_gpu_gemm_digests as cases  # noqa: E402

if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    native.lib()
    out = cases.digests(native)
    print(f"{native.LIB_PATH}: {len(out)} digests")
    with open(sys.argv[1], "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
