"""The wgmma GEMM keeps the tensor pipe fed across k tiles: in the SASS of every gemm_packed_kernel instantiation the
first wait after a k tile's wgmmas is WARPGROUP.DEPBAR.LE gsb0, 0x1 (that k tile stays in flight while the stage of the
one before is released), and the kernel has no local-memory traffic.  ptxas -v must report no spills for these kernels
and at most 112 registers, so that two 288-thread CTAs fit on one SM."""
from sass_report import functions, library_sass, ops, ptxas_report

KERNEL = "gemm_packed_kernel"


def test_gemm_main_loop_keeps_one_k_tile_in_flight():
    funcs = functions(library_sass(), KERNEL)
    assert len(funcs) == 3, f"expected the NT, NN and TN instantiations of {KERNEL}, found {sorted(funcs)}"
    for name, body in funcs.items():
        body_ops = ops(body)
        mma = [i for i, (op, _) in enumerate(body_ops) if op.startswith("HGMMA")]
        assert mma, f"no HGMMA in {name}"
        waits = [args for op, args in body_ops[mma[0]:] if op == "WARPGROUP.DEPBAR.LE"]
        assert waits and waits[0] == "gsb0, 0x1", f"{name}: first wait after the k tile's wgmmas is {waits[:1]}"
        assert not [op for op, _ in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"


def test_gemm_kernels_do_not_spill_and_fit_two_ctas_per_sm():
    report, stderr = ptxas_report("gemm_tc.cu")
    found = 0
    for m in report:
        if KERNEL in m.group(1):
            found += 1
            assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
            assert int(m.group(5)) <= 112, m.group(0)
    assert found == 3, stderr[-2000:]
