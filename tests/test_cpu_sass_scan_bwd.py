"""The BPTT scan's step loop reads its per-step activations (gates, c_prev, dh_head) through cp.async copies issued one
step ahead, not through loads that the pointwise phase waits on.  In the SASS of lstm_scan_bwd_kernel<512,16> (the
cfg-3 instantiation), from the step loop's first mbarrier wait on, the only global loads are LDGSTS (the stage copies)
and the LDG.E.STRONG.SYS status read of the bounded wait's slow path."""
import re

from sass_report import functions, library_sass

KERNEL = "lstm_scan_bwd_kernelILi512ELi16E"


def test_bwd_scan_step_loop_has_no_blocking_global_loads():
    from r2d2_b200 import native
    body = next(iter(functions(library_sass(), KERNEL).values()), None)
    assert body is not None, f"{KERNEL} not found in {native.LIB_PATH}"
    ops = [m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s*(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", body)]
    first_wait = next((i for i, op in enumerate(ops) if op.startswith("SYNCS.PHASECHK")), None)
    assert first_wait is not None, "no mbarrier wait in the BPTT kernel"
    loads = [op for op in ops[first_wait:] if op.startswith("LDG") and op != "LDGDEPBAR"]
    blocking = sorted({op for op in loads if not op.startswith("LDGSTS") and op != "LDG.E.STRONG.SYS"})
    assert not blocking, f"global loads on the BPTT step loop's critical path: {blocking}"
    assert any(op.startswith("LDGSTS") for op in loads), "the stage copies (LDGSTS) are missing from the step loop"
    assert not [op for op in ops[first_wait:] if op.startswith(("LDL", "STL"))], "local-memory traffic in the step loop"
