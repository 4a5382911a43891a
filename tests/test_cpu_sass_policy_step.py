"""The actor-step kernels keep their accumulators in registers: ptxas -v reports no stack frame and no spills for the
five policy_phase_kernel instantiations, and their SASS in the shipped library has no local-memory traffic."""
from sass_report import functions, library_sass, ops, ptxas_report

KERNEL = "policy_phase_kernel"


def test_policy_step_kernels_do_not_spill():
    report, stderr = ptxas_report("policy.cu")
    found = 0
    for m in report:
        if KERNEL in m.group(1):
            found += 1
            assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert found == 5, stderr[-2000:]


def test_policy_step_sass_has_no_local_memory():
    funcs = functions(library_sass(), KERNEL)
    assert len(funcs) == 5, sorted(funcs)
    for name, body in funcs.items():
        body_ops = [op for op, _ in ops(body)]
        assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
        assert any(op.startswith("FFMA") for op in body_ops), name
