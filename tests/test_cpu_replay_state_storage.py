"""fp16 recurrent-state storage of the replay shard, host side: the option takes exactly "float32" and "float16" (in
PathConfig and in R2D2_REPLAY_STATE_DTYPE), the default ring size follows the row width of each mode, and the new
gather, range-check and conversion kernels keep everything in registers."""
import pytest

from learner_harness import fake_engine_learner
from sass_report import functions, library_sass, ops, ptxas_report

GB = 1 << 30


def test_path_config_accepts_exactly_the_two_dtypes():
    from r2d2_b200 import engine
    assert engine.PathConfig(obs=3, act=1).replay_state_dtype == "float32"
    for v in ("float32", "float16"):
        assert engine.PathConfig(obs=3, act=1, replay_state_dtype=v).replay_state_dtype == v
    for bad in ("bfloat16", "fp16", "half", "float64", "", None, 16, ["float16"]):
        with pytest.raises(ValueError, match="replay_state_dtype"):
            engine.PathConfig(obs=3, act=1, replay_state_dtype=bad)


def test_environment_variable(monkeypatch, tmp_path):
    assert fake_engine_learner(monkeypatch, tmp_path).engine.cfg.replay_state_dtype == "float32"
    lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_STATE_DTYPE="float16")
    assert lr.engine.cfg.replay_state_dtype == "float16" and lr.memory.state_dtype == "float16"
    lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_STATE_DTYPE="float32")
    assert lr.engine.cfg.replay_state_dtype == "float32" and lr.memory.state_dtype == "float32"
    for bad in ("bfloat16", "float", "FLOAT16", "16", ""):
        with pytest.raises(ValueError, match="R2D2_REPLAY_STATE_DTYPE"):
            fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_STATE_DTYPE=bad)


def test_replay_memory_rejects_other_dtypes():
    from replay_memory import LearnerReplayMemory
    with pytest.raises(ValueError, match="replay_state_dtype"):
        LearnerReplayMemory(obs_size=3, n_actions=1, hidden=8, state_dtype="bfloat16")


def _capacity(monkeypatch, dtype, free, O, A, H, seqs=5_000_000):
    import torch
    from replay_memory import LearnerReplayMemory
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (free, 80 * GB))
    m = LearnerReplayMemory(memory_sequence_size=seqs, obs_size=O, n_actions=A, hidden=H, state_dtype=dtype)
    return m._default_capacity_rows(O, A, H)


@pytest.mark.parametrize("O, A, H", [(376, 17, 512), (17, 6, 256), (24, 6, 128), (5, 2, 33)])
def test_default_capacity_follows_the_row_width(monkeypatch, capsys, O, A, H):
    free = 70 * GB
    want = int(5_000_000 * 1.3) + 4096
    for dtype, per_h in (("float32", 32), ("float16", 16)):
        row = 4 * (O + A + 2) + per_h * H + 5
        fit = int(0.6 * free / row)
        got = _capacity(monkeypatch, dtype, free, O, A, H)
        assert got == (fit if fit < want else want), (dtype, got, fit, want)
        note = capsys.readouterr().out
        assert (dtype in note) == (fit < want), note


def test_fp16_fits_at_least_1_83x_the_rows_at_cfg3(monkeypatch):
    free = 40 * GB                                   # the cap applies in both modes
    r32 = _capacity(monkeypatch, "float32", free, 376, 17, 512)
    r16 = _capacity(monkeypatch, "float16", free, 376, 17, 512)
    assert r16 >= 1.83 * r32, (r16, r32)


def test_fp32_capacity_is_unchanged(monkeypatch):
    """float32 keeps the earlier row width 4 (O + A + 2 + 8 H) + 5, so the default ring is what it was."""
    for O, A, H in ((376, 17, 512), (24, 6, 128)):
        free = 50 * GB
        row = 4 * (O + A + 2 + 8 * H) + 5
        want = int(5_000_000 * 1.3) + 4096
        assert _capacity(monkeypatch, "float32", free, O, A, H) == min(int(0.6 * free / row), want)


NEW_KERNELS = ("gather_batch_kernelILb0ELb1E", "gather_batch_kernelILb1ELb1E", "count_f16_overflow_kernel",
               "states_to_f16_kernel")


def test_new_kernels_do_not_spill():
    report, stderr = ptxas_report("replay.cu")
    seen = set()
    for m in report:
        for k in NEW_KERNELS:
            if k in m.group(1):
                seen.add(k)
                assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert seen == set(NEW_KERNELS), stderr[-2000:]


def test_new_kernels_sass_has_no_local_memory():
    sass = library_sass()
    for k in NEW_KERNELS:
        funcs = functions(sass, k)
        assert len(funcs) == 1, (k, sorted(funcs))
        for name, body in funcs.items():
            body_ops = [op for op, _ in ops(body)]
            assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
