"""Recurrent states in pinned host memory, host side: R2D2_REPLAY_HOST_GB's parsing and refusals, PathConfig's
replay_state_memory, the host tier's ring sizing (each of the wanted rows, the HBM fit and the host budget binding in
turn, in both state types) and the host-tier gather kernels' registers."""
import pytest

from learner_harness import fake_engine_learner
from sass_report import functions, library_sass, ops, ptxas_report

GB = 1 << 30
WANT_5M = int(5_000_000 * 1.3) + 4096          # 6,504,096 ring rows for the reference's memory_sequence_size


def test_path_config_accepts_exactly_device_and_host():
    from r2d2_b200 import engine
    assert engine.PathConfig(obs=3, act=1).replay_state_memory == "device"
    for v in ("device", "host"):
        assert engine.PathConfig(obs=3, act=1, replay_state_memory=v).replay_state_memory == v
    for bad in ("HOST", "pinned", "hbm", "", None, 1, True, ["host"]):
        with pytest.raises(ValueError, match="replay_state_memory"):
            engine.PathConfig(obs=3, act=1, replay_state_memory=bad)


def test_native_options_keep_positional_construction():
    from r2d2_b200 import native as nv
    assert (nv.STATE_MEMORY_DEVICE, nv.STATE_MEMORY_HOST) == (0, 1)
    o = nv.ReplayOptions(nv.STATE_F16)
    assert (o.state_storage, o.state_memory) == (nv.STATE_F16, nv.STATE_MEMORY_DEVICE)
    assert "r2d2_replay_host_bytes" in nv.SIGNATURES


def test_environment_variable(monkeypatch, tmp_path):
    lr = fake_engine_learner(monkeypatch, tmp_path)
    assert lr.replay_host_gb == 0.0 and lr.memory.host_gb == 0.0
    assert lr.engine.cfg.replay_state_memory == "device" and lr.memory._cfg().replay_state_memory == "device"
    for v, gb in (("0", 0.0), ("53.5", 53.5), ("1e2", 100.0), (" 7 ", 7.0)):
        lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_HOST_GB=v)
        assert lr.replay_host_gb == gb and lr.memory.host_gb == gb, v
        mem = "host" if gb > 0 else "device"
        assert lr.engine.cfg.replay_state_memory == mem and lr.memory._cfg().replay_state_memory == mem
    lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_HOST_GB="8", R2D2_REPLAY_STATE_DTYPE="float16")
    assert lr.memory._cfg().replay_state_dtype == "float16" and lr.memory._cfg().replay_state_memory == "host"
    for bad in ("-1", "-0.5", "nan", "inf", "-inf", "", "8GB", "eight", "1,5"):
        with pytest.raises(ValueError, match="R2D2_REPLAY_HOST_GB"):
            fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_HOST_GB=bad)


def test_replay_memory_refuses_bad_budgets():
    from replay_memory import LearnerReplayMemory
    for bad in (-1, -1e-9, float("nan"), float("inf"), "8", None, True):
        with pytest.raises(ValueError, match="host_gb"):
            LearnerReplayMemory(obs_size=3, n_actions=1, hidden=8, host_gb=bad)


def _capacity(monkeypatch, dtype, free, O, A, H, host_gb, seqs=5_000_000):
    import torch
    from replay_memory import LearnerReplayMemory
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (free, 80 * GB))
    m = LearnerReplayMemory(memory_sequence_size=seqs, obs_size=O, n_actions=A, hidden=H, state_dtype=dtype,
                            host_gb=host_gb)
    return m._default_capacity_rows(O, A, H)


@pytest.mark.parametrize("dtype, per_h", [("float32", 32), ("float16", 16)])
@pytest.mark.parametrize("O, A, H", [(376, 17, 512), (17, 6, 256)])
def test_each_limit_binds_in_turn(monkeypatch, capsys, dtype, per_h, O, A, H):
    hbm_row, host_row = 4 * (O + A + 2) + 5, per_h * H
    # want binds: plenty of HBM and host memory
    assert _capacity(monkeypatch, dtype, 70 * GB, O, A, H, 1e4) == WANT_5M
    note = capsys.readouterr().out
    assert "limited by memory_sequence_size=5000000" in note and "FIFO" not in note, note
    assert "%.2f GB of HBM" % (WANT_5M * hbm_row / 1e9) in note, note
    assert "%.2f GB of pinned host memory" % (WANT_5M * host_row / 1e9) in note, note
    # the HBM fit binds
    free = GB // 2
    fit = int(0.6 * free / hbm_row)
    assert fit < WANT_5M
    assert _capacity(monkeypatch, dtype, free, O, A, H, 1e4) == fit
    note = capsys.readouterr().out
    assert "limited by 60 % of the free HBM" in note and "FIFO eviction starts earlier" in note, note
    # the host budget binds
    host = int(3.0 * 1e9 / host_row)
    assert host < WANT_5M
    assert _capacity(monkeypatch, dtype, 70 * GB, O, A, H, 3.0) == host
    note = capsys.readouterr().out
    assert "limited by the host budget host_gb=3" in note and dtype in note and "FIFO" in note, note


def test_the_issue_figures_at_cfg3_and_cfg2(monkeypatch, capsys):
    """The full 5 M-sequence ring: 1,585 HBM bytes per cfg-3 row, 10.3 GB of HBM, 53.3 GB (fp16) or 106.6 GB (fp32) of
    host memory; at cfg-2 0.68 GB of HBM and 26.6 / 53.3 GB of host memory."""
    assert 4 * (376 + 17 + 2) + 5 == 1585
    for (O, A, H), hbm_gb, host in (((376, 17, 512), "10.31", {"float16": "53.28", "float32": "106.56"}),
                                    ((17, 6, 256), "0.68", {"float16": "26.64", "float32": "53.28"})):
        for dtype in ("float16", "float32"):
            assert _capacity(monkeypatch, dtype, 70 * GB, O, A, H, 200.0) == WANT_5M
            note = capsys.readouterr().out
            assert "%s GB of HBM" % hbm_gb in note and "%s GB of pinned host memory" % host[dtype] in note, note


def test_host_tier_beats_the_device_cap_at_cfg3(monkeypatch, capsys):
    """In the 40 GB budget of DESIGN section 7 the device tier holds a third of the rows the reference keeps; the host
    tier holds all of them."""
    free = int(40e9 / 0.6)
    dev = _capacity(monkeypatch, "float32", free, 376, 17, 512, 0)
    assert dev < 0.35 * WANT_5M
    assert _capacity(monkeypatch, "float32", free, 376, 17, 512, 110.0) == WANT_5M


def test_a_budget_below_one_row_is_refused(monkeypatch):
    with pytest.raises(ValueError, match="holds no replay row"):
        _capacity(monkeypatch, "float32", 70 * GB, 376, 17, 512, 1e-6)


def test_zero_budget_keeps_the_device_arithmetic(monkeypatch, capsys):
    """host_gb = 0 is the earlier sizing, note included."""
    for dtype, per_h in (("float32", 32), ("float16", 16)):
        free = 40 * GB
        row = 4 * (376 + 17 + 2) + per_h * 512 + 5
        assert _capacity(monkeypatch, dtype, free, 376, 17, 512, 0) == int(0.6 * free / row)
        note = capsys.readouterr().out
        assert note.startswith("LearnerReplayMemory: ring capped at") and "of HBM, %s recurrent states" % dtype in note


HOST_KERNELS = ("gather_host_states_kernelILb0ELb0E", "gather_host_states_kernelILb0ELb1E",
                "gather_host_states_kernelILb1ELb0E", "gather_host_states_kernelILb1ELb1E")


def test_host_tier_gathers_do_not_spill():
    report, stderr = ptxas_report("replay.cu")
    seen = set()
    for m in report:
        for k in HOST_KERNELS:
            if k in m.group(1):
                seen.add(k)
                assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert seen == set(HOST_KERNELS), stderr[-2000:]


def test_host_tier_gathers_have_no_local_memory():
    sass = library_sass()
    for k in HOST_KERNELS:
        funcs = functions(sass, k)
        assert len(funcs) == 1, (k, sorted(funcs))
        for name, body in funcs.items():
            body_ops = [op for op, _ in ops(body)]
            assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
