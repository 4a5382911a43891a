"""Observation normalisation on the host: the oracle's merge against one-shot float64 statistics, the float32 transform
against torch.clamp bit for bit, the environment options, the exchange schedule of the training loop, and the training
state record."""
import numpy as np
import pytest
import torch

from obs_norm_oracle import merge, moments, normalize, pair
from r2d2_b200 import obs_norm, run_loop


@pytest.mark.parametrize("seed", range(5))
def test_merge_equals_one_shot_statistics(seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((997, 7)) * rng.uniform(0.01, 100, 7) + rng.uniform(-50, 50, 7)
    cuts = np.sort(rng.choice(np.arange(1, 997), size=rng.integers(1, 9), replace=False))
    acc = np.zeros(1 + 2 * 7)
    for part in np.split(x, cuts):
        acc = merge(acc, moments(part))
    ref = moments(x)
    assert acc[0] == ref[0]
    np.testing.assert_allclose(acc[1:8], ref[1:8], rtol=1e-12, atol=1e-12 * np.abs(ref[1:8]).max())
    np.testing.assert_allclose(acc[8:], ref[8:], rtol=1e-12)


def test_merge_with_an_empty_side_is_the_other_side():
    b = moments(np.random.default_rng(0).standard_normal((5, 3)))
    assert np.array_equal(merge(np.zeros(7), b), b)
    assert np.array_equal(merge(b, np.zeros(7)), b)
    m, s = pair(np.zeros(7))
    assert np.array_equal(m, np.zeros(3, np.float32)) and np.array_equal(s, np.ones(3, np.float32))


def test_transform_equals_torch_clamp_bit_for_bit():
    rng = np.random.default_rng(1)
    O, c = 9, 5.0
    m = rng.standard_normal(O).astype(np.float32)
    s = rng.uniform(0.01, 10, O).astype(np.float32)
    x = (rng.standard_normal((64, O)) * 10).astype(np.float32)
    x[0] = [np.nan, np.inf, -np.inf, 0.0, -0.0, 1e38, -1e38, 0.0, 0.0]
    x[1] = m + np.float32(c) / s          # around +-c after the transform
    x[2] = m - np.float32(c) / s
    x[3] = m
    ref = torch.clamp((torch.from_numpy(x) - torch.from_numpy(m)) * torch.from_numpy(s), -c, c).numpy()
    got = normalize(x, m, s, c)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    assert np.isnan(got[0, 0]) and got[0, 1] == c and got[0, 2] == -c
    t = obs_norm.normalize_torch(torch.from_numpy(x), torch.from_numpy(m), torch.from_numpy(s), c).numpy()
    assert np.array_equal(t.view(np.uint32), ref.view(np.uint32))


def test_environment_options():
    assert obs_norm.from_environ({}) == (False, 5.0)
    assert obs_norm.from_environ({"R2D2_OBS_NORM": "1", "R2D2_OBS_NORM_CLIP": "3.5"}) == (True, 3.5)
    for bad in ({"R2D2_OBS_NORM": "yes"}, {"R2D2_OBS_NORM": "2"}, {"R2D2_OBS_NORM_CLIP": "0"},
                {"R2D2_OBS_NORM_CLIP": "-1"}, {"R2D2_OBS_NORM_CLIP": "inf"}, {"R2D2_OBS_NORM_CLIP": "nan"},
                {"R2D2_OBS_NORM_CLIP": "five"}):
        with pytest.raises(ValueError):
            obs_norm.from_environ(bad)


def test_path_config_validates_the_options():
    from r2d2_b200.engine import PathConfig
    assert PathConfig(obs=3, act=1).obs_norm is False
    for kw in (dict(obs_norm=1), dict(obs_norm_clip=0.0), dict(obs_norm_clip=float("nan")), dict(obs_norm_clip=True)):
        with pytest.raises(ValueError):
            PathConfig(obs=3, act=1, **kw)


class _Engine:
    def __init__(self, calls):
        self.calls, self.leaf_idx, self.priority = calls, None, None

    def step(self, prefetch=None):
        self.calls.append("step")
        if prefetch is not None:
            prefetch(self, self)


class _Replay:
    def __init__(self, calls):
        self.calls = calls

    def sample_into(self, eng):
        self.calls.append("sample")

    def update_priorities(self, leaf, prio):
        self.calls.append("write_back")


@pytest.mark.parametrize("warm", [(1, 7), (3, 2)])
def test_exchange_schedule_is_the_same_on_every_rank(warm):
    """Two ranks whose warm-up gates pass after different numbers of ingests make the same collectives, each right after
    an ingest (or before the first step) and never with a batch drawn ahead of it."""
    logs = []
    for n_warm in warm:
        calls = []
        left = [n_warm]

        def ready():
            return left[0] == 0

        def local_ingest():
            calls.append("ingest")
            left[0] -= 1
        assert run_loop.warm_up(local_ingest, ready) == n_warm
        calls.clear()
        run_loop.run_learner_loop(_Engine(calls), _Replay(calls), max_steps=120, ingest_every=50, save_every=50,
                                  ingest=lambda: calls.append("ingest"), save=lambda: None,
                                  exchange=lambda: calls.append("exchange"))
        logs.append(calls)
        assert calls[0] == "exchange" and calls[1] == "sample"
        for i, c in enumerate(calls):
            if c == "exchange" and i:
                assert calls[i - 1] == "ingest"
            if c == "ingest":
                assert calls[i + 1] == "exchange"
        # nothing drawn ahead of an exchange: no sample between the last step and the exchange after it
        for i in [i for i, c in enumerate(calls) if c == "exchange"][1:]:
            last_step = max(j for j in range(i) if calls[j] == "step")
            assert "sample" not in calls[last_step:i]
    assert [c for c in logs[0] if c == "exchange"] == [c for c in logs[1] if c == "exchange"]
    assert logs[0].count("exchange") == 1 + 120 // 50


def test_load_training_state_checks_the_obs_norm_record():
    """load_training_state refuses an on / off mismatch either way and another clip, before it loads anything (host
    stand-ins for the engine and its device statistics; the round trip itself runs on the GPU)."""
    from r2d2_b200 import engine as E

    class _Stats:
        clip = 5.0

        def __init__(self):
            self.loaded = None

        def load_state(self, st):
            self.loaded = st

    class _Eng:
        obs_norm = None

    rec = {"enabled": True, "clip": 5.0, "n": 10.0, "mean": np.arange(3.0), "M2": np.ones(3)}
    off, on = _Eng(), _Eng()
    on.obs_norm = _Stats()
    with pytest.raises(ValueError, match="obs_norm="):
        E.LearnerEngine.load_training_state(off, {"obs_norm": rec})
    with pytest.raises(ValueError, match="obs_norm="):
        E.LearnerEngine.load_training_state(on, {})
    with pytest.raises(ValueError, match="obs_norm_clip"):
        E.LearnerEngine.load_training_state(on, {"obs_norm": dict(rec, clip=4.0)})
    assert on.obs_norm.loaded is None
