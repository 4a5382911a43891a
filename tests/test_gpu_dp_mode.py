"""R2D2_DP_MODE selects the data-parallel gradient exchange: "peer" (default) or "defer".  Any other value is an error
when the engine is built: a mode that matched no exchange used to train every rank on its own gradients."""
import pytest

pytestmark = pytest.mark.gpu


def _cfg(engine):
    return engine.PathConfig(obs=6, act=2, hidden=64, batch=16, burn_in=4, learning=6, n_step=2)


@pytest.mark.parametrize("value", ["serial", "peers"])
def test_unknown_dp_mode_is_rejected(monkeypatch, value):
    from r2d2_b200 import engine, native
    monkeypatch.setenv("R2D2_DP_MODE", value)
    with pytest.raises(native.NativeError, match="peer.*defer"):
        engine.LearnerEngine(_cfg(engine))


def test_default_dp_mode_is_peer(monkeypatch):
    from r2d2_b200 import engine
    monkeypatch.delenv("R2D2_DP_MODE", raising=False)
    eng = engine.LearnerEngine(_cfg(engine))
    assert eng._dp_mode == "peer"
    eng.close()
