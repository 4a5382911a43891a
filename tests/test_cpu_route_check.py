"""The profiler retry loop of tests/route_check.py (observe) on scripted sessions: an incomplete session is repeated, the
agreement mode waits for two equal sessions in a row, and running out of sessions fails."""
import functools

import pytest

import route_check as rc

ROUTE = "void thin_tn_kernel<8>(float const*, int)"
OTHER = "void thin_tn_kernel<24>(float const*, int)"
FILL = "void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<float>>(int)"
SESSIONS = len(rc.PAUSES) + 1


class Scripted:
    """A session(fn) that runs fn and returns the next scripted list of kernel names (the last one repeats)."""

    def __init__(self, *names):
        self.names, self.calls = list(names), 0

    def __call__(self, fn):
        out = fn()
        self.calls += 1
        return out, self.names[min(self.calls, len(self.names)) - 1]


@pytest.fixture(autouse=True)
def pauses(monkeypatch):
    slept = []
    monkeypatch.setattr(rc.time, "sleep", slept.append)
    return slept


def test_incomplete_sessions_are_repeated(pauses):
    s, lost = Scripted([], [FILL], [ROUTE, FILL]), []
    assert rc.observe("c", lambda: 7, rc.recorded_route, lost=lost, session=s) == (7, [ROUTE, FILL])
    assert s.calls == 3 and lost == ["c", "c"] and pauses == list(rc.PAUSES[:2])


def test_sentinel_completes_a_session_without_route_kernels():
    s = Scripted([ROUTE], ["td_elem_kernel<true>", FILL])
    assert rc.observe("c", lambda: None, rc.recorded_sentinel, session=s)[1] == ["td_elem_kernel<true>", FILL]
    assert s.calls == 2


def test_agreement_waits_for_two_equal_sessions_in_a_row():
    s = Scripted([ROUTE], [ROUTE, ROUTE], [], [ROUTE, ROUTE], [ROUTE, ROUTE, OTHER], [ROUTE, ROUTE, OTHER])
    assert rc.observe("c", lambda: None, rc.recorded_route, agree=True, session=s)[1] == [ROUTE, ROUTE, OTHER]
    assert s.calls == 6
    s = Scripted([ROUTE, FILL], [ROUTE])                    # the sentinel is not a launch count to agree on
    assert rc.observe("c", lambda: None, rc.recorded_route, agree=True, session=s) is not None and s.calls == 2


def test_running_out_of_sessions_fails(monkeypatch, pauses):
    s, lost = Scripted([FILL]), []
    assert rc.observe("c", lambda: None, rc.recorded_route, lost=lost, session=s) is None
    assert s.calls == SESSIONS == 8 and len(lost) == SESSIONS and pauses == list(rc.PAUSES)
    alternating = Scripted(*([ROUTE], [ROUTE, ROUTE]) * SESSIONS)
    assert rc.observe("c", lambda: None, rc.recorded_route, agree=True, session=alternating) is None
    assert alternating.calls == SESSIONS

    monkeypatch.setattr(rc, "observe", functools.partial(rc.observe, session=Scripted([FILL])))
    with pytest.raises(AssertionError, match="no route kernel in 8 sessions"):
        rc.RouteLog().profile("c", lambda: None)
    with pytest.raises(AssertionError, match="no route kernel in 8 sessions"):
        rc.launch_counts("c", lambda: None)
    monkeypatch.setattr(rc, "observe", functools.partial(rc.observe, session=Scripted(*([ROUTE], [OTHER]) * 4)))
    with pytest.raises(AssertionError, match="no two profiler sessions in a row"):
        rc.launch_counts("c", lambda: None, agree=True)


def test_route_log_and_launch_counts_keep_route_kernels(monkeypatch):
    monkeypatch.setattr(rc, "observe", functools.partial(rc.observe, session=Scripted([ROUTE, OTHER, ROUTE, FILL])))
    log = rc.RouteLog()
    assert log.profile("c", lambda: 3) == (3, sorted({ROUTE, OTHER}))
    assert log.seen == {"c": sorted({ROUTE, OTHER})} and log.lost == []
    assert rc.launch_counts("c", lambda: None) == {ROUTE: 2, OTHER: 1}
