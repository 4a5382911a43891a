"""R2D2's n-step target options on the GPU: the invertible value rescaling h_eps(R + gamma^n (1-d) h_eps^-1(Q')) and the
absolute-TD-error priorities, through the C ABI, the learner engine, the actor side and the drop-in learner.

 * the defaults give the bits of the entries without options and of an engine that never heard of them;
 * h_eps(h_eps^-1(q')) = q' on the device over 36 decades, on both TD routes;
 * the TD kernels against float64 (oracle/learner_oracle.py) in every mode x metric, weighted and not, on both sides of
   the 48 KB shared-memory switch, each case asserting the kernel instantiation that served it (observed under
   torch.profiler in a fresh process, the `routes` fixture);
 * the actor-side kernel against float64, and ActorPool's memory files in the environment's mode;
 * multi-iteration learner runs against the float64 oracle, also with importance weights, Polyak targets and clipping;
 * pipelined = sequential, seeded runs and resumed runs bit for bit; the drop-in learner with the variables set."""
import json
import os
import re

import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import dev, f64, nv, ptr  # noqa: F401
from learner_harness import (SMALL, assert_pipelined_matches_sequential, assert_resumed_run_is_bit_identical,
                             assert_same_bits, check_against_oracle, col_err, golden_case, port_case, replay_fed_run,
                             snapshot, trained_dropin_learner)
from oracle import actor_oracle
from oracle import learner_oracle as lo
from oracle import ref_port
from route_check import observe, observe_in_fresh_process, recorded_sentinel

pytestmark = pytest.mark.gpu

MODES = [(r, m) for r in ("reference", "invertible") for m in ("squared", "abs")]
NATIVE = {"reference": 0, "invertible": 1, "squared": 0, "abs": 1}
NEW = dict(value_rescaling="invertible", rescaling_eps=1e-3, priority_metric="abs")


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


# ------------------------------------------------------------------------------------------------ helpers
def td_inputs(L, B, A, Bn, n, seed):
    """q' log-uniform in magnitude 1e-6 .. 1e4 with both signs and exact zeros; terminals anywhere.  Not
    kernel_harness.td_inputs: h_eps and its inverse are exercised over many decades of |q'|, not around 1."""
    rng = np.random.default_rng(seed)
    T = Bn + L + n
    qn = 10.0 ** rng.uniform(-6, 4, (L, B, A)) * rng.choice([-1.0, 1.0], (L, B, A))
    qn[rng.uniform(size=qn.shape) < 0.03] = 0.0
    q = rng.standard_normal((L, B, A)) * 3
    rew = rng.standard_normal((T, B)) * 3
    term = (rng.uniform(size=(T, B)) < 0.15).astype(np.float64)
    return q, qn, rew, term


def options(nv, rescaling, eps, metric):
    return nv.TdOptions(NATIVE[rescaling], eps, NATIVE[metric])


def td_call(nv, inputs, L, B, A, Bn, n, *, opts="null", w=None, entry="ex", gamma=0.997,
            want=("y", "dq", "td", "p", "loss")):
    """One TD call; entry "plain" / "weighted" are the entries without options, "ex" takes opts (a TdOptions, or
    "null" for a NULL pointer).  Requested outputs start as NaN so that an unwritten element fails every bound."""
    shapes = {"y": (L, B, A), "dq": (L, B, A), "td": (L, B), "p": (B,), "loss": (1,)}
    o = {k: torch.full(s, float("nan"), device="cuda") for k, s in shapes.items() if k in want}
    q, qn, rew, term = (dev(x) for x in inputs)
    wt = None if w is None else dev(w)
    lib, P = nv.lib(), lambda k: ptr(o.get(k))                      # noqa: E731
    st = nv.current_stream()
    if entry == "plain":
        rc = lib.r2d2_td_priority(ptr(q), ptr(qn), ptr(rew), ptr(term), L, B, A, Bn, n, gamma, 0.9, P("y"), P("dq"),
                                  P("td"), P("p"), P("loss"), st)
    elif entry == "weighted":
        rc = lib.r2d2_td_priority_weighted(ptr(q), ptr(qn), ptr(rew), ptr(term), ptr(wt), L, B, A, Bn, n, gamma, 0.9,
                                           P("y"), P("dq"), P("td"), P("p"), P("loss"), st)
    else:
        rc = lib.r2d2_td_priority_ex(ptr(q), ptr(qn), ptr(rew), ptr(term), ptr(wt), L, B, A, Bn, n, gamma, 0.9, P("y"),
                                     P("dq"), P("td"), P("p"), P("loss"), None if opts == "null" else nv.byref(opts), st)
    nv.check(rc)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k


def expected_kernels(A, td_sq, rescaling, metric):
    inv, ab = int(rescaling == "invertible"), int(metric == "abs")
    if td_sq and 8 * 2 * 32 * A * 4 <= 48 * 1024:
        return {"td_elem_kernel": (inv,), "td_reduce_kernel": (ab,)}
    return {"td_priority_column_kernel": (inv, ab)}


def _flags(name, base):
    """Template flags of kernel `base` in a demangled (<true, false>) or mangled (ILb1ELb0E) name, else None."""
    m = re.search(re.escape(base) + r"<([^>]*)>", name)
    if m:
        return tuple(int(x.strip() == "true") for x in m.group(1).split(","))
    m = re.search(re.escape(base) + r"I((?:Lb[01]E)+)E", name)
    return tuple(int(x) for x in re.findall(r"Lb([01])E", m.group(1))) if m else None


def td_route_key(A, td_sq, weighted, rescaling, metric):
    return f"td/A={A}/td_sq={int(td_sq)}/w={int(weighted)}/{rescaling}/{metric}"


def actor_route_key(rescaling, metric):
    return f"actor/{rescaling}/{metric}"


def _route_cases(nv):
    """key -> the launch each profiled case below makes (the same entry point, shapes, options and outputs)."""
    cases = {}
    for A, td_sq in TD_CASES:
        for weighted in (False, True):
            for r, m in MODES:
                L, B, Bn, n = 33, 77, 3, 5
                inputs = td_inputs(L, B, A, Bn, n, seed=A * 31 + weighted)
                w = np.ones(B, np.float32) if weighted else None
                want = ("y", "dq", "td", "p", "loss") if td_sq else ("y", "dq", "p", "loss")
                cases[td_route_key(A, td_sq, weighted, r, m)] = (
                    lambda inputs=inputs, L=L, B=B, A=A, Bn=Bn, n=n, w=w, want=want, r=r, m=m:
                    td_call(nv, inputs, L, B, A, Bn, n, opts=options(nv, r, 1e-3, m), w=w, want=want))
    for r, m in MODES:
        cases[actor_route_key(r, m)] = lambda r=r, m=m: actor_call(nv, *actor_inputs(), r, m)
    return cases


def route_child(out_path):
    """Entry point of the fresh process behind the `routes` fixture: every case once under the profiler, from a session
    that recorded the sentinel -> {base name: sorted [template flags]} of the TD / actor-priority kernels, or None."""
    from r2d2_b200 import native
    native.lib()
    bases = ("td_elem_kernel", "td_reduce_kernel", "td_priority_column_kernel", "actor_priority_kernel")
    lost, out = [], {}
    for key, fn in _route_cases(native).items():
        got = observe(key, fn, recorded_sentinel, lost=lost)
        seen = {}
        for n in (got[1] if got else ()):
            for b in bases:
                f = _flags(n, b)
                if f is not None:
                    seen.setdefault(b, set()).add(f)
        out[key] = None if got is None else {k: sorted(list(f) for f in v) for k, v in seen.items()}
    out["lost_sessions"] = len(lost)
    with open(out_path, "w") as f:
        json.dump(out, f)


@pytest.fixture(scope="module")
def routes():
    """Which kernel instantiation served each profiled case, observed in a fresh Python process.  torch.profiler's
    collection in a long-lived test process can stop for several sessions in a row after the hundreds of sessions other
    test files run (seen on an H100 with torch 2.11 / CUDA 12.8, never in a fresh process), which says nothing about this
    library; a fresh process gives every case a complete session.  The values are checked in this process."""
    got = observe_in_fresh_process("test_gpu_value_rescaling", timeout=900)
    print(f"\nprofiler sessions repeated in the route process: {got.pop('lost_sessions')}")
    return got


def assert_route(routes, key, expect):
    got = routes[key]
    assert got is not None, f"{key}: torch.profiler recorded no kernel at all in eight sessions"
    assert got == {k: [list(v)] for k, v in expect.items()}, f"{key}: expected {expect}, ran {got}"


# ------------------------------------------------------------------------------------------------ 1. defaults
@pytest.mark.parametrize("A", [6, 38])
@pytest.mark.parametrize("weighted", [False, True])
def test_ex_defaults_are_the_plain_entries_bits(nv, A, weighted):
    L, B, Bn, n = 33, 77, 3, 5
    inputs = td_inputs(L, B, A, Bn, n, seed=A)
    w = np.random.default_rng(A).uniform(0.05, 1.0, B).astype(np.float32) if weighted else None
    base = td_call(nv, inputs, L, B, A, Bn, n, entry="weighted" if weighted else "plain", w=w)
    for opts in ("null", options(nv, "reference", 0.0, "squared"), options(nv, "reference", 0.5, "squared")):
        _bits(base, td_call(nv, inputs, L, B, A, Bn, n, opts=opts, w=w))


def test_engine_default_setters_keep_the_bits(eng_mod):
    def setters(eng):
        assert eng.lib.r2d2_learner_set_value_rescaling(eng._h, 0, 0.0) == 0
        assert eng.lib.r2d2_learner_set_priority_metric(eng._h, 0) == 0
    kw = dict(target_interval=3)
    assert_same_bits(replay_fed_run(eng_mod, 5, **kw), replay_fed_run(eng_mod, 5, setup=setters, **kw))


def test_launch_count_is_the_same_in_every_mode(eng_mod):
    counts = set()
    for r, m in MODES:
        eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL, value_rescaling=r, priority_metric=m), seed=1)
        eng.set_batch(ref_port.synthetic_batch(ref_port.PathConfig(**SMALL), seed=1))
        eng.step()
        counts.add(eng.launches_per_iteration)
        eng.close()
    assert len(counts) == 1, counts


def test_library_rejects_bad_values(eng_mod, nv):
    eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL))
    lib = eng.lib
    for mode, eps in ((2, 1e-3), (-1, 1e-3), (1, float("nan")), (1, float("inf")), (1, -1e-6), (1, 1.5)):
        assert lib.r2d2_learner_set_value_rescaling(eng._h, mode, eps) == -2           # R2D2_ERR_ARG
    for metric in (2, -1):
        assert lib.r2d2_learner_set_priority_metric(eng._h, metric) == -2
    assert lib.r2d2_learner_set_value_rescaling(eng._h, 0, float("nan")) == 0           # the reference ignores eps
    assert lib.r2d2_learner_set_value_rescaling(eng._h, 1, 1.0) == 0 and lib.r2d2_learner_set_priority_metric(eng._h, 1) == 0
    L, B, A = 4, 3, 2
    z = torch.zeros(16, device="cuda")
    for o in (options(nv, "invertible", float("nan"), "squared"), nv.TdOptions(3, 0.0, 0), nv.TdOptions(0, 0.0, 7)):
        assert lib.r2d2_td_priority_ex(ptr(z), ptr(z), ptr(z), ptr(z), None, L, B, A, 0, 1, 0.9, 0.9, None, None, None,
                                       None, None, nv.byref(o), nv.current_stream()) == -2
    eng.close()


# ------------------------------------------------------------------------------------------------ 2. round trip
@pytest.mark.parametrize("A", [6, 38])
@pytest.mark.parametrize("eps", [0.0, 1e-3, 1e-2])
def test_invertible_target_round_trips_on_device(nv, routes, A, eps):
    """gamma = 1, r = 0, d = 0: y = h_eps(h_eps^-1(q')) must give q' back (on the route of the unweighted TD case at
    this A: the kernel choice depends on the shape and options only)."""
    assert_route(routes, td_route_key(A, True, False, "invertible", "squared"),
                 expected_kernels(A, True, "invertible", "squared"))
    L, B, Bn, n = 8, 40, 2, 1
    mag = np.logspace(-30, 6, L * B * A // 2)
    qn = np.concatenate((mag, -mag))
    qn[:4] = 0.0
    qn = qn.astype(np.float32).reshape(L, B, A)
    inputs = (np.zeros((L, B, A)), qn, np.zeros((Bn + L + n, B)), np.zeros((Bn + L + n, B)))
    o = td_call(nv, inputs, L, B, A, Bn, n, opts=options(nv, "invertible", eps, "squared"), gamma=1.0)
    y, q = o["y"].astype(np.float64), qn.astype(np.float64)
    nz = q != 0
    assert (y[~nz] == 0).all()
    rel = np.abs(y[nz] - q[nz]) / np.abs(q[nz])
    assert rel.max() < 1e-6, (rel.max(), q[nz][rel.argmax()])
    ref = td_call(nv, inputs, L, B, A, Bn, n, opts=options(nv, "reference", eps, "squared"), gamma=1.0)["y"]
    assert (np.abs(ref[nz] - q[nz]) / np.abs(q[nz])).max() > 0.5          # h0 alone does not give q' back


# ------------------------------------------------------------------------------------------------ 3. TD vs float64
TD_CASES = [(A, True) for A in (1, 6, 17, 24, 25, 38, 64)] + [(6, False)]


@pytest.mark.parametrize("rescaling,metric", MODES)
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("A,td_sq", TD_CASES)
def test_td_against_float64(nv, routes, A, td_sq, weighted, rescaling, metric):
    L, B, Bn, n, eps = 33, 77, 3, 5, 1e-3
    inputs = td_inputs(L, B, A, Bn, n, seed=A * 31 + weighted)
    w = np.random.default_rng(A + 1).uniform(0.05, 1.0, B).astype(np.float32) if weighted else None
    ref = lo.td_targets_and_priorities(*(f64(x) for x in inputs), burn_in=Bn, learning=L, n_step=n, gamma=0.997,
                                       rescaling=rescaling, eps=float(np.float32(eps)), metric=metric,
                                       is_weight=None if w is None else f64(w))
    want = ("y", "dq", "td", "p", "loss") if td_sq else ("y", "dq", "p", "loss")
    assert_route(routes, td_route_key(A, td_sq, weighted, rescaling, metric),
                 expected_kernels(A, td_sq, rescaling, metric))
    o = td_call(nv, inputs, L, B, A, Bn, n, opts=options(nv, rescaling, eps, metric), w=w, want=want)
    y, loss, dq, tdsq, prio = ref
    for name, got, exp, ax in (("target", o["y"], y, A), ("dq", o["dq"], dq, A), ("priority", o["p"], prio, None)) + \
            ((("td_sq", o["td"], tdsq, None),) if td_sq else ()):
        assert rel_l2(got, exp) < 1e-5, (name, rel_l2(got, exp))
        if ax:
            assert col_err(got, exp, ax) < 1e-5, (name, col_err(got, exp, ax))
    assert abs(o["loss"][0] / loss - 1) < 1e-5, (o["loss"][0], loss)


# ------------------------------------------------------------------------------------------------ 4. actor side
ACTOR = dict(A=6, Bn=20, L=40, n=5, gamma=0.997, eps=1e-2, lens=(65, 66, 90, 131))


def actor_inputs():
    """q [T-n,B,A] online, qt [T,B,A] target, rew, term [T,B] of four zero-padded episodes (host, float64)."""
    c = ACTOR
    rng = np.random.default_rng(9)
    A, n, lens = c["A"], c["n"], c["lens"]
    B, T = len(lens), max(lens)
    q = np.zeros((T - n, B, A))
    qt = 10.0 ** rng.uniform(-4, 3, (T, B, A)) * rng.choice([-1.0, 1.0], (T, B, A))
    rew = np.zeros((T, B))
    term = np.ones((T, B))
    for b, N in enumerate(lens):
        E = N - n
        q[:E, b] = rng.standard_normal((E, A)) * 4
        rew[:N, b] = rng.standard_normal(N) * 3
        term[:E, b] = 0
    return q, qt, rew, term


def actor_call(nv, q, qt, rew, term, rescaling, metric):
    """r2d2_actor_priorities_ex on the inputs: prio [B, p_max] (host)."""
    c = ACTOR
    A, Bn, L, n, lens = c["A"], c["Bn"], c["L"], c["n"], c["lens"]
    B, T = len(lens), max(lens)
    p_max = T - n - (Bn + L)
    prio = torch.full((B, p_max), float("nan"), device="cuda")
    n_rows = torch.tensor(lens, dtype=torch.int32, device="cuda")
    qd, qtd, rd, td_ = dev(q), dev(qt), dev(rew), dev(term)
    nv.check(nv.lib().r2d2_actor_priorities_ex(ptr(qd), ptr(qtd), ptr(rd), ptr(td_), ptr(n_rows), B, A, Bn, L, n,
                                               c["gamma"], 0.9, p_max, ptr(prio),
                                               nv.byref(options(nv, rescaling, c["eps"], metric)), nv.current_stream()))
    torch.cuda.synchronize()
    return prio.cpu().numpy()


@pytest.mark.parametrize("rescaling,metric", MODES)
def test_actor_priorities_ex_against_float64(nv, routes, rescaling, metric):
    c = ACTOR
    inv, ab = int(rescaling == "invertible"), int(metric == "abs")
    assert_route(routes, actor_route_key(rescaling, metric), {"actor_priority_kernel": (inv, ab)})
    q, qt, rew, term = actor_inputs()
    got = actor_call(nv, q, qt, rew, term, rescaling, metric)
    for b, N in enumerate(c["lens"]):
        E = N - c["n"]
        want = actor_oracle.window_priorities(f64(q[:E, b]), f64(qt[:N, b]), f64(rew[:N, b]), f64(term[:N, b]), burn_in=c["Bn"],
                                              learning=c["L"], n_step=c["n"], gamma=c["gamma"], rescaling=rescaling,
                                              eps=float(np.float32(c["eps"])), metric=metric)
        assert rel_l2(got[b, :want.size], want) < 1e-5, (b, rel_l2(got[b, :want.size], want))
        assert (got[b, want.size:] == 0).all()


def test_actor_pool_files_use_the_environment_mode(monkeypatch, tmp_path):
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="32", R2D2_VALUE_RESCALING="invertible",
                     R2D2_RESCALING_EPS="0.01", R2D2_PRIORITY_METRIC="abs").items():
        monkeypatch.setenv(k, v)
    monkeypatch.chdir(tmp_path)
    os.makedirs("memory_data")
    os.makedirs("model_data")
    from actor_pool import ActorPool
    from r2d2_b200 import actor_priority as ap
    pool = ActorPool([0, 1], seed=2)
    with torch.no_grad():                                            # critic outputs of a few units
        for net in ("critic", "target_critic"):
            pool.model_dict[net]["l3.weight"].mul_(300.0)
            pool.model_dict[net]["l3.bias"].fill_(2.0)
        pool.stepper.load(pool.model_dict)
    for env in pool.envs:
        env.episode_len = 70
    pool.run(max_steps=4 * 71)
    payload = torch.load("memory_data/memory0.pt", weights_only=False)
    from replay_memory import pack_episode
    checked = 0
    for rows, states, prio in zip(payload["replay_memory"], payload["recurrent_state"], payload["priority"]):
        obs, act, rew, term, _ = pack_episode(rows, states, hidden=32)
        kw = dict(hidden=32, burn_in=20, learning=40, n_step=5, gamma=0.997)
        want, _ = ap.episode_priorities(pool.model_dict["critic"], pool.model_dict["target_actor"],
                                        pool.model_dict["target_critic"], [(obs, act, rew, term)], **kw,
                                        rescaling="invertible", eps=0.01, priority_metric="abs")
        other, _ = ap.episode_priorities(pool.model_dict["critic"], pool.model_dict["target_actor"],
                                         pool.model_dict["target_critic"], [(obs, act, rew, term)], **kw)
        assert rel_l2(prio, want[0]) < 1e-6, rel_l2(prio, want[0])
        assert rel_l2(prio, other[0]) > 1e-2                             # not the default mode's numbers
        checked += 1
    assert checked >= 3


# ------------------------------------------------------------------------------------------------ 5. learner vs oracle
def _check_learner(eng_mod, kw, actor, critic, batches, iters, *, tau=1.0, interval=500, clip=0.0, beta=False):
    """From the second iteration on, with fresh importance weights every iteration when beta."""
    rng = np.random.default_rng(3)
    weights = (lambda it: rng.uniform(0.05, 1.0, kw["batch"]).astype(np.float32)) if beta else None
    return check_against_oracle(eng_mod, dict(kw, **NEW, target_tau=tau, target_interval=interval, grad_clip_norm=clip,
                                              is_exponent=0.6 if beta else 0.0),
                                actor, critic, batches, iters, weights=weights, first=1)


@pytest.mark.parametrize("extras", [False, True], ids=["plain", "weights_polyak_clip"])
@pytest.mark.parametrize("name", ["ref_pend_h128.npz", "ref_walker_h128.npz"])
def test_learner_against_oracle_on_goldens(eng_mod, name, extras):
    kw, actor, critic, batches = golden_case(name)
    extra = dict(tau=0.05, interval=1, clip=0.5, beta=True) if extras else {}
    worst = _check_learner(eng_mod, kw, actor, critic, batches, 12, **extra)
    print(f"{name} extras={extras}: worst relative error {worst:.3e}")


def test_learner_against_oracle_cfg2(eng_mod):
    kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    worst = _check_learner(eng_mod, kw, *port_case(kw), 6)
    print(f"cfg-2: worst relative error {worst:.3e}")


# ------------------------------------------------------------------------------------------------ 6. determinism
def test_pipelined_step_matches_sequential_bit_for_bit(eng_mod):
    assert_pipelined_matches_sequential(eng_mod, eng_mod.PathConfig(**SMALL, **NEW, target_interval=1000), 6)


def test_replay_fed_runs_are_bitwise_reproducible(eng_mod):
    a, b = replay_fed_run(eng_mod, 7, target_interval=3, **NEW), replay_fed_run(eng_mod, 7, target_interval=3, **NEW)
    assert_same_bits(a, b)
    assert not torch.equal(a["priority"], replay_fed_run(eng_mod, 7, target_interval=3)["priority"])   # the options matter


def test_resumed_run_is_bit_identical(eng_mod):
    def check_state(st):
        assert (st["value_rescaling"], st["priority_metric"]) == ("invertible", "abs")
        with pytest.raises(ValueError, match="invertible"):
            eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL), seed=1).load_training_state(st)
    assert_resumed_run_is_bit_identical(eng_mod, eng_mod.PathConfig(**SMALL, **NEW, target_interval=3), check_state)


def test_options_may_change_between_iterations(eng_mod):
    """An engine switched to the new options after two iterations matches one that ran three iterations from a state
    saved after two and loaded under those options."""
    pc = ref_port.PathConfig(**SMALL)
    a = eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL), seed=4)
    for it in range(2):
        a.set_batch(ref_port.synthetic_batch(pc, seed=it))
        a.step()
    st = a.training_state()
    st.update(NEW)
    b = eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL, **NEW), seed=5)
    b.load_training_state(st)
    a.set_td_options(**NEW)
    for it in range(2, 5):
        batch = ref_port.synthetic_batch(pc, seed=it)
        for e in (a, b):
            e.set_batch(batch)
            e.step()
    assert_same_bits(snapshot(a), snapshot(b))


# ------------------------------------------------------------------------------------------------ 7. drop-in
def test_dropin_learner_trains_with_the_options(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_VALUE_RESCALING="invertible", R2D2_RESCALING_EPS="0.001",
                                R2D2_PRIORITY_METRIC="abs") as (lr, actors):
        c = lr.engine.cfg
        assert (c.value_rescaling, c.rescaling_eps, c.priority_metric) == ("invertible", 0.001, "abs")
        for a in actors:
            assert a.td_options == lr.td_options
        p = lr.engine.priority.cpu().numpy()
        assert np.isfinite(p).all() and (p > 0).all()
        st = torch.load("model_data/learner_state.pt", weights_only=False)
        assert (st["value_rescaling"], st["priority_metric"]) == ("invertible", "abs")
