"""Sequence geometry on the GPU: every kernel route that the learning window (burn-in Bn, learning length L, n-step n,
T = Bn + L + n rows) and the batch B select, checked against float64, at the windows the other suites never run: burn-in
0, n-step 1, L = 2 and L not a multiple of 8, n > L, and windows of hundreds of rows.

 1. The TD / priority kernels through the C ABI (grid rows ceil(L / 8), warps striding over L, the [b:-1:B] quirk)
    on both routes, with NULL outputs, importance weights and the R2D2 target / priority options.
 2. The weight-gradient products of r2d2_lstm_net_backward, which contract over T·B rows: the row count turns split-K
    on, and split-K moves the products with one side <= 32 (dW3, the obs and action blocks of dW1) from the mma.sync
    kernel to thin_tn_kernel.  The switch points are found by bisection on T·B and printed; each product runs just below
    and just above its own.  The wide products (dW_hh, dW_ih) run below the split, with a ragged last slice and at a
    400-row window.
 3. Scan step counts through r2d2_lstm_net_forward / _backward on the cluster scans (H = 128, 512) and the per-step
    path (H = 96): S = T·repeat in every residue mod 4 (the hand-off parity), long chains, first_row 0 and T - 1.
 4. Learner iterations at edge windows against the float64 oracle and the CPU port; one replay-fed run and one
    twin-critic run at burn-in 0.
 5. The replay gather at episodes with 0, 1 and 2 sequence starts, and the actor-side n-step rewards and priorities.
 6. L = 1: every entry that computes a priority refuses it; the TD kernel without a priority output still runs.

Every time-major output is bounded per time row (step_err) as well as over the whole tensor: a whole-tensor norm over
hundreds of rows dilutes an error confined to one step.  Which kernel served each case is observed under torch.profiler
in one fresh process (the `routes` fixture); the values are checked here.  Run with -s for the switch points, the routes
seen and the worst errors per group."""
import json

import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import WorstLog, dev, f64, make_params, ptr, scan_status, td_inputs
from kernel_harness import nv_routes as nv  # noqa: F401
from learner_harness import TOL, check_against_oracle, episode, oracle_for, port_case, step_err
from oracle import actor_oracle
from oracle import learner_oracle as lo
from oracle import ref_port
from oracle.sumtree import SumTreeOracle
from route_check import ROUTE_KERNELS, RouteLog, launch_counts, observe_in_fresh_process, ran, template_args

pytestmark = pytest.mark.gpu

TOL_FWD, TOL_BWD = 2e-5, 5e-5
ERR_ARG = -2
NATIVE = {"reference": 0, "invertible": 1, "squared": 0, "abs": 1}
B_MAX = 1 << 14          # bisection ceiling in rows: far beyond the split-K switch of any product here

ROUTES = RouteLog()
WORST = WorstLog()


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    WORST.report()
    ROUTES.report()


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


def count(counts, key, args=None):
    """Launches of route `key` (with trailing template arguments `args`, None: any) in a launch_counts result."""
    base = ROUTE_KERNELS[key]
    return sum(k for n, k in counts.items() if base in n and (args is None or any(
        a[len(a) - len(args):] == tuple(args) for a in template_args(n, base) if len(a) >= len(args))))


# ------------------------------------------------------------------------------------------------ 1. TD / priority
def td_call(nv, inputs, L, B, A, Bn, n, want=("y", "dq", "td", "p", "loss"), w=None, opts=None, check=True):
    """r2d2_td_priority (w and opts None), _weighted (w given) or _ex (opts = (rescaling, eps, metric)) with the
    outputs in `want`, NULL for the others; requested outputs start as NaN.  Returns ({output: host array}, rc)."""
    shapes = {"y": (L, B, A), "dq": (L, B, A), "td": (L, B), "p": (B,), "loss": (1,)}
    o = {k: torch.full(s, float("nan"), device="cuda") for k, s in shapes.items() if k in want}
    q, qn, rew, term = (dev(x) for x in inputs)
    wt = None if w is None else dev(w)
    lib, P = nv.lib(), lambda k: ptr(o.get(k))                      # noqa: E731
    if opts is not None:
        to = nv.TdOptions(NATIVE[opts[0]], opts[1], NATIVE[opts[2]])
        rc = lib.r2d2_td_priority_ex(ptr(q), ptr(qn), ptr(rew), ptr(term), ptr(wt), L, B, A, Bn, n, 0.997, 0.9, P("y"),
                                     P("dq"), P("td"), P("p"), P("loss"), nv.byref(to), nv.current_stream())
    elif w is not None:
        rc = lib.r2d2_td_priority_weighted(ptr(q), ptr(qn), ptr(rew), ptr(term), ptr(wt), L, B, A, Bn, n, 0.997, 0.9,
                                           P("y"), P("dq"), P("td"), P("p"), P("loss"), nv.current_stream())
    else:
        rc = lib.r2d2_td_priority(ptr(q), ptr(qn), ptr(rew), ptr(term), L, B, A, Bn, n, 0.997, 0.9, P("y"), P("dq"),
                                  P("td"), P("p"), P("loss"), nv.current_stream())
    if check:
        nv.check(rc)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}, rc


def td_ref(inputs, L, Bn, n, w=None, opts=None):
    kw = {} if opts is None else dict(rescaling=opts[0], eps=float(np.float32(opts[1])), metric=opts[2])
    return lo.td_targets_and_priorities(*(f64(x) for x in inputs), burn_in=Bn, learning=L, n_step=n, gamma=0.997,
                                        is_weight=None if w is None else f64(w), **kw)


def check_td(group, case, o, ref, opts=None):
    y, loss, dq, td_sq, prio = ref
    # y to 1e-6 over the whole tensor, 1e-5 per time row: at B = 1 a row is A targets, and r + gamma^n q' can cancel
    tol_y = 1e-6 if opts is None or opts[0] == "reference" else 1e-5
    for k, got, want, tol, ax in (("y", o.get("y"), y, tol_y, 0), ("dq", o.get("dq"), dq, 1e-5, 0),
                                  ("td", o.get("td"), td_sq, 1e-5, 0), ("p", o.get("p"), prio, 1e-5, None)):
        if got is not None:
            WORST.bound(f"td {group} {k}", f"{case} {k}", got, want, tol, time_axis=ax, step_tol=1e-5)
    if "loss" in o:
        e = abs(o["loss"][0] / loss - 1.0)
        WORST.note(f"td {group} loss", e)
        assert e < 1e-5, (case, o["loss"][0], loss)


# (L, Bn, n, B, A, route): every L with two (Bn, n, B) of the chosen grid per route; "two_pass" A = 6 with td_sq,
# "column" A = 6 with td_sq NULL, "wide" A = 38 (past the 48 KB shared-memory switch) with every output
TD_L, TD_B, TD_BN, TD_N = (2, 3, 7, 8, 9, 16, 17, 33, 160, 400), (1, 2, 31, 32, 33, 257), (0, 1, 80), (1, 2, 5, 10)
TD_CASES = [(L, TD_BN[(i + j) % 3], TD_N[(i + 2 * j) % 4], TD_B[(i + 3 * j) % 6], 38 if r == "wide" else 6, r)
            for i, L in enumerate(TD_L) for j, r in enumerate(("two_pass", "column", "wide"))]
TD_WANT = {"two_pass": ("y", "dq", "td", "p", "loss"), "column": ("y", "dq", "p", "loss"),
           "wide": ("y", "dq", "td", "p", "loss")}
TD_ROUTE = {"two_pass": "td_two_pass", "column": "td_column", "wide": "td_column"}


def td_key(L, Bn, n, B, A, route):
    return f"td L={L} Bn={Bn} n={n} B={B} A={A} {route}"


@pytest.mark.parametrize("L,Bn,n,B,A,route", TD_CASES)
def test_td_window(nv, routes, L, Bn, n, B, A, route):
    key = td_key(L, Bn, n, B, A, route)
    ROUTES.assert_route(key, TD_ROUTE[route], list(routes[key]))
    inputs = td_inputs(L, B, A, Bn, n, seed=L * 1009 + B * 17 + n * 3 + A)
    o, _ = td_call(nv, inputs, L, B, A, Bn, n, want=TD_WANT[route])
    check_td(route, key, o, td_ref(inputs, L, Bn, n))


# a few points of the grid with importance weights, the R2D2 options (invertible target, abs priority) on both routes,
# and outputs left NULL: ("y", "p") takes the column kernel, ("dq", "td") the element pass without the reduction
TD_VARIANT_POINTS = [(2, 0, 10, 33), (17, 80, 1, 257), (400, 1, 5, 2)]
TD_VARIANTS = {"weighted": (6, ("y", "dq", "td", "p", "loss"), True, None, "td_two_pass"),
               "options": (6, ("y", "dq", "td", "p", "loss"), True, ("invertible", 1e-2, "abs"), "td_two_pass"),
               "options_wide": (38, ("y", "dq", "td", "p", "loss"), True, ("invertible", 1e-2, "abs"), "td_column"),
               "y_p_only": (6, ("y", "p"), False, None, "td_column"),
               "dq_td_only": (6, ("dq", "td"), False, None, "td_two_pass")}
TD_VARIANT_CASES = [(L, Bn, n, B, v) for (L, Bn, n, B) in TD_VARIANT_POINTS for v in TD_VARIANTS]


def td_variant_key(L, Bn, n, B, v):
    return f"td L={L} Bn={Bn} n={n} B={B} {v}"


@pytest.mark.parametrize("L,Bn,n,B,variant", TD_VARIANT_CASES)
def test_td_window_variants(nv, routes, L, Bn, n, B, variant):
    A, want, weighted, opts, route = TD_VARIANTS[variant]
    key = td_variant_key(L, Bn, n, B, variant)
    ROUTES.assert_route(key, route, list(routes[key]))
    inputs = td_inputs(L, B, A, Bn, n, seed=L * 7 + B + n)
    w = np.random.default_rng(B).uniform(0.05, 1.0, B).astype(np.float32) if weighted else None
    o, _ = td_call(nv, inputs, L, B, A, Bn, n, want=want, w=w, opts=opts)
    assert set(o) == set(want)
    check_td(variant, key, o, td_ref(inputs, L, Bn, n, w=w, opts=opts), opts)


@pytest.mark.parametrize("L,B,A", [(2, 1, 6), (2, 33, 38), (9, 32, 6), (160, 2, 38), (3, 257, 6)])
def test_td_quirk_drops_the_last_element(nv, L, B, A):
    """A huge TD at (L-1, B-1), the element learner.py:137's [b:-1:B] drops: no priority moves, the loss does."""
    Bn, n = 1, 2
    inputs = td_inputs(L, B, A, Bn, n, seed=L + B + A)
    base, _ = td_call(nv, inputs, L, B, A, Bn, n)
    q = inputs[0].copy()
    q[L - 1, B - 1] += 1e4
    big, _ = td_call(nv, (q,) + inputs[1:], L, B, A, Bn, n)
    assert np.array_equal(big["p"].view(np.uint32), base["p"].view(np.uint32))
    assert big["loss"][0] > 1e3 * base["loss"][0]
    assert big["td"][L - 1, B - 1] > 1e7 and np.array_equal(big["td"][:L - 1], base["td"][:L - 1])
    check_td("quirk", f"quirk L={L} B={B} A={A}", big, td_ref((q,) + inputs[1:], L, Bn, n))


# ------------------------------------------------------------------------------------------------ nets
class NetRun:
    """Device buffers of one r2d2_lstm_net_forward / _backward case (zero inputs without a seed); out and d_act start
    as NaN so that an unwritten element fails every bound."""

    def __init__(self, nv, O, A, H, critic, T, B, repeat, first_row, seed=None):
        self.nv, self.critic, self.T, self.B, self.repeat, self.first_row = nv, critic, T, B, repeat, first_row
        self.O, self.A, self.H = O, A, H
        rng = np.random.default_rng(seed)
        if seed is None:
            z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
            self.p = {k: np.zeros_like(v) for k, v in make_params(rng, O, A, H, critic).items()}
            self.obs, self.act, self.h0, self.c0 = z(T, B, O), z(T, B, A), z(B, H), z(B, H)
            self.d_out = z(T - first_row, B, A)
        else:
            self.p = make_params(rng, O, A, H, critic)
            self.obs = rng.standard_normal((T, B, O)).astype(np.float32)
            self.act = rng.uniform(-1, 1, (T, B, A)).astype(np.float32)
            self.h0 = (0.3 * rng.standard_normal((B, H))).astype(np.float32)
            self.c0 = (0.3 * rng.standard_normal((B, H))).astype(np.float32)
            self.d_out = rng.standard_normal((T - first_row, B, A)).astype(np.float32)
        lib = nv.lib()
        self.shape = nv.NetShape(O, A, H, int(critic))
        flat = np.concatenate([self.p[k].reshape(-1) for k in lo.PARAM_KEYS])
        assert lib.r2d2_net_param_count(nv.byref(self.shape)) == flat.size
        self.ws = torch.zeros(lib.r2d2_net_workspace_floats(nv.byref(self.shape), T, B, repeat), device="cuda")
        self.dparams, self.dobs, self.dact, self.dh0, self.dc0 = (dev(a) for a in (flat, self.obs, self.act, self.h0,
                                                                                    self.c0))
        self.dd_out = dev(self.d_out)
        self.out = torch.full((T - first_row, B, A), float("nan"), device="cuda")
        self.grads = torch.zeros(flat.size, device="cuda")
        self.d_act = torch.full((T, B, A), float("nan"), device="cuda") if critic else None

    def forward(self):
        nv = self.nv
        nv.check(nv.lib().r2d2_lstm_net_forward(
            nv.byref(self.shape), nv.dptr(self.dparams), nv.dptr(self.dobs), nv.dptr(self.dact) if self.critic else None,
            nv.dptr(self.dh0), nv.dptr(self.dc0), self.T, self.B, self.repeat, self.first_row, nv.dptr(self.out),
            nv.dptr(self.ws), nv.current_stream()))

    def backward(self):
        nv = self.nv
        self.grads.zero_()                                    # the weight-gradient products add into the block
        nv.check(nv.lib().r2d2_lstm_net_backward(
            nv.byref(self.shape), nv.dptr(self.dparams), nv.dptr(self.dobs), nv.dptr(self.dact) if self.critic else None,
            nv.dptr(self.dd_out), self.T, self.B, self.repeat, self.first_row, nv.dptr(self.grads),
            nv.dptr(self.d_act), nv.dptr(self.ws), nv.current_stream()))

    def check(self, group, case, tol_fwd=TOL_FWD, tol_bwd=TOL_BWD):
        """Forward and backward against lo.net_forward / net_backward: out and d_act per time row, every gradient."""
        nv, critic, repeat, fr = self.nv, self.critic, self.repeat, self.first_row
        self.forward()
        self.backward()
        torch.cuda.synchronize()
        assert scan_status(nv) == 0, f"{case}: a bounded hand-off wait expired inside a scan kernel"
        p = {k: f64(v) for k, v in self.p.items()}
        x = np.concatenate((self.obs, self.act), 2) if critic else self.obs
        sv = lo.net_forward(p, f64(x), f64(self.h0), f64(self.c0), critic=critic, repeat=repeat)
        d_full = np.zeros_like(sv["out"])
        d_full[repeat - 1::repeat][fr:] = f64(self.d_out)
        g_ref, dx_ref, _ = lo.net_backward(p, sv, d_full, critic=critic, want_wgrad=True, want_dx=critic)
        WORST.bound(f"{group} out", f"{case} out", self.out.cpu().numpy(), sv["out"][repeat - 1::repeat][fr:], tol_fwd,
              time_axis=0)
        if critic:
            WORST.bound(f"{group} d_act", f"{case} d_act", self.d_act.cpu().numpy(), dx_ref[:, :, self.O:], tol_bwd,
                  time_axis=0)
        g, off = self.grads.cpu().numpy(), 0
        for k in lo.PARAM_KEYS:
            n = g_ref[k].size
            WORST.bound(f"{group} grad", f"{case} grad {k}", g[off:off + n].reshape(g_ref[k].shape), g_ref[k], tol_bwd)
            off += n


# ------------------------------------------------------------------------------------------------ 2. wgrad routes
# O = 20 and A = 3 put the obs block of dW1 (N = O) into thin_tn_kernel<24> and dW3 (M = A) and the action block
# (N = A) into thin_tn_kernel<8>; a product that stays on split_k = 1 runs the mma.sync kernel.  H = 128: cluster scans.
WG = dict(O=20, A=3, H=128)
WG_PRODUCTS = ("dW3", "dW1 obs", "dW1 act")


def wgrad_launches(critic, M, Mh, switch):
    """Expected launches {thin_tn<8>, thin_tn<24>, mma} of a backward over M = T·B rows, Mh = (T - first_row)·B of them
    under the head, given the switch points (first row count on thin_tn) of the three products."""
    t8 = int(Mh >= switch["dW3"]) + (int(M >= switch["dW1 act"]) if critic else 0)
    t24 = int(M >= switch["dW1 obs"])
    return {"thin_tn<8>": t8, "thin_tn<24>": t24, "mma": (3 if critic else 2) - t8 - t24}


def observed_wgrad(counts):
    return {"thin_tn<8>": count(counts, "thin_tn", (8,)), "thin_tn<24>": count(counts, "thin_tn", (24,)),
            "mma": count(counts, "mma")}


def probe_wgrad(nv, critic, rows, cache):
    """observed_wgrad of the backward of a one-row window (T = 1, first_row 0) of `rows` batch rows."""
    key = (critic, rows)
    if key not in cache:
        run = NetRun(nv, WG["O"], WG["A"], WG["H"], critic, 1, rows, 1, 0)
        run.forward()
        cache[key] = observed_wgrad(launch_counts(f"probe critic={critic} rows={rows}", run.backward))
    return cache[key]


def first_rows(pred):
    """Smallest row count with pred (monotone, false at 1), by doubling then bisection; None if not by B_MAX."""
    lo_r, hi = 1, 2
    while not pred(hi):
        lo_r = hi
        if hi >= B_MAX:
            return None
        hi = min(2 * hi, B_MAX)
    while hi - lo_r > 1:
        mid = (lo_r + hi) // 2
        if pred(mid):
            hi = mid
        else:
            lo_r = mid
    return hi


def find_wgrad_switches(nv):
    """{product: first T·B on thin_tn}: dW3 and the obs block from the actor (thin_tn<8> / <24>), the action block from
    the critic's second thin_tn<8> launch beyond dW3's."""
    cache = {}
    out = {"dW3": first_rows(lambda r: probe_wgrad(nv, False, r, cache)["thin_tn<8>"] >= 1),
           "dW1 obs": first_rows(lambda r: probe_wgrad(nv, False, r, cache)["thin_tn<24>"] >= 1)}
    out["dW1 act"] = first_rows(lambda r: probe_wgrad(nv, True, r, cache)["thin_tn<8>"] - int(r >= out["dW3"]) >= 1)
    return out, len(cache)


def wgrad_switch_cases(switch):
    """(product, side, critic, T, B, first_row): one-row windows just below and at each product's switch point."""
    out = []
    for prod in WG_PRODUCTS:
        for side, rows in (("below", switch[prod] - 1), ("above", switch[prod])):
            out.append((prod, side, prod == "dW1 act", 1, rows, 0))
    return out


# the wide products dW_hh (K = S·B) and dW_ih (K = T·B) on the wgmma kernel: 480 rows (15 k tiles of 32, just below
# the 16 that turn split-K on), 525 rows (17 k tiles in 2 slices of 9 and 8), and a 400-row window (800 k tiles in 62
# slices of 13, the last one 7) with 40 burn-in rows
WIDE_CASES = [(2, 240, 1), (3, 175, 0), (400, 64, 40)]


def wgrad_key(critic, T, B, first_row):
    return f"wgrad critic={int(critic)} T={T} B={B} first_row={first_row}"


def test_wgrad_switch_points_found(routes):
    sw = routes["wgrad_switch"]
    missing = [p for p in WG_PRODUCTS if sw.get(p) is None or sw[p] < 2]
    assert not missing, f"no switch from mma to thin_tn found below {B_MAX} rows for {missing}: {sw}"


@pytest.mark.parametrize("which", range(6))
def test_wgrad_at_switch(nv, routes, which):
    sw = routes["wgrad_switch"]
    prod, side, critic, T, B, fr = wgrad_switch_cases(sw)[which]
    key = wgrad_key(critic, T, B, fr)
    got, want = observed_wgrad(routes[key]), wgrad_launches(critic, T * B, (T - fr) * B, sw)
    assert got == want, f"{key}: launches {got}, expected {want} (switch points {sw})"
    on_thin = (T * B if prod != "dW3" else (T - fr) * B) >= sw[prod]
    assert on_thin == (side == "above")
    NetRun(nv, WG["O"], WG["A"], WG["H"], critic, T, B, 1, fr, seed=B * 3 + critic).check(
        "wgrad", f"{prod} {side} ({key})")


@pytest.mark.parametrize("T,B,first_row", WIDE_CASES)
def test_wgrad_wide_products(nv, routes, T, B, first_row):
    key = wgrad_key(True, T, B, first_row)
    sw = routes["wgrad_switch"]
    assert ran(list(routes[key]), ROUTE_KERNELS["wgmma"]), f"{key}: dW_hh / dW_ih not on wgmma: {routes[key]}"
    got, want = observed_wgrad(routes[key]), wgrad_launches(True, T * B, (T - first_row) * B, sw)
    assert got == want, f"{key}: launches {got}, expected {want}"
    NetRun(nv, WG["O"], WG["A"], WG["H"], True, T, B, 1, first_row, seed=T + B).check("wgrad wide", key)


# ------------------------------------------------------------------------------------------------ 3. scan steps
# (H, critic, T, repeat, first_row, B): S = T·repeat = 1, 2, 3, 4, 5 and 6 (every residue of the hand-off parity's
# period 4), first_row 0 and T - 1 (head_first_step = first_row·repeat), long chains of 160 and 320 steps
def _scan_cases():
    out = []
    for H in (128, 512, 96):
        for T in (1, 2, 3, 4, 5):
            for fr in sorted({0, T - 1}):
                out.append((H, True, T, 1, fr, 5))
        for T, fr in ((1, 0), (3, 2), (2, 0)):
            out.append((H, False, T, 2, fr, 7))
        out += [(H, True, 160, 1, 0, 9), (H, True, 160, 1, 159, 9), (H, False, 160, 2, 80, 9)]
    return out


SCAN_CASES = _scan_cases()
SCAN_O, SCAN_A = 7, 3


def scan_key(H, critic, T, repeat, first_row, B, d):
    return f"scan {d} H={H} critic={int(critic)} T={T} repeat={repeat} first_row={first_row} B={B}"


@pytest.mark.parametrize("H,critic,T,repeat,first_row,B", SCAN_CASES)
def test_scan_steps(nv, routes, H, critic, T, repeat, first_row, B):
    for d in ("fwd", "bwd"):
        case = scan_key(H, critic, T, repeat, first_row, B, d)
        names = list(routes[case])
        ROUTES.seen.setdefault(case, names)
        base = ROUTE_KERNELS[f"scan_{d}"]
        if H == 96:
            assert ran(names, ROUTE_KERNELS[f"cell_{d}"]) and not ran(names, base), (case, names)
        else:
            assert any(a[0] == H for n in names for a in template_args(n, base)), (case, names)
    run = NetRun(nv, SCAN_O, SCAN_A, H, critic, T, B, repeat, first_row, seed=H * 31 + T * 7 + first_row + repeat)
    long = T * repeat > 100
    run.check("scan long" if long else "scan", f"H={H} critic={critic} S={T * repeat} first_row={first_row}",
              tol_bwd=1e-4 if long else TOL_BWD)


# ------------------------------------------------------------------------------------------------ 4. learner
LEARNER_WINDOWS = [(0, 2, 1), (0, 8, 5), (1, 3, 1), (2, 2, 10), (17, 33, 3), (80, 80, 5), (40, 160, 10)]
LEARNER_CASES = [(Bn, L, n, B) for (Bn, L, n) in LEARNER_WINDOWS for B in (1, 2, 33)] + [(80, 80, 5, 130),
                                                                                        (40, 160, 10, 96)]


def _sd(m):
    return {k: v.detach().numpy().copy() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("Bn,L,n,B", LEARNER_CASES)
def test_learner_window(eng_mod, Bn, L, n, B):
    """Three iterations against the float64 oracle and the CPU port: q and the target per time row, the priorities,
    both losses, the final weights."""
    kw = dict(obs=5, act=2, hidden=32, batch=B, burn_in=Bn, learning=L, n_step=n)
    pc = ref_port.PathConfig(**kw)
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    port = ref_port.PortLearner(pc, seed=Bn + L + n + B)
    actor, critic = _sd(port.actor), _sd(port.critic)
    eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**kw))
    eng.load_state_dicts(actor, critic)
    ol = oracle_for(eng.cfg, actor, critic)
    errs = {}
    for it in range(3):
        batch = ref_port.synthetic_batch(pc, seed=700 + it, terminal_frac=0.3)
        eng.set_batch(batch)
        eng.step()
        ref_o, ref_p = ol.iteration(batch), port.iteration(batch)
        torch.cuda.synchronize()
        for name, ref in (("oracle", ref_o), ("port", ref_p)):
            for k in ("q_value", "target_q_value"):
                got = getattr(eng, k).cpu().numpy().reshape(L, B, 2)
                want = np.asarray(ref[k]).reshape(L, B, 2)
                errs[f"{name}/{k}/{it}"] = max(rel_l2(got, want), step_err(got, want))
            errs[f"{name}/priority/{it}"] = rel_l2(eng.priority.cpu().numpy(), ref["priority"])
            for i, k in enumerate(("critic_loss", "actor_loss")):
                errs[f"{name}/{k}/{it}"] = abs(eng.losses[i].item() / ref[k] - 1.0)
    for net in ("actor", "critic"):
        mine = {k: v.detach().cpu().numpy() for k, v in eng.views(net).items()}
        port_after = _sd(getattr(port, net))
        for k in lo.PARAM_KEYS:
            errs[f"oracle/{net}/{k}"] = rel_l2(mine[k], getattr(ol, net)[k])
            errs[f"port/{net}/{k}"] = rel_l2(mine[k], port_after[k])
    eng.close()
    WORST.note("learner", *errs.values())
    bad = {k: f"{v:.2e}" for k, v in errs.items() if not v < TOL}
    assert not bad, bad


def test_replay_fed_learner_at_burn_in_zero(eng_mod):
    """Batches drawn from a replay shard at burn-in 0 (episodes with 1 to 20 starts): each gathered batch through the
    engine and through the float64 oracle."""
    E = eng_mod
    cfg = E.PathConfig(obs=5, act=2, hidden=32, batch=16, burn_in=0, learning=8, n_step=3)
    rng = np.random.default_rng(8)
    rp = E.DeviceReplay(cfg, capacity_rows=4000)
    rp.add_episodes([episode(rng, cfg, int(e)) for e in rng.integers(cfg.learning + 1, cfg.learning + 21, size=30)])
    eng = E.LearnerEngine(cfg, seed=4)
    ol = oracle_for(cfg, {k: v.cpu().numpy() for k, v in eng.views("actor").items()},
                    {k: v.cpu().numpy() for k, v in eng.views("critic").items()})
    gen = torch.Generator(device="cuda").manual_seed(2)
    for it in range(3):
        rp.sample_into(eng, generator=gen)
        torch.cuda.synchronize()
        st = eng.states.cpu().numpy()
        batch = {"obs": eng.obs.cpu().numpy(), "act": eng.act.cpu().numpy(), "rew": eng.rew.cpu().numpy(),
                 "term": eng.term.cpu().numpy(), "a_state": st[0], "ta_state": st[1], "c_state": st[2],
                 "tc_state": st[3]}
        eng.step()
        ref = ol.iteration(batch)
        torch.cuda.synchronize()
        errs = {k: rel_l2(getattr(eng, k).cpu().numpy(), ref[k]) for k in ("q_value", "target_q_value", "priority")}
        WORST.note("learner replay-fed", *errs.values())
        assert all(v < TOL for v in errs.values()), (it, errs)
        rp.update_priorities(eng.leaf_idx, eng.priority)
    rp.close()
    eng.close()


@pytest.mark.parametrize("L,n,B", [(3, 1, 2), (8, 10, 33)])
def test_twin_critic_at_burn_in_zero(eng_mod, L, n, B):
    """Critic 2 and its target start from the zero state at row 0: with no burn-in rows at all."""
    kw = dict(obs=5, act=2, hidden=32, batch=B, burn_in=0, learning=L, n_step=n)
    actor, critic, batches = port_case(kw, seed=3, n_batches=2, batch_seed=40)
    worst = check_against_oracle(eng_mod, dict(kw, twin_critic=True), actor, critic, batches, 2)
    WORST.note("learner twin", worst)


# ------------------------------------------------------------------------------------------------ 5. replay, actor side
# (burn_in, learning, n_step): starts per episode E - (Bn + L) = 0, 1, 2 and a few more
REPLAY_WINDOWS = [(0, 2, 1), (2, 2, 10), (0, 33, 5), (80, 80, 5)]


@pytest.mark.parametrize("Bn,L,n", REPLAY_WINDOWS)
def test_replay_gather_at_few_starts(eng_mod, Bn, L, n):
    """Episodes with exactly 0, 1, 2 (and 5) sequence starts: the sum tree bit for bit against the C oracle, an episode
    without starts holds rows but no probability mass and is never drawn, and every gathered window and stored state
    bit for bit (episode-wise and file-wise ingest build the same tree)."""
    E = eng_mod
    cfg = E.PathConfig(obs=4, act=2, hidden=8, batch=48, burn_in=Bn, learning=L, n_step=n)
    rng = np.random.default_rng(Bn + L + n)
    starts = [1, 0, 2, 1, 5, 0, 2, 1, 2, 0, 1, 2]
    eps = [episode(rng, cfg, Bn + L + k) for k in starts]
    cap = sum(e[0].shape[0] for e in eps) + 7
    rp, rp2, oracle = E.DeviceReplay(cfg, capacity_rows=cap), E.DeviceReplay(cfg, capacity_rows=cap), SumTreeOracle(cap)
    rows0, row = [], 0
    for ep in eps:
        rp.add_episode(*ep)
        n_rows, k = ep[0].shape[0], len(ep[5])
        if k:
            oracle.set_range(row, ep[5])
        oracle.set_range(row + k, None, n_rows - k)
        rows0.append(row)
        row += n_rows
    rp2.add_episodes(eps)
    assert rp.stats()["n_episodes"] == len(eps)
    for lvl in range(oracle.levels):
        want = oracle.level(lvl)
        assert np.array_equal(rp.tree_level(lvl).cpu().numpy()[:len(want)], want), f"level {lvl}"
        assert np.array_equal(rp2.tree_level(lvl).cpu().numpy()[:len(want)], want), f"level {lvl} (add_episodes)"
    leaves = oracle.level(0)
    for ep, r0 in zip(eps, rows0):
        n_rows, k = ep[0].shape[0], len(ep[5])
        assert (leaves[r0 + k:r0 + n_rows] == 0).all() and (leaves[r0:r0 + k] > 0).all()
    u = np.concatenate([rng.uniform(size=4000).astype(np.float32), np.float32([0.0, np.nextafter(np.float32(1),
                                                                                                  np.float32(0))])])
    leaf = rp.sample_indices(torch.as_tensor(u).cuda()).cpu().numpy()
    assert np.array_equal(leaf, oracle.sample(u)) and (leaves[leaf] > 0).all()
    eng = E.LearnerEngine(cfg)
    rp.sample_into(eng, u=torch.as_tensor(u[:cfg.batch]).cuda())
    torch.cuda.synchronize()
    li = eng.leaf_idx.cpu().numpy()
    assert np.array_equal(li, oracle.sample(u[:cfg.batch]))
    ep_i, seq_i = rp.decode(li)
    obs, act, rew, term, states = (t.cpu().numpy() for t in (eng.obs, eng.act, eng.rew, eng.term, eng.states))
    for b in range(cfg.batch):
        ep, s = eps[ep_i[b]], seq_i[b]
        assert rows0[ep_i[b]] + s == li[b] and s < len(ep[5])
        for got, src in ((obs, ep[0]), (act, ep[1]), (rew, ep[2]), (term, ep[3])):
            assert np.array_equal(got[:, b], src[s:s + cfg.rows])
        assert np.array_equal(states[:, :, b], ep[4][s])
    eng.close()
    rp.close()
    rp2.close()


# (Bn, L, n): n-step 1, burn-in 0, long windows; episode lengths E give E - (Bn + L) = 0, 1, 2 and more starts
ACTOR_WINDOWS = [(0, 2, 1), (0, 160, 5), (3, 7, 1), (80, 400, 10)]


@pytest.mark.parametrize("rescaling,metric", [("reference", "squared"), ("invertible", "abs")])
@pytest.mark.parametrize("Bn,L,n", ACTOR_WINDOWS)
def test_actor_side_windows(nv, Bn, L, n, rescaling, metric):
    """r2d2_nstep_rewards and r2d2_actor_priorities(_ex) against oracle/actor_oracle.py, p_max beyond every episode's
    start count: the padding is 0."""
    rng = np.random.default_rng(Bn + L + n)
    lens = [Bn + L + k + n for k in (0, 1, 2, 9, 37)]
    B, T, A, gamma = len(lens), max(lens), 3, float(np.float32(0.997))   # the library takes gamma in float32
    p_max = T - n - (Bn + L) + 5
    raw = np.zeros((T, B), np.float32)
    q = np.zeros((T, B, A), np.float32)
    qt = (rng.standard_normal((T, B, A)) * 3).astype(np.float32)
    term = np.ones((T, B), np.float32)
    for b, N in enumerate(lens):
        raw[:N, b] = rng.standard_normal(N)
        q[:N - n, b] = rng.standard_normal((N - n, A)) * 2
        term[:N - n, b] = 0
    n_rows = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rew = torch.full((T, B), float("nan"), device="cuda")
    nv.check(nv.lib().r2d2_nstep_rewards(ptr(dev(raw)), ptr(n_rows), T, B, n, gamma, ptr(rew), nv.current_stream()))
    prio = torch.full((B, p_max), float("nan"), device="cuda")
    dq, dqt, dterm = dev(q), dev(qt), dev(term)
    if rescaling == "reference":
        rc = nv.lib().r2d2_actor_priorities(ptr(dq), ptr(dqt), ptr(rew), ptr(dterm), ptr(n_rows), B, A, Bn, L, n,
                                            gamma, 0.9, p_max, ptr(prio), nv.current_stream())
    else:
        o = nv.TdOptions(NATIVE[rescaling], 1e-2, NATIVE[metric])
        rc = nv.lib().r2d2_actor_priorities_ex(ptr(dq), ptr(dqt), ptr(rew), ptr(dterm), ptr(n_rows), B, A, Bn, L, n,
                                               gamma, 0.9, p_max, ptr(prio), nv.byref(o), nv.current_stream())
    nv.check(rc)
    torch.cuda.synchronize()
    rew_h, prio_h = rew.cpu().numpy(), prio.cpu().numpy()
    for b, N in enumerate(lens):
        want_r = actor_oracle.nstep_rewards(raw[:N, b], n, gamma)
        WORST.bound("actor nstep", f"b={b} rewards", rew_h[:N, b], want_r, 1e-6, time_axis=0)
        assert (rew_h[N:, b] == 0).all()
        want = actor_oracle.window_priorities(f64(q[:N - n, b]), f64(qt[:N, b]), f64(rew_h[:N, b]), f64(term[:N, b]),
                                              burn_in=Bn, learning=L, n_step=n, gamma=gamma, rescaling=rescaling,
                                              eps=float(np.float32(1e-2)), metric=metric)
        assert want.size == N - n - (Bn + L)
        if want.size:
            WORST.bound("actor priority", f"b={b} priorities", prio_h[b, :want.size], want, 1e-5)
        assert (prio_h[b, want.size:] == 0).all(), f"b={b}: padding past {want.size} starts is not 0"


# ------------------------------------------------------------------------------------------------ 6. L = 1
@pytest.mark.parametrize("entry", ["plain", "weighted", "ex"])
def test_td_refuses_one_step_window_with_priority(nv, entry):
    """At L = 1 the [b:-1:B] series of the last batch element is empty: a priority output is refused (the library
    used to write eta * max(empty) + (1 - eta) * 0 / 0 = NaN there)."""
    L, B, A, Bn, n = 1, 4, 6, 2, 3
    inputs = td_inputs(L, B, A, Bn, n, seed=1)
    w = np.ones(B, np.float32) if entry != "plain" else None
    opts = ("reference", 0.0, "squared") if entry == "ex" else None
    for want in (("y", "dq", "td", "p", "loss"), ("y", "dq", "p", "loss"), ("p",)):
        o, rc = td_call(nv, inputs, L, B, A, Bn, n, want=want, w=w, opts=opts, check=False)
        assert rc == ERR_ARG, f"{entry} {want}: L = 1 accepted with a priority output, priority = {o['p']}"
        assert "L >= 2" in nv.lib().r2d2_last_error().decode()


@pytest.mark.parametrize("A,want", [(6, ("y", "dq", "td", "loss")), (38, ("y", "dq", "td", "loss")),
                                    (6, ("y", "dq", "loss"))])
def test_td_one_step_window_without_priority(nv, A, want):
    """Critic 2's TD at L = 1 asks for no priority: target, dq, td_sq and the loss stay defined and finite."""
    L, B, Bn, n = 1, 33, 0, 1
    inputs = td_inputs(L, B, A, Bn, n, seed=A)
    o, _ = td_call(nv, inputs, L, B, A, Bn, n, want=want)
    q, qn, rew, term = (f64(x) for x in inputs)
    y = lo.n_step_target(rew[Bn:Bn + L, :, None], 0.997 ** n * (1.0 - term[Bn + n - 1:Bn + n - 1 + L, :, None]), qn)
    diff = q - y
    assert all(np.isfinite(v).all() for v in o.values())
    WORST.bound("td L=1 y", "y", o["y"], y, 1e-6)
    WORST.bound("td L=1 dq", "dq", o["dq"], 2.0 * diff / diff.size, 1e-5)
    if "td" in o:
        WORST.bound("td L=1 td_sq", "td_sq", o["td"], np.mean(diff * diff, axis=2), 1e-5)
    assert abs(o["loss"][0] / np.mean(diff * diff) - 1.0) < 1e-5


def test_learner_refuses_one_step_window(eng_mod, nv):
    """PathConfig refuses L = 1, and so does r2d2_learner_create when it is reached around it."""
    with pytest.raises(ValueError, match="learning"):
        eng_mod.PathConfig(obs=3, act=2, hidden=32, batch=4, burn_in=2, learning=1, n_step=2)
    for twin in (False, True):
        cfg = eng_mod.PathConfig(obs=3, act=2, hidden=32, batch=4, burn_in=2, learning=2, n_step=2, twin_critic=twin)
        cfg.learning = 1
        with pytest.raises(nv.NativeError, match="learning >= 2"):
            eng_mod.LearnerEngine(cfg)


# ------------------------------------------------------------------------------------------------ route observation
def route_child(out_path):
    """Entry point of the fresh process behind the `routes` fixture: the wgrad switch points and every case's launches
    (same entry points and shapes, zero inputs: no route depends on values) once under the profiler."""
    from r2d2_b200 import native as nv
    nv.lib().r2d2_set_scan_impl(1)
    switch, probes = find_wgrad_switches(nv)
    seen = {}
    for L, Bn, n, B, A, route in TD_CASES:
        z = td_inputs(L, B, A, Bn, n, 0)
        z = tuple(np.zeros_like(x) for x in z)
        seen[td_key(L, Bn, n, B, A, route)] = launch_counts(
            route, lambda: td_call(nv, z, L, B, A, Bn, n, want=TD_WANT[route]))
    for L, Bn, n, B, v in TD_VARIANT_CASES:
        A, want, weighted, opts, _ = TD_VARIANTS[v]
        z = tuple(np.zeros_like(x) for x in td_inputs(L, B, A, Bn, n, 0))
        w = np.ones(B, np.float32) if weighted else None
        seen[td_variant_key(L, Bn, n, B, v)] = launch_counts(
            v, lambda: td_call(nv, z, L, B, A, Bn, n, want=want, w=w, opts=opts))
    for _, _, critic, T, B, fr in wgrad_switch_cases(switch):
        run = NetRun(nv, WG["O"], WG["A"], WG["H"], critic, T, B, 1, fr)
        run.forward()
        seen[wgrad_key(critic, T, B, fr)] = launch_counts("wgrad", run.backward)
    for T, B, fr in WIDE_CASES:
        run = NetRun(nv, WG["O"], WG["A"], WG["H"], True, T, B, 1, fr)
        run.forward()
        seen[wgrad_key(True, T, B, fr)] = launch_counts("wgrad", run.backward)
    for c in SCAN_CASES:
        run = NetRun(nv, SCAN_O, SCAN_A, c[0], c[1], c[2], c[5], c[3], c[4])
        seen[scan_key(*c, "fwd")] = launch_counts("scan fwd", run.forward)
        seen[scan_key(*c, "bwd")] = launch_counts("scan bwd", run.backward)
    with open(out_path, "w") as f:
        json.dump({"switch": switch, "probes": probes, "seen": seen}, f)


@pytest.fixture(scope="module")
def routes(nv):
    """{case: {route kernel: launches}} and "wgrad_switch": {product: first T·B on thin_tn}, observed in a fresh Python
    process (route_child).  Prints the switch points."""
    got = observe_in_fresh_process("test_gpu_sequence_geometry", timeout=1200)
    routes = dict(got["seen"])
    routes["wgrad_switch"] = got["switch"]
    print(f"\nroute process: {got['probes']} bisection probes")
    print("weight-gradient switch points (first T·B on thin_tn_kernel; below it the mma.sync kernel), "
          f"O = {WG['O']}, A = {WG['A']}, H = {WG['H']}:")
    for p in WG_PRODUCTS:
        print(f"  {p:8s} from T·B = {got['switch'][p]}")
    return routes
