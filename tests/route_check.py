"""Which kernel served a call: run it under torch.profiler and assert the route kernel that ran, so that a dispatch
change that moves a test case off its route fails by name instead of silently dropping the coverage.

A route is a key of ROUTE_KERNELS, optionally followed by ":" and comma-separated template arguments, which must match
the kernel's trailing template arguments (bool arguments as 0 / 1): "smalln:16" is thin_smalln_kernel<*, 16>,
"scan_fwd:128,32" is lstm_scan_fwd_kernel<128, 32>.  Each test module keeps its own RouteLog for its report."""
import json
import os
import re
import subprocess
import sys
import tempfile
import time
from collections import Counter

# route name -> kernel (base name) that serves it
ROUTE_KERNELS = {
    "td_column": "td_priority_column_kernel",
    "td_two_pass": "td_elem_kernel",
    "smallk": "thin_smallk_kernel",
    "smalln": "thin_smalln_kernel",
    "rowdot4": "thin_rowdot4_kernel",
    "thin_tn": "thin_tn_kernel",
    "mma": "gemm_bf16x3_kernel",
    "wgmma": "gemm_packed_kernel",
    "scan_fwd": "lstm_scan_fwd_kernel",
    "scan_bwd": "lstm_scan_bwd_kernel",
    "cell_fwd": "lstm_cell_fwd_pointwise",
    "cell_bwd": "lstm_cell_bwd_pointwise",
    "policy": "policy_phase_kernel",
}


def template_args(name, base):
    """Integer template arguments of every instance of kernel `base` in profiler name `name` (demangled or
    Itanium-mangled; true / false -> 1 / 0), one tuple per instance."""
    out = []
    for m in re.finditer(re.escape(base) + r"<([^<>]*)>", name):
        args = [a.strip() for a in m.group(1).split(",")]
        out.append(tuple(1 if a == "true" else 0 if a == "false" else int((re.findall(r"-?\d+", a) or ["-1"])[-1])
                         for a in args))
    for m in re.finditer(re.escape(base) + r"I((?:L[bi]-?\d+E)+)E", name):
        out.append(tuple(int(v) for v in re.findall(r"L[bi](-?\d+)E", m.group(1))))
    return out


def ran(names, base, args=None):
    """Did a kernel `base` whose trailing template arguments are `args` (None: any) run?"""
    for n in names:
        if base not in n:
            continue
        if args is None:
            return True
        if any(a[len(a) - len(args):] == tuple(args) for a in template_args(n, base) if len(a) >= len(args)):
            return True
    return False


def parse_route(route):
    key, _, spec = route.partition(":")
    return key, (tuple(int(v) for v in spec.split(",")) if spec else None)


SENTINEL = "FillFunctor"                      # the kernel of cuda_session's fill
PAUSES = (0.1, 0.3, 1.0, 2.0, 4.0, 8.0, 8.0)  # seconds between the sessions of observe: eight sessions in all


def route_names(names):
    """The names in `names` that belong to a route kernel."""
    return [n for n in names if any(b in n for b in ROUTE_KERNELS.values())]


def recorded_route(names):
    return bool(route_names(names))


def recorded_sentinel(names):
    return any(SENTINEL in n for n in names)


def cuda_session(fn):
    """fn() and then a fill kernel of torch's own (the sentinel) under torch.profiler -> (fn's result, the name of every
    CUDA kernel launch recorded)."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.empty(256, device="cuda").fill_(1.0)
        torch.cuda.synchronize()
    return out, [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]


def observe(case, fn, complete, *, agree=False, lost=None, session=cuda_session):
    """session(fn) until one is complete -> (fn's result, kernel names) of that session, or None when none of
    len(PAUSES) + 1 sessions was.  Every session runs fn in full, so fn must be idempotent.

    torch.profiler now and then returns a session without some or all of the kernels it ran (on an H100 with torch
    2.11 / CUDA 12.8, about one session in a hundred, and then often the next few sessions too; in a long-lived test
    process, after the hundreds of sessions other test files run, collection can stop altogether, which is why the route
    suites observe in a fresh process).  complete(names) tells a usable session: recorded_route or recorded_sentinel.
    agree: the caller asserts launch counts exactly, so a session that kept only part of the kernels must not be taken:
    a complete session counts only when the complete session just before it recorded the same route kernel launches.
    Each repeated session appends `case` to `lost` and is preceded by a growing pause."""
    prev = None
    for pause in PAUSES + (None,):
        out, names = session(fn)
        counts = Counter(route_names(names)) if complete(names) else None
        if counts is not None and (not agree or counts == prev):
            return out, names
        prev = counts
        if lost is not None:
            lost.append(case)
        if pause is not None:
            time.sleep(pause)
    return None


def launch_counts(case, fn, agree=False):
    """{profiler name of a route kernel: launches} of fn, from a session that recorded a route kernel (observe)."""
    got = observe(case, fn, recorded_route, agree=agree)
    assert got is not None, (f"{case}: no two profiler sessions in a row recorded the same launches" if agree else
                             f"{case}: the profiler recorded no route kernel in {len(PAUSES) + 1} sessions")
    return dict(Counter(route_names(got[1])))


def observe_in_fresh_process(module, timeout):
    """The JSON that tests/<module>.py's route_child(path) writes, run in a new Python interpreter: route kernels are
    observed there because a long-lived test process can stop recording them (observe)."""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "routes.json")
        code = ("import sys; sys.path[:0] = %r; import %s as t; t.route_child(%r)"
                % ([here, root, os.path.join(root, "pytorch-r2d2-dpg_b200")], module, out))
        res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, cwd=root)
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
        with open(out) as f:
            return json.load(f)


class RouteLog:
    """Profiled calls of one test module: `seen` maps a case to the route kernels that ran, `lost` lists the cases whose
    profiler session had to be repeated."""

    def __init__(self):
        self.seen = {}
        self.lost = []

    def profile(self, case, fn):
        """Run fn (idempotent) under the CUDA profiler (observe) -> (fn's result in the last session, sorted names of
        the route kernels that ran)."""
        got = observe(case, fn, recorded_route, lost=self.lost)
        assert got is not None, f"{case}: the profiler recorded no route kernel in {len(PAUSES) + 1} sessions"
        routed = sorted(set(route_names(got[1])))
        self.seen[case] = routed
        return got[0], routed

    def run_routed(self, case, route, fn):
        """profile(), then assert that of the route kernels exactly the expected one served the call (a session that
        recorded a different route kernel fails at once).  Returns fn's result."""
        out, names = self.profile(case, fn)
        self.assert_route(case, route, names)
        return out

    def assert_route(self, case, route, names, others=()):
        """Of the route kernels in `names` (profiler kernel names), exactly the one of `route` and those of the route
        keys `others` ran, and the `route` kernel with its template arguments."""
        key, args = parse_route(route)
        self.seen.setdefault(case, route_names(names))
        keys = sorted(k for k in ROUTE_KERNELS if any(ROUTE_KERNELS[k] in n for n in names))
        assert keys == sorted({key, *others}), f"{case}: expected route {key} ({ROUTE_KERNELS[key]}), ran: {names}"
        assert ran(names, ROUTE_KERNELS[key], args), f"{case}: expected {ROUTE_KERNELS[key]} {args}: {names}"

    def report(self, title="routes seen"):
        print(f"profiler sessions repeated: {len(self.lost)} {self.lost}")
        print(f"{title}:")
        for case, names in self.seen.items():
            print(f"  {case}: {names}")
