"""Which kernel served a call: run it under torch.profiler and assert the route kernel that ran, so that a dispatch
change that moves a test case off its route fails by name instead of silently dropping the coverage.

A route is a key of ROUTE_KERNELS, optionally followed by ":" and comma-separated template arguments, which must match
the kernel's trailing template arguments (bool arguments as 0 / 1): "smalln:16" is thin_smalln_kernel<*, 16>,
"scan_fwd:128,32" is lstm_scan_fwd_kernel<128, 32>.  Each test module keeps its own RouteLog for its report."""
import re
import time

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


class RouteLog:
    """Profiled calls of one test module: `seen` maps a case to the route kernels that ran, `lost` lists the cases whose
    profiler session had to be repeated."""

    def __init__(self):
        self.seen = {}
        self.lost = []

    def profile(self, case, fn):
        """Run fn (idempotent) under the CUDA profiler -> (fn's result, sorted names of the route kernels that ran).
        torch.profiler now and then returns a session without any of the kernels it ran (on an H100 with torch 2.11 /
        CUDA 12.8, about one session in a hundred, and then often the next few sessions too): a session that recorded
        no route kernel at all is repeated after a growing pause, five sessions in all, and then fails.  Every session
        runs fn in full; the caller checks the values of the last one.  In a long-lived test process, after the hundreds
        of sessions other test files run, collection can stop altogether (tests/test_gpu_value_rescaling.py): a module
        with many cases observes them in a fresh process instead (tests/test_gpu_hidden_size.py)."""
        import torch
        from torch.autograd import DeviceType
        from torch.profiler import ProfilerActivity, profile
        for pause in (0.1, 0.3, 1.0, 3.0, None):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                out = fn()
                torch.cuda.synchronize()
            names = sorted({e.name for e in prof.events() if e.device_type == DeviceType.CUDA})
            routed = [n for n in names if any(b in n for b in ROUTE_KERNELS.values())]
            if routed or pause is None:
                break
            self.lost.append(case)
            time.sleep(pause)
        assert routed, f"{case}: the profiler recorded no route kernel in five sessions (kernels recorded: {names})"
        self.seen[case] = routed
        return out, routed

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
        self.seen.setdefault(case, [n for n in names if any(b in n for b in ROUTE_KERNELS.values())])
        keys = sorted(k for k in ROUTE_KERNELS if any(ROUTE_KERNELS[k] in n for n in names))
        assert keys == sorted({key, *others}), f"{case}: expected route {key} ({ROUTE_KERNELS[key]}), ran: {names}"
        assert ran(names, ROUTE_KERNELS[key], args), f"{case}: expected {ROUTE_KERNELS[key]} {args}: {names}"

    def report(self, title="routes seen"):
        print(f"profiler sessions repeated: {len(self.lost)} {self.lost}")
        print(f"{title}:")
        for case, names in self.seen.items():
            print(f"  {case}: {names}")
