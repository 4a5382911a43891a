"""Helpers shared by the GPU kernel and route suites: the `nv` fixtures, device and float64 conversions, the scan status
flag, device properties the dispatch reads, the standard inputs of a TD call and of one net, and the worst-error log
behind each suite's bounds and -s report.

A suite takes a fixture into its own namespace (`from kernel_harness import nv_routes as nv`); pytest registers it
under that name."""
import ctypes
from collections import defaultdict

import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import col_err, step_err, tile_err, unit_group_err


@pytest.fixture(scope="module")
def nv():
    """The native library, loaded."""
    from r2d2_b200 import native
    native.lib()
    return native


@pytest.fixture(scope="module")
def nv_routes():
    """The native library in the default GEMM implementation with the cluster scans on: the routes a route suite
    asserts are that configuration's."""
    from r2d2_b200 import native
    lib = native.lib()
    assert lib.r2d2_get_gemm_impl() == 1, "these routes are the default implementation's"
    lib.r2d2_set_scan_impl(1)
    return native


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def f64(a):
    """a as the library sees it (float32), in float64."""
    return np.asarray(a, np.float32).astype(np.float64)


def ptr(t, offset_floats=0):
    """Device address of tensor t (None for None), offset_floats floats in."""
    return None if t is None else t.data_ptr() + 4 * offset_floats


def scan_status(nv, stream=None):
    """The scans' device-wide flag (sticky until read): nonzero when a bounded hand-off wait of a scan expired."""
    status = ctypes.c_int(0)
    nv.check(nv.lib().r2d2_scan_status(ctypes.byref(status), nv.current_stream() if stream is None else stream))
    return status.value


def num_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def smem_optin():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).shared_memory_per_block_optin


def td_inputs(L, B, A, Bn, n, seed):
    """q, q' [L, B, A], rewards and terminals [Bn + L + n, B]: standard normal, terminals anywhere (the window's middle
    included)."""
    rng = np.random.default_rng(seed)
    T = Bn + L + n
    q, qn = rng.standard_normal((L, B, A)) * 2, rng.standard_normal((L, B, A)) * 5
    rew = rng.standard_normal((T, B)) * 3
    term = (rng.uniform(size=(T, B)) < 0.15).astype(np.float64)
    return q, qn, rew, term


def make_params(rng, O, A, H, critic):
    """One net's weights (float32), uniform at about the scale of PyTorch's initialisation."""
    I = O + (A if critic else 0)
    u = lambda shp, b: rng.uniform(-b, b, shp).astype(np.float32)  # noqa: E731
    return {"l1.weight": u((H, I), 1 / np.sqrt(I)), "l1.bias": u((H,), 0.2),
            "l2.weight_ih": u((4 * H, H), 2 / np.sqrt(4 * H)), "l2.weight_hh": u((4 * H, H), 2 / np.sqrt(4 * H)),
            "l2.bias_ih": u((4 * H,), 0.1), "l2.bias_hh": u((4 * H,), 0.1),
            "l3.weight": u((A, H), 1 / np.sqrt(H)), "l3.bias": u((A,), 0.1)}


class WorstLog:
    """The worst error seen per "<group> <measure>" in one test module, for its -s report."""

    def __init__(self):
        self.worst = defaultdict(float)

    def note(self, key, *errs):
        self.worst[key] = max(self.worst[key], *errs)

    def bound(self, group, name, x, ref, tol, *, cols=None, tile=None, tile_axis=-2, H=None, unit_axis=-1,
              time_axis=None, step_tol=None):
        """rel_l2 < tol, and each measure asked for: with `cols` the worst of that many columns (col_err), with `tile`
        the worst tile of that many indices along tile_axis (tile_err), with H the worst 32-unit group along unit_axis
        (unit_group_err), with time_axis the worst single time row (step_err < step_tol, default tol)."""
        errs = {"rel_l2": (rel_l2(x, ref), tol)}
        if cols:
            errs["col_err"] = (col_err(x, ref, cols), tol)
        if tile:
            errs["tile_err"] = (tile_err(x, ref, tile, axis=tile_axis), tol)
        if H:
            errs["unit_group_err"] = (unit_group_err(x, ref, H, unit_axis), tol)
        if time_axis is not None:
            errs["step_err"] = (step_err(x, ref, time_axis), step_tol or tol)
        for k, (e, _) in errs.items():
            self.note(f"{group} {k}", e)
        bad = {k: f"{e:.3e} (bound {t:.0e})" for k, (e, t) in errs.items() if not e < t}
        assert not bad, f"{name}: {bad}"

    def report(self):
        print("\nworst errors per group:")
        for g, e in sorted(self.worst.items()):
            print(f"  {g:34s} {e:.2e}")
