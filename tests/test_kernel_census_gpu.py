"""Every kernel the library compiles, launched by its census case (tests/kernel_census.py) and held to
that case's float64 or exact reference.

The launch census runs every case under torch.profiler in a spawned child process (many profiling
sessions in the test process leave later sessions in it without kernel records; see
tests/test_coefficients_batch_gpu.py) and returns the kernels each case launched: each row's case
must launch the row's kernel.  The parity test runs each case in this process, parametrised by
instantiation, and holds every result to its bar.  A case shared by several rows runs once.
"""
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import kernel_census as K

pytestmark = pytest.mark.gpu


def _launched(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {K.normalise(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and not e.name.startswith(("Memcpy", "Memset"))}


def _census_child(case_ids):
    """{case id: kernels it launched} (run in a spawned process).  Each case runs once first, so that
    one-time work (weight preparation, packing, module loading) is outside the profiled call; kernels
    of that first run count too, a call's cache being part of it."""
    out = {}
    for cid in case_ids:
        first = _launched(K.CASES[cid])
        out[cid] = sorted(first | _launched(K.CASES[cid]))
    return out


@pytest.fixture(scope="module")
def census():
    with mp.get_context("spawn").Pool(1) as pool:
        return pool.apply(_census_child, (sorted(K.CASES),))


def test_every_case_launches_its_kernels(census):
    missed = [f"{src}: {k} (case {cid} launched {census[cid]})" for (src, k), cid in sorted(K.ROWS.items())
              if k not in census[cid]]
    print(f"\n{len(K.ROWS)} kernels, {len(K.CASES)} cases; "
          f"{len(K.ROWS) - len(missed)} launched by their case")
    assert not missed, f"{len(missed)} rows not launched by their case: " + "; ".join(missed)


_results = {}


def _run(cid):
    if cid not in _results:
        torch.manual_seed(0)
        check = K.CASES[cid]()
        torch.cuda.synchronize()
        _results[cid] = check()
    return _results[cid]


@pytest.mark.parametrize("key", sorted(K.ROWS), ids=lambda k: f"{k[0][:-3]}:{k[1]}")
def test_kernel_against_its_reference(key):
    res = _run(K.ROWS[key])
    for what, err, bar in res:
        print(f"{key[1]} [{K.ROWS[key]}] {what}: {err:.3e} (bar {bar:.0e})")
    over = [f"{what}: {err:.3e} > {bar:.0e}" for what, err, bar in res if not err <= bar]
    assert not over, f"{key[1]} (case {K.ROWS[key]}): " + "; ".join(over)
    assert res and all(np.isfinite(err) for _, err, _ in res)
