"""Times the reference's own JAX file (jax/bilateral_slice.py:299-380, imported unmodified under the
numpy stand-in, oracle/jax_shim.py) + the reference's `apply` (hdrnet/layers.py:153-198) on THIS
machine's host cores: BASELINE.md section 3's "R-JAX" row.  It needs a google/hdrnet checkout
(HDRNET_REFERENCE); bench.py's CPU legs time the reference's compiled C++ loops (or the C
restatement) instead, so this is a reported-only number.

    HDRNET_REFERENCE=<checkout> python tests/golden/time_reference_jax.py [H W]   # default: one 1080 x 1920 frame
"""
import os
import platform
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.normpath(os.path.join(HERE, "..", "..")))

import oracle  # noqa: E402
from oracle import jax_shim  # noqa: E402


def main():
    H, W = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (1080, 1920)
    rng = np.random.RandomState(1234)
    grid = rng.rand(1, 16, 16, 8, 12).astype(np.float32)
    guide = rng.rand(1, H, W).astype(np.float32)
    inp = rng.rand(1, H, W, 3).astype(np.float32)
    t = time.perf_counter()
    out = jax_shim.bilateral_slice_apply(grid, guide, inp, True)
    dt = time.perf_counter() - t
    t = time.perf_counter()
    ref = oracle.best().bilateral_slice_apply(grid, guide, inp, True)
    dc = time.perf_counter() - t
    err = float(np.abs(out - ref).max() / np.abs(ref).max())
    cpu = platform.processor() or platform.machine()
    try:
        with open("/proc/cpuinfo") as f:
            cpu = next(line.split(":", 1)[1].strip() for line in f if line.startswith("model name"))
    except Exception:
        pass
    print(f"host: {os.cpu_count()} CPUs, {cpu}")
    print(f"reference jax/bilateral_slice.py (numpy stand-in, one process) + apply, 1 x {H} x {W}, grid 16x16x8x12: "
          f"{dt:.2f} s = {H * W / dt / 1e6:.3f} MP/s")
    print(f"reference C++ loops ({oracle.best().kind}, {oracle.best().num_threads()} threads available, one frame = one thread): "
          f"{dc:.3f} s = {H * W / dc / 1e6:.2f} MP/s; max |jax - c++| / max |c++| = {err:.2e}")


if __name__ == "__main__":
    main()
